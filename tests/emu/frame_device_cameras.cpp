// frame_device_cameras.cpp -- device cameras (meao_bind_device_cameras) through the HOST-compiled camera kernel (TEST INFRASTRUCTURE ONLY,
// see cuda_emu.h).  Built by device_cameras.py into libmeao_emu_cameras.so together with the camera unit (build.py CAMERA_SOURCES),
// linked against libmeao_emu.so: every other kernel, the surface-access counter and the launch ledger are that library's.  The camera
// stage is launched the way libmeao launches it (csrc/frame_record.h launch_cameras, camera_args), and a bound frame runs the schedule
// with the camera stage first and the layered kernels at every layer count (FrameIO.cams).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

namespace {

void whole_frame(FrameState &f)
{
    f.band0 = 0; f.band1 = f.H;
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
}

// meao_api.cu sample_thickness (AO.cs:577-590): Mathf.Sqrt is (float)Math.Sqrt((double)x)
float mathf_sqrt(float f) { return (float)std::sqrt((double)f); }
void sample_thickness(float t[12])
{
    t[0] = mathf_sqrt(1 - 0.2f * 0.2f);                 t[1] = mathf_sqrt(1 - 0.4f * 0.4f);
    t[2] = mathf_sqrt(1 - 0.6f * 0.6f);                 t[3] = mathf_sqrt(1 - 0.8f * 0.8f);
    t[4] = mathf_sqrt(1 - 0.2f * 0.2f - 0.2f * 0.2f);   t[5] = mathf_sqrt(1 - 0.2f * 0.2f - 0.4f * 0.4f);
    t[6] = mathf_sqrt(1 - 0.2f * 0.2f - 0.6f * 0.6f);   t[7] = mathf_sqrt(1 - 0.2f * 0.2f - 0.8f * 0.8f);
    t[8] = mathf_sqrt(1 - 0.4f * 0.4f - 0.4f * 0.4f);   t[9] = mathf_sqrt(1 - 0.4f * 0.4f - 0.6f * 0.6f);
    t[10] = mathf_sqrt(1 - 0.4f * 0.4f - 0.8f * 0.8f);  t[11] = mathf_sqrt(1 - 0.6f * 0.6f - 0.6f * 0.6f);
}

DeviceCameras device_cameras(const float *cams, uint32_t *status)
{
    DeviceCameras dc;
    dc.cams = cams; dc.status = status;
    sample_thickness(dc.thick);
    return dc;
}

}  // namespace

extern "C" {

// Gives the plan of the frame `h` (frame_driver.cpp frame_create / frame_set_plan, whose frame type derives from FrameState, first and
// only base) what meao_api.cu build_plan adds besides the getters' constants: single_pass_stereo, and the layers' projections `proj`
// (MeaoProjection per layer) -- Plan.orthographic / FrameState::layer_ortho, and for each orthographic layer the atlas padding of levels
// 1-2, fma(zbx, 0, zby) (reversed Z: 1e5).  The arena's camera tables are then camera_tables() of that plan, as libmeao uploads them.
void frame_cams_plan(void *h, int stereo, const int32_t *proj)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.plan.variants.single_pass_stereo = stereo;
    for (int l = 0; l < f.layers; l++) {
        if (proj[l] != MEAO_PROJECTION_ORTHOGRAPHIC) continue;
        CamConsts &cc = f.layer_consts[l];
        for (int k = 1; k <= 2; k++) cc.pad[k] = f.plan.reversed_z ? 1e5f : std::fmaf(cc.zb[0], 0.0f, cc.zb[1]);
    }
    memcpy(f.plan.pad, f.layer_consts[0].pad, sizeof f.plan.pad);
    plan_projections(f, [proj](int l) { return proj[l] == MEAO_PROJECTION_ORTHOGRAPHIC; });
    std::vector<LayerZ> tz;
    std::vector<LayerRender> tr;
    camera_tables(f, tz, tr);
    memcpy(f.layer_zb, tz.data(), tz.size() * sizeof(LayerZ));
    memcpy(f.layer_ren, tr.data(), tr.size() * sizeof(LayerRender));
}

// camera_tables() of the plan (the host planner's bytes): L LayerZ into zb, 8 L LayerRender into ren
void frame_cams_expected(void *h, void *zb, void *ren)
{
    const FrameState &f = *static_cast<FrameState *>(h);
    std::vector<LayerZ> tz;
    std::vector<LayerRender> tr;
    camera_tables(f, tz, tr);
    memcpy(zb, tz.data(), tz.size() * sizeof(LayerZ));
    memcpy(ren, tr.data(), tr.size() * sizeof(LayerRender));
}

// The arena's camera tables as they stand: L LayerZ into zb, 8 L LayerRender into ren
void frame_cams_tables(void *h, void *zb, void *ren)
{
    const FrameState &f = *static_cast<FrameState *>(h);
    memcpy(zb, f.layer_zb, (size_t)f.layers * sizeof(LayerZ));
    memcpy(ren, f.layer_ren, (size_t)8 * f.layers * sizeof(LayerRender));
}

// Fills the arena's camera tables with the byte `fill`, so that a derivation that skips an entry shows
void frame_cams_clobber(void *h, int fill)
{
    const FrameState &f = *static_cast<FrameState *>(h);
    memset(f.layer_zb, fill, (size_t)f.layers * sizeof(LayerZ));
    memset(f.layer_ren, fill, (size_t)8 * f.layers * sizeof(LayerRender));
}

// The camera stage alone: the tables derived from cams ([layers][3] floats) into the arena; status: the kernel's kCameraStatusWords
// words.  Returns the launch's cudaError_t.
int frame_cams_derive(void *h, const float *cams, uint32_t *status)
{
    const FrameState &f = *static_cast<FrameState *>(h);
    return (int)launch_cameras(f, device_cameras(cams, status), nullptr);
}

// One whole bound frame: the schedule with the camera stage first (frame_schedule(variants, true)), every other launch through the
// launcher libmeao picks for the plan (launch_entry_mixed, launch_entry_ortho or launch_entry) with FrameIO.cams set.  fused and ao as
// frame_mixed.cpp frame_run_mixed.  ren_tile: render_tile_variant's force (-1: the planner's rule).  Returns the first launch error (a
// cudaError_t), 0 when every launch was made.
int frame_cams_run(void *h, const float *cams, uint32_t *status, const void *depth, int kind, int fused, void *ao, int ren_tile)
{
    FrameState &f = *static_cast<FrameState *>(h);
    whole_frame(f);
    const DeviceCameras dc = device_cameras(cams, status);
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, depth, kind);
    io.low_only = io.fused = fused != 0; io.ao = fused ? ao : nullptr;
    io.cams = &dc;
    for (const FrameLaunch &l : frame_schedule(f.plan.variants, true)) {
        cudaError_t e;
        if (l.stage == kStageCamera) e = launch_cameras(f, dc, nullptr);
        else if (!f.layer_ortho.empty()) e = launch_entry_mixed(f, l, io, ren_tile, nullptr);
        else if (f.plan.orthographic) e = launch_entry_ortho(f, l, io, ren_tile, nullptr);
        else e = launch_entry(f, l, io, ren_tile, nullptr);
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

// TiledDepth<k> (debug buffer 5 + k) of layer `layer` into out, with the padding value of the layer's camera table row for depth kind
// `kind` -- what meao_get_buffer reads back while a device camera buffer is bound, since the host plan's value is the host camera's
void frame_cams_tiled(void *h, int k, int layer, int kind, void *out)
{
    const FrameState &f = *static_cast<FrameState *>(h);
    const float pad = f.layer_ren[(size_t)2 * (k - 1) * f.layers + layer].pad;
    launch_tiled_atlas(f, k, layer, kind, static_cast<__half *>(out), nullptr, &pad);
}

// The camera unit as this library builds it (kernels.h kCameraKernelUnits, which only libmeao lists): its file name into name (32
// bytes); returns its kernel count.
int frame_cams_kernel_unit(char *name)
{
    std::snprintf(name, 32, "%s", kCameraTablesUnit.file);
    return kCameraTablesUnit.walk(nullptr);
}

}  // extern "C"
