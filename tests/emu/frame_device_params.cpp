// frame_device_params.cpp -- device parameters (meao_bind_device_params) through the HOST-compiled parameter stage and render twins (TEST
// INFRASTRUCTURE ONLY, see cuda_emu.h).  Built by device_params.py into libmeao_emu_params.so together with the device-parameter units
// (build.py PARAM_SOURCES), linked against libmeao_emu_cameras.so and the libraries it links: every other kernel, the surface-access
// counter and the launch ledger are the emulator's.  The stage and the renders are launched the way libmeao launches them
// (csrc/frame_record.h launch_render_params, launch_render_params_entry), and a frame runs the schedule libmeao records for its bindings.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

namespace {

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

// slot: the context's allocation as meao_bind_device_params makes it, {reject_fadeoff, intensity} then kParamStatusWords status words
RenderParamArgs param_args(const float *params, float *slot)
{
    RenderParamArgs a{};
    a.params = params; a.derived = slot; a.status = reinterpret_cast<uint32_t *>(slot + 2);
    return a;
}

}  // namespace

extern "C" {

// The parameter stage alone: {thickness_modifier, intensity} at params into the slot (4 words).  Returns the launch's cudaError_t.
int frame_params_derive(const float *params, float *slot)
{
    return (int)launch_render_params(param_args(params, slot), nullptr);
}

// One whole frame of the plan in `h` (frame_driver.cpp frame_create / frame_set_plan; device_cameras.py frame for projections and
// stereo): the schedule of its bindings, frame_schedule(variants, cams != nullptr, params != nullptr), every launch through the launcher
// libmeao picks -- the camera stage, the parameter stage, the *_params_layered renders while parameters are bound (FrameIO.params), and
// otherwise launch_entry_mixed, launch_entry_ortho or launch_entry with FrameIO.cams set while cameras are bound.  params == nullptr:
// the host parameters of the plan (the reference frame).  fused and ao as frame_device_cameras.cpp frame_cams_run.  Returns the first
// launch error (a cudaError_t), 0 when every launch was made.
int frame_params_run(void *h, const float *params, float *slot, const float *cams, uint32_t *cam_status, const void *depth, int kind,
                     int fused, void *ao, int ren_tile)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    DeviceCameras dc;
    dc.cams = cams; dc.status = cam_status;
    sample_thickness(dc.thick);
    const RenderParamArgs pa = param_args(params, slot);
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, depth, kind);
    io.low_only = io.fused = fused != 0; io.ao = fused ? ao : nullptr;
    io.cams = cams ? &dc : nullptr;
    io.params = params ? &pa : nullptr;
    for (const FrameLaunch &l : frame_schedule(f.plan.variants, cams != nullptr, params != nullptr)) {
        const bool render = l.stage == kStageRender || l.stage == kStageRenderWide;
        cudaError_t e;
        if (l.stage == kStageCamera) e = launch_cameras(f, dc, nullptr);
        else if (l.stage == kStageParams) e = launch_render_params(pa, nullptr);
        else if (io.params && render) e = launch_render_params_entry(f, l, io, ren_tile, nullptr);
        else if (!f.layer_ortho.empty()) e = launch_entry_mixed(f, l, io, ren_tile, nullptr);
        else if (f.plan.orthographic) e = launch_entry_ortho(f, l, io, ren_tile, nullptr);
        else e = launch_entry(f, l, io, ren_tile, nullptr);
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

// The device-parameter units as this library builds them (kernels.h kParamKernelUnits, which only libmeao lists): up to `cap` file names
// (48 bytes each) into names and kernel counts into counts; returns the number of units.
int frame_params_kernel_units(char *names, int *counts, int cap)
{
    const KernelUnit *units[] = {&kRenderParamsUnit, &kRenderAoParamsLayeredUnit, &kRenderAoOrthoParamsLayeredUnit, &kRenderAoMixedParamsLayeredUnit};
    int n = 0;
    for (const KernelUnit *u : units) {
        if (n >= cap) break;
        std::snprintf(names + 48 * n, 48, "%s", u->file);
        counts[n++] = u->walk(nullptr);
    }
    return n;
}

}  // extern "C"
