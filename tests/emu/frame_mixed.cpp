// frame_mixed.cpp -- layered frames whose layers mix both projections (meao_set_layer_projections) through the HOST-compiled kernel
// sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  Built by mixed.py into libmeao_emu_mixed.so together with the mixed kernels'
// translation units (build.py MIXED_SOURCES), linked against libmeao_emu.so: every other kernel, the surface-access counter and the
// launch ledger are that library's.  A frame is launched the way libmeao launches it: the frame schedule, argument blocks and launcher
// choice of csrc/frame_record.h (launch_entry_mixed).
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

}  // namespace

extern "C" {

// Gives the plan of the frame `h` (frame_driver.cpp frame_create / frame_set_plan, whose frame type derives from FrameState, first and
// only base) the layers' projections `proj` (MeaoProjection per layer), as meao_api.cu build_plan plans them: Plan.orthographic /
// FrameState::layer_ortho (plan_projections), and for each orthographic layer the atlas padding of levels 1-2 -- the orthographic
// linearisation of raw depth 0, fma(zbx, 0, zby) (reversed Z: 1e5) -- in its constants and the arena's camera tables.  The other
// constants are the plan's: frame_set_plan takes each layer's from a plan-only libmeao context with the same projection table.
void frame_mixed_set(void *h, const int32_t *proj)
{
    FrameState &f = *static_cast<FrameState *>(h);
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
    if (f.layer_zb) memcpy(f.layer_zb, tz.data(), tz.size() * sizeof(LayerZ));
    if (f.layer_ren) memcpy(f.layer_ren, tr.data(), tr.size() * sizeof(LayerRender));
}

// 1: the plan mixes both projections (launch_entry_mixed's frames), 0: it does not
int frame_mixed_is_mixed(void *h) { return static_cast<FrameState *>(h)->layer_ortho.empty() ? 0 : 1; }

// One whole frame from the tight depth `depth` (kind: MEAO_DEPTH_*).  fused: low-only prepare_depth and the final upsample that reads
// and linearises the depth, storing the AO into `ao` (what meao_render records); 0: prepare_depth -> LinearDepth -> final upsample into
// the result buffer (the stage API's frame).  ren_tile: render_tile_variant's force (-1: the planner's rule).  Returns the first launch
// error (a cudaError_t), 0 when every launch was made.
int frame_run_mixed(void *h, const void *depth, int kind, int fused, void *ao, int ren_tile)
{
    FrameState &f = *static_cast<FrameState *>(h);
    whole_frame(f);
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, depth, kind);
    io.low_only = io.fused = fused != 0; io.ao = fused ? ao : nullptr;
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) {
        const cudaError_t e = launch_entry_mixed(f, l, io, ren_tile, nullptr);
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

// A CUDA-array frame: depth an emulated array of shape depth_shape (0 2-D, 1 layered, 2 cube) of L images of W x H elements (4 bytes:
// f32, 2 bytes: D16 codes) with rows depth_pitch bytes apart; ao the same for the AO (1 byte per texel).  Returns as frame_run_mixed.
int frame_run_arrays_mixed(void *h, void *depth, int kind, int depth_shape, long long depth_pitch, void *ao, int ao_shape, long long ao_pitch,
                           int ren_tile)
{
    FrameState &f = *static_cast<FrameState *>(h);
    whole_frame(f);
    const meao_emu::Surface ds{depth, (int)depth_esize(kind), f.W, f.H, f.layers, (size_t)depth_pitch, depth_shape};
    const meao_emu::Surface as{ao, 1, f.W, f.H, f.layers, (size_t)ao_pitch, ao_shape};
    auto surf_kind = [](int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : shape == meao_emu::SURF_LAYERED ? kSurfLayered : kSurfCube; };
    ArrayIO aio{(cudaSurfaceObject_t)&ds, (cudaSurfaceObject_t)&as, surf_kind(depth_shape), surf_kind(ao_shape), ao};
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, nullptr, kind);
    io.aio = &aio;
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) {
        const cudaError_t e = launch_entry_mixed(f, l, io, ren_tile, nullptr);
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

// TiledDepth<k> (debug buffer 5 + k) of layer `layer` in the reference layout (16 slices of f16) into out, with the layer's atlas padding
// for depth kind `kind` -- frame_driver.cpp's readback takes the kind of the last frame it ran itself, not of these frames.
void frame_mixed_tiled(void *h, int k, int layer, int kind, void *out)
{
    launch_tiled_atlas(*static_cast<FrameState *>(h), k, layer, kind, static_cast<__half *>(out), nullptr);
}

// The mixed units as this library builds them (kernels.h kMixedKernelUnits, which only libmeao lists): file names 32 bytes apart in
// names, kernel counts in counts; returns the number of units.
int frame_mixed_kernel_units(char *names, int *counts, int cap)
{
    static const KernelUnit *const units[] = {&kPrepareDepthMixedLayeredUnit, &kPrepareDepthArrayMixedUnit, &kRenderAoMixedLayeredUnit,
                                              &kBlurUpsampleLinMixedUnit};
    int n = 0;
    for (const KernelUnit *u : units) {
        if (n >= cap) break;
        std::snprintf(names + 32 * n, 32, "%s", u->file);
        counts[n++] = u->walk(nullptr);
    }
    return n;
}

}  // extern "C"
