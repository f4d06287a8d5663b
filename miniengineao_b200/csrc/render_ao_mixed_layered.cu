// render_ao_mixed_layered.cu -- render_ao_ortho_layered.cu's kernels for a layered frame whose layers mix both projections
// (meao_set_layer_projections): render_ao_kernel.inc with MEAO_LAYERED 1 and MEAO_ORTHO 2.  Each CTA reads its layer's bit of the
// LayerProjections parameter once and runs the sampling loop of render_ao_layered.cu (perspective) or render_ao_ortho_layered.cu
// (orthographic); the tile load before it is the one all three share.  A layer's constants are its LayerRender entries, computed with its
// own projection.  A translation unit of its own (build.py MIXED_SOURCES).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 2
#define MEAO_LAYERED 1
#define render_ao_layered_kernel render_ao_mixed_layered_kernel
#include "render_ao_kernel.inc"
#undef render_ao_layered_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [render_slot]
const Kernel<CUtensorMap, RenderArgs, int, const LayerRender *, int, LayerProjections> kKernels[kRenderSlots] =
    MEAO_RENDER_SLOTS(render_ao_mixed_layered_kernel);

}  // namespace

cudaError_t launch_render_ao_mixed_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                           const LayerRender *cam, int pad, const LayerProjections &proj)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || !cam) return cudaErrorInvalidValue;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h), layers);
    MEAO_LAUNCH((kKernels[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0, cam, pad, proj);
    return cudaGetLastError();
}

const KernelUnit kRenderAoMixedLayeredUnit = {"render_ao_mixed_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
