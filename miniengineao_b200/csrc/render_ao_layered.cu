// render_ao_layered.cu -- stage 2 for a layered frame (meao_set_layers): one launch renders level k of all L layers.
// The kernel body is render_ao.cu's (render_ao_kernel.inc); the layer is blockIdx.z and selects the LowDepth<k> /
// Occlusion<k> (or HighQuality<k>) image of that layer (kernels.h "layered frames").  A translation unit of its own so that
// render_ao.cu compiles to exactly the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#include "render_ao_kernel.inc"
#undef MEAO_LAYERED

// [render_slot]
const Kernel<CUtensorMap, RenderArgs, int, const LayerRender *, int> kKernels[kRenderSlots] = MEAO_RENDER_SLOTS(render_ao_layered_kernel);

}  // namespace

cudaError_t launch_render_ao_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                     const LayerRender *cam, int pad)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h), layers);
    MEAO_LAUNCH((kKernels[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0, cam, pad);
    return cudaGetLastError();
}

const KernelUnit kRenderAoLayeredUnit = {"render_ao_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
