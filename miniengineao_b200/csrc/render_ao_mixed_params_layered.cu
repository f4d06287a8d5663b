// render_ao_mixed_params_layered.cu -- render_ao_mixed_layered.cu's kernels for a bound device parameter buffer (meao_bind_device_params):
// render_ao_kernel.inc with MEAO_LAYERED 1, MEAO_ORTHO 2 and MEAO_DEVICE_PARAMS 1 (render_ao_params_layered.cu).  A translation unit of
// its own (build.py PARAM_SOURCES).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_DEVICE_PARAMS 1
#define MEAO_ORTHO 2
#define MEAO_LAYERED 1
#define render_ao_layered_kernel render_ao_mixed_params_layered_kernel
#include "render_ao_kernel.inc"
#undef render_ao_layered_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO
#undef MEAO_DEVICE_PARAMS

// [render_slot]
const Kernel<CUtensorMap, RenderArgs, int, const LayerRender *, int, const float *, LayerProjections> kKernels[kRenderSlots] =
    MEAO_RENDER_SLOTS(render_ao_mixed_params_layered_kernel);

}  // namespace

cudaError_t launch_render_ao_mixed_params_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                                  const LayerRender *cam, int pad, const float *params, const LayerProjections &proj)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || !cam || !params) return cudaErrorInvalidValue;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h), layers);
    MEAO_LAUNCH((kKernels[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0, cam, pad, params, proj);
    return cudaGetLastError();
}

const KernelUnit kRenderAoMixedParamsLayeredUnit = {"render_ao_mixed_params_layered.cu",
                                                    [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
