// render_ao_params_layered.cu -- render_ao_layered.cu's kernels for a bound device parameter buffer (meao_bind_device_params):
// render_ao_kernel.inc with MEAO_LAYERED 1 and MEAO_DEVICE_PARAMS 1.  Each CTA reads the frame's {reject_fadeoff, intensity} from the
// slot render_params.cu derived ahead of the renders, so a recorded frame follows the buffer at every replay.  A bound single-layer frame
// takes these kernels with one layer.  A translation unit of its own (build.py PARAM_SOURCES), so every other kernel keeps its code.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_DEVICE_PARAMS 1
#define MEAO_LAYERED 1
#define render_ao_layered_kernel render_ao_params_layered_kernel
#include "render_ao_kernel.inc"
#undef render_ao_layered_kernel
#undef MEAO_LAYERED
#undef MEAO_DEVICE_PARAMS

// [render_slot]
const Kernel<CUtensorMap, RenderArgs, int, const LayerRender *, int, const float *> kKernels[kRenderSlots] =
    MEAO_RENDER_SLOTS(render_ao_params_layered_kernel);

}  // namespace

cudaError_t launch_render_ao_params_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                            const LayerRender *cam, int pad, const float *params)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || !params) return cudaErrorInvalidValue;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h), layers);
    MEAO_LAUNCH((kKernels[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0, cam, pad, params);
    return cudaGetLastError();
}

const KernelUnit kRenderAoParamsLayeredUnit = {"render_ao_params_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
