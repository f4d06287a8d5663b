// prepare_depth_views.cu -- stage 1 of a layered pointer frame with a layer-viewport table (meao_set_layer_viewports): layer l reads
// the W x H rectangle of its table entry (kernels.h LayerView) from the caller's pitched depth, ONE launch for all layers.  Only the
// low-only form: such a frame is always fused (its final upsample linearises the full-resolution depth, blur_upsample_lin_views.cu).
// The kernel body is prepare_depth_layered.cu's (prepare_depth_kernel.inc with MEAO_LAYERED 1 and MEAO_VIEWS 1): only the base of each
// layer's depth and its vector-load test differ.  A translation unit of its own so that prepare_depth_layered.cu compiles to exactly
// the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#define MEAO_VIEWS 1
#include "prepare_depth_kernel.inc"
#undef MEAO_VIEWS
#undef MEAO_LAYERED

// [prepare_slot]
const Kernel<PrepareArgs, const LayerView *, const LayerZ *> kKernels[kPrepareSlots] = MEAO_PREPARE_SLOTS(prepare_depth_low_views_kernel, MEAO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_views(const PrepareArgs &a_in, const LayerView *views, int layers, cudaStream_t s, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    if (layers < 1 || layers > kMaxLayers || !views) return cudaErrorInvalidValue;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepLowTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, views, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthViewsUnit = {"prepare_depth_views.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
