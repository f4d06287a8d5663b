// prepare_depth_layered.cu -- stage 1 for a layered frame (meao_set_layers): L same-size depth images stacked at a stride of
// PrepareArgs.depth_layer_pitch (tight: one W x H image), ONE launch for all of them.  The kernel body is prepare_depth.cu's (prepare_depth_kernel.inc); the
// layer is blockIdx.z and selects the input image and the output images of every level (kernels.h "layered frames").
// A translation unit of its own so that prepare_depth.cu compiles to exactly the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#include "prepare_depth_kernel.inc"
#undef MEAO_LAYERED

}  // namespace

cudaError_t launch_prepare_depth_layered(const PrepareArgs &a_in, int layers, cudaStream_t s, bool low_only, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH), layers);
#define MEAO_PREP_K(...) (low_only ? prepare_depth_low_layered_kernel<__VA_ARGS__> : prepare_depth_layered_kernel<__VA_ARGS__>)
    if (!a.raw) {
        MEAO_LAUNCH((MEAO_PREP_K(false, true, IN_F32)), grid, kPrepThreads, 0, s, a, layer_zb);
    } else if (a.in_format == IN_D16) {
        if (a.reversed_z) MEAO_LAUNCH((MEAO_PREP_K(true, true, IN_D16)), grid, kPrepThreads, 0, s, a, layer_zb);
        else              MEAO_LAUNCH((MEAO_PREP_K(true, false, IN_D16)), grid, kPrepThreads, 0, s, a, layer_zb);
    } else if (a.in_format == IN_D24S8) {
        if (a.reversed_z) MEAO_LAUNCH((MEAO_PREP_K(true, true, IN_D24S8)), grid, kPrepThreads, 0, s, a, layer_zb);
        else              MEAO_LAUNCH((MEAO_PREP_K(true, false, IN_D24S8)), grid, kPrepThreads, 0, s, a, layer_zb);
    } else {
        if (a.reversed_z) MEAO_LAUNCH((MEAO_PREP_K(true, true, IN_F32)), grid, kPrepThreads, 0, s, a, layer_zb);
        else              MEAO_LAUNCH((MEAO_PREP_K(true, false, IN_F32)), grid, kPrepThreads, 0, s, a, layer_zb);
    }
#undef MEAO_PREP_K
    return cudaGetLastError();
}

#ifndef MEAO_EMULATE
cudaError_t preload_prepare_depth_layered()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(prepare_depth_layered_kernel<false, true, IN_F32>);
    t(prepare_depth_layered_kernel<true, true, IN_F32>); t(prepare_depth_layered_kernel<true, false, IN_F32>);
    t(prepare_depth_layered_kernel<true, true, IN_D16>); t(prepare_depth_layered_kernel<true, false, IN_D16>);
    t(prepare_depth_layered_kernel<true, true, IN_D24S8>); t(prepare_depth_layered_kernel<true, false, IN_D24S8>);
    t(prepare_depth_low_layered_kernel<false, true, IN_F32>);
    t(prepare_depth_low_layered_kernel<true, true, IN_F32>); t(prepare_depth_low_layered_kernel<true, false, IN_F32>);
    t(prepare_depth_low_layered_kernel<true, true, IN_D16>); t(prepare_depth_low_layered_kernel<true, false, IN_D16>);
    t(prepare_depth_low_layered_kernel<true, true, IN_D24S8>); t(prepare_depth_low_layered_kernel<true, false, IN_D24S8>);
    return e;
}
#endif

}  // namespace meao
