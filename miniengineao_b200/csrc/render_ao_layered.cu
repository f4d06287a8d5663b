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

}  // namespace

template <int MODE, bool EXH, int TH>
static void launch_render_layered_variant(const CUtensorMap &low_map, int t, const RenderArgs &a, dim3 grid, cudaStream_t s, const LayerRender *cam, int pad)
{
    const size_t smem = (size_t)Geo<MODE, TH>::kSW * Geo<MODE, TH>::kSH * sizeof(float);
    MEAO_LAUNCH((render_ao_layered_kernel<MODE, EXH, TH>), grid, kThreads, smem, s, low_map, a, t, cam, pad);
}
template <int MODE, bool EXH>
static cudaError_t launch_render_layered_th(const CUtensorMap &low_map, int t, const RenderArgs &a, int gx, int rows, int layers, cudaStream_t s,
                                            const LayerRender *cam, int pad)
{
    switch (a.tile_h) {
        case kRenderTileHs[0]: launch_render_layered_variant<MODE, EXH, kRenderTileHs[0]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[0]), layers), s, cam, pad); break;
        case kRenderTileHs[1]: launch_render_layered_variant<MODE, EXH, kRenderTileHs[1]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[1]), layers), s, cam, pad); break;
        case kRenderTileHs[2]: launch_render_layered_variant<MODE, EXH, kRenderTileHs[2]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[2]), layers), s, cam, pad); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_render_ao_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                     const LayerRender *cam, int pad)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const int gx = ceil_div(a.lw, kTW), rows = a.row1 - ybase;
    const int t = use_tma ? 1 : 0;
    if (!a.wide) return a.exhaustive ? launch_render_layered_th<0, true>(low_map, t, a, gx, rows, layers, s, cam, pad)
                                     : launch_render_layered_th<0, false>(low_map, t, a, gx, rows, layers, s, cam, pad);
    return a.exhaustive ? launch_render_layered_th<1, true>(low_map, t, a, gx, rows, layers, s, cam, pad)
                        : launch_render_layered_th<1, false>(low_map, t, a, gx, rows, layers, s, cam, pad);
}

#ifndef MEAO_EMULATE
cudaError_t preload_render_ao_layered()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(render_ao_layered_kernel<0, false, 32>); t(render_ao_layered_kernel<0, false, 16>); t(render_ao_layered_kernel<0, false, 8>);
    t(render_ao_layered_kernel<0, true, 32>); t(render_ao_layered_kernel<0, true, 16>); t(render_ao_layered_kernel<0, true, 8>);
    t(render_ao_layered_kernel<1, false, 32>); t(render_ao_layered_kernel<1, false, 16>); t(render_ao_layered_kernel<1, false, 8>);
    t(render_ao_layered_kernel<1, true, 32>); t(render_ao_layered_kernel<1, true, 16>); t(render_ao_layered_kernel<1, true, 8>);
    return e;
}
#endif

}  // namespace meao
