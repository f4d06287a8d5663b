// render_ao.cu -- stage 2 of the SSAO pipe: volumetric-obscurance sampling at one mip level.
//
// Replaces Render.compute kernel main_interleaved (TestSamplePair :60-75, TestSamples :77-110,
// MAIN :112-177) for TiledDepth<k> -> Occlusion<k>.
//
// Design (not a port): the reference deinterleaves depth into 16 slices so that its sparse taps
// become unit-stride texture fetches.  Here the level-k depth stays in NATURAL layout: one CTA
// stages a (64+32) x (32+32) f32 tile of LowDepth<k> in shared memory with a single TMA box load,
// rounds it to f16 in place (the reference samples an RHalf atlas), and every thread then reads
// its 36 taps at stride 4 texels -- which, across a warp of consecutive pixels, is unit-stride and
// bank-conflict free.  A thread owns two horizontally adjacent pixels so each tap is one LDS.64.
//
// Virtual atlas semantics that must be preserved (SURVEY.md P3): pixel (X,Y) of level k lives in
// slice (X&3, Y&3) at slice texel (X>>2, Y>>2); a tap (di,dj) reads slice texel
// (clamp(i+di, 0, sw-1), clamp(j+dj, 0, sh-1)), i.e. natural pixel (4*ci + (X&3), 4*cj + (Y&3)),
// which is a padding texel (value `pad`) when it lies outside level k.  Tiles whose footprint is
// entirely inside the level need none of this and take the TMA path; border tiles resolve the
// clamp/padding per texel with a gather from global memory.
//
// Bound: instruction issue (estimated from the source: about 250 thread-instructions per output, 2 B + 1 B of HBM traffic).
//
// Variants (SURVEY.md 8f.2; shipped in Render.compute but never dispatched by AmbientOcclusion.cs):
//   MODE 1 = kernel `main` (WIDE_SAMPLING, REN:27-29,46-50,79-82,115-116,125,136,174): plain f32 Texture2D
//            source (LowDepth<k> itself, no f16 rounding, no atlas), taps at 2x the offsets, per-texel
//            clamp-to-edge in level space, output at the same resolution -> HighQuality<k>.  Same CTA
//            shape; the apron shrinks to 8 texels (TMA box 80 x 48) and the tap stride to 2.
//   EXH      = #define SAMPLE_EXHAUSTIVELY (REN:144-159): twelve TestSamples calls (68 taps) instead of seven (36).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 0
#include "render_ao_kernel.inc"
#undef MEAO_LAYERED

// debug view: TiledDepth<k>[slice][j][i] exactly as Downsample1/2 would have written it
__global__ void synth_tiled_kernel(const float *low, int lw, int lh, int lpitch, int sw, int sh, float pad, __half *out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y, s = blockIdx.z;
    if (i >= sw) return;
    const int x = 4 * i + (s & 3), y = 4 * j + (s >> 2);                     // inverse of DS1:69,71
    float v = pad;
    if (x < lw && y < lh) v = low[(size_t)y * lpitch + x];
    out[((size_t)s * sh + j) * sw + i] = __float2half_rn(v);
}

}  // namespace

template <int MODE, bool EXH, int TH>
static void launch_render_variant(const CUtensorMap &low_map, int t, const RenderArgs &a, dim3 grid, cudaStream_t s)
{
    const size_t smem = (size_t)Geo<MODE, TH>::kSW * Geo<MODE, TH>::kSH * sizeof(float);
    MEAO_LAUNCH((render_ao_kernel<MODE, EXH, TH>), grid, kThreads, smem, s, low_map, a, t);
}
template <int MODE, bool EXH>
static cudaError_t launch_render_th(const CUtensorMap &low_map, int t, const RenderArgs &a, int gx, int rows, cudaStream_t s)
{
    switch (a.tile_h) {
        case kRenderTileHs[0]: launch_render_variant<MODE, EXH, kRenderTileHs[0]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[0])), s); break;
        case kRenderTileHs[1]: launch_render_variant<MODE, EXH, kRenderTileHs[1]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[1])), s); break;
        case kRenderTileHs[2]: launch_render_variant<MODE, EXH, kRenderTileHs[2]>(low_map, t, a, dim3(gx, ceil_div(rows, kRenderTileHs[2])), s); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_render_ao(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, cudaStream_t s)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    const int ybase = a.row0 & ~3;
    const int gx = ceil_div(a.lw, kTW), rows = a.row1 - ybase;
    const int t = use_tma ? 1 : 0;
    if (!a.wide) return a.exhaustive ? launch_render_th<0, true>(low_map, t, a, gx, rows, s) : launch_render_th<0, false>(low_map, t, a, gx, rows, s);
    return a.exhaustive ? launch_render_th<1, true>(low_map, t, a, gx, rows, s) : launch_render_th<1, false>(low_map, t, a, gx, rows, s);
}

cudaError_t launch_synth_tiled(const float *low, int lw, int lh, int lpitch, int sw, int sh, float pad,
                               __half *out, cudaStream_t s)
{
    dim3 grid(ceil_div(sw, 128), sh, 16);
    MEAO_LAUNCH((synth_tiled_kernel), grid, 128, 0, s, low, lw, lh, lpitch, sw, sh, pad, out);
    return cudaGetLastError();
}

#ifndef MEAO_EMULATE
cudaError_t preload_render_ao()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(render_ao_kernel<0, false, 32>); t(render_ao_kernel<0, false, 16>); t(render_ao_kernel<0, false, 8>);
    t(render_ao_kernel<0, true, 32>); t(render_ao_kernel<0, true, 16>); t(render_ao_kernel<0, true, 8>);
    t(render_ao_kernel<1, false, 32>); t(render_ao_kernel<1, false, 16>); t(render_ao_kernel<1, false, 8>);
    t(render_ao_kernel<1, true, 32>); t(render_ao_kernel<1, true, 16>); t(render_ao_kernel<1, true, 8>);
    t(synth_tiled_kernel);
    return e;
}
#endif

}  // namespace meao
