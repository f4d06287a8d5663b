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

const struct {
    Kernel<CUtensorMap, RenderArgs, int> render[kRenderSlots];      // [render_slot]
    Kernel<const float *, int, int, int, int, int, float, __half *> synth_tiled;
} kKernels = {MEAO_RENDER_SLOTS(render_ao_kernel), synth_tiled_kernel};

}  // namespace

cudaError_t launch_render_ao(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, cudaStream_t s)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h));
    MEAO_LAUNCH((kKernels.render[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0);
    return cudaGetLastError();
}

cudaError_t launch_synth_tiled(const float *low, int lw, int lh, int lpitch, int sw, int sh, float pad,
                               __half *out, cudaStream_t s)
{
    dim3 grid(ceil_div(sw, 128), sh, 16);
    MEAO_LAUNCH((synth_tiled_kernel), grid, 128, 0, s, low, lw, lh, lpitch, sw, sh, pad, out);
    return cudaGetLastError();
}

const KernelUnit kRenderAoUnit = {"render_ao.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels.render, kKernels.synth_tiled); }};

}  // namespace meao
