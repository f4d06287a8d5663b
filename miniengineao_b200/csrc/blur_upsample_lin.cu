// blur_upsample_lin.cu -- the final blur_upsample level (Upsample.compute main / main_premin, L1 -> L0) of a whole frame, reading
// the caller's raw depth instead of LinearDepth.  Each thread loads the raw depth of its own eight pixels, linearises it with
// prepare_depth's arithmetic (depth_in.cuh), rounds it to f16 -- the values LinearDepth would hold -- stores those to LinearDepth and
// upsamples with them.  prepare_depth then runs low_only: it loads only the even depth rows and does not write LinearDepth.
//
// Why: prepare_depth is bound by HBM bandwidth and the final upsample by instruction issue, so the full-resolution LinearDepth
// round trip (written by the one, read back by the other) is moved to the kernel with bandwidth to spare.  Every output bit stays
// the same.  Kernels that run apart from their frame's prepare_depth (the stage API, split band frames, CUDA-array frames, the AO
// regeneration of meao_get_buffer) keep the pair prepare_depth -> LinearDepth -> blur_upsample.
//
// The kernel bodies are blur_upsample.cu's (blur_upsample_kernel.inc with MEAO_UPS_LIN 1), single-image and layered, templated on
// the input format; the linear-input case and reversed Z are run-time (warp-uniform) values of `din`.  A translation unit of its own
// so that blur_upsample.cu and blur_upsample_layered.cu compile to exactly the code they did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#include "blur_upsample_device.inc"
#include "blur_upsample_layer_args.inc"
#include "depth_in.cuh"

// The LinearDepth values of pixels px0 .. px0 + 7 of row py of layer `layer` (those inside the row: all eight when `full`): load
// their raw depth, linearise it (DS1:37-48), round it to f16 and store it to LinearDepth at `lin` (this thread's first pixel; the
// 16-byte store is aligned because px0 % 8 == 0 and rows are 128-byte pitched).  Returns the packed halves (pixel 0 in the low half
// of .x): what the 128-bit LinearDepth load of the kernel that reads LinearDepth returns.
// LAYERED: the layer's ZBufferParams come from din.layer_zb when it is set (per-layer cameras).
template <int IN, bool LAYERED = false>
__device__ __forceinline__ uint4 linearize_pixels8(const DepthIn &din, int layer, int py, int px0, int hiw, int hih, bool full, __half *lin)
{
    const void *depth = reinterpret_cast<const char *>(din.depth) + (size_t)layer * din.depth_layer_pitch * (IN == IN_D16 ? 2 : 4);
    float v[8], d[8];
    load8<IN>(depth, (size_t)(py - din.depth_row0) * din.depth_pitch + px0, full && din.vec_ok, hiw - px0, v);
    float zbx = din.zbx, zby = din.zby;
    if (LAYERED && din.layer_zb) { zbx = __ldg(&din.layer_zb[layer].zbx); zby = __ldg(&din.layer_zb[layer].zby); }
    if (!din.raw) linearize8<false, true>(v, zbx, zby, d);
    else if (din.reversed_z) linearize8<true, true>(v, zbx, zby, d);
    else linearize8<true, false>(v, zbx, zby, d);
    const __half2 h0 = __floats2half2_rn(d[0], d[1]), h1 = __floats2half2_rn(d[2], d[3]);
    const __half2 h2 = __floats2half2_rn(d[4], d[5]), h3 = __floats2half2_rn(d[6], d[7]);
    uint4 pk;
    pk.x = *reinterpret_cast<const uint32_t *>(&h0); pk.y = *reinterpret_cast<const uint32_t *>(&h1);
    pk.z = *reinterpret_cast<const uint32_t *>(&h2); pk.w = *reinterpret_cast<const uint32_t *>(&h3);
    if (full) {
        *reinterpret_cast<uint4 *>(lin) = pk;                                            // DS1:46
    } else {
#pragma unroll
        for (int e = 0; e < 8; e++) {
            if (px0 + e >= hiw) break;
            lin[e] = __float2half_rn(d[e]);
        }
    }
    return pk;
}

// layer_args of the fused layered kernels: the caller's AO advances by its own layer pitch (DepthIn.ao_layer_pitch, bytes) instead of
// hih x out_pitch, so a layered AO view keeps the layer pitch of the tensor or allocation it lives in
__device__ __forceinline__ UpsampleArgs layer_args(const UpsampleArgs &a, int l, long long ao_layer_pitch)
{
    UpsampleArgs r = layer_args(a, l);
    r.out = a.out + (size_t)l * ao_layer_pitch;
    return r;
}
__device__ __forceinline__ UpsamplePreminArgs layer_args(const UpsamplePreminArgs &pa, int l, long long ao_layer_pitch)
{
    UpsamplePreminArgs r = layer_args(pa, l);
    r.base.out = pa.base.out + (size_t)l * ao_layer_pitch;
    return r;
}

#define MEAO_UPS_LIN 1
#define MEAO_UPS_PREMIN 0
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_PREMIN 1
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_LAYERED 1
#define MEAO_UPS_PREMIN 0
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_PREMIN 1
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#undef MEAO_UPS_LAYERED
#undef MEAO_UPS_LIN

template <int IN>
void launch_lin(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, const UpsampleArgs &a,
                const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din, int t, int layers, dim3 grid, cudaStream_t s)
{
    const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
    if (layers == 1) {
        if (!lo_ao2) MEAO_LAUNCH((blur_upsample_lin_kernel<IN>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, din);
        else         MEAO_LAUNCH((blur_upsample_premin_lin_kernel<IN>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, din);
    } else {
        if (!lo_ao2) MEAO_LAUNCH((blur_upsample_lin_layered_kernel<IN>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, din);
        else         MEAO_LAUNCH((blur_upsample_premin_lin_layered_kernel<IN>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, din);
    }
}

}  // namespace

cudaError_t launch_blur_upsample_lin(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                     const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din_in, int layers, int sm_count,
                                     cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    if (!a_in.hi_is_half || a_in.hi_ao || (lo_ao2 && !lo_ao2_map)) return cudaErrorInvalidValue;      // the final level only
    UpsampleArgs a = a_in;
    const int ybase = a.row0 & ~1;
    a.tiles_x = ceil_div(a.hiw, kHW); a.tiles_y = ceil_div(a.row1 - ybase, kHH);
    const long long ntiles_ll = (long long)a.tiles_x * a.tiles_y * layers;
    if (ntiles_ll > 0x7fffffffLL) return cudaErrorInvalidValue;        // the tile index is a 32-bit int
    const int ntiles = (int)ntiles_ll;
    // the rule of launch_blur_upsample(_layered): the persistent tile loop from two tiles per CTA slot
    const int kWave = sm_count * MEAO_UPS_MINB;
    const char *force = getenv("MEAO_UPS_PERSIST_MIN_WAVES");
    const double min_waves = force ? atof(force) : 2.0;
    const bool persist = a.tile_ctr && ntiles >= (int)(min_waves * kWave);
    if (!persist) a.tile_ctr = nullptr;
    const dim3 grid(persist ? kWave : ntiles);
    const int t = use_tma ? 1 : 0;
    DepthIn din = din_in;           // zero pitches: the tight values
    if (!din.depth_pitch) din.depth_pitch = a.hiw;
    if (!din.depth_layer_pitch) din.depth_layer_pitch = (long long)din.depth_pitch * a.hih;
    if (!din.ao_layer_pitch) din.ao_layer_pitch = (long long)a.hih * a.out_pitch;
    if (din.in_format == IN_D16)       launch_lin<IN_D16>(lo_depth_map, lo_ao_map, lo_ao2_map, a, lo_ao2, lo_a2pitch, din, t, layers, grid, s);
    else if (din.in_format == IN_D24S8) launch_lin<IN_D24S8>(lo_depth_map, lo_ao_map, lo_ao2_map, a, lo_ao2, lo_a2pitch, din, t, layers, grid, s);
    else                                launch_lin<IN_F32>(lo_depth_map, lo_ao_map, lo_ao2_map, a, lo_ao2, lo_a2pitch, din, t, layers, grid, s);
    return cudaGetLastError();
}

#ifndef MEAO_EMULATE
cudaError_t preload_blur_upsample_lin()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(blur_upsample_lin_kernel<IN_F32>); t(blur_upsample_lin_kernel<IN_D16>); t(blur_upsample_lin_kernel<IN_D24S8>);
    t(blur_upsample_premin_lin_kernel<IN_F32>); t(blur_upsample_premin_lin_kernel<IN_D16>); t(blur_upsample_premin_lin_kernel<IN_D24S8>);
    t(blur_upsample_lin_layered_kernel<IN_F32>); t(blur_upsample_lin_layered_kernel<IN_D16>); t(blur_upsample_lin_layered_kernel<IN_D24S8>);
    t(blur_upsample_premin_lin_layered_kernel<IN_F32>); t(blur_upsample_premin_lin_layered_kernel<IN_D16>);
    t(blur_upsample_premin_lin_layered_kernel<IN_D24S8>);
    return e;
}
#endif

}  // namespace meao
