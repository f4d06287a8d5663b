// blur_upsample_lin_views.cu -- the fused final blur_upsample level of a layered pointer frame with a layer-viewport table
// (meao_set_layer_viewports): each tile reads the raw depth of its layer's rectangle (kernels.h LayerView) in the caller's pitched
// depth, linearises it, writes LinearDepth and stores its AO into the layer's rectangle of the caller's pitched AO.  The kernel bodies
// are blur_upsample_lin.cu's layered ones (blur_upsample_kernel.inc with MEAO_UPS_LIN 1, MEAO_UPS_LAYERED 1 and MEAO_UPS_VIEWS 1): only
// the bases of a layer's depth and AO and their vector-access tests differ.  A translation unit of its own so that
// blur_upsample_lin.cu compiles to exactly the code it did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#include "blur_upsample_device.inc"
#include "blur_upsample_layer_args.inc"
#include "depth_in.cuh"
#include "blur_upsample_lin_device.inc"

// The arguments of layer l with the caller's AO at the layer's rectangle: slice ao_slice (ao_layer_pitch bytes each), row ao_y, column
// ao_x.  The 64-bit stores need the host's rows test (a.out_vec_ok: out_pitch % 8 == 0) and this layer's base; a misaligned layer
// stores byte by byte, with the same codes.
__device__ __forceinline__ uint8_t *view_out(const UpsampleArgs &a, long long ao_layer_pitch, const LayerView *v)
{
    return a.out + (long long)__ldg(&v->ao_slice) * ao_layer_pitch + (long long)__ldg(&v->ao_y) * a.out_pitch + __ldg(&v->ao_x);
}
__device__ __forceinline__ UpsampleArgs layer_args(const UpsampleArgs &a, int l, long long ao_layer_pitch, const LayerView *views)
{
    UpsampleArgs r = layer_args(a, l);
    r.out = view_out(a, ao_layer_pitch, views + l);
    r.out_vec_ok = a.out_vec_ok && (reinterpret_cast<uintptr_t>(r.out) & 7) == 0;
    return r;
}
__device__ __forceinline__ UpsamplePreminArgs layer_args(const UpsamplePreminArgs &pa, int l, long long ao_layer_pitch, const LayerView *views)
{
    UpsamplePreminArgs r = layer_args(pa, l);
    r.base.out = view_out(pa.base, ao_layer_pitch, views + l);
    r.base.out_vec_ok = pa.base.out_vec_ok && (reinterpret_cast<uintptr_t>(r.base.out) & 7) == 0;
    return r;
}
// din with layer l's depth as a layer of pitch 0 at its rectangle (slice depth_slice, row depth_y, column depth_x, in elements), so
// that linearize_pixels8 reads the rectangle; vec_ok: the host's rows test (depth row pitch % 16 == 0) and this layer's base
template <int IN>
__device__ __forceinline__ DepthIn view_depth(const DepthIn &din, const LayerView *views, int l)
{
    DepthIn r = din;
    const LayerView *v = views + l;
    r.depth = reinterpret_cast<const char *>(din.depth) + ((long long)__ldg(&v->depth_slice) * din.depth_layer_pitch +
              (long long)__ldg(&v->depth_y) * din.depth_pitch + __ldg(&v->depth_x)) * (IN == IN_D16 ? 2 : 4);
    r.depth_layer_pitch = 0;
    r.vec_ok = din.vec_ok && (reinterpret_cast<uintptr_t>(r.depth) & 15) == 0;
    return r;
}

#define MEAO_UPS_LIN 1
#define MEAO_UPS_LAYERED 1
#define MEAO_UPS_VIEWS 1
#define MEAO_UPS_PREMIN 0
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_PREMIN 1
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#undef MEAO_UPS_VIEWS
#undef MEAO_UPS_LAYERED
#undef MEAO_UPS_LIN

const struct {      // [depth_format_slot]
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, int, DepthIn, const LayerView *> plain[kDepthFormatSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, int, DepthIn, const LayerView *> premin[kDepthFormatSlots];
} kKernels = {MEAO_LIN_SLOTS(blur_upsample_lin_views_kernel), MEAO_LIN_SLOTS(blur_upsample_premin_lin_views_kernel)};

}  // namespace

cudaError_t launch_blur_upsample_lin_views(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                           const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din, int layers,
                                           int sm_count, const LayerView *views, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || !views) return cudaErrorInvalidValue;
    if (!a_in.hi_is_half || a_in.hi_ao || (lo_ao2 && !lo_ao2_map)) return cudaErrorInvalidValue;      // the final level only
    if (!din.depth_pitch) return cudaErrorInvalidValue;    // the caller's pitches, always explicit here
    UpsampleArgs a = a_in;
    dim3 grid;
    if (!ups_tile_grid(a, layers, sm_count, &grid)) return cudaErrorInvalidValue;
    const int t = use_tma ? 1 : 0, k = depth_format_slot(din.in_format);
    if (!lo_ao2) {
        MEAO_LAUNCH((kKernels.plain[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, din, views);
    } else {
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        MEAO_LAUNCH((kKernels.premin[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, din, views);
    }
    return cudaGetLastError();
}

const KernelUnit kBlurUpsampleLinViewsUnit = {"blur_upsample_lin_views.cu",
                                              [](cudaError_t *load) { return walk_kernels(load, kKernels.plain, kKernels.premin); }};

}  // namespace meao
