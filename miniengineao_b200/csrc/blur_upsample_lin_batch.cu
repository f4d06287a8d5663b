// blur_upsample_lin_batch.cu -- the fused final blur_upsample level of a batch over device buffers (meao_render_batch): each tile reads
// the raw depth of its layer's own buffer, linearises it, writes LinearDepth and stores its AO into the layer's own AO buffer, each at
// its own row pitch: entry l of the batch table (kernels.h BatchPointers, a kernel parameter).  The kernel bodies are blur_upsample_lin.cu's
// layered ones (blur_upsample_kernel.inc with MEAO_UPS_LIN 1, MEAO_UPS_LAYERED 1 and MEAO_UPS_BATCH 1): only the bases and pitches of a
// layer's depth and AO and their vector-access tests differ.  A translation unit of its own so that blur_upsample_lin.cu compiles to
// exactly the code it did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#include "blur_upsample_device.inc"
#include "blur_upsample_layer_args.inc"
#include "depth_in.cuh"
#include "blur_upsample_lin_device.inc"

// The arguments of layer l with the layer's own AO buffer and row pitch.  The 64-bit stores need its base and row pitch 8-byte aligned
// (out_vec_ok); a misaligned layer stores byte by byte, with the same codes.  Read where the tile starts, not held from the prologue:
// the entry lives in the parameter bank.
__device__ __forceinline__ UpsampleArgs layer_args(const UpsampleArgs &a, int l, const BatchPointers &batch)
{
    UpsampleArgs r = layer_args(a, l);
    r.out = batch.e[l].ao;
    r.out_pitch = batch.e[l].ao_pitch;
    r.out_vec_ok = ((reinterpret_cast<uintptr_t>(r.out) | (uintptr_t)r.out_pitch) & 7) == 0;
    return r;
}
__device__ __forceinline__ UpsamplePreminArgs layer_args(const UpsamplePreminArgs &pa, int l, const BatchPointers &batch)
{
    UpsamplePreminArgs r = layer_args(pa, l);
    r.base.out = batch.e[l].ao;
    r.base.out_pitch = batch.e[l].ao_pitch;
    r.base.out_vec_ok = ((reinterpret_cast<uintptr_t>(r.base.out) | (uintptr_t)r.base.out_pitch) & 7) == 0;
    return r;
}
// din with layer l's own depth as a layer of pitch 0, so that linearize_pixels8 reads it; vec_ok: its base and row pitch (in bytes)
// 16-byte multiples
template <int IN>
__device__ __forceinline__ DepthIn batch_depth(const DepthIn &din, const BatchPointers &batch, int l)
{
    DepthIn r = din;
    r.depth = batch.e[l].depth;
    r.depth_pitch = batch.e[l].depth_pitch;
    r.depth_layer_pitch = 0;
    r.vec_ok = ((reinterpret_cast<uintptr_t>(r.depth) | (uintptr_t)r.depth_pitch * (IN == IN_D16 ? 2 : 4)) & 15) == 0;
    return r;
}

#define MEAO_UPS_LIN 1
#define MEAO_UPS_LAYERED 1
#define MEAO_UPS_BATCH 1
#define MEAO_UPS_PREMIN 0
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_PREMIN 1
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#undef MEAO_UPS_BATCH
#undef MEAO_UPS_LAYERED
#undef MEAO_UPS_LIN

const struct {      // [depth_format_slot]
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, int, DepthIn, BatchPointers> plain[kDepthFormatSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, int, DepthIn, BatchPointers> premin[kDepthFormatSlots];
} kKernels = {MEAO_LIN_SLOTS(blur_upsample_lin_batch_kernel), MEAO_LIN_SLOTS(blur_upsample_premin_lin_batch_kernel)};

}  // namespace

cudaError_t launch_blur_upsample_lin_batch(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                           const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din_in, int layers,
                                           int sm_count, const BatchPointers &io, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxBatch) return cudaErrorInvalidValue;
    if (!a_in.hi_is_half || a_in.hi_ao || (lo_ao2 && !lo_ao2_map)) return cudaErrorInvalidValue;      // the final level only
    if (a_in.row0 != 0 || a_in.row1 != a_in.hih || din_in.depth_row0 != 0) return cudaErrorInvalidValue;     // the whole frame
    UpsampleArgs a = a_in;
    a.out = nullptr; a.out_pitch = 0; a.out_row_origin = 0; a.out_vec_ok = 0;      // each layer's come from its entry
    DepthIn din = din_in;
    din.depth = nullptr; din.depth_pitch = 0; din.depth_layer_pitch = 0; din.ao_layer_pitch = 0; din.vec_ok = 0;
    dim3 grid;
    if (!ups_tile_grid(a, layers, sm_count, &grid)) return cudaErrorInvalidValue;
    const int t = use_tma ? 1 : 0, k = depth_format_slot(din.in_format);
    if (!lo_ao2) {
        MEAO_LAUNCH((kKernels.plain[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, din, io);
    } else {
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        MEAO_LAUNCH((kKernels.premin[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, din, io);
    }
    return cudaGetLastError();
}

const KernelUnit kBlurUpsampleLinBatchUnit = {"blur_upsample_lin_batch.cu",
                                              [](cudaError_t *load) { return walk_kernels(load, kKernels.plain, kKernels.premin); }};

}  // namespace meao
