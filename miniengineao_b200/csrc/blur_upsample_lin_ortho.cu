// blur_upsample_lin_ortho.cu -- blur_upsample_lin.cu's kernels (the fused final upsample that linearises the caller's raw depth) under
// an orthographic projection (meao_set_projection): the same bodies with MEAO_ORTHO 1, whose linearize8 (depth_in.cuh) is the affine
// one.  The upsample itself works on the stored linear depth and does not depend on the projection; linear ingest stays with
// blur_upsample_lin.cu's kernels.  A translation unit of its own (build.py ORTHO_SOURCES).
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 1
#include "blur_upsample_device.inc"
#include "blur_upsample_layer_args.inc"
#include "depth_in.cuh"

#include "blur_upsample_lin_device.inc"

#define blur_upsample_lin_kernel blur_upsample_lin_ortho_kernel              // the names of the orthographic instantiations
#define blur_upsample_premin_lin_kernel blur_upsample_premin_lin_ortho_kernel
#define blur_upsample_lin_layered_kernel blur_upsample_lin_ortho_layered_kernel
#define blur_upsample_premin_lin_layered_kernel blur_upsample_premin_lin_ortho_layered_kernel
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
#undef blur_upsample_premin_lin_layered_kernel
#undef blur_upsample_lin_layered_kernel
#undef blur_upsample_premin_lin_kernel
#undef blur_upsample_lin_kernel
#undef MEAO_ORTHO

const struct {      // [depth_format_slot]
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, DepthIn> plain[kDepthFormatSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, DepthIn> premin[kDepthFormatSlots];
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, int, DepthIn> layered[kDepthFormatSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, int, DepthIn> premin_layered[kDepthFormatSlots];
} kKernels = {MEAO_LIN_SLOTS(blur_upsample_lin_ortho_kernel), MEAO_LIN_SLOTS(blur_upsample_premin_lin_ortho_kernel),
              MEAO_LIN_SLOTS(blur_upsample_lin_ortho_layered_kernel), MEAO_LIN_SLOTS(blur_upsample_premin_lin_ortho_layered_kernel)};

}  // namespace

cudaError_t launch_blur_upsample_lin_ortho(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                           const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din_in, int layers,
                                           int sm_count, cudaStream_t s, bool layered)
{
    if (!din_in.raw)
        return launch_blur_upsample_lin(lo_depth_map, lo_ao_map, lo_ao2_map, use_tma, a_in, lo_ao2, lo_a2pitch, din_in, layers, sm_count, s, layered);
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    if (!a_in.hi_is_half || a_in.hi_ao || (lo_ao2 && !lo_ao2_map)) return cudaErrorInvalidValue;      // the final level only
    UpsampleArgs a = a_in;
    dim3 grid;
    if (!ups_tile_grid(a, layers, sm_count, &grid)) return cudaErrorInvalidValue;
    const int t = use_tma ? 1 : 0;
    DepthIn din = din_in;           // zero pitches: the tight values
    if (!din.depth_pitch) din.depth_pitch = a.hiw;
    if (!din.depth_layer_pitch) din.depth_layer_pitch = (long long)din.depth_pitch * a.hih;
    if (!din.ao_layer_pitch) din.ao_layer_pitch = (long long)a.hih * a.out_pitch;
    const int k = depth_format_slot(din.in_format);
    const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
    if (layers == 1 && !layered) {
        if (!lo_ao2) MEAO_LAUNCH((kKernels.plain[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, din);
        else         MEAO_LAUNCH((kKernels.premin[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, din);
    } else {
        if (!lo_ao2) MEAO_LAUNCH((kKernels.layered[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, din);
        else         MEAO_LAUNCH((kKernels.premin_layered[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, din);
    }
    return cudaGetLastError();
}

const KernelUnit kBlurUpsampleLinOrthoUnit = {"blur_upsample_lin_ortho.cu", [](cudaError_t *load) {
    return walk_kernels(load, kKernels.plain, kKernels.premin, kKernels.layered, kKernels.premin_layered);
}};

}  // namespace meao
