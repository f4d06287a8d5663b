// blur_upsample_array_batch.cu -- the final blur_upsample level of a batch over CUDA arrays (meao_render_arrays_batch): each tile stores
// its AO at the top-left corner of its layer's own 2-D array, entry l of the batch table (kernels.h BatchArrays, a kernel parameter).
// The kernel bodies are blur_upsample_array.cu's (blur_upsample_kernel.inc with MEAO_UPS_ARRAY 1 and MEAO_UPS_BATCH 1); everything but
// the surface of the stores is the existing code.  A translation unit of its own so that blur_upsample_array.cu compiles to exactly the
// code it did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_UPS_ARRAY 1
#define MEAO_UPS_BATCH 1
#include "blur_upsample_device.inc"
#include "blur_upsample_layer_args.inc"

#define MEAO_UPS_LAYERED 1
#define MEAO_UPS_PREMIN 0
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#define MEAO_UPS_PREMIN 1
#include "blur_upsample_kernel.inc"
#undef MEAO_UPS_PREMIN
#undef MEAO_UPS_LAYERED
#undef MEAO_UPS_BATCH
#undef MEAO_UPS_ARRAY

const struct {      // [upsample_slot]: the final level's slot only
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, int, BatchArrays> plain[kUpsampleSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, int, BatchArrays> premin[kUpsampleSlots];
} kKernels = {MEAO_UPSAMPLE_SLOTS(blur_upsample_array_batch_kernel, MEAO_NO_SLOT),
              MEAO_UPSAMPLE_SLOTS(blur_upsample_premin_array_batch_kernel, MEAO_NO_SLOT)};

}  // namespace

cudaError_t launch_blur_upsample_array_batch(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map,
                                             bool use_tma, const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count,
                                             const BatchArrays &ao, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxBatch) return cudaErrorInvalidValue;
    if (a_in.hi_ao || !a_in.hi_is_half || a_in.row0 != 0 || a_in.row1 != a_in.hih) return cudaErrorInvalidValue;     // the final level, whole frame
    UpsampleArgs a = a_in;
    a.out = nullptr; a.out_pitch = 0; a.out_row_origin = 0;
    a.out_vec_ok = 1;               // surface stores have no alignment requirement
    dim3 grid;
    if (!ups_tile_grid(a, layers, sm_count, &grid)) return cudaErrorInvalidValue;
    const int t = use_tma ? 1 : 0, k = upsample_slot(a);
    if (!lo_ao2) {
        MEAO_LAUNCH((kKernels.plain[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, ao);
    } else {        // main_premin
        if (!lo_ao2_map) return cudaErrorInvalidValue;
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        MEAO_LAUNCH((kKernels.premin[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, ao);
    }
    return cudaGetLastError();
}

const KernelUnit kBlurUpsampleArrayBatchUnit = {"blur_upsample_array_batch.cu",
                                                [](cudaError_t *load) { return walk_kernels(load, kKernels.plain, kKernels.premin); }};

}  // namespace meao
