// blur_upsample_layered.cu -- stage 3 for a layered frame (meao_set_layers): one launch blurs and upsamples one level of all
// L layers.  The kernel bodies are blur_upsample.cu's (blur_upsample_kernel.inc with MEAO_UPS_LAYERED 1): the tile index runs
// over tiles_x x tiles_y x L tiles, layer-major, and each tile reads and writes the images of its own layer (kernels.h "layered
// frames").  A translation unit of its own so that blur_upsample.cu compiles to exactly the code it did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

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

const struct {      // [upsample_slot]
    Kernel<CUtensorMap, CUtensorMap, UpsampleArgs, int, int> plain[kUpsampleSlots];
    Kernel<CUtensorMap, CUtensorMap, CUtensorMap, UpsamplePreminArgs, int, int> premin[kUpsampleSlots];
} kKernels = {MEAO_UPSAMPLE_SLOTS(blur_upsample_layered_kernel, MEAO_SLOT), MEAO_UPSAMPLE_SLOTS(blur_upsample_premin_layered_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_blur_upsample_layered(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                         const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    UpsampleArgs a = a_in;
    dim3 grid;
    if (!ups_tile_grid(a, layers, sm_count, &grid)) return cudaErrorInvalidValue;
    const int t = use_tma ? 1 : 0, k = upsample_slot(a);
    if (!kKernels.plain[k]) return cudaErrorInvalidValue;          // a blend / hi-res depth pairing upsample_args never makes
    if (!lo_ao2) {
        MEAO_LAUNCH((kKernels.plain[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers);
    } else {        // main_premin / main_premin_blendout
        if (!lo_ao2_map) return cudaErrorInvalidValue;
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        MEAO_LAUNCH((kKernels.premin[k]), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers);
    }
    return cudaGetLastError();
}

const KernelUnit kBlurUpsampleLayeredUnit = {"blur_upsample_layered.cu",
                                             [](cudaError_t *load) { return walk_kernels(load, kKernels.plain, kKernels.premin); }};

}  // namespace meao
