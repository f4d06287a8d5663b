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

}  // namespace

cudaError_t launch_blur_upsample_layered(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                         const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    UpsampleArgs a = a_in;
    const int ybase = a.row0 & ~1;
    a.tiles_x = ceil_div(a.hiw, kHW); a.tiles_y = ceil_div(a.row1 - ybase, kHH);
    const long long ntiles_ll = (long long)a.tiles_x * a.tiles_y * layers;
    if (ntiles_ll > 0x7fffffffLL) return cudaErrorInvalidValue;        // the tile index is a 32-bit int
    const int ntiles = (int)ntiles_ll;
    // the same rule as launch_blur_upsample, on the tiles of ALL layers: the persistent tile loop from two tiles per CTA slot
    const int kWave = sm_count * MEAO_UPS_MINB;
    const char *force = getenv("MEAO_UPS_PERSIST_MIN_WAVES");
    const double min_waves = force ? atof(force) : 2.0;
    const bool persist = a.tile_ctr && ntiles >= (int)(min_waves * kWave);
    if (!persist) a.tile_ctr = nullptr;
    dim3 grid(persist ? kWave : ntiles);
    const int t = use_tma ? 1 : 0;
    if (!lo_ao2) {
        if (a.hi_ao) {
            if (a.hi_is_half) MEAO_LAUNCH((blur_upsample_layered_kernel<true, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers);
            else              MEAO_LAUNCH((blur_upsample_layered_kernel<true, false>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers);
        } else {
            if (a.hi_is_half) MEAO_LAUNCH((blur_upsample_layered_kernel<false, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers);
            else              MEAO_LAUNCH((blur_upsample_layered_kernel<false, false>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers);
        }
    } else {        // main_premin / main_premin_blendout
        if (!lo_ao2_map) return cudaErrorInvalidValue;
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        if (a.hi_ao) {
            if (a.hi_is_half) MEAO_LAUNCH((blur_upsample_premin_layered_kernel<true, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers);
            else              MEAO_LAUNCH((blur_upsample_premin_layered_kernel<true, false>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers);
        } else {
            if (a.hi_is_half) MEAO_LAUNCH((blur_upsample_premin_layered_kernel<false, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers);
            else              MEAO_LAUNCH((blur_upsample_premin_layered_kernel<false, false>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers);
        }
    }
    return cudaGetLastError();
}

#ifndef MEAO_EMULATE
cudaError_t preload_blur_upsample_layered()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(blur_upsample_layered_kernel<true, true>); t(blur_upsample_layered_kernel<true, false>);
    t(blur_upsample_layered_kernel<false, true>); t(blur_upsample_layered_kernel<false, false>);
    t(blur_upsample_premin_layered_kernel<true, true>); t(blur_upsample_premin_layered_kernel<true, false>);
    t(blur_upsample_premin_layered_kernel<false, true>); t(blur_upsample_premin_layered_kernel<false, false>);
    return e;
}
#endif

}  // namespace meao
