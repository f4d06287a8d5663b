// blur_upsample_array.cu -- the final blur_upsample level (Upsample.compute main / main_premin, LinearDepth as HiResDB, no hi-res
// AO) with the AO written into a CUDA array (meao_render_arrays): a 2-D, layered or cube-map array of L layers, one launch.  The
// kernel bodies are blur_upsample.cu's in their layered tile-loop form (blur_upsample_kernel.inc with MEAO_UPS_LAYERED 1 and
// MEAO_UPS_ARRAY 1): the 64-bit store of the fast path and the stores of upsample8_slow become one-byte surface stores at
// (x, y, layer) (surface_io.cuh); everything else, including every read of the intermediates, is the existing code.  The coarse
// levels run the existing kernels on the context's arena.  A translation unit of its own so that blur_upsample.cu and
// blur_upsample_layered.cu compile to exactly the code they did before.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_UPS_ARRAY 1
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
#undef MEAO_UPS_ARRAY

}  // namespace

cudaError_t launch_blur_upsample_array(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                       const UpsampleArgs &a_in, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count,
                                       cudaSurfaceObject_t out, int surf_kind, cudaStream_t s)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    if (a_in.hi_ao || !a_in.hi_is_half || a_in.row0 != 0 || a_in.row1 != a_in.hih) return cudaErrorInvalidValue;     // the final level, whole frame
    UpsampleArgs a = a_in;
    a.out = nullptr; a.out_pitch = 0; a.out_row_origin = 0;
    a.out_vec_ok = 1;               // surface stores have no alignment requirement
    const int ybase = a.row0 & ~1;
    a.tiles_x = ceil_div(a.hiw, kHW); a.tiles_y = ceil_div(a.row1 - ybase, kHH);
    const long long ntiles_ll = (long long)a.tiles_x * a.tiles_y * layers;
    if (ntiles_ll > 0x7fffffffLL) return cudaErrorInvalidValue;        // the tile index is a 32-bit int
    const int ntiles = (int)ntiles_ll;
    // the rule of launch_blur_upsample(_layered), on the tiles of all layers: the persistent tile loop from two tiles per CTA slot
    const int kWave = sm_count * MEAO_UPS_MINB;
    const char *force = getenv("MEAO_UPS_PERSIST_MIN_WAVES");
    const double min_waves = force ? atof(force) : 2.0;
    const bool persist = a.tile_ctr && ntiles >= (int)(min_waves * kWave);
    if (!persist) a.tile_ctr = nullptr;
    dim3 grid(persist ? kWave : ntiles);
    const int t = use_tma ? 1 : 0;
    if (!lo_ao2) {
        MEAO_LAUNCH((blur_upsample_array_kernel<false, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, a, t, layers, out, surf_kind);
    } else {        // main_premin
        if (!lo_ao2_map) return cudaErrorInvalidValue;
        const UpsamplePreminArgs pa{a, lo_ao2, lo_a2pitch};
        MEAO_LAUNCH((blur_upsample_premin_array_kernel<false, true>), grid, kThreads, 0, s, lo_depth_map, lo_ao_map, *lo_ao2_map, pa, t, layers, out, surf_kind);
    }
    return cudaGetLastError();
}

#ifndef MEAO_EMULATE
cudaError_t preload_blur_upsample_array()
{
    cudaError_t e = cudaSuccess;
    auto t = [&](auto k) { if (e == cudaSuccess) e = preload_kernel(k); };
    t(blur_upsample_array_kernel<false, true>); t(blur_upsample_premin_array_kernel<false, true>);
    return e;
}
#endif

}  // namespace meao
