// pitched_driver.cpp -- runs a fused frame (lin_driver.cpp) whose depth and AO are VIEWS with their own row and layer pitch, through
// the host-compiled kernel sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h), with the argument blocks filled the way meao_api.cu's
// recorders fill them for meao_render_pitched: PrepareArgs / DepthIn carry the depth pitches (elements) and DepthIn the AO layer pitch,
// UpsampleArgs.out_pitch the AO row pitch, and the vector-path flags follow the pitched rules.  All four pitches 0: the new fields stay
// zero, as in the drivers written before them (the launchers then use the tight values).
#include "lin_driver.cpp"

namespace {

struct Pitch { long long depth_row, depth_layer, ao_row, ao_layer; };      // bytes

bool zero_pitch(const Pitch &p) { return !p.depth_row && !p.depth_layer && !p.ao_row && !p.ao_layer; }

PrepareArgs pitched_prepare_args(LEmu *e, const void *depth, int in_format, int row0, int row1, const Pitch &p)
{
    PrepareArgs a = prepare_args(e, depth, in_format, row0, row1);     // tight vec_ok, zero pitches
    if (zero_pitch(p)) return a;
    const int es = in_format == 1 ? 2 : 4;
    a.depth_pitch = (int)(p.depth_row / es);
    a.depth_layer_pitch = p.depth_layer / es;
    a.vec_ok = (((uintptr_t)depth & 15) == 0) && (p.depth_row % 16 == 0) && (e->L == 1 || p.depth_layer % 16 == 0);
    return a;
}

// the final level, rows [row0, row1), reading the raw depth view (its row row0 at `depth`) and storing into the AO view (its row row0 at `ao`)
void run_upsample_pitched(LEmu *e, const void *depth, int in_format, int row0, int row1, uint8_t *ao, const Pitch &p)
{
    const PrepareArgs pa = pitched_prepare_args(e, depth, in_format, row0, row1, p);
    DepthIn din{};
    din.depth = depth; din.in_format = in_format; din.depth_row0 = row0; din.zbx = pa.zbx; din.zby = pa.zby;
    din.raw = pa.raw; din.reversed_z = pa.reversed_z; din.vec_ok = pa.vec_ok;
    din.depth_pitch = pa.depth_pitch; din.depth_layer_pitch = pa.depth_layer_pitch; din.ao_layer_pitch = p.ao_layer;
    UpsampleArgs a{};
    a.lo_depth = e->low[1]; a.low = e->lw[1]; a.loh = e->lh[1]; a.lo_dpitch = e->low_pitch[1];
    a.lo_ao = e->single_scale ? e->occ[1] : e->comb[1]; a.lo_apitch = e->occ_pitch[1];
    a.hi_depth = e->lin; a.hi_is_half = 1; a.hi_dpitch = e->lin_pitch; a.hi_ao = nullptr; a.hi_apitch = 0;
    a.out = ao; a.out_pitch = p.ao_row ? (int)p.ao_row : e->W; a.out_row_origin = row0;
    a.out_vec_ok = (((uintptr_t)ao & 7) == 0) && (a.out_pitch % 8 == 0) && (e->L == 1 || (p.ao_layer ? p.ao_layer : (long long)e->H * a.out_pitch) % 8 == 0);
    a.hiw = e->lw[0]; a.hih = e->lh[0];
    a.noise_filter_strength = e->nfs[1]; a.step_size = e->step[1]; a.blur_tolerance = e->kblur[1]; a.upsample_tolerance = e->tol[1];
    a.fast_div_ok = upsample_fast_div_ok(a.upsample_tolerance, a.noise_filter_strength);
    a.row0 = row0; a.row1 = row1;
    a.tile_ctr = e->tile_ctr;
    const bool premin = (e->hq_mask & 1) != 0;
    const int rows = e->L * e->lh[1];
    const CUtensorMap md = make_map(e->low[1], 4, e->lw[1], rows, e->low_pitch[1], kUpsDepthBoxW, kUpsDepthBoxH);
    const CUtensorMap ma = make_map(a.lo_ao, 1, e->lw[1], rows, e->occ_pitch[1], kUpsAoBoxW, kUpsAoBoxH);
    const CUtensorMap mh = make_map(e->hq[1], 1, e->lw[1], rows, e->occ_pitch[1], kUpsAoBoxW, kUpsAoBoxH);
    launch_blur_upsample_lin(md, ma, &mh, e->use_tma != 0, a, premin ? e->hq[1] : nullptr, e->occ_pitch[1], din, e->L, e->sm_count, nullptr);
}

}  // namespace

extern "C" {

// One fused frame from the depth view at `depth` into the AO view at `ao` (pitches in bytes; all 0: zero pitches in the argument
// blocks, tight views).  row1 > row0: a row band, as femu_run -- prepare_depth runs in its full form over the whole depth view
// (LowDepth1..4 with the band's halo), and the final level's rows [row0, row1) read the depth view from its row row0 on and store
// into `ao`, the band's AO view (its first row is row0).
void pemu_run(void *h, const void *depth, int in_format, long long depth_row, long long depth_layer, uint8_t *ao, long long ao_row,
              long long ao_layer, int row0, int row1)
{
    LEmu *e = (LEmu *)h;
    const Pitch p{depth_row, depth_layer, ao_row, ao_layer};
    const bool band = row1 > row0;
    if (!band) { row0 = 0; row1 = e->H; }
    const long long row_bytes = depth_row ? depth_row : (long long)e->W * (in_format == 1 ? 2 : 4);
    const void *band_depth = (const char *)depth + (size_t)row0 * row_bytes;
    const PrepareArgs a = pitched_prepare_args(e, depth, in_format, 0, e->H, p);
    if (e->L == 1) launch_prepare_depth(a, nullptr, !band);
    else launch_prepare_depth_layered(a, e->L, nullptr, !band);
    if (e->single_scale) { run_render(e, 1, false); run_upsample_pitched(e, band_depth, in_format, row0, row1, ao, p); return; }
    for (int k = 1; k <= 4; k++) run_render(e, k, false);
    for (int k = 1; k <= 4; k++) if ((e->hq_mask >> (k - 1)) & 1) run_render(e, k, true);
    for (int lo = 4; lo >= 2; lo--) run_upsample(e, lo);
    run_upsample_pitched(e, band_depth, in_format, row0, row1, ao, p);
}

}  // extern "C"
