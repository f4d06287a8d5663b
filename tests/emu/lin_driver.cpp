// lin_driver.cpp -- runs a frame in its fused form through the host-compiled kernel sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h):
// prepare_depth low-only (LowDepth1..4 from the even rows, no LinearDepth) and the final blur_upsample reading the raw depth and writing
// LinearDepth (blur_upsample_lin.cu), as meao_api.cu's record_frame_dag records a whole frame.  The arena, the constants, the renders
// and the coarse upsamples are layered_driver.cpp's (included: one translation unit); one layer takes the single-image prepare_depth and
// final-upsample kernels, L > 1 the layered ones, and a row band [row0, row1) runs the single-image kernels on those rows only.
#include "layered_driver.cpp"

namespace {

PrepareArgs prepare_args(LEmu *e, const void *depth, int in_format, int row0, int row1)
{
    PrepareArgs a{};
    a.depth = depth; a.in_format = in_format; a.W = e->W; a.H = e->H; a.depth_row0 = row0; a.row0 = row0; a.row1 = row1;
    a.lin = e->lin; a.lin_pitch = e->lin_pitch;
    for (int k = 1; k <= 4; k++) { a.low[k - 1] = e->low[k]; a.low_pitch[k - 1] = e->low_pitch[k]; }
    a.zbx = e->zbx; a.zby = e->zby; a.raw = e->raw; a.reversed_z = e->reversed_z;
    a.vec_ok = (((uintptr_t)depth & 15) == 0) && (e->W % (in_format == 1 ? 8 : 4) == 0);
    return a;
}

void run_prepare_low(LEmu *e, const void *depth, int in_format, int row0, int row1)
{
    const PrepareArgs a = prepare_args(e, depth, in_format, row0, row1);
    if (e->L == 1) launch_prepare_depth(a, nullptr, true);
    else launch_prepare_depth_layered(a, e->L, nullptr, true);
}

// run_upsample(e, 1) with the raw depth: rows [row0, row1) of the final level
void run_upsample_lin(LEmu *e, const void *depth, int in_format, int row0, int row1)
{
    const PrepareArgs p = prepare_args(e, depth, in_format, row0, row1);
    DepthIn din{};
    din.depth = depth; din.in_format = in_format; din.depth_row0 = row0; din.zbx = p.zbx; din.zby = p.zby;
    din.raw = p.raw; din.reversed_z = p.reversed_z; din.vec_ok = p.vec_ok;
    UpsampleArgs a{};
    a.lo_depth = e->low[1]; a.low = e->lw[1]; a.loh = e->lh[1]; a.lo_dpitch = e->low_pitch[1];
    a.lo_ao = e->single_scale ? e->occ[1] : e->comb[1]; a.lo_apitch = e->occ_pitch[1];
    a.hi_depth = e->lin; a.hi_is_half = 1; a.hi_dpitch = e->lin_pitch; a.hi_ao = nullptr; a.hi_apitch = 0;
    a.out = e->result; a.out_pitch = e->result_pitch; a.out_row_origin = 0; a.out_vec_ok = 1;
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

// LinearDepth of every layer := NaN (f16 0x7e00)
void femu_poison_lin(void *h)
{
    LEmu *e = (LEmu *)h;
    const uint16_t nan = 0x7e00;
    for (size_t i = 0, n = (size_t)e->L * e->lin_pitch * e->H; i < n; i++) memcpy(&e->lin[i], &nan, 2);
}

// the low-only prepare_depth alone, whole frame
void femu_prepare_low(void *h, const void *depth, int in_format)
{
    LEmu *e = (LEmu *)h;
    run_prepare_low(e, depth, in_format, 0, e->H);
}

// one fused frame.  row1 > row0: only the final level's rows [row0, row1) take the fused kernel (single layer; row0 % 16 == 0),
// the other levels of the frame are whole -- what the rows of one band compute once its LowDepth halo rows have arrived
void femu_run(void *h, const void *depth, int in_format, int row0, int row1)
{
    LEmu *e = (LEmu *)h;
    const bool band = row1 > row0;
    if (!band) { row0 = 0; row1 = e->H; }
    const void *band_depth = (const char *)depth + (size_t)row0 * e->W * (in_format == 1 ? 2 : 4);
    if (band) run_downsample(e, depth, in_format);             // LowDepth1..4 of the whole frame (the band's halo included)
    else run_prepare_low(e, depth, in_format, 0, e->H);
    if (e->single_scale) { run_render(e, 1, false); run_upsample_lin(e, band_depth, in_format, row0, row1); return; }
    for (int k = 1; k <= 4; k++) run_render(e, k, false);
    for (int k = 1; k <= 4; k++) if ((e->hq_mask >> (k - 1)) & 1) run_render(e, k, true);
    for (int lo = 4; lo >= 2; lo--) run_upsample(e, lo);
    run_upsample_lin(e, band_depth, in_format, row0, row1);
}

}  // extern "C"
