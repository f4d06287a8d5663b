// array_driver.cpp -- runs one CUDA-ARRAY frame (meao_render_arrays) through the host-compiled kernel sources (TEST INFRASTRUCTURE
// ONLY, see cuda_emu.h).  The depth is read from, and the AO written into, emulated arrays through emulated surface objects (2-D,
// layered or cube), by the kernels of prepare_depth_array.cu and blur_upsample_array.cu; the render levels and the coarse upsamples
// are the layered kernels on the arena, as meao_api.cu records them.  The arena, the constants and the other launches are
// layered_driver.cpp's (included: one frame layout for both drivers).
#include "layered_driver.cpp"

namespace meao_emu { long long surface_accesses = 0; }

namespace {

// what meao_api.cu check_array derives from an array: how the kernels address its layers
int surf_kind_of(int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : shape == meao_emu::SURF_LAYERED ? kSurfLayered : kSurfCube; }

void run_downsample_array(LEmu *e, const meao_emu::Surface *depth, int in_format)
{
    PrepareArgs a{};
    a.in_format = in_format; a.W = e->W; a.H = e->H; a.depth_row0 = 0; a.row0 = 0; a.row1 = e->H;
    a.lin = e->lin; a.lin_pitch = e->lin_pitch;
    for (int k = 1; k <= 4; k++) { a.low[k - 1] = e->low[k]; a.low_pitch[k - 1] = e->low_pitch[k]; }
    a.zbx = e->zbx; a.zby = e->zby; a.raw = e->raw; a.reversed_z = e->reversed_z;
    launch_prepare_depth_array(a, (cudaSurfaceObject_t)depth, surf_kind_of(depth->shape), e->L, nullptr);
}

// run_upsample(e, 1) with the AO stored into the array
void run_final_upsample_array(LEmu *e, const meao_emu::Surface *ao)
{
    UpsampleArgs a{};
    a.lo_depth = e->low[1]; a.low = e->lw[1]; a.loh = e->lh[1]; a.lo_dpitch = e->low_pitch[1];
    a.lo_ao = e->single_scale ? e->occ[1] : e->comb[1]; a.lo_apitch = e->occ_pitch[1];
    a.hi_depth = e->lin; a.hi_is_half = 1; a.hi_dpitch = e->lin_pitch; a.hi_ao = nullptr; a.hi_apitch = 0;
    a.hiw = e->lw[0]; a.hih = e->lh[0];
    a.noise_filter_strength = e->nfs[1]; a.step_size = e->step[1]; a.blur_tolerance = e->kblur[1]; a.upsample_tolerance = e->tol[1];
    a.fast_div_ok = upsample_fast_div_ok(a.upsample_tolerance, a.noise_filter_strength);
    a.row0 = 0; a.row1 = e->lh[0];
    a.tile_ctr = e->tile_ctr;
    const bool premin = (e->hq_mask & 1) != 0;
    const int rows = e->L * e->lh[1];
    const CUtensorMap md = make_map(e->low[1], 4, e->lw[1], rows, e->low_pitch[1], kUpsDepthBoxW, kUpsDepthBoxH);
    const CUtensorMap ma = make_map(a.lo_ao, 1, e->lw[1], rows, e->occ_pitch[1], kUpsAoBoxW, kUpsAoBoxH);
    const CUtensorMap mh = make_map(e->hq[1], 1, e->lw[1], rows, e->occ_pitch[1], kUpsAoBoxW, kUpsAoBoxH);
    launch_blur_upsample_array(md, ma, &mh, e->use_tma != 0, a, premin ? e->hq[1] : nullptr, e->occ_pitch[1], e->L, e->sm_count,
                               (cudaSurfaceObject_t)ao, surf_kind_of(ao->shape), nullptr);
}

}  // namespace

extern "C" {

// depth: `layers` images of W x H elements (4 bytes: f32, 2 bytes: D16 codes) with rows depth_pitch bytes apart, in an emulated array of
// shape depth_shape (0 2-D, 1 layered, 2 cube); ao: the same for the AO (1 byte per pixel).  The pitches are chosen by the test, wider
// than a row, so a kernel that ignored the array's own addressing would read or write the wrong bytes.
void aemu_run(void *h, void *depth, int in_format, int depth_shape, long long depth_pitch, void *ao, int ao_shape, long long ao_pitch)
{
    LEmu *e = (LEmu *)h;
    const meao_emu::Surface ds{depth, in_format == 1 ? 2 : 4, e->W, e->H, depth_shape == 2 ? 6 : e->L, (size_t)depth_pitch, depth_shape};
    const meao_emu::Surface as{ao, 1, e->W, e->H, ao_shape == 2 ? 6 : e->L, (size_t)ao_pitch, ao_shape};
    run_downsample_array(e, &ds, in_format);
    if (e->single_scale) { run_render(e, 1, false); run_final_upsample_array(e, &as); return; }     // record_frame_dag, single_scale branch
    for (int k = 1; k <= 4; k++) run_render(e, k, false);
    for (int k = 1; k <= 4; k++) if ((e->hq_mask >> (k - 1)) & 1) run_render(e, k, true);
    for (int lo = 4; lo >= 2; lo--) run_upsample(e, lo);
    run_final_upsample_array(e, &as);
}

long long aemu_surface_accesses() { return meao_emu::surface_accesses; }

}  // extern "C"
