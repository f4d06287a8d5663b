// layer_cameras_driver.cpp -- runs one LAYERED frame with PER-LAYER CAMERAS (meao_set_layer_cameras) through the host-compiled kernel
// sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  layered_driver.cpp's buffers and argument blocks, plus the per-layer tables
// (kernels.h LayerZ / LayerRender) filled from each layer's constants -- read by the test from a plan-only libmeao context through
// meao_render_constants_layer / meao_zbuffer_params_layer -- and handed to the kernels the way meao_api.cu's recorders do.  A frame
// runs either the whole-frame form (low-only prepare_depth + the fused final upsample that linearises the raw depth, optionally
// from a pitched depth view and into a pitched AO view) or the pair prepare_depth -> LinearDepth -> layered upsample.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/kernels.h"

using namespace meao;

namespace {

inline int align_up(int x, int a) { return (x + a - 1) / a * a; }
template <class T> T *alloc(size_t n) { void *p = nullptr; if (posix_memalign(&p, 256, (n * sizeof(T) + 255) / 256 * 256 + 256)) abort(); memset(p, 0, n * sizeof(T)); return (T *)p; }

struct LEmu {
    int W, H, L, lw[7], lh[7];
    __half *lin; int lin_pitch;
    float *low[5]; int low_pitch[5];
    uint8_t *occ[5], *comb[4], *hq[5]; int occ_pitch[5];
    uint8_t *result; int result_pitch;
    float zbx = 0, zby = 1; int raw = 1, reversed_z = 1;
    float inv_thickness[5][12], inv_thickness_wide[5][12], sample_weight[5][12];
    float reject_fadeoff = -1, intensity = 1, pad[5] = {0, 0, 0, 0, 0};
    float nfs[5], step[5], kblur[5], tol[5];
    int hq_mask = 0, exhaustive = 0, single_scale = 0;
    int use_tma = 1;        // 1: interior tiles take the kernels' TMA path (emulated box loads), 0: every tile gathers
    int sm_count = 132;     // SMs of the device the planner's rules are evaluated for (an H100 SXM)
    uint32_t tile_ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // per-layer cameras: layer_zb[l], layer_ren[(2 (k - 1) + wide) L + l], layer_pad12[l] (meao_api.cu upload_camera_tables)
    std::vector<LayerZ> layer_zb;
    std::vector<LayerRender> layer_ren;
    std::vector<float> layer_pad12;
    int fused = 1;                          // 1: low-only prepare + fused final upsample (a whole frame); 0: prepare -> LinearDepth -> upsample
    // the caller's AO view of the fused form (nullptr: the context's result buffer) and its pitches in bytes
    uint8_t *ao_out = nullptr; long long ao_row = 0, ao_layer = 0;
    long long depth_row = 0, depth_layer = 0;   // the depth view's pitches in elements (0: tight)
    int in_format = 0; const void *depth = nullptr;
};

// what MeaoCtx::make_map hands to cuTensorMapEncodeTiled: one map over all layers, height L x h
CUtensorMap make_map(const void *base, int elem, int w, int h, int pitch_elems, int bw, int bh)
{
    CUtensorMap m{};
    m.base = base; m.elem = elem; m.w = w; m.h = h; m.pitch_bytes = (size_t)pitch_elems * elem; m.bw = bw; m.bh = bh;
    return m;
}

void run_downsample(LEmu *e, const void *depth, int in_format)
{
    PrepareArgs a{};
    a.depth = depth; a.in_format = in_format; a.W = e->W; a.H = e->H; a.depth_row0 = 0; a.row0 = 0; a.row1 = e->H;
    a.lin = e->lin; a.lin_pitch = e->lin_pitch;
    for (int k = 1; k <= 4; k++) { a.low[k - 1] = e->low[k]; a.low_pitch[k - 1] = e->low_pitch[k]; }
    a.zbx = e->zbx; a.zby = e->zby; a.raw = e->raw; a.reversed_z = e->reversed_z;
    const int es = in_format == 1 ? 2 : 4;
    a.depth_pitch = (int)e->depth_row; a.depth_layer_pitch = e->depth_layer;
    const long long rp = e->depth_row ? e->depth_row : e->W, lp = e->depth_layer ? e->depth_layer : rp * e->H;
    a.vec_ok = (((uintptr_t)depth & 15) == 0) && (rp * es % 16 == 0) && (lp * es % 16 == 0);
    launch_prepare_depth_layered(a, e->L, nullptr, e->fused != 0, e->layer_zb.data());
}

void run_render(LEmu *e, int k, bool wide)
{
    static const int idx_checker[7] = {1, 3, 4, 8, 11, 6, 10}, idx_exh[12] = {0, 1, 2, 3, 4, 8, 11, 5, 6, 7, 9, 10};
    const int n = e->exhaustive ? 12 : 7; const int *idx = e->exhaustive ? idx_exh : idx_checker;
    RenderArgs a{};
    a.low = e->low[k]; a.lw = e->lw[k]; a.lh = e->lh[k]; a.lpitch = e->low_pitch[k];
    a.occ = wide ? e->hq[k] : e->occ[k]; a.opitch = e->occ_pitch[k];
    a.sw = e->lw[k + 2]; a.sh = e->lh[k + 2];
    a.pad = __half2float(__float2half_rn(e->pad[k]));
    const float *it = wide ? e->inv_thickness_wide[k] : e->inv_thickness[k];
    for (int i = 0; i < n; i++) { a.inv_thickness[i] = it[idx[i]]; a.neg_front[i] = -(a.inv_thickness[i] - 0.5f); a.weight[i] = e->sample_weight[k][idx[i]]; }
    a.reject_fadeoff = e->reject_fadeoff; a.intensity = e->intensity;
    a.row0 = 0; a.row1 = e->lh[k]; a.wide = wide; a.exhaustive = e->exhaustive;
    int tv;                 // meao_api.cu render_tile_variant: the CTAs of ALL layers count
    for (tv = 0; tv < kRenderTileVariants - 1; tv++)
        if ((long long)e->L * ((e->lw[k] + 63) / 64) * ((a.row1 + kRenderTileHs[tv] - 1) / kRenderTileHs[tv]) >= e->sm_count) break;
    a.tile_h = kRenderTileHs[tv];
    const CUtensorMap map = make_map(e->low[k], 4, e->lw[k], e->L * e->lh[k], e->low_pitch[k], wide ? kRenderWideBoxW : kRenderBoxW, render_box_h(a.tile_h, wide));
    launch_render_ao_layered(map, e->use_tma != 0, a, e->L, nullptr, e->layer_ren.data() + (size_t)(2 * (k - 1) + (wide ? 1 : 0)) * e->L, e->raw);
}

void run_upsample(LEmu *e, int lo)
{
    const int hi = lo - 1;
    UpsampleArgs a{};
    a.lo_depth = e->low[lo]; a.low = e->lw[lo]; a.loh = e->lh[lo]; a.lo_dpitch = e->low_pitch[lo];
    a.lo_ao = (e->single_scale && lo == 1) ? e->occ[1] : (lo == 4) ? e->occ[4] : e->comb[lo]; a.lo_apitch = e->occ_pitch[lo];
    if (hi == 0) { a.hi_depth = e->lin; a.hi_is_half = 1; a.hi_dpitch = e->lin_pitch; a.hi_ao = nullptr; a.out = e->result; a.out_pitch = e->result_pitch; }
    else { a.hi_depth = e->low[hi]; a.hi_is_half = 0; a.hi_dpitch = e->low_pitch[hi]; a.hi_ao = e->occ[hi]; a.hi_apitch = e->occ_pitch[hi]; a.out = e->comb[hi]; a.out_pitch = e->occ_pitch[hi]; }
    a.out_row_origin = 0; a.out_vec_ok = 1;
    a.hiw = e->lw[hi]; a.hih = e->lh[hi];
    a.noise_filter_strength = e->nfs[lo]; a.step_size = e->step[lo]; a.blur_tolerance = e->kblur[lo]; a.upsample_tolerance = e->tol[lo];
    a.fast_div_ok = upsample_fast_div_ok(a.upsample_tolerance, a.noise_filter_strength);
    a.row0 = 0; a.row1 = e->lh[hi];
    a.tile_ctr = e->tile_ctr + 2 * (lo - 1);
    const bool premin = ((e->hq_mask >> (lo - 1)) & 1) != 0;
    const int rows = e->L * e->lh[lo];
    const CUtensorMap md = make_map(e->low[lo], 4, e->lw[lo], rows, e->low_pitch[lo], kUpsDepthBoxW, kUpsDepthBoxH);
    const CUtensorMap ma = make_map(a.lo_ao, 1, e->lw[lo], rows, e->occ_pitch[lo], kUpsAoBoxW, kUpsAoBoxH);
    const CUtensorMap mh = make_map(e->hq[lo], 1, e->lw[lo], rows, e->occ_pitch[lo], kUpsAoBoxW, kUpsAoBoxH);
    if (hi == 0 && e->fused) {
        DepthIn d{};
        d.depth = e->depth; d.in_format = e->in_format; d.depth_row0 = 0; d.zbx = e->zbx; d.zby = e->zby; d.raw = e->raw; d.reversed_z = e->reversed_z;
        const int es = e->in_format == 1 ? 2 : 4;
        d.depth_pitch = (int)e->depth_row; d.depth_layer_pitch = e->depth_layer;
        const long long rp = e->depth_row ? e->depth_row : e->W, lp = e->depth_layer ? e->depth_layer : rp * e->H;
        d.vec_ok = (((uintptr_t)e->depth & 15) == 0) && (rp * es % 16 == 0) && (lp * es % 16 == 0);
        if (e->ao_out) {
            a.out = e->ao_out; a.out_pitch = (int)e->ao_row; d.ao_layer_pitch = e->ao_layer;
            a.out_vec_ok = (((uintptr_t)a.out & 7) == 0) && (a.out_pitch % 8 == 0) && (e->ao_layer % 8 == 0);
        }
        d.layer_zb = e->layer_zb.data();
        launch_blur_upsample_lin(md, ma, &mh, e->use_tma != 0, a, premin ? e->hq[lo] : nullptr, e->occ_pitch[lo], d, e->L, e->sm_count, nullptr);
        if (e->ao_out)      // the context's own copy, as meao_get_buffer(17) regenerates it after a frame into the caller's AO
            { a.out = e->result; a.out_pitch = e->result_pitch; a.out_vec_ok = 1; launch_blur_upsample_layered(md, ma, &mh, e->use_tma != 0, a, premin ? e->hq[lo] : nullptr, e->occ_pitch[lo], e->L, e->sm_count, nullptr); }
        return;
    }
    launch_blur_upsample_layered(md, ma, &mh, e->use_tma != 0, a, premin ? e->hq[lo] : nullptr, e->occ_pitch[lo], e->L, e->sm_count, nullptr);
}

}  // namespace

extern "C" {

void *lcemu_create(int W, int H, int layers)
{
    LEmu *e = new LEmu();
    e->W = W; e->H = H; e->L = layers;
    const size_t L = (size_t)layers;
    for (int l = 0; l < 7; l++) { const int d = 1 << l; e->lw[l] = (W + d - 1) / d; e->lh[l] = (H + d - 1) / d; }
    e->lin_pitch = align_up(W, 64); e->lin = alloc<__half>(L * e->lin_pitch * H);
    e->result_pitch = align_up(W, 128); e->result = alloc<uint8_t>(L * e->result_pitch * H);
    for (int k = 1; k <= 4; k++) {
        e->low_pitch[k] = align_up(e->lw[k], 32); e->occ_pitch[k] = align_up(e->lw[k], 128);
        e->low[k] = alloc<float>(L * e->low_pitch[k] * e->lh[k]);
        e->occ[k] = alloc<uint8_t>(L * e->occ_pitch[k] * e->lh[k]);
        e->hq[k] = alloc<uint8_t>(L * e->occ_pitch[k] * e->lh[k]);
        if (k <= 3) e->comb[k] = alloc<uint8_t>(L * e->occ_pitch[k] * e->lh[k]);
    }
    return e;
}

void lcemu_destroy(void *h)
{
    LEmu *e = (LEmu *)h;
    free(e->lin); free(e->result);
    for (int k = 1; k <= 4; k++) { free(e->low[k]); free(e->occ[k]); free(e->hq[k]); if (k <= 3) free(e->comb[k]); }
    delete e;
}

// the same constant layout as emu_set_constants (emu_driver.cpp)
void lcemu_set_constants(void *h, const float *rc, const float *rcw, const float *uc, const float *zb, float pad12,
                        int raw, int reversed_z, int hq_mask, int exhaustive, int single_scale, int use_tma)
{
    LEmu *e = (LEmu *)h;
    for (int k = 1; k <= 4; k++) {
        memcpy(e->inv_thickness[k], rc + 28 * (k - 1), 48);
        memcpy(e->sample_weight[k], rc + 28 * (k - 1) + 12, 48);
        memcpy(e->inv_thickness_wide[k], rcw + 28 * (k - 1), 48);
        e->pad[k] = (k <= 2) ? pad12 : 0.0f;
        const float *u = uc + 8 * (k - 1);
        e->nfs[k] = u[4]; e->step[k] = u[5]; e->kblur[k] = u[6]; e->tol[k] = u[7];
    }
    e->reject_fadeoff = rc[26]; e->intensity = rc[27];
    e->zbx = zb[0]; e->zby = zb[1]; e->raw = raw; e->reversed_z = reversed_z; e->hq_mask = hq_mask; e->exhaustive = exhaustive;
    e->single_scale = single_scale; e->use_tma = use_tma;
}

// layer l's constants (the layouts of meao_render_constants_layer / meao_zbuffer_params_layer) -> the per-layer tables; pad12: the
// layer's Linearize(0) of levels 1-2.  Call after lcemu_set_constants, for every layer.
void lcemu_set_layer(void *h, int l, const float *rc, const float *rcw, const float *zb, float pad12)
{
    static const int idx_checker[7] = {1, 3, 4, 8, 11, 6, 10}, idx_exh[12] = {0, 1, 2, 3, 4, 8, 11, 5, 6, 7, 9, 10};
    LEmu *e = (LEmu *)h;
    const int L = e->L;
    e->layer_zb.resize(L); e->layer_ren.resize((size_t)8 * L); e->layer_pad12.resize(L);
    e->layer_zb[l] = LayerZ{zb[0], zb[1]};
    e->layer_pad12[l] = pad12;
    const int n = e->exhaustive ? 12 : 7; const int *idx = e->exhaustive ? idx_exh : idx_checker;
    for (int k = 1; k <= 4; k++)
        for (int w = 0; w < 2; w++) {
            LayerRender r{};
            const float *it = (w ? rcw : rc) + 28 * (k - 1);
            for (int i = 0; i < n; i++) { r.it_nf[i].x = it[idx[i]]; r.it_nf[i].y = -(r.it_nf[i].x - 0.5f); }
            r.pad = __half2float(__float2half_rn(k <= 2 ? pad12 : 0.0f));
            e->layer_ren[(size_t)(2 * (k - 1) + w) * L + l] = r;
        }
}

// fused: see LEmu::fused.  depth_row / depth_layer: the depth view's pitches in elements (0: tight); ao (may be null): the caller's
// AO view with byte pitches ao_row / ao_layer
void lcemu_set_views(void *h, int fused, long long depth_row, long long depth_layer, void *ao, long long ao_row, long long ao_layer)
{
    LEmu *e = (LEmu *)h;
    e->fused = fused; e->depth_row = depth_row; e->depth_layer = depth_layer; e->ao_out = (uint8_t *)ao; e->ao_row = ao_row; e->ao_layer = ao_layer;
}

long long lcemu_tma_box_loads() { return meao_emu::tma_box_loads; }

// depth: L images of W x H (at the pitches of lcemu_set_views); in_format 0 = f32, 1 = D16 codes, 2 = D24S8 words; 16-byte aligned
void lcemu_run(void *h, const void *depth, int in_format)
{
    LEmu *e = (LEmu *)h;
    e->depth = depth; e->in_format = in_format;
    run_downsample(e, depth, in_format);
    if (e->single_scale) { run_render(e, 1, false); run_upsample(e, 1); return; }    // record_frame_dag, single_scale branch
    for (int k = 1; k <= 4; k++) run_render(e, k, false);
    for (int k = 1; k <= 4; k++) if ((e->hq_mask >> (k - 1)) & 1) run_render(e, k, true);
    for (int lo = 4; lo >= 1; lo--) run_upsample(e, lo);
}

// buffer <id> (1..21) of layer `layer` in the reference layout / native type, like one layer of meao_get_buffer
int lcemu_get_buffer(void *h, int id, int layer, void *out)
{
    LEmu *e = (LEmu *)h;
    if (layer < 0 || layer >= e->L) return -1;
    auto copy2d = [&](const void *src, size_t pitch_bytes, int w, int hgt, int elem) {
        src = (const char *)src + (size_t)layer * hgt * pitch_bytes;       // layer l starts l x rows x pitch after layer 0
        for (int y = 0; y < hgt; y++) memcpy((char *)out + (size_t)y * w * elem, (const char *)src + (size_t)y * pitch_bytes, (size_t)w * elem);
    };
    if (id == 1) copy2d(e->lin, (size_t)e->lin_pitch * 2, e->lw[0], e->lh[0], 2);
    else if (id >= 2 && id <= 5) copy2d(e->low[id - 1], (size_t)e->low_pitch[id - 1] * 4, e->lw[id - 1], e->lh[id - 1], 4);
    else if (id >= 6 && id <= 9) {
        const int k = id - 5;
        launch_synth_tiled(e->low[k] + (size_t)layer * e->lh[k] * e->low_pitch[k], e->lw[k], e->lh[k], e->low_pitch[k], e->lw[k + 2], e->lh[k + 2],
                           __half2float(__float2half_rn(k <= 2 && e->raw ? e->layer_pad12[layer] : 0.0f)), (__half *)out, nullptr);
    }
    else if (id >= 10 && id <= 13) copy2d(e->occ[id - 9], e->occ_pitch[id - 9], e->lw[id - 9], e->lh[id - 9], 1);
    else if (id >= 14 && id <= 16) copy2d(e->comb[id - 13], e->occ_pitch[id - 13], e->lw[id - 13], e->lh[id - 13], 1);
    else if (id == 17) copy2d(e->result, e->result_pitch, e->lw[0], e->lh[0], 1);
    else if (id >= 18 && id <= 21) copy2d(e->hq[id - 17], e->occ_pitch[id - 17], e->lw[id - 17], e->lh[id - 17], 1);
    else return -1;
    return 0;
}

}  // extern "C"
