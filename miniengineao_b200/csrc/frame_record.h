// frame_record.h -- what a frame's kernels are launched with: the frame state a recorder reads, where the buffers of a size sit in the
// arena, the TMA maps over them, the argument blocks of the three stages and which launcher runs each stage, and around the frame the
// debug buffers' table and views and the segments a row band sends to its neighbours.  Host code only, with no
// CUDA runtime call: meao_api.cu records its frames with it, and tests/emu/frame_driver.cpp runs the host-compiled kernels with it
// (-DMEAO_EMULATE), so the CPU tests launch the kernels exactly as libmeao does.
#ifndef MEAO_FRAME_RECORD_H
#define MEAO_FRAME_RECORD_H

#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/meao.h"
#include "kernels.h"
#include "arena_layout.h"

namespace meao {

struct Range { int lo, hi; };   // [lo, hi)

// The plan's variants: MeaoVariants as set (meao_set_variants) and the hierarchy depth as set (meao_set_hierarchy_depth, 1..4).
// Together they decide the levels a frame runs (effective_depth), so they travel as one value.
struct PlanVariants : MeaoVariants {
    int levels = 4;
    PlanVariants() : MeaoVariants{0, 0, 0, 0} {}
    PlanVariants(const MeaoVariants &v, int levels_ = 4) : MeaoVariants(v), levels(levels_) {}
};

// The levels 1..n a frame renders and upsamples; the first upsample reads Occlusion<n>.  single_scale (BASELINE.json configs[0]) is
// n = 1.  The one place the depth in effect is derived: the schedule, the upsample wiring and the launch counts all read it.
inline int effective_depth(const PlanVariants &v) { return v.single_scale ? 1 : v.levels; }

struct Plan {
    // Render (per level 1..4) -- AO.cs:660-734
    float inv_thickness[5][12];
    float sample_weight[5][12];
    float inv_slice_dim[5][2];
    float reject_fadeoff;
    float intensity;
    float pad[5];
    float inv_thickness_wide[5][12];       // the same for a NON-tiled source LowDepth<k> (kernel "main", AO.cs:679)
    float inv_slice_dim_wide[5][2];
    // Upsample (per lo level 1..4) -- AO.cs:750-771
    float inv_low[5][2], inv_high[5][2];
    float noise_filter_strength[5], step_size[5], blur_tolerance[5], upsample_tolerance[5];
    float zb[4];
    // the plan inputs the recorders read besides the constants: the variants with the hierarchy depth, and the cameras' Z direction
    PlanVariants variants;
    int reversed_z;
    int orthographic;                       // every layer MEAO_PROJECTION_ORTHOGRAPHIC: launch_entry_ortho's kernels
};

// The camera-dependent part of the plan, for one camera: ZBufferParams, both inv_thickness tables of every level and the atlas
// padding value.  Plan holds it for the first layer; FrameState::layer_consts holds it for every layer.
struct CamConsts {
    float zb[2];
    float inv_thickness[5][12], inv_thickness_wide[5][12];
    float pad[5];
};

// The TMA maps of a frame size: one 2-D map per buffer over all layers (height L x lh: the kernels fetch a box only when it lies
// inside one layer), each with the box of the kernel that reads it.
struct FrameMaps {
    CUtensorMap low_ren[kRenderTileVariants][5];    // LowDepth<k> with the render box of tile height kRenderTileHs[t]
    CUtensorMap low_wide[kRenderTileVariants][5];   // LowDepth<k> with the wide-render box
    CUtensorMap low_ups[5];                 // LowDepth<k> with the upsample depth box
    CUtensorMap comb_ups[4];                // Combined<k> (k = 1..3) as LoResAO1 of upsample lo level k below the frame's depth
    CUtensorMap occ_ups[5];                 // Occlusion<k> as LoResAO1 of upsample lo level k = the frame's depth (its first upsample)
    CUtensorMap hq_ups[5];                  // HighQuality<k> as LoResAO2 of upsample lo level k
};

// What the recorders read: the geometry and rows of one frame size, where its buffers are, its maps, its plan and its camera tables.
struct FrameState {
    int W = 0, H = 0;
    int layers = 1;                         // every image holds `layers` same-size views stacked at a stride of one image
    int lw[7] = {0}, lh[7] = {0};
    int band0 = 0, band1 = 0;               // global L0 rows of the band (the whole frame without one)
    Range need_c[5];                        // rows of Occlusion<k>/Combined<k> to produce (k=1..4); [0] = final rows

    // device buffers (natural layout, pitched, global coordinates): arena_layout(W, H, layers)
    __half *lin = nullptr; int lin_pitch = 0;
    float *low[5] = {nullptr}; int low_pitch[5] = {0};
    uint8_t *occ[5] = {nullptr}; int occ_pitch[5] = {0};
    uint8_t *comb[4] = {nullptr};           // same pitch as occ of that level
    uint8_t *hq[5] = {nullptr};             // HighQuality<k> (kernel "main" output), same pitch as occ of that level
    uint8_t *result = nullptr; int result_pitch = 0;
    uint32_t *tile_ctr = nullptr;           // 2 words per upsample level: tile cursor + finished-CTA count of the persistent blur_upsample grid
    // the per-layer camera tables (kernels.h LayerZ / LayerRender): layer_zb[l]; layer_ren[(2 (k - 1) + wide) L + l]
    LayerZ *layer_zb = nullptr;
    LayerRender *layer_ren = nullptr;
    LayerView *layer_views = nullptr;       // the layer-viewport table (meao_set_layer_viewports), read by the frames that have one set

    int sm_count = 132;                     // SMs of the device (132 = H100 SXM for plan-only contexts)
    bool tma_ok = false;
    FrameMaps maps;

    Plan plan;
    std::vector<CamConsts> layer_consts;    // the plan's camera constants of every layer (all alike without a layer-camera table)
    // the layers' projections when they mix both (meao_set_layer_projections): bit l of word l / 32 set = layer l orthographic, the
    // kernels.h LayerProjections table of launch_entry_mixed; empty when every layer has the same projection (Plan.orthographic).
    // proj_key: 0 for an all-perspective frame, else a hash of the layers' projections (the graph cache keeps frames of other kernels apart)
    std::vector<uint32_t> layer_ortho;
    uint64_t proj_key = 0;
};

// The layers' projections of a plan: Plan.orthographic, FrameState::layer_ortho and proj_key from ortho(l), layer l orthographic
template <class F> inline void plan_projections(FrameState &f, F &&ortho)
{
    const int L = f.layers;
    std::vector<uint32_t> bits((size_t)(L + 31) / 32, 0u);
    int n = 0;
    for (int l = 0; l < L; l++)
        if (ortho(l)) { bits[l >> 5] |= 1u << (l & 31); n++; }
    f.plan.orthographic = n == L;
    f.proj_key = 0;
    if (n) {
        uint64_t h = 1469598103934665603ull;                // FNV-1a over the words
        for (uint32_t w : bits) { h ^= w; h *= 1099511628211ull; }
        f.proj_key = h | 1;
    }
    if (n > 0 && n < L) f.layer_ortho.swap(bits);
    else f.layer_ortho.clear();
}

inline float host_f16_round(float x) { return __half2float(__float2half_rn(x)); }

// The buffers of a W x H frame (layout `a` = arena_layout(W, H, layers)) in the arena at `base`, with the camera tables of slot `slot`.
// base == nullptr (no arena): the geometry and pitches only.
inline void place_frame(FrameState &f, const ArenaLayout &a, char *base, int slot)
{
    for (int l = 0; l < 7; l++) { f.lw[l] = a.lw[l]; f.lh[l] = a.lh[l]; }
    f.lin_pitch = a.lin_pitch;
    f.result_pitch = a.result_pitch;
    for (int k = 1; k <= 4; k++) { f.low_pitch[k] = a.low_pitch[k]; f.occ_pitch[k] = a.occ_pitch[k]; }
    if (!base) return;
    f.lin = (__half *)(base + a.lin);
    f.result = (uint8_t *)(base + a.result);
    for (int k = 1; k <= 4; k++) {
        f.low[k] = (float *)(base + a.low[k]);
        f.occ[k] = (uint8_t *)(base + a.occ[k]);
        if (k <= 3) f.comb[k] = (uint8_t *)(base + a.comb[k]);
        f.hq[k] = (uint8_t *)(base + a.hq[k]);
    }
    f.tile_ctr = (uint32_t *)(base + a.ctr);
    f.layer_zb = (LayerZ *)(base + a.table0 + (size_t)slot * a.table_stride);
    f.layer_ren = (LayerRender *)((char *)f.layer_zb + a.table_ren);
    f.layer_views = (LayerView *)(base + a.views);
}

// One TMA map: w x h elements of elem bytes (4: f32, 1: u8) at base, rows pitch_elems apart, box bw x bh
struct MapSpec { void *base; int elem, w, h, pitch_elems, bw, bh; };

// Encodes every map of the frame with enc(CUtensorMap &, const MapSpec &) -> bool; false if any failed.
template <class Enc> bool encode_maps(FrameState &f, Enc &&enc)
{
    bool ok = true;
    FrameMaps &m = f.maps;
    for (int k = 1; k <= 4; k++) {
        const int mh = f.layers * f.lh[k];
        for (int t = 0; t < kRenderTileVariants; t++) {
            ok &= enc(m.low_ren[t][k], MapSpec{f.low[k], 4, f.lw[k], mh, f.low_pitch[k], kRenderBoxW, render_box_h(kRenderTileHs[t], false)});
            ok &= enc(m.low_wide[t][k], MapSpec{f.low[k], 4, f.lw[k], mh, f.low_pitch[k], kRenderWideBoxW, render_box_h(kRenderTileHs[t], true)});
        }
        ok &= enc(m.low_ups[k], MapSpec{f.low[k], 4, f.lw[k], mh, f.low_pitch[k], kUpsDepthBoxW, kUpsDepthBoxH});
        if (k <= 3) ok &= enc(m.comb_ups[k], MapSpec{f.comb[k], 1, f.lw[k], mh, f.occ_pitch[k], kUpsAoBoxW, kUpsAoBoxH});
        ok &= enc(m.occ_ups[k], MapSpec{f.occ[k], 1, f.lw[k], mh, f.occ_pitch[k], kUpsAoBoxW, kUpsAoBoxH});
        ok &= enc(m.hq_ups[k], MapSpec{f.hq[k], 1, f.lw[k], mh, f.occ_pitch[k], kUpsAoBoxW, kUpsAoBoxH});
    }
    return ok;
}

inline bool hq_level(const FrameState &f, int k) { return ((f.plan.variants.high_quality_mask >> (k - 1)) & 1) != 0; }

// The f16-rounded atlas padding value of layer l at render level k for depth kind `kind` (linear ingest pads with 0)
inline float layer_pad(const FrameState &f, int l, int k, int kind)
{
    return host_f16_round((kind != MEAO_DEPTH_LINEAR_F32) ? f.layer_consts[l].pad[k] : 0.0f);
}

// The call-order tables of the render stage: Render.compute:162-168 (checker) and :148-159 (exhaustive) table slots
constexpr int kIdxChecker[7] = {1, 3, 4, 8, 11, 6, 10};
constexpr int kIdxExh[12] = {0, 1, 2, 3, 4, 8, 11, 5, 6, 7, 9, 10};

// The LayerRender entry of camera constants `cc` at render level k (wide: kernel "main"): what render_args puts into RenderArgs
inline LayerRender layer_render(const FrameState &f, const CamConsts &cc, int k, bool wide)
{
    const bool exh = f.plan.variants.sample_exhaustively != 0;
    const int n = exh ? 12 : 7;
    const int *idx = exh ? kIdxExh : kIdxChecker;
    const float *it = wide ? cc.inv_thickness_wide[k] : cc.inv_thickness[k];
    LayerRender r{};
    for (int i = 0; i < n; i++) {
        r.it_nf[i].x = it[idx[i]];
        r.it_nf[i].y = -(r.it_nf[i].x - 0.5f);                                                      // Render.compute:85
    }
    r.pad = host_f16_round(cc.pad[k]);
    return r;
}

// The per-layer camera tables of the plan, as they go into the arena
inline void camera_tables(const FrameState &f, std::vector<LayerZ> &zb, std::vector<LayerRender> &ren)
{
    const int L = f.layers;
    zb.resize(L);
    ren.resize((size_t)8 * L);
    for (int l = 0; l < L; l++) {
        const CamConsts &cc = f.layer_consts[l];
        zb[l] = LayerZ{cc.zb[0], cc.zb[1]};
        for (int k = 1; k <= 4; k++)
            for (int w = 0; w < 2; w++) ren[(size_t)(2 * (k - 1) + w) * L + l] = layer_render(f, cc, k, w != 0);
    }
}

// Tile-height variant (index into kRenderTileHs = {32, 16, 8}) of a render launch.  The big levels keep the 64 x 32 tile
// (least apron overhead: throughput); a level whose grid would not even put one CTA on every SM is latency-bound -- one
// CTA's serial time IS the kernel time -- so it takes the tallest tile that still gives at least one CTA per SM, else 64 x 8.
// A layered launch counts the CTAs of all its layers.  force >= 0: that variant for every level (a tuning aid).
inline int render_tile_variant(const FrameState &f, int k, int rows, int force)
{
    if (force >= 0 && force < kRenderTileVariants) return force;
    for (int t = 0; t < kRenderTileVariants; t++) {
        const long long ctas = (long long)f.layers * ((f.lw[k] + 63) / 64) * ((rows + kRenderTileHs[t] - 1) / kRenderTileHs[t]);
        if (ctas >= f.sm_count) return t;
    }
    return kRenderTileVariants - 1;
}

// A CUDA-array frame (meao_render_arrays): the surfaces of the depth and AO arrays and how their layers are addressed (surface_io.cuh).
// The frame reads the depth array's texels [depth_x, depth_x + W) x [depth_y, depth_y + H) and writes the AO array's at (ao_x, ao_y)
// (meao_render_arrays_at; all 0 for meao_render_arrays).
struct ArrayIO { cudaSurfaceObject_t depth, ao; int depth_surf, ao_surf; const void *ao_array; int depth_x = 0, depth_y = 0, ao_x = 0, ao_y = 0; };

// The byte pitches of the caller's depth and AO views (meao_render_pitched).  A view is `layers` images of rows [band0, band1) of
// the frame, W pixels per row.
struct ViewPitch { int64_t depth_row, depth_layer, ao_row, ao_layer; };
inline int64_t depth_esize(int kind) { return kind == MEAO_DEPTH_RAW_D16_UNORM ? 2 : 4; }
// meao_render's views: tight rows, tight layers
inline ViewPitch tight_pitch(const FrameState &f, int kind)
{
    const int64_t es = depth_esize(kind), rows = f.band1 - f.band0;
    return ViewPitch{f.W * es, rows * f.W * es, f.W, rows * f.W};
}

// The caller's depth as the kernels read it: rows [band0, band1) of the frame of every layer, at the pitches of `vp` (nullptr: tight).
inline DepthIn depth_in(const FrameState &f, const void *depth, int kind, const ViewPitch *vp = nullptr)
{
    const ViewPitch p = vp ? *vp : tight_pitch(f, kind);
    const int64_t es = depth_esize(kind);
    DepthIn d{};
    d.depth = depth;
    d.in_format = (kind == MEAO_DEPTH_RAW_D16_UNORM) ? 1 : (kind == MEAO_DEPTH_RAW_D24S8 ? 2 : 0);
    d.depth_row0 = f.band0;
    d.zbx = f.plan.zb[0]; d.zby = f.plan.zb[1];
    d.raw = (kind != MEAO_DEPTH_LINEAR_F32);
    d.reversed_z = f.plan.reversed_z;
    // 128-bit loads: every row (and layer) start 16-byte aligned.  Tight views: W % 4 == 0 (4-byte kinds), W % 8 == 0 (D16)
    d.vec_ok = (((uintptr_t)depth & 15) == 0) && (p.depth_row % 16 == 0) && (f.layers == 1 || p.depth_layer % 16 == 0);
    d.depth_pitch = (int)(p.depth_row / es);
    d.depth_layer_pitch = p.depth_layer / es;
    d.ao_layer_pitch = p.ao_layer;
    d.layer_zb = f.layer_zb;
    return d;
}

// PushDownsampleCommands, AO.cs:604-658: prepare_depth of rows [band0, band1) from the depth `d` describes
inline PrepareArgs prepare_args(const FrameState &f, const DepthIn &d)
{
    PrepareArgs a{};
    a.depth = d.depth;
    a.in_format = d.in_format;
    a.W = f.W; a.H = f.H;
    a.depth_row0 = d.depth_row0;
    a.row0 = f.band0; a.row1 = f.band1;
    a.lin = f.lin; a.lin_pitch = f.lin_pitch;
    for (int k = 1; k <= 4; k++) { a.low[k - 1] = f.low[k]; a.low_pitch[k - 1] = f.low_pitch[k]; }
    a.zbx = d.zbx; a.zby = d.zby;
    a.raw = d.raw;
    a.reversed_z = d.reversed_z;
    a.vec_ok = d.vec_ok;
    a.depth_pitch = d.depth_pitch; a.depth_layer_pitch = d.depth_layer_pitch;
    return a;
}

// aio: read the depth from a CUDA array instead of a.depth.  low_only: LowDepth1..4 only -- the frame's final upsample is launched
// with the same depth (launch_upsample's `fused`) and writes LinearDepth itself.  layered: the layered kernel at layers == 1 too, which
// reads the camera table (a device camera buffer is bound: FrameIO.cams)
inline cudaError_t launch_prepare(const FrameState &f, const PrepareArgs &a, const ArrayIO *aio, bool low_only, cudaStream_t s, bool layered = false)
{
    if (aio) return launch_prepare_depth_array(a, aio->depth, aio->depth_surf, aio->depth_x, aio->depth_y, f.layers, s, f.layer_zb);
    if (f.layers > 1 || layered) return launch_prepare_depth_layered(a, f.layers, s, low_only, f.layer_zb);
    return launch_prepare_depth(a, s, low_only);
}

// PushRenderCommands, AO.cs:660-748, of level k.  wide = false: the call AmbientOcclusion.cs makes (tiled source, kernel
// main_interleaved); wide = true: the same recorder for the non-tiled source LowDepth<k> (kernel main) -> HighQuality<k>.
// force_tile: render_tile_variant's force.
inline RenderArgs render_args(const FrameState &f, int k, int kind, bool wide, int force_tile)
{
    const bool exh = f.plan.variants.sample_exhaustively != 0;
    const int n = exh ? 12 : 7;
    const int *idx = exh ? kIdxExh : kIdxChecker;
    RenderArgs a{};
    a.low = f.low[k]; a.lw = f.lw[k]; a.lh = f.lh[k]; a.lpitch = f.low_pitch[k];
    a.occ = wide ? f.hq[k] : f.occ[k]; a.opitch = f.occ_pitch[k];
    a.sw = f.lw[k + 2]; a.sh = f.lh[k + 2];
    a.pad = host_f16_round((kind != MEAO_DEPTH_LINEAR_F32) ? f.plan.pad[k] : 0.0f);
    const float *it = wide ? f.plan.inv_thickness_wide[k] : f.plan.inv_thickness[k];
    for (int i = 0; i < n; i++) {
        a.inv_thickness[i] = it[idx[i]];
        a.neg_front[i] = -(a.inv_thickness[i] - 0.5f);                                               // Render.compute:85
        a.weight[i] = f.plan.sample_weight[k][idx[i]];
    }
    a.reject_fadeoff = f.plan.reject_fadeoff;
    a.intensity = f.plan.intensity;
    a.row0 = f.need_c[k].lo; a.row1 = f.need_c[k].hi;
    a.wide = wide ? 1 : 0;
    a.exhaustive = exh ? 1 : 0;
    a.tile_h = kRenderTileHs[render_tile_variant(f, k, a.row1 - (a.row0 & ~3), force_tile)];
    return a;
}

// The TMA map of render launch `a` of level k (its tile height and source) and its layers' camera table entries (nullptr: none)
inline const CUtensorMap &render_map(const FrameState &f, const RenderArgs &a, int k)
{
    int tv = 0;
    while (tv + 1 < kRenderTileVariants && kRenderTileHs[tv] != a.tile_h) tv++;
    return a.wide ? f.maps.low_wide[tv][k] : f.maps.low_ren[tv][k];
}
inline const LayerRender *render_layer_cams(const FrameState &f, const RenderArgs &a, int k)
{
    return f.layer_ren ? f.layer_ren + (size_t)(2 * (k - 1) + a.wide) * f.layers : nullptr;
}

// The render launch of level k with the map of a.tile_h; a layered frame (and, with `layered`, a single layer) takes its layers'
// camera table entries
inline cudaError_t launch_render(const FrameState &f, const RenderArgs &a, int k, int kind, cudaStream_t s, bool layered = false)
{
    const CUtensorMap &map = render_map(f, a, k);
    if (f.layers == 1 && !layered) return launch_render_ao(map, f.tma_ok, a, s);
    return launch_render_ao_layered(map, f.tma_ok, a, f.layers, s, render_layer_cams(f, a, k), kind != MEAO_DEPTH_LINEAR_F32 ? 1 : 0);
}

// PushUpsampleCommands with the wiring of AO.cs:528-531, lo level `lo`.  ao_out (final level only): the caller's AO at the pitches
// of vp (nullptr: tight), its first row band0; nullptr: the context's result buffer.  The frame's first upsample (lo = effective_depth)
// reads Occlusion<lo> as LoResAO1, since no coarser level contributes; every later one the Combined<lo> the one before wrote.
inline UpsampleArgs upsample_args(const FrameState &f, int lo, void *ao_out, const ViewPitch *vp)
{
    const int hi = lo - 1;
    UpsampleArgs a{};
    a.lo_depth = f.low[lo]; a.low = f.lw[lo]; a.loh = f.lh[lo]; a.lo_dpitch = f.low_pitch[lo];
    a.lo_ao = lo == effective_depth(f.plan.variants) ? f.occ[lo] : f.comb[lo]; a.lo_apitch = f.occ_pitch[lo];
    if (hi == 0) { a.hi_depth = f.lin; a.hi_is_half = 1; a.hi_dpitch = f.lin_pitch; a.hi_ao = nullptr; a.hi_apitch = 0; }
    else { a.hi_depth = f.low[hi]; a.hi_is_half = 0; a.hi_dpitch = f.low_pitch[hi]; a.hi_ao = f.occ[hi]; a.hi_apitch = f.occ_pitch[hi]; }
    if (hi == 0) {
        if (ao_out) { a.out = (uint8_t *)ao_out; a.out_pitch = vp ? (int)vp->ao_row : f.W; a.out_row_origin = f.band0; }
        else { a.out = f.result; a.out_pitch = f.result_pitch; a.out_row_origin = 0; }
    } else { a.out = f.comb[hi]; a.out_pitch = f.occ_pitch[hi]; a.out_row_origin = 0; }
    // 64-bit stores: every row (and, in the caller's layered AO, layer) start 8-byte aligned.  A tight AO: W % 8 == 0
    a.out_vec_ok = (((uintptr_t)a.out & 7) == 0) && (a.out_pitch % 8 == 0) && !(vp && ao_out && f.layers > 1 && vp->ao_layer % 8 != 0);
    a.hiw = f.lw[hi]; a.hih = f.lh[hi];
    a.noise_filter_strength = f.plan.noise_filter_strength[lo];
    a.step_size = f.plan.step_size[lo];
    a.blur_tolerance = f.plan.blur_tolerance[lo];
    a.upsample_tolerance = f.plan.upsample_tolerance[lo];
    a.fast_div_ok = upsample_fast_div_ok(a.upsample_tolerance, a.noise_filter_strength);
    a.row0 = f.need_c[hi].lo; a.row1 = f.need_c[hi].hi;
    a.tile_ctr = f.tile_ctr + 2 * (lo - 1);
    return a;
}

// The upsample launch of lo level `lo`.  aio (final level only): store the AO into a CUDA array.  fused (final level only): read and
// linearise the raw depth and write LinearDepth, after a low_only prepare of the same depth.
// The LoResAO1 map of the upsample of lo level `lo`, and its LoResAO2 (HighQuality<lo>: kernels main_premin / main_premin_blendout; nullptr:
// main / main_blendout)
inline const CUtensorMap &upsample_ao_map(const FrameState &f, int lo)
{
    return lo == effective_depth(f.plan.variants) ? f.maps.occ_ups[lo] : f.maps.comb_ups[lo];
}
inline const uint8_t *upsample_lo_ao2(const FrameState &f, int lo) { return hq_level(f, lo) ? f.hq[lo] : nullptr; }

// layered: a fused final upsample reads the camera table at layers == 1 too.
inline cudaError_t launch_upsample(const FrameState &f, int lo, const UpsampleArgs &a, const ArrayIO *aio, const DepthIn *fused, cudaStream_t s,
                                   bool layered = false)
{
    const bool final_level = lo == 1;
    const uint8_t *lo_ao2 = upsample_lo_ao2(f, lo);
    const CUtensorMap &ao_map = upsample_ao_map(f, lo);
    const CUtensorMap &dm = f.maps.low_ups[lo], *hm = &f.maps.hq_ups[lo];
    if (fused && final_level)
        return launch_blur_upsample_lin(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], *fused, f.layers, f.sm_count, s, layered);
    if (aio && final_level)
        return launch_blur_upsample_array(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.layers, f.sm_count, aio->ao, aio->ao_surf,
                                          aio->ao_x, aio->ao_y, s);
    if (f.layers > 1) return launch_blur_upsample_layered(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.layers, f.sm_count, s);
    return launch_blur_upsample(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.sm_count, s);
}

// ---- the frame schedule: which kernels a frame launches, in what order, on which stream and after which other launch ----------
// kStageCamera: the camera tables derived from a bound device camera buffer (launch_camera_tables), ahead of the prepare.
// kStageParams: reject_fadeoff and intensity derived from a bound device parameter buffer (launch_render_params), ahead of the prepare.
enum FrameStage { kStagePrepare, kStageRender, kStageRenderWide, kStageUpsample, kStageCamera, kStageParams };
// PDL (DESIGN.md 2.5): a launch whose only predecessor is the launch before it on its stream carries the programmatic-dependent-launch
// attribute from PDL level 1 on; one that also waits for another branch, from level 2; the first launch of a branch never.
enum PdlClass { kPdlNever = 0, kPdlFrom1 = 1, kPdlFrom2 = 2 };

struct FrameLaunch {
    int stage;      // FrameStage
    int level;      // render level k, or the upsample's lo level (1 = the final upsample); 0 for the prepare
    int branch;     // 0: the caller's stream; 1..3: the context's forked streams
    int wait;       // index of an earlier launch on another branch that this one waits for; -1: none
    int pdl;        // PdlClass
};

inline bool pdl_on(const FrameLaunch &l, int pdl_level) { return l.pdl != kPdlNever && pdl_level >= l.pdl; }

// The launches of one frame of depth n in serial order (RebuildCommandBuffers, AO.cs:511-531): prepare, render 1..n, the wide renders
// of the high_quality_mask levels up to n, upsamples n..1.  The branches make it a DAG: the render levels are independent (SURVEY.md
// 3.2), a level's wide render rides on its branch, the coarse upsample chain n->..->2 runs on level n's branch and only needs
// Occlusion2..n, and only the last two upsamples wait for the big level-1 render.  The first upsample reads Occlusion<n> (and
// HighQuality<n>); at n = 1 it is the final upsample, on the caller's stream behind render 1.  Mask bits above n launch nothing.
// device_cameras (meao_bind_device_cameras): the camera stage first, on the caller's stream; every other launch follows it through the
// prepare.  device_params (meao_bind_device_params): the parameter stage next, on the caller's stream and without PDL, so every render
// follows it through the prepare as well; it sits on the frame's critical path, ahead of a prepare that waits for it in full.
inline std::vector<FrameLaunch> frame_schedule(const PlanVariants &v, bool device_cameras = false, bool device_params = false)
{
    const int hq_mask = v.high_quality_mask, n = effective_depth(v);
    std::vector<FrameLaunch> s;
    int last[4] = {0, 0, 0, 0};             // the last launch on each branch so far
    auto add = [&](int stage, int level, int branch, int wait, int pdl) {
        last[branch] = (int)s.size();
        s.push_back(FrameLaunch{stage, level, branch, wait, pdl});
    };
    if (device_cameras) add(kStageCamera, 0, 0, -1, kPdlNever);
    if (device_params) add(kStageParams, 0, 0, -1, kPdlNever);
    const int prep = (int)s.size();
    add(kStagePrepare, 0, 0, -1, kPdlNever);
    for (int k = 1; k <= n; k++) add(kStageRender, k, k - 1, k == 1 ? -1 : prep, k == 1 ? kPdlFrom1 : kPdlNever);
    for (int k = 1; k <= n; k++)
        if ((hq_mask >> (k - 1)) & 1) add(kStageRenderWide, k, k - 1, -1, kPdlFrom1);
    // lo >= 3 on level n's branch, waiting for Occlusion<lo - 1>; lo = 2 on the caller's stream (Occlusion1), waiting for the chain
    for (int lo = n; lo >= 3; lo--) add(kStageUpsample, lo, n - 1, last[lo - 2], kPdlFrom2);
    if (n >= 2) add(kStageUpsample, 2, 0, last[n - 1], kPdlFrom2);
    add(kStageUpsample, 1, 0, -1, kPdlFrom1);
    return s;
}

// The launch's name in meao_profile_frame: "prepare_depth", "render_ao L1", "render_ao_wide L1", "blur_upsample L2->L1"
inline std::string launch_name(const FrameLaunch &l)
{
    const std::string k = std::to_string(l.level);
    switch (l.stage) {
        case kStagePrepare: return "prepare_depth";
        case kStageCamera: return "camera_tables";
        case kStageParams: return "render_params";
        case kStageRender: return "render_ao L" + k;
        case kStageRenderWide: return "render_ao_wide L" + k;
        default: return "blur_upsample L" + k + "->L" + std::to_string(l.level - 1);
    }
}

// What a frame form puts into the first and the last launch of its schedule.
struct FrameIO {
    int kind = MEAO_DEPTH_RAW_F32;
    DepthIn depth{};                    // the caller's depth (depth_in), read by the prepare and by a fused final upsample
    const ArrayIO *aio = nullptr;       // read the depth from, and store the AO into, CUDA arrays
    bool low_only = false;              // the prepare writes LowDepth1..4 only
    bool fused = false;                 // the final upsample reads and linearises `depth` and writes LinearDepth
    void *ao = nullptr;                 // the final upsample's AO at the pitches of vp (nullptr: tight); nullptr: the result buffer
    const ViewPitch *vp = nullptr;
    const LayerView *views = nullptr;   // layer l reads and writes the rectangles and slices of views[l] (launch_entry_views)
    const struct BatchIO *batch = nullptr;  // layer l reads and writes its own resources (launch_entry_batch)
    // a bound device camera buffer (meao_bind_device_cameras): the schedule's camera stage derives the tables from it, and every launch
    // that reads a camera takes the layered kernel at layers == 1 too, so that it reads the tables rather than its argument block
    const struct DeviceCameras *cams = nullptr;
    // a bound device parameter buffer (meao_bind_device_params): the schedule's parameter stage derives the slot from it, and every render
    // takes the *_params_layered kernel, at layers == 1 too (launch_render_params_entry)
    const RenderParamArgs *params = nullptr;
};

// A bound device camera buffer: cams[l] = {near_clip, far_clip, tan_half_fov_h} of layer l, the kernel's status words (kernels.h
// CameraTableArgs) and SampleThickness in table order (meao_api.cu sample_thickness).
struct DeviceCameras {
    const float *cams = nullptr;
    uint32_t *status = nullptr;
    float thick[12] = {0};
};

// The camera stage's arguments: the tables of the frame's slot, and what camera_consts / layer_render read besides the camera
inline CameraTableArgs camera_args(const FrameState &f, const DeviceCameras &dc)
{
    const bool exh = f.plan.variants.sample_exhaustively != 0;
    const int *idx = exh ? kIdxExh : kIdxChecker;
    CameraTableArgs a{};
    a.cams = dc.cams; a.zb = f.layer_zb; a.ren = f.layer_ren; a.status = dc.status;
    a.layers = f.layers;
    for (int l = 0; l < 7; l++) a.lw[l] = f.lw[l];
    a.stereo = f.plan.variants.single_pass_stereo != 0;
    a.reversed_z = f.plan.reversed_z != 0;
    a.ortho = f.plan.orthographic != 0;
    a.n = exh ? 12 : 7;
    for (int i = 0; i < a.n; i++) a.thick[i] = dc.thick[idx[i]];
    return a;
}

// The camera stage of a frame (kStageCamera): with the layers' projections as a kernel parameter when they mix both.  Apart from
// launch_entry so that a recorder that never binds a camera buffer does not link the camera kernels.
inline cudaError_t launch_cameras(const FrameState &f, const DeviceCameras &dc, cudaStream_t s)
{
    if (f.layer_ortho.empty()) return launch_camera_tables(camera_args(f, dc), nullptr, s);
    LayerProjections proj{};
    for (size_t i = 0; i < f.layer_ortho.size(); i++) proj.ortho[i] = f.layer_ortho[i];
    return launch_camera_tables(camera_args(f, dc), &proj, s);
}

// A render of a frame with a bound device parameter buffer (FrameIO.params): the kernel for the plan's projections that reads reject_fadeoff
// and intensity from the derived slot.  The layers' camera table entries as the layered launch takes them (launch_render,
// launch_entry_ortho, launch_entry_mixed); a single layer without device cameras reads its argument block, as the single-image kernels
// do.  Apart from launch_entry so that a recorder that never binds a parameter buffer does not link these kernels.
inline cudaError_t launch_render_params_entry(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    if (!io.params || (l.stage != kStageRender && l.stage != kStageRenderWide)) return cudaErrorInvalidValue;
    const RenderArgs a = render_args(f, l.level, io.kind, l.stage == kStageRenderWide, force_tile);
    const CUtensorMap &map = render_map(f, a, l.level);
    const LayerRender *cam = f.layers > 1 || io.cams ? render_layer_cams(f, a, l.level) : nullptr;
    const int pad = io.kind != MEAO_DEPTH_LINEAR_F32 ? 1 : 0;
    if (!f.layer_ortho.empty()) {
        LayerProjections proj{};
        for (size_t i = 0; i < f.layer_ortho.size(); i++) proj.ortho[i] = f.layer_ortho[i];
        return launch_render_ao_mixed_params_layered(map, f.tma_ok, a, f.layers, s, cam, pad, io.params->derived, proj);
    }
    if (f.plan.orthographic) return launch_render_ao_ortho_params_layered(map, f.tma_ok, a, f.layers, s, cam, pad, io.params->derived);
    return launch_render_ao_params_layered(map, f.tma_ok, a, f.layers, s, cam, pad, io.params->derived);
}

// A batch (meao_render_arrays_batch / meao_render_batch): the kernel-parameter tables of its first and last launch.  arrays: layer l
// reads depth.e[l] and writes ao.e[l]; otherwise layer l reads and writes its own buffers, ptr.e[l].
struct BatchIO {
    bool arrays = false;
    BatchArrays depth{}, ao{};
    BatchPointers ptr{};
};

// Launches schedule entry l of a frame on stream s.  force_tile: render_tile_variant's force.
inline cudaError_t launch_entry(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    const bool final_level = l.stage == kStageUpsample && l.level == 1;
    const bool layered = io.cams != nullptr;
    switch (l.stage) {
        case kStageCamera: return cudaErrorInvalidValue;       // launch_cameras, apart so that a recorder without the stage does not link it
        case kStagePrepare: return launch_prepare(f, prepare_args(f, io.depth), io.aio, io.low_only, s, layered);
        case kStageRender:
        case kStageRenderWide:
            return launch_render(f, render_args(f, l.level, io.kind, l.stage == kStageRenderWide, force_tile), l.level, io.kind, s, layered);
        default:
            return launch_upsample(f, l.level, upsample_args(f, l.level, final_level ? io.ao : nullptr, final_level ? io.vp : nullptr),
                                   io.aio, io.fused ? &io.depth : nullptr, s, layered);
    }
}

// launch_entry for a frame that may have a layer-viewport table (FrameIO.views): its prepare and its final upsample are the table
// kernels, every other launch is launch_entry's.  A CUDA-array frame (io.aio) or a fused pointer frame (what meao_render_pitched
// records).  Apart from launch_entry so that a recorder that never sets a table does not link the table kernels.
inline cudaError_t launch_entry_views(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    const bool final_level = l.stage == kStageUpsample && l.level == 1;
    if (!io.views || (l.stage != kStagePrepare && !final_level)) return launch_entry(f, l, io, force_tile, s);
    // the vector accesses of a pointer frame: the host tests the rows (depth row pitch % 16, AO row pitch % 8), each layer its base
    DepthIn d = io.depth;
    d.vec_ok = (int64_t)d.depth_pitch * (d.in_format == 1 ? 2 : 4) % 16 == 0;
    if (l.stage == kStagePrepare) {
        PrepareArgs a = prepare_args(f, d);
        if (io.aio) return launch_prepare_depth_array_views(a, io.aio->depth, io.aio->depth_surf, io.views, f.layers, s, f.layer_zb);
        if (!io.fused) return cudaErrorInvalidValue;
        return launch_prepare_depth_views(a, io.views, f.layers, s, f.layer_zb);
    }
    UpsampleArgs a = upsample_args(f, 1, io.aio ? nullptr : io.ao, io.aio ? nullptr : io.vp);
    const uint8_t *lo_ao2 = upsample_lo_ao2(f, 1);
    const CUtensorMap &ao_map = upsample_ao_map(f, 1);
    if (io.aio)
        return launch_blur_upsample_array_views(f.maps.low_ups[1], ao_map, &f.maps.hq_ups[1], f.tma_ok, a, lo_ao2, f.occ_pitch[1], f.layers,
                                                f.sm_count, io.aio->ao, io.aio->ao_surf, io.views, s);
    a.out_vec_ok = a.out_pitch % 8 == 0;
    return launch_blur_upsample_lin_views(f.maps.low_ups[1], ao_map, &f.maps.hq_ups[1], f.tma_ok, a, lo_ao2, f.occ_pitch[1], d, f.layers,
                                          f.sm_count, io.views, s);
}

// launch_entry for a batch (FrameIO.batch): its prepare and its final upsample are the batch kernels, every other launch is launch_entry's.
// A CUDA-array batch, or a pointer batch recorded fused (io.low_only and io.fused: the prepare reads the even rows, the final upsample
// linearises every pixel).  Perspective and whole frames only (meao_api.cu refuses an orthographic projection and a row band).  Apart
// from launch_entry so that a recorder that never renders a batch does not link the batch kernels.
inline cudaError_t launch_entry_batch(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    const bool final_level = l.stage == kStageUpsample && l.level == 1;
    if (!io.batch || (l.stage != kStagePrepare && !final_level)) return launch_entry(f, l, io, force_tile, s);
    if (f.plan.orthographic || io.aio || io.views || (!io.batch->arrays && !(io.low_only && io.fused))) return cudaErrorInvalidValue;
    if (l.stage == kStagePrepare) {
        const PrepareArgs a = prepare_args(f, io.depth);
        if (io.batch->arrays) return launch_prepare_depth_array_batch(a, io.batch->depth, f.layers, s, f.layer_zb);
        return launch_prepare_depth_batch(a, io.batch->ptr, f.layers, s, f.layer_zb);
    }
    const UpsampleArgs a = upsample_args(f, 1, nullptr, nullptr);
    const uint8_t *lo_ao2 = upsample_lo_ao2(f, 1);
    const CUtensorMap &ao_map = upsample_ao_map(f, 1);
    if (io.batch->arrays)
        return launch_blur_upsample_array_batch(f.maps.low_ups[1], ao_map, &f.maps.hq_ups[1], f.tma_ok, a, lo_ao2, f.occ_pitch[1], f.layers,
                                                f.sm_count, io.batch->ao, s);
    return launch_blur_upsample_lin_batch(f.maps.low_ups[1], ao_map, &f.maps.hq_ups[1], f.tma_ok, a, lo_ao2, f.occ_pitch[1], io.depth, f.layers,
                                          f.sm_count, io.batch->ptr, s);
}

// launch_entry for a frame under an orthographic projection (Plan.orthographic): the launches whose arithmetic depends on the projection
// -- the prepare of raw depth, every render and the fused final upsample of raw depth -- are the orthographic kernels (kernels.h), every
// other launch is launch_entry's.  No layer-viewport table and no row band go with an orthographic projection (meao_set_projection).
// Apart from launch_entry so that a recorder that never sets the projection does not link the orthographic kernels.
inline cudaError_t launch_entry_ortho(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    if (!f.plan.orthographic || io.views) return cudaErrorInvalidValue;
    const bool layered = f.layers > 1 || io.cams;
    if (l.stage == kStagePrepare) {
        const PrepareArgs a = prepare_args(f, io.depth);
        if (io.aio) return launch_prepare_depth_array_ortho(a, io.aio->depth, io.aio->depth_surf, io.aio->depth_x, io.aio->depth_y, f.layers, s, f.layer_zb);
        if (layered) return launch_prepare_depth_ortho_layered(a, f.layers, s, io.low_only, f.layer_zb);
        return launch_prepare_depth_ortho(a, s, io.low_only);
    }
    if (l.stage == kStageRender || l.stage == kStageRenderWide) {
        const RenderArgs a = render_args(f, l.level, io.kind, l.stage == kStageRenderWide, force_tile);
        const CUtensorMap &map = render_map(f, a, l.level);
        if (!layered) return launch_render_ao_ortho(map, f.tma_ok, a, s);
        return launch_render_ao_ortho_layered(map, f.tma_ok, a, f.layers, s, render_layer_cams(f, a, l.level),
                                              io.kind != MEAO_DEPTH_LINEAR_F32 ? 1 : 0);
    }
    if (l.level == 1 && io.fused) {
        return launch_blur_upsample_lin_ortho(f.maps.low_ups[1], upsample_ao_map(f, 1), &f.maps.hq_ups[1], f.tma_ok,
                                              upsample_args(f, 1, io.ao, io.vp), upsample_lo_ao2(f, 1), f.occ_pitch[1], io.depth, f.layers,
                                              f.sm_count, s, layered);
    }
    return launch_entry(f, l, io, force_tile, s);
}

// launch_entry for a layered frame whose layers mix both projections (FrameState::layer_ortho): the launches whose arithmetic depends on
// the projection -- the prepare of raw depth, every render and the fused final upsample of raw depth -- are the mixed kernels (kernels.h),
// which take the layers' projections as a parameter; every other launch is launch_entry's.  No layer-viewport table, batch or row band
// goes with an orthographic layer (meao_set_layer_projections).  Apart from launch_entry so that a recorder that never sets a projection
// table does not link the mixed kernels.
inline cudaError_t launch_entry_mixed(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    if (f.layer_ortho.empty() || f.layers < 2 || io.views || io.batch) return cudaErrorInvalidValue;
    const bool render = l.stage == kStageRender || l.stage == kStageRenderWide;
    if (!render && l.stage != kStagePrepare && !(l.level == 1 && io.fused)) return launch_entry(f, l, io, force_tile, s);
    LayerProjections proj{};
    for (size_t i = 0; i < f.layer_ortho.size(); i++) proj.ortho[i] = f.layer_ortho[i];
    if (l.stage == kStagePrepare) {
        const PrepareArgs a = prepare_args(f, io.depth);
        if (io.aio)
            return launch_prepare_depth_array_mixed(a, io.aio->depth, io.aio->depth_surf, io.aio->depth_x, io.aio->depth_y, f.layers, s, f.layer_zb, proj);
        return launch_prepare_depth_mixed_layered(a, f.layers, s, io.low_only, f.layer_zb, proj);
    }
    if (render) {
        const RenderArgs a = render_args(f, l.level, io.kind, l.stage == kStageRenderWide, force_tile);
        return launch_render_ao_mixed_layered(render_map(f, a, l.level), f.tma_ok, a, f.layers, s, render_layer_cams(f, a, l.level),
                                              io.kind != MEAO_DEPTH_LINEAR_F32 ? 1 : 0, proj);
    }
    return launch_blur_upsample_lin_mixed(f.maps.low_ups[1], upsample_ao_map(f, 1), &f.maps.hq_ups[1], f.tma_ok, upsample_args(f, 1, io.ao, io.vp),
                                          upsample_lo_ao2(f, 1), f.occ_pitch[1], io.depth, f.layers, f.sm_count, proj, s);
}

// ---- the debug buffers (meao_get_buffer, meao_set_buffer, meao_debug_view) ---------------------------------------------------
// Buffer `id` (include/meao.h MEAO_BUF_*, 1..21) of a frame: its reference layout (slices x lh[level] x lw[level] elements of elem
// bytes per layer) and where layer 0 of it sits in the arena, every layer `layer` bytes after the one before.  TiledDepth<k> (16 slices
// of level k + 2) exists only as a view of LowDepth<k>, so its base, pitch and layer are LowDepth<k>'s.  Without an arena: null base.
struct BufferRef { int level, slices, elem; char *base; size_t pitch, layer; };

inline bool buffer_ref(const FrameState &f, int id, BufferRef &b)
{
    auto ref = [&](int level, int slices, int elem, void *base, size_t pitch, int k) { b = BufferRef{level, slices, elem, (char *)base, pitch, pitch * f.lh[k]}; };
    if (id == 1) ref(0, 1, 2, f.lin, (size_t)f.lin_pitch * 2, 0);
    else if (id >= 2 && id <= 5) { const int k = id - 1; ref(k, 1, 4, f.low[k], (size_t)f.low_pitch[k] * 4, k); }
    else if (id >= 6 && id <= 9) { const int k = id - 5; ref(k + 2, 16, 2, f.low[k], (size_t)f.low_pitch[k] * 4, k); }
    else if (id >= 10 && id <= 13) { const int k = id - 9; ref(k, 1, 1, f.occ[k], f.occ_pitch[k], k); }
    else if (id >= 14 && id <= 16) { const int k = id - 13; ref(k, 1, 1, f.comb[k], f.occ_pitch[k], k); }
    else if (id == 17) ref(0, 1, 1, f.result, f.result_pitch, 0);
    else if (id >= 18 && id <= 21) { const int k = id - 17; ref(k, 1, 1, f.hq[k], f.occ_pitch[k], k); }    // HighQuality1..4 (extension)
    else return false;
    return true;
}

// TiledDepth<k> of layer l in the reference layout (16 slices of lw[k + 2] x lh[k + 2] f16) into out, synthesised from LowDepth<k> with
// the layer's atlas padding for depth kind `kind`.  table_pad: the raw-ingest padding value of the layer's camera table entry, read back
// from the device (a bound device camera buffer derived it); nullptr: the plan's.
inline cudaError_t launch_tiled_atlas(const FrameState &f, int k, int l, int kind, __half *out, cudaStream_t s, const float *table_pad = nullptr)
{
    const float pad = table_pad ? (kind != MEAO_DEPTH_LINEAR_F32 ? *table_pad : 0.0f) : layer_pad(f, l, k, kind);
    return launch_synth_tiled(f.low[k] + (size_t)l * f.lh[k] * f.low_pitch[k], f.lw[k], f.lh[k], f.low_pitch[k], f.lw[k + 2], f.lh[k + 2],
                              pad, out, s);
}

// The debug view of layer l of buffer `id` into the W x H R8 image at out: TiledDepth<k> through Blit.shader pass 4 (AO.cs:810-814)
// with the layer's atlas padding for depth kind `kind`, every other buffer point-sampled (AO.cs:815-819).  false: no such buffer.
inline bool debug_view_args(const FrameState &f, int id, int l, int kind, uint8_t *out, DebugViewArgs &a)
{
    BufferRef b;
    if (!buffer_ref(f, id, b)) return false;
    a = DebugViewArgs{};
    a.W = f.W; a.H = f.H; a.out = out; a.out_pitch = f.W;
    a.src = b.base + (size_t)l * b.layer;
    a.sw = f.lw[b.level]; a.sh = f.lh[b.level];
    if (b.slices == 16) {
        const int k = b.level - 2;
        a.tiled = 1; a.elem = 4; a.spitch = f.low_pitch[k]; a.lw = f.lw[k]; a.lh = f.lh[k]; a.pad = layer_pad(f, l, k, kind);
    } else {
        a.elem = b.elem; a.spitch = (int)(b.pitch / b.elem);
    }
    return true;
}

// ---- row bands: what moves between neighbouring bands -------------------------------------------------------------------------
// The halo message of one side (meao_halo_pack): rows[k] of LowDepth<k>, level 1 first, in tight rows from `packed` on.  Appends one
// segment per non-empty level to a: pack copies the arena into the message, unpack the message into the arena.
inline void halo_segments(const FrameState &f, const Range rows[5], float *packed, bool pack, HaloArgs &a)
{
    for (int k = 1; k <= 4; k++) {
        const int n = rows[k].hi - rows[k].lo;
        if (n <= 0) continue;
        float *buf = f.low[k] + (size_t)rows[k].lo * f.low_pitch[k];
        a.seg[a.nseg++] = pack ? HaloSeg{buf, packed, f.low_pitch[k], f.lw[k], f.lw[k], n} : HaloSeg{packed, buf, f.lw[k], f.low_pitch[k], f.lw[k], n};
        packed += (size_t)n * f.lw[k];
    }
}

// The neighbour exchange towards `side` (band_exchange_kernel): rows[k] of LowDepth<k> go to the same byte offset in the neighbour's
// arena at `peer`, laid out like the local one at `arena`.  Whole pitched rows, so each level is one contiguous, 128-byte aligned copy.
inline void exchange_segments(const FrameState &f, const char *arena, char *peer, int side, const Range rows[5], XchgArgs &a)
{
    for (int k = 1; k <= 4; k++) {
        const int n = rows[k].hi - rows[k].lo;
        if (n <= 0) continue;
        const size_t off = (size_t)((const char *)(f.low[k] + (size_t)rows[k].lo * f.low_pitch[k]) - arena);
        a.seg[a.nseg++] = XchgSeg{(const uint4 *)(arena + off), (uint4 *)(peer + off), (uint32_t)((size_t)n * f.low_pitch[k] * sizeof(float) / 16), side};
    }
}

}  // namespace meao

#endif  // MEAO_FRAME_RECORD_H
