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
    // the plan inputs the recorders read besides the constants: the variants and the cameras' Z direction
    MeaoVariants variants;
    int reversed_z;
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
    CUtensorMap ao_ups[5];                  // lo AO of upsample lo level k (Occlusion4 / Combined k)
    CUtensorMap hq_ups[5];                  // HighQuality<k> as LoResAO2 of upsample lo level k
    CUtensorMap occ1_ups;                   // Occlusion1 as LoResAO1 of the final upsample (MeaoVariants.single_scale)
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

    int sm_count = 132;                     // SMs of the device (132 = H100 SXM for plan-only contexts)
    bool tma_ok = false;
    FrameMaps maps;

    Plan plan;
    std::vector<CamConsts> layer_consts;    // the plan's camera constants of every layer (all alike without a layer-camera table)
};

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
        ok &= enc(m.ao_ups[k], MapSpec{(k == 4) ? f.occ[4] : f.comb[k], 1, f.lw[k], mh, f.occ_pitch[k], kUpsAoBoxW, kUpsAoBoxH});
        ok &= enc(m.hq_ups[k], MapSpec{f.hq[k], 1, f.lw[k], mh, f.occ_pitch[k], kUpsAoBoxW, kUpsAoBoxH});
    }
    ok &= enc(m.occ1_ups, MapSpec{f.occ[1], 1, f.lw[1], f.layers * f.lh[1], f.occ_pitch[1], kUpsAoBoxW, kUpsAoBoxH});
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
struct ArrayIO { cudaSurfaceObject_t depth, ao; int depth_surf, ao_surf; const void *ao_array; };

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
// with the same depth (launch_upsample's `fused`) and writes LinearDepth itself.
inline cudaError_t launch_prepare(const FrameState &f, const PrepareArgs &a, const ArrayIO *aio, bool low_only, cudaStream_t s)
{
    if (aio) return launch_prepare_depth_array(a, aio->depth, aio->depth_surf, f.layers, s, f.layer_zb);
    if (f.layers > 1) return launch_prepare_depth_layered(a, f.layers, s, low_only, f.layer_zb);
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

// The render launch of level k with the map of a.tile_h; a layered frame takes its layers' camera table entries
inline cudaError_t launch_render(const FrameState &f, const RenderArgs &a, int k, int kind, cudaStream_t s)
{
    int tv = 0;
    while (tv + 1 < kRenderTileVariants && kRenderTileHs[tv] != a.tile_h) tv++;
    const CUtensorMap &map = a.wide ? f.maps.low_wide[tv][k] : f.maps.low_ren[tv][k];
    if (f.layers == 1) return launch_render_ao(map, f.tma_ok, a, s);
    const LayerRender *ren = f.layer_ren ? f.layer_ren + (size_t)(2 * (k - 1) + a.wide) * f.layers : nullptr;
    return launch_render_ao_layered(map, f.tma_ok, a, f.layers, s, ren, kind != MEAO_DEPTH_LINEAR_F32 ? 1 : 0);
}

// PushUpsampleCommands with the wiring of AO.cs:528-531, lo level `lo`.  ao_out (final level only): the caller's AO at the pitches
// of vp (nullptr: tight), its first row band0; nullptr: the context's result buffer.
inline UpsampleArgs upsample_args(const FrameState &f, int lo, void *ao_out, const ViewPitch *vp)
{
    const int hi = lo - 1;
    const bool single = f.plan.variants.single_scale != 0 && lo == 1;     // LoResAO1 = Occlusion1: no coarser level contributes
    UpsampleArgs a{};
    a.lo_depth = f.low[lo]; a.low = f.lw[lo]; a.loh = f.lh[lo]; a.lo_dpitch = f.low_pitch[lo];
    a.lo_ao = single ? f.occ[1] : (lo == 4) ? f.occ[4] : f.comb[lo]; a.lo_apitch = f.occ_pitch[lo];
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
inline cudaError_t launch_upsample(const FrameState &f, int lo, const UpsampleArgs &a, const ArrayIO *aio, const DepthIn *fused, cudaStream_t s)
{
    const bool final_level = lo == 1;
    const uint8_t *lo_ao2 = hq_level(f, lo) ? f.hq[lo] : nullptr;                   // kernels main_premin / main_premin_blendout
    const CUtensorMap &ao_map = (f.plan.variants.single_scale != 0 && final_level) ? f.maps.occ1_ups : f.maps.ao_ups[lo];
    const CUtensorMap &dm = f.maps.low_ups[lo], *hm = &f.maps.hq_ups[lo];
    if (fused && final_level)
        return launch_blur_upsample_lin(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], *fused, f.layers, f.sm_count, s);
    if (aio && final_level)
        return launch_blur_upsample_array(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.layers, f.sm_count, aio->ao, aio->ao_surf, s);
    if (f.layers > 1) return launch_blur_upsample_layered(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.layers, f.sm_count, s);
    return launch_blur_upsample(dm, ao_map, hm, f.tma_ok, a, lo_ao2, f.occ_pitch[lo], f.sm_count, s);
}

// ---- the frame schedule: which kernels a frame launches, in what order, on which stream and after which other launch ----------
enum FrameStage { kStagePrepare, kStageRender, kStageRenderWide, kStageUpsample };
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

// The launches of one frame in serial order (RebuildCommandBuffers, AO.cs:511-531): prepare, render 1..k, the wide renders of the
// high_quality_mask levels, upsamples k..1.  The branches make it a DAG: the four render levels are independent (SURVEY.md 3.2), a
// level's wide render rides on its branch, the coarse upsample chain 4->3->2 only needs Occlusion2..4, and only the last two upsamples
// wait for the big level-1 render.  single_scale (BASELINE.json configs[0]): prepare, render 1 and the final-style upsample on Occlusion1.
inline std::vector<FrameLaunch> frame_schedule(const MeaoVariants &v)
{
    const int kmax = v.single_scale ? 1 : 4;
    std::vector<FrameLaunch> s;
    int last[4] = {0, 0, 0, 0};             // the last launch on each branch so far
    auto add = [&](int stage, int level, int branch, int wait, int pdl) {
        last[branch] = (int)s.size();
        s.push_back(FrameLaunch{stage, level, branch, wait, pdl});
    };
    add(kStagePrepare, 0, 0, -1, kPdlNever);
    for (int k = 1; k <= kmax; k++) add(kStageRender, k, k - 1, k == 1 ? -1 : 0, k == 1 ? kPdlFrom1 : kPdlNever);
    for (int k = 1; k <= kmax; k++)
        if ((v.high_quality_mask >> (k - 1)) & 1) add(kStageRenderWide, k, k - 1, -1, kPdlFrom1);
    if (kmax == 4) {
        add(kStageUpsample, 4, 3, last[2], kPdlFrom2);
        add(kStageUpsample, 3, 3, last[1], kPdlFrom2);
        add(kStageUpsample, 2, 0, last[3], kPdlFrom2);
    }
    add(kStageUpsample, 1, 0, -1, kPdlFrom1);
    return s;
}

// The launch's name in meao_profile_frame: "prepare_depth", "render_ao L1", "render_ao_wide L1", "blur_upsample L2->L1"
inline std::string launch_name(const FrameLaunch &l)
{
    const std::string k = std::to_string(l.level);
    switch (l.stage) {
        case kStagePrepare: return "prepare_depth";
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
};

// Launches schedule entry l of a frame on stream s.  force_tile: render_tile_variant's force.
inline cudaError_t launch_entry(const FrameState &f, const FrameLaunch &l, const FrameIO &io, int force_tile, cudaStream_t s)
{
    const bool final_level = l.stage == kStageUpsample && l.level == 1;
    switch (l.stage) {
        case kStagePrepare: return launch_prepare(f, prepare_args(f, io.depth), io.aio, io.low_only, s);
        case kStageRender:
        case kStageRenderWide:
            return launch_render(f, render_args(f, l.level, io.kind, l.stage == kStageRenderWide, force_tile), l.level, io.kind, s);
        default:
            return launch_upsample(f, l.level, upsample_args(f, l.level, final_level ? io.ao : nullptr, final_level ? io.vp : nullptr),
                                   io.aio, io.fused ? &io.depth : nullptr, s);
    }
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
// the layer's atlas padding for depth kind `kind`
inline cudaError_t launch_tiled_atlas(const FrameState &f, int k, int l, int kind, __half *out, cudaStream_t s)
{
    return launch_synth_tiled(f.low[k] + (size_t)l * f.lh[k] * f.low_pitch[k], f.lw[k], f.lh[k], f.low_pitch[k], f.lw[k + 2], f.lh[k + 2],
                              layer_pad(f, l, k, kind), out, s);
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
