// frame_driver.cpp -- runs frames through the HOST-compiled kernel sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h), launched the
// way libmeao launches them: buffer placement, TMA maps, the frame schedule, argument blocks and launcher choice, and the buffer
// table, debug views, halo and exchange segments around the frame, all come from csrc/frame_record.h, the code meao_api.cu records
// its frames and serves its debug reads and row bands with.  What this driver adds is a host arena, the plan (the constants a
// plan-only libmeao context reports, handed in by the test) and what each frame form puts into its first and last launch.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

namespace meao_emu { long long surface_accesses = 0; }

namespace {

struct Frame : FrameState {
    char *arena = nullptr;
    size_t bytes = 0;
    int Wmax = 0, Hmax = 0;
    int use_tma = 1;        // 1: interior tiles take the kernels' TMA path (emulated box loads), 0: every tile gathers
    int ren_tile = -1;      // render_tile_variant's force (-1: the planner's rule)
    int zero_pitches = 0;   // pins the launchers' convention that zero pitches in PrepareArgs / DepthIn mean the tight views
    int kind = MEAO_DEPTH_RAW_F32;          // depth kind of the last prepare (the atlas padding of the tiled views)
    bool ao_elsewhere = false;              // the last final upsample stored into the caller's AO or an array, not the result buffer
    uint32_t host_error = 0;
    BandFlags &flags() { return *(BandFlags *)arena; }
};

Frame *F(void *h) { return (Frame *)h; }

// what meao_api.cu hands to cuTensorMapEncodeTiled
bool emu_map(CUtensorMap &m, const MapSpec &s)
{
    m = CUtensorMap{};
    m.base = s.base; m.elem = s.elem; m.w = s.w; m.h = s.h; m.pitch_bytes = (size_t)s.pitch_elems * s.elem; m.bw = s.bw; m.bh = s.bh;
    return true;
}

void whole_frame(Frame *f)
{
    f->band0 = 0; f->band1 = f->H;
    for (int k = 0; k <= 4; k++) f->need_c[k] = Range{0, f->lh[k]};
}

// The caller's depth (pitches vp, nullptr: tight) as the frame's first launch reads it
FrameIO frame_io(Frame *f, const void *depth, int kind, const ViewPitch *vp = nullptr)
{
    FrameIO io;
    io.kind = kind; io.depth = depth_in(*f, depth, kind, vp);
    if (f->zero_pitches) { io.depth.depth_pitch = 0; io.depth.depth_layer_pitch = 0; io.depth.ao_layer_pitch = 0; }
    return io;
}

// Launches [first, end) of the frame schedule, serially, through the shared launcher
void run_schedule(Frame *f, const FrameIO &io, size_t first, size_t end = SIZE_MAX)
{
    const std::vector<FrameLaunch> s = frame_schedule(f->plan.variants);
    end = std::min(end, s.size());
    if (first == 0) f->kind = io.kind;
    if (end == s.size()) f->ao_elsewhere = io.ao || io.aio;
    for (size_t i = first; i < end; i++) launch_entry(*f, s[i], io, f->ren_tile, nullptr);
}

}  // namespace

extern "C" {

// An arena laid out for Wmax x Hmax at `layers` layers, zeroed like a fresh context's; frame_resize places a frame in it.
void *frame_create(int Wmax, int Hmax, int layers)
{
    Frame *f = new Frame();
    f->layers = layers; f->Wmax = Wmax; f->Hmax = Hmax;
    f->bytes = arena_layout(Wmax, Hmax, layers).bytes;
    void *p = nullptr;
    if (posix_memalign(&p, 256, f->bytes)) abort();
    memset(p, 0, f->bytes);
    f->arena = (char *)p;
    f->flags().epoch = 1;
    return f;
}

void frame_destroy(void *h) { free(F(h)->arena); delete F(h); }

size_t frame_arena_bytes(void *h) { return F(h)->bytes; }

// The buffers of a W x H frame where meao_api.cu's place_size puts them; -1 if the size lies outside the arena's
int frame_resize(void *h, int W, int H)
{
    Frame *f = F(h);
    if (W < 1 || H < 1 || W > f->Wmax || H > f->Hmax) return -1;
    const ArenaLayout a = arena_layout(W, H, f->layers);
    if (a.bytes > f->bytes) return -1;
    f->W = W; f->H = H;
    place_frame(*f, a, f->arena, 0);
    encode_maps(*f, emu_map);
    whole_frame(f);
    return 0;
}

// The plan of the current size.  Per layer l: rc / rcw + 28 (4 l + k - 1) = meao_render_constants_layer(l, k, wide = 0 / 1),
// zb + 4 l = meao_zbuffer_params_layer(l), pad12[l] = the atlas padding value of levels 1-2 (Linearize(0)).  uc + 8 (lo - 1) =
// meao_upsample_constants(lo).  The camera tables go into the arena, as meao_api.cu uploads them.
void frame_set_plan(void *h, const float *rc, const float *rcw, const float *uc, const float *zb, const float *pad12, int reversed_z,
                    int hq_mask, int exhaustive, int single_scale, int use_tma, int ren_tile)
{
    Frame *f = F(h);
    Plan &p = f->plan;
    p = Plan{};
    p.variants.high_quality_mask = hq_mask; p.variants.sample_exhaustively = exhaustive; p.variants.single_scale = single_scale;
    p.reversed_z = reversed_z;
    f->layer_consts.assign(f->layers, CamConsts{});
    for (int l = 0; l < f->layers; l++) {
        CamConsts &cc = f->layer_consts[l];
        cc.zb[0] = zb[4 * l]; cc.zb[1] = zb[4 * l + 1];
        for (int k = 1; k <= 4; k++) {
            memcpy(cc.inv_thickness[k], rc + 28 * (4 * l + k - 1), 48);
            memcpy(cc.inv_thickness_wide[k], rcw + 28 * (4 * l + k - 1), 48);
            cc.pad[k] = k <= 2 ? pad12[l] : 0.0f;
        }
    }
    const CamConsts &c0 = f->layer_consts[0];          // the plan's camera constants are the first layer's
    memcpy(p.zb, zb, sizeof p.zb);
    memcpy(p.inv_thickness, c0.inv_thickness, sizeof p.inv_thickness);
    memcpy(p.inv_thickness_wide, c0.inv_thickness_wide, sizeof p.inv_thickness_wide);
    memcpy(p.pad, c0.pad, sizeof p.pad);
    for (int k = 1; k <= 4; k++) {
        memcpy(p.sample_weight[k], rc + 28 * (k - 1) + 12, 48);
        const float *u = uc + 8 * (k - 1);
        p.noise_filter_strength[k] = u[4]; p.step_size[k] = u[5]; p.blur_tolerance[k] = u[6]; p.upsample_tolerance[k] = u[7];
    }
    p.reject_fadeoff = rc[26]; p.intensity = rc[27];
    std::vector<LayerZ> tz;
    std::vector<LayerRender> tr;
    camera_tables(*f, tz, tr);
    memcpy(f->layer_zb, tz.data(), tz.size() * sizeof(LayerZ));
    memcpy(f->layer_ren, tr.data(), tr.size() * sizeof(LayerRender));
    f->use_tma = use_tma; f->ren_tile = ren_tile;
    f->tma_ok = use_tma != 0;
}

// ---- convention pins: what the launchers do with argument blocks libmeao itself no longer produces ---------------------------
// The layered and array kernels' null-table path (every layer takes the argument block's constants); until the next frame_resize.
void frame_null_tables(void *h) { F(h)->layer_zb = nullptr; F(h)->layer_ren = nullptr; }
// Zero depth / AO pitches in PrepareArgs and DepthIn, which the launchers resolve to the tight views.
void frame_zero_pitches(void *h, int on) { F(h)->zero_pitches = on; }

// ---- frame forms -----------------------------------------------------------------------------------------------------------------
// One frame from `depth` (kind: MEAO_DEPTH_*) into `ao` (NULL: the result buffer).  depth_row != 0: the depth and the AO are views
// with these byte pitches (meao_render_pitched); 0: tight.  fused: low-only prepare_depth and the final upsample that reads the raw
// depth (what meao_render records); 0: prepare_depth -> LinearDepth -> final upsample (the stage API, and array frames).
// row1 > row0 (fused, one layer): prepare_depth runs its full form over the whole depth (LowDepth1..4 with a band's halo) and only
// the final level's rows [row0, row1) take the fused kernel, reading the depth from its row row0 on and storing into `ao`, whose first
// row is row0 -- what the rows of one band compute once its halo rows have arrived.
void frame_run(void *h, const void *depth, int kind, int fused, long long depth_row, long long depth_layer, void *ao, long long ao_row,
               long long ao_layer, int row0, int row1)
{
    Frame *f = F(h);
    whole_frame(f);
    const ViewPitch v{depth_row, depth_layer, ao_row, ao_layer}, *vp = depth_row ? &v : nullptr;
    const bool band = fused && row1 > row0;
    FrameIO io = frame_io(f, depth, kind, vp);
    io.low_only = fused && !band; io.fused = fused != 0; io.ao = ao; io.vp = vp;
    if (!band) { run_schedule(f, io, 0); return; }
    const size_t n = frame_schedule(f->plan.variants).size();
    run_schedule(f, io, 0, n - 1);
    f->band0 = f->need_c[0].lo = row0; f->band1 = f->need_c[0].hi = row1;
    io.depth = frame_io(f, (const char *)depth + (size_t)row0 * (depth_row ? depth_row : f->W * depth_esize(kind)), kind, vp).depth;
    run_schedule(f, io, n - 1);
    whole_frame(f);
}

// the low-only prepare_depth alone, whole frame
void frame_prepare_low(void *h, const void *depth, int kind)
{
    whole_frame(F(h));
    FrameIO io = frame_io(F(h), depth, kind);
    io.low_only = true;
    run_schedule(F(h), io, 0, 1);
}

// A CUDA-array frame (meao_render_arrays): depth: `layers` images of W x H elements (4 bytes: f32, 2 bytes: D16 codes) with rows
// depth_pitch bytes apart, in an emulated array of shape depth_shape (0 2-D, 1 layered, 2 cube); ao: the same for the AO (1 byte per pixel).
void frame_run_arrays(void *h, void *depth, int kind, int depth_shape, long long depth_pitch, void *ao, int ao_shape, long long ao_pitch)
{
    Frame *f = F(h);
    whole_frame(f);
    const meao_emu::Surface ds{depth, (int)depth_esize(kind), f->W, f->H, depth_shape == 2 ? 6 : f->layers, (size_t)depth_pitch, depth_shape};
    const meao_emu::Surface as{ao, 1, f->W, f->H, ao_shape == 2 ? 6 : f->layers, (size_t)ao_pitch, ao_shape};
    // what meao_api.cu check_array derives from an array: how the kernels address its layers
    auto surf_kind = [](int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : shape == meao_emu::SURF_LAYERED ? kSurfLayered : kSurfCube; };
    const ArrayIO aio{(cudaSurfaceObject_t)&ds, (cudaSurfaceObject_t)&as, surf_kind(depth_shape), surf_kind(ao_shape), ao};
    FrameIO io = frame_io(f, nullptr, kind);
    io.aio = &aio;
    run_schedule(f, io, 0);
}

// ---- row bands: the two phases of meao_band_phase_a / _b around the neighbour exchange ----------------------------------
// produce10 = meao_band_rows()[0..9]: rows of level k = 0..4 to produce; [row0, row1) = the band itself
void frame_set_band(void *h, int row0, int row1, const int *produce10)
{
    Frame *f = F(h);
    f->band0 = row0; f->band1 = row1;
    for (int k = 0; k <= 4; k++) f->need_c[k] = Range{produce10[2 * k], produce10[2 * k + 1]};
}

// depth_band: the band's rows only (row1 - row0 rows), like meao_render_band_prepare
void frame_band_phase_a(void *h, const void *depth_band, int kind) { run_schedule(F(h), frame_io(F(h), depth_band, kind), 0, 1); }

// the launches after the prepare into the result buffer, like meao_band_phase_b and meao_render_band_finish
void frame_band_phase_b(void *h) { run_schedule(F(h), frame_io(F(h), nullptr, F(h)->kind), 1); }

// rows8 = meao_halo_rows(side, send): {lo1,hi1, ..., lo4,hi4}, as the rows[k] of LowDepth<k> frame_record.h's segment builders take
static void halo_rows(const int *rows8, Range rows[5])
{
    rows[0] = Range{0, 0};
    for (int k = 1; k <= 4; k++) rows[k] = Range{rows8[2 * (k - 1)], rows8[2 * (k - 1) + 1]};
}

// meao_halo_pack / meao_halo_unpack of the side rows8 describes, through the segments of meao_band_phase_a / _b's halo_copy_kernel
void frame_halo(void *h, const int *rows8, float *packed, int pack)
{
    Range rows[5]; halo_rows(rows8, rows);
    HaloArgs a{};
    halo_segments(*F(h), rows, packed, pack != 0, a);
    launch_halo_copy(a, nullptr);
}

// ---- native neighbour exchange: band_exchange_kernel with the segments meao_api.cu's record_exchange builds.  up / down: the
// neighbours' handles (NULL = none), frames of the same size; rows_up8 / rows_down8 = meao_halo_rows(side, send = 1).  The fiber
// emulator runs one grid at a time, so the test presets the flags a concurrently running neighbour would have written
// (frame_band_flags).  Returns the kernel's sticky error.
int frame_band_exchange(void *h, void *up, void *down, const int *rows_up8, const int *rows_down8, int timeout_polls)
{
    Frame *f = F(h);
    Frame *peer[2] = {F(up), F(down)};
    const int *rows8[2] = {rows_up8, rows_down8};
    XchgArgs a{};
    a.local = &f->flags(); a.host_error = &f->host_error;
    a.timeout_ns = (unsigned long long)timeout_polls * 1000ull;       // the emulated global timer advances 1000 "ns" per read
    for (int side = 0; side < 2; side++) {
        if (!peer[side]) continue;
        a.peer[side] = &peer[side]->flags();
        Range rows[5]; halo_rows(rows8[side], rows);
        exchange_segments(*f, f->arena, peer[side]->arena, side, rows, a);
    }
    launch_band_exchange(a, nullptr);
    return (int)f->flags().error;
}

// out8 = ready[2], ack[2], epoch, done, error, host_error;  set_ready_ack4 (may be NULL) overwrites ready / ack first
void frame_band_flags(void *h, const int *set_ready_ack4, int *out8)
{
    Frame *f = F(h);
    BandFlags &b = f->flags();
    if (set_ready_ack4) { for (int i = 0; i < 2; i++) { b.ready[i] = set_ready_ack4[i]; b.ack[i] = set_ready_ack4[2 + i]; } }
    if (out8) {
        out8[0] = b.ready[0]; out8[1] = b.ready[1]; out8[2] = b.ack[0]; out8[3] = b.ack[1];
        out8[4] = b.epoch; out8[5] = b.done; out8[6] = b.error; out8[7] = f->host_error;
    }
}

// ---- poison and fill: what a kernel must never read -------------------------------------------------------------------------------
// what = 0: every image byte of the arena := 0xFF (stale data where a fresh context holds zeros); 1: LinearDepth := NaN;
// 2: LowDepth1..4 := NaN (rows a band neither produces nor receives must never reach an output)
void frame_poison(void *h, int what)
{
    Frame *f = F(h);
    const size_t L = f->layers;
    if (what == 0) { const size_t off = arena_layout(f->Wmax, f->Hmax, f->layers).lin; memset(f->arena + off, 0xFF, f->bytes - off); }
    if (what == 1) { const uint16_t nan = 0x7e00; for (size_t i = 0; i < L * f->lin_pitch * f->H; i++) memcpy(&f->lin[i], &nan, 2); }
    if (what == 2)
        for (int k = 1; k <= 4; k++) for (size_t i = 0; i < L * f->low_pitch[k] * f->lh[k]; i++) f->low[k][i] = __uint_as_float(0x7fc00000u);
}

// ---- reading the buffers back ------------------------------------------------------------------------------------------------------
// buffer <id> (1..21) of layer `layer` in the reference layout / native type, like one layer of meao_get_buffer
int frame_get_buffer(void *h, int id, int layer, void *out)
{
    Frame *f = F(h);
    BufferRef b;
    if (layer < 0 || layer >= f->layers || !buffer_ref(*f, id, b)) return -1;
    if (id == 17 && f->ao_elsewhere)                    // meao_get_buffer: the context's own copy of an AO stored elsewhere
        launch_entry(*f, frame_schedule(f->plan.variants).back(), FrameIO{}, f->ren_tile, nullptr);
    if (b.slices == 16) { launch_tiled_atlas(*f, b.level - 2, layer, f->kind, (__half *)out, nullptr); return 0; }
    const size_t wb = (size_t)f->lw[b.level] * b.elem;
    for (int y = 0; y < f->lh[b.level]; y++) memcpy((char *)out + y * wb, b.base + layer * b.layer + y * b.pitch, wb);
    return 0;
}

// the debug view of buffer <id> of a single-layer frame (meao_debug_view) into out[W * H]
int frame_debug_view(void *h, int id, uint8_t *out)
{
    DebugViewArgs a;
    if (!debug_view_args(*F(h), id, 0, F(h)->kind, out, a)) return -1;
    launch_debug_view(a, nullptr);
    return 0;
}

// Blit.shader passes 1 / 2 on host buffers (launch_composite): color updated in place
void frame_composite(const uint8_t *ao, void *color, long long npix, int half, int rgb, int alpha, int one_minus)
{
    launch_composite(ao, color, npix, half, rgb, alpha, one_minus, nullptr);
}

void frame_composite_debug(const uint8_t *view, void *color, long long npix, int half) { launch_debug_composite(view, color, npix, half, nullptr); }

// ---- the frame schedule ------------------------------------------------------------------------------------------------------------
// frame_schedule of variants4 = MeaoVariants {single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale}: launch i as
// out5[5 i .. 5 i + 4] = stage, level, branch, wait, PDL class, and its meao_profile_frame name at names + 32 i.  Returns the count.
int frame_schedule_export(const int *variants4, int *out5, char *names, int cap)
{
    const MeaoVariants v{variants4[0], variants4[1], variants4[2], variants4[3]};
    const std::vector<FrameLaunch> s = frame_schedule(v);
    for (size_t i = 0; i < s.size() && (int)i < cap; i++) {
        const FrameLaunch &l = s[i];
        const int row[5] = {l.stage, l.level, l.branch, l.wait, l.pdl};
        memcpy(out5 + 5 * i, row, sizeof row);
        snprintf(names + 32 * i, 32, "%s", launch_name(l).c_str());
    }
    return (int)s.size();
}

// ---- the kernel units (kernels.h kKernelUnits): unit i's file at names + 32 i, the kernel count of its table in counts[i] ----------
int frame_kernel_units(char *names, int *counts, int cap)
{
    int n = 0;
    for (const KernelUnit *u : kKernelUnits) {
        if (n < cap) { snprintf(names + 32 * n, 32, "%s", u->file); counts[n] = u->walk(nullptr); }
        n++;
    }
    return n;
}

// ---- counters and self-checks -----------------------------------------------------------------------------------------------------
long long frame_tma_box_loads() { return meao_emu::tma_box_loads; }
long long frame_surface_accesses() { return meao_emu::surface_accesses; }

// the launch ledger (cuda_emu.h): which kernels ran since the reset, how often, with how many TMA box loads and over how many CTAs
void frame_ledger_reset() { meao_emu::ledger_reset(); }
int frame_ledger_read(unsigned long long *offset, long long *launches, long long *tma_loads, long long *ctas, int cap)
{
    return meao_emu::ledger_read(offset, launches, tma_loads, ctas, cap);
}

// aborts (on purpose) with the emulated TMA's alignment complaint: an f32 box starting at x = 3
int emu_selfcheck_unaligned_tma()
{
    alignas(128) static float src[64 * 8], dst[16 * 4];
    CUtensorMap m;
    emu_map(m, MapSpec{src, 4, 64, 8, 64, 16, 4});
    meao_emu::tma_load_2d(dst, &m, 3, 0);
    return 0;
}

}  // extern "C"
