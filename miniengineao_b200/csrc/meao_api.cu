// meao_api.cu -- context, planner and C ABI of libmeao.so (see include/meao.h).
//
// Host-side mirror of the parts of AmbientOcclusion.cs that own the hot path:
//   RTHandle geometry/formats (AO.cs:124-282), the CPU constant math of the three Push*Commands
//   recorders (AO.cs:561-593, 660-734, 750-771), the record order of RebuildCommandBuffers
//   (AO.cs:511-531) and the re-plan triggers of LateUpdate (AO.cs:329-350).
// "Plan once, replay per frame" maps to: constants + TMA descriptors are rebuilt only when a
// parameter, the camera or the size changes; a frame is then ten kernel launches (or one CUDA
// graph launch) on one stream.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <unistd.h>

#include <nvtx3/nvToolsExt.h>

#include "../../include/meao.h"
#include "common.cuh"
#include "kernels.h"
#include "arena_layout.h"
#include "frame_record.h"

using namespace meao;

namespace {

thread_local std::string g_create_error;

inline Range clampr(Range r, int n) { Range o{r.lo < 0 ? 0 : r.lo, r.hi > n ? n : r.hi}; if (o.hi < o.lo) o.hi = o.lo; return o; }

// cuTensorMapEncodeTiled is fetched through the runtime so libmeao.so has no link-time
// dependency on libcuda (it must load on a machine without a driver for the ABI tests).
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Everything of a context that depends on the frame size: what the recorders read (frame_record.h FrameState) plus the band's
// neighbours and row ranges and the state of the per-layer camera table slot.  A reserved context (meao_reserve) keeps one of these
// per recently used size (MeaoCtx::size_slots) and swaps it in on a resize to that size, so a return to a planned size is host bookkeeping only.
struct SizeState : FrameState {
    int prev0 = -1, next1 = -1;             // the neighbour bands' extents (meao_set_row_band)
    Range need_low[5];                      // rows of LowDepth<k> required by this band
    Range own_low[5];                       // rows of LowDepth<k> this band produces
    bool cam_table_stale = true;            // a structural re-plan changed layer_consts (ensure_ready uploads them after a device synchronise)
    int slot = 0;                           // the arena slot of this size's camera tables (FrameState::layer_zb / layer_ren)
    bool table_pending = false;             // the slot's tables are not written yet: the next frame writes them on its own stream
    uint64_t plan_gen = 0;                  // the frame-constant generation (MeaoCtx::consts_gen) this size's plan was built at
};

}  // namespace

struct MeaoCtx : SizeState {
    int device = 0;
    bool plan_only = false;                 // device < 0: host-side planning only (no CUDA calls at all)
    uint32_t flags = 0;
    std::string error;
    cudaStream_t stream = nullptr;
    cudaStream_t branch[3] = {nullptr, nullptr, nullptr};   // forked capture streams: the graph runs independent levels side by side
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    PFN_encodeTiled encode = nullptr;

    MeaoParams params;
    MeaoCamera camera;
    std::vector<MeaoCamera> layer_cams;     // meao_set_layer_cameras: one camera per layer, or empty (every layer uses `camera`)
    MeaoVariants variants = {0, 0, 0, 0};
    bool plan_dirty = true;                 // a structural input changed: the next frame re-plans (replan)
    // Frame constants (include/meao.h): bumped by every change of MeaoParams or of a camera that keeps the Z direction.  A size whose
    // plan_gen is older re-plans its constants on the host (refresh_constants); a graph captured at an older one re-targets (launch_cached).
    uint64_t consts_gen = 0;

    // meao_reserve: the arena is laid out for res_w x res_h (0 x 0: for the current size) and every size inside it keeps its plan
    int res_w = 0, res_h = 0;
    struct SizeSlot { bool valid = false; uint64_t last_use = 0; SizeState s; };
    SizeSlot size_slots[kSizeSlots];        // slot i: the parked state of a planned size whose camera tables live in arena slot i
    uint64_t size_clock = 0;
    int64_t arena_allocations = 0, graph_instantiations = 0;

    void *arena = nullptr;
    size_t arena_bytes = 0;
    // staging for the host path: two slots so that the H2D copy of frame i+1 overlaps the kernels and the
    // D2H copy of frame i (meao_render_host_async).  At the offsets of the arena's own size (the reservation's when reserved), so no
    // size's intermediates ever share bytes with them.
    float *depth_stage[2] = {nullptr, nullptr};     // device, layers*W*H each
    uint8_t *ao_stage[2] = {nullptr, nullptr};      // device, layers*W*H each
    cudaStream_t slot_stream[2] = {nullptr, nullptr};
    cudaEvent_t slot_done[2] = {nullptr, nullptr};
    cudaEvent_t compute_done = nullptr;
    bool compute_done_valid = false;

    // native neighbour exchange (meao_band_export / _connect / _step)
    BandFlags *band_flags = nullptr;        // first 256 bytes of the arena
    void *peer_base[2] = {nullptr, nullptr};    // the neighbours' arenas through a peer mapping (same layout as ours)
    bool peer_ipc[2] = {false, false};      // mapping came from cudaIpcOpenMemHandle (must be closed)
    unsigned long long band_timeout_ns = 2000000000ull;
    uint32_t *host_error = nullptr;         // pinned + mapped: the exchange kernel mirrors its sticky error here (read by meao_band_step without a CUDA call)
    uint32_t *host_error_dev = nullptr;     // device alias of host_error
    int pdl_level = -1;                     // programmatic dependent launch in the captured graphs: -1 untried, 0 none, 1 plain chains, 2 all same-stream edges

    int64_t launches = 0;

    // CUDA graph cache: one instantiated graph per (depth, out, kind), LRU; when it is full the least recently used
    // executable graph is RE-TARGETED in place with cudaGraphExecUpdate (same topology, new pointers: no device
    // synchronisation, launches already enqueued are unaffected), and so is a graph captured before the frame constants last
    // changed, at its next launch (new kernel arguments).  Dropped as a whole only when a structural plan input changes.
    // kind: the depth kind of a pointer frame; 100+ / 200+ / 300+ band graphs; kArrayGraphKind+ array frames (the key holds
    // cudaArray_t handles, so a pointer equal to a handle value never finds an array frame's graph, nor the reverse).
    // pitch: the byte pitches of a pointer frame's depth and AO views (meao_render_pitched; 0 for the other kinds) -- a frame at the
    // same pointers with other pitches is another graph, never a replay that reads the wrong rows.
    // size: the frame size and camera table slot the graph was captured at (launch_cached fills it in) -- a reserved context keeps the
    // graphs of every size it has visited, and a size re-planned into another slot never replays a graph that reads the old slot.
    struct GraphKey { const void *p[4]; int kind; int64_t pitch[4] = {0, 0, 0, 0}; int size[3] = {0, 0, 0}; bool operator<(const GraphKey &o) const {
        for (int i = 0; i < 4; i++) if (p[i] != o.p[i]) return p[i] < o.p[i];
        if (kind != o.kind) return kind < o.kind;
        for (int i = 0; i < 4; i++) if (pitch[i] != o.pitch[i]) return pitch[i] < o.pitch[i];
        for (int i = 0; i < 3; i++) if (size[i] != o.size[i]) return size[i] < o.size[i];
        return false; } };
    // launches: the kernels its capture recorded; gen: the plan_gen of the constants it launches with
    struct GraphEntry { cudaGraphExec_t exec; uint64_t last_use; int launches; uint64_t gen; };
    std::map<GraphKey, GraphEntry> graphs;
    // executable graphs that cudaGraphExecUpdate could not re-target while they were possibly in flight; `done` is recorded after the
    // frame that replaced them, so once it has completed (and, frames of a context running in order, every earlier frame) the graph
    // is destroyed without a device synchronise (reclaim_retired)
    struct Retired { cudaGraphExec_t exec; cudaEvent_t done; };
    std::vector<Retired> retired;
    uint64_t graph_clock = 0;
    bool graphs_stale = false;              // set by the device-less getters: dropped by the next ensure_ready (on the right device)
    void *last_out = nullptr;               // where the last final upsample wrote (nullptr: c->result; an array frame: its AO array)
    // CUDA-array frames (meao_render_arrays): one surface object per cudaArray_t this context has rendered with, made on first use.
    // A surface object describes the memory of its array, so it lives exactly as long as the graphs that launch with it: it is
    // destroyed by meao_release_array (that array) and drop_graph (all), both after a device synchronise -- never while a launch
    // that uses it may still be in flight.
    std::map<const void *, cudaSurfaceObject_t> surfaces;
    int last_kind = MEAO_DEPTH_RAW_F32;     // ingest kind of the last downsample (selects the atlas padding value)

    std::vector<std::pair<std::string, float>> last_profile;
    int profile_repeats = 1;                // launches per kernel inside one event pair of meao_profile_frame
};

namespace {

int fail(MeaoCtx *c, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (c) c->error = buf; else g_create_error = buf;
    return code;
}
// Row bands and layered frames exclude each other: a band's halo rows are whole rows of ONE image.
int refuse_layered(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands need a single-layer context (this one has %d layers, meao_set_layers)", what, c->layers);
}
// Row bands and reservations exclude each other too: every arena of one frame size must have one layout (DESIGN.md 4).
int refuse_reserved(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands need an unreserved context (this one reserves %dx%d, meao_reserve)", what, c->res_w, c->res_h);
}
#define BAND_GUARD(c, what) do { if ((c) && (c)->layers > 1) return refuse_layered((c), (what)); \
    if ((c) && (c)->res_w > 0) return refuse_reserved((c), (what)); } while (0)
#define CUDA_TRY(c, expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) \
    return fail((c), MEAO_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); } while (0)

// Mathf.Sqrt / Mathf.Pow are (float)Math.X((double)...) in Unity
float mathf_sqrt(float f) { return (float)std::sqrt((double)f); }
float mathf_pow(float f, float p) { return (float)std::pow((double)f, (double)p); }

// AO.cs:577-590
void sample_thickness(float t[12])
{
    t[0] = mathf_sqrt(1 - 0.2f * 0.2f);                 t[1] = mathf_sqrt(1 - 0.4f * 0.4f);
    t[2] = mathf_sqrt(1 - 0.6f * 0.6f);                 t[3] = mathf_sqrt(1 - 0.8f * 0.8f);
    t[4] = mathf_sqrt(1 - 0.2f * 0.2f - 0.2f * 0.2f);   t[5] = mathf_sqrt(1 - 0.2f * 0.2f - 0.4f * 0.4f);
    t[6] = mathf_sqrt(1 - 0.2f * 0.2f - 0.6f * 0.6f);   t[7] = mathf_sqrt(1 - 0.2f * 0.2f - 0.8f * 0.8f);
    t[8] = mathf_sqrt(1 - 0.4f * 0.4f - 0.4f * 0.4f);   t[9] = mathf_sqrt(1 - 0.4f * 0.4f - 0.6f * 0.6f);
    t[10] = mathf_sqrt(1 - 0.4f * 0.4f - 0.8f * 0.8f);  t[11] = mathf_sqrt(1 - 0.6f * 0.6f - 0.6f * 0.6f);
}

// Z direction of the context's cameras (meao_set_layer_cameras requires one for all layers)
inline int ctx_reversed_z(const MeaoCtx *c) { return c->layer_cams.empty() ? c->camera.reversed_z : c->layer_cams[0].reversed_z; }

// A change of the cameras in effect.  Their near and far planes and fields of view are frame constants; their Z direction selects
// kernel instantiations (prepare_slot), so a change of it re-plans like any structural input.
void note_camera_change(MeaoCtx *c, int old_reversed_z, int new_reversed_z)
{
    if (old_reversed_z != new_reversed_z) c->plan_dirty = true;
    else c->consts_gen++;
}

// The camera-dependent constants of camera `cam` (the part of build_plan that reads the camera).
void camera_consts(const MeaoCtx *c, const MeaoCamera &cam, CamConsts &p)
{
    // AO.cs:561-568
    const float fpn = cam.far_clip / cam.near_clip;
    if (cam.reversed_z) { p.zb[0] = fpn - 1; p.zb[1] = 1; } else { p.zb[0] = 1 - fpn; p.zb[1] = fpn; }

    float thick[12];
    sample_thickness(thick);
    for (int k = 1; k <= 4; k++) {
        const int src_w = c->lw[k + 2];
        const float ScreenspaceDiameter = 10;                                                        // AO.cs:669
        float ThicknessMultiplier = 2 * cam.tan_half_fov_h * ScreenspaceDiameter / src_w;           // AO.cs:678
        if (c->variants.single_pass_stereo) ThicknessMultiplier *= 2;                                // AO.cs:680
        float InverseRangeFactor = 1 / ThicknessMultiplier;                                          // AO.cs:683
        for (int i = 0; i < 12; i++) p.inv_thickness[k][i] = InverseRangeFactor / thick[i];          // AO.cs:687-688
        {   // the same recorder fed a non-tiled source (LowDepth<k>): kernel "main"
            float tm = 2 * cam.tan_half_fov_h * ScreenspaceDiameter / c->lw[k];                     // AO.cs:678
            tm *= 2;                                                                                 // AO.cs:679 (!source.isTiled)
            if (c->variants.single_pass_stereo) tm *= 2;                                             // AO.cs:680
            const float irf = 1 / tm;                                                                // AO.cs:683
            for (int i = 0; i < 12; i++) p.inv_thickness_wide[k][i] = irf / thick[i];
        }
        // value of the atlas padding texels (SURVEY.md P3): Downsample1 writes Linearize(OOB load = 0),
        // Downsample2 writes 0 (its OOB load of DS4x)
        float pad = 0.0f;
        if (k <= 2) {
            // raw depth 0 through Linearize (DS1:40-45); linear ingest: 0
            pad = cam.reversed_z ? 1e5f : 1.0f / std::fmaf(p.zb[0], 0.0f, p.zb[1]);
        }
        p.pad[k] = pad;   // the depth-kind dependent part (linear ingest -> 0) is applied at launch
    }
}

// Rebuild the per-dispatch constants (the CPU half of RebuildCommandBuffers, AO.cs:496-540).
void build_plan(MeaoCtx *c)
{
    Plan &p = c->plan;
    // every layer's camera constants: one entry per distinct camera computed, copied to the layers that share it
    const int L = c->layers;
    c->layer_consts.resize(L);
    if (c->layer_cams.empty()) {
        camera_consts(c, c->camera, c->layer_consts[0]);
        for (int l = 1; l < L; l++) c->layer_consts[l] = c->layer_consts[0];
    } else {
        for (int l = 0; l < L; l++) {
            if (l > 0 && memcmp(&c->layer_cams[l], &c->layer_cams[l - 1], sizeof(MeaoCamera)) == 0) c->layer_consts[l] = c->layer_consts[l - 1];
            else camera_consts(c, c->layer_cams[l], c->layer_consts[l]);
        }
    }
    // the Plan's own camera constants: the first layer's
    const CamConsts &cc = c->layer_consts[0];
    p.zb[0] = cc.zb[0]; p.zb[1] = cc.zb[1];
    p.zb[2] = p.zb[3] = 0;
    p.variants = c->variants;
    p.reversed_z = ctx_reversed_z(c);
    memcpy(p.inv_thickness, cc.inv_thickness, sizeof p.inv_thickness);
    memcpy(p.inv_thickness_wide, cc.inv_thickness_wide, sizeof p.inv_thickness_wide);
    memcpy(p.pad, cc.pad, sizeof p.pad);

    float thick[12];
    sample_thickness(thick);
    for (int k = 1; k <= 4; k++) {
        const int src_w = c->lw[k + 2], src_h = c->lh[k + 2];
        p.inv_slice_dim_wide[k][0] = 1.0f / c->lw[k]; p.inv_slice_dim_wide[k][1] = 1.0f / c->lh[k];
        static const float mult[12] = {4, 4, 4, 4, 4, 8, 8, 8, 4, 8, 8, 4};                          // AO.cs:696-707
        float *w = p.sample_weight[k];
        for (int i = 0; i < 12; i++) w[i] = mult[i] * thick[i];
        if (!c->variants.sample_exhaustively) { w[0] = 0; w[2] = 0; w[5] = 0; w[7] = 0; w[9] = 0; }  // AO.cs:709-715
        float total = 0.0f;
        for (int i = 0; i < 12; i++) total += w[i];                                                  // AO.cs:718-721
        for (int i = 0; i < 12; i++) w[i] /= total;                                                  // AO.cs:723-724
        p.inv_slice_dim[k][0] = 1.0f / src_w; p.inv_slice_dim[k][1] = 1.0f / src_h;                  // AO.cs:732
    }
    p.reject_fadeoff = -1 / c->params.thickness_modifier;                                            // AO.cs:733
    p.intensity = c->params.intensity;                                                               // AO.cs:734

    for (int lo = 1; lo <= 4; lo++) {
        const int lo_w = c->lw[lo], lo_h = c->lh[lo], hi_w = c->lw[lo - 1], hi_h = c->lh[lo - 1];
        float stepSize = 1920.0f / lo_w;                                                             // AO.cs:760
        float blurTolerance = 1 - mathf_pow(10, c->params.blur_tolerance) * stepSize;                // AO.cs:761
        blurTolerance *= blurTolerance;                                                              // AO.cs:762
        float upsampleTolerance = mathf_pow(10, c->params.upsample_tolerance);                       // AO.cs:763
        float noiseFilterWeight = 1 / (mathf_pow(10, c->params.noise_filter_tolerance) + upsampleTolerance);   // AO.cs:764
        p.inv_low[lo][0] = 1.0f / lo_w; p.inv_low[lo][1] = 1.0f / lo_h;                              // AO.cs:766
        p.inv_high[lo][0] = 1.0f / hi_w; p.inv_high[lo][1] = 1.0f / hi_h;                            // AO.cs:767
        p.noise_filter_strength[lo] = noiseFilterWeight;
        p.step_size[lo] = stepSize;
        p.blur_tolerance[lo] = blurTolerance;
        p.upsample_tolerance[lo] = upsampleTolerance;
    }
    c->plan_dirty = false;
    c->plan_gen = c->consts_gen;
}

// Caller must have made c->device current (ensure_ready / meao_resize / meao_destroy do).
void drop_graph(MeaoCtx *c)
{
    c->graphs_stale = false;
    if (c->graphs.empty() && c->retired.empty() && c->surfaces.empty()) return;
    cudaDeviceSynchronize();            // a re-plan is rare; never destroy an executable graph (or surface) that may still be in flight
    for (auto &kv : c->graphs) cudaGraphExecDestroy(kv.second.exec);
    for (auto &r : c->retired) { cudaGraphExecDestroy(r.exec); cudaEventDestroy(r.done); }
    for (auto &kv : c->surfaces) cudaDestroySurfaceObject(kv.second);
    c->graphs.clear();
    c->retired.clear();
    c->surfaces.clear();
}

void disconnect_peers(MeaoCtx *c)
{
    for (int side = 0; side < 2; side++) {
        if (c->peer_base[side] && c->peer_ipc[side]) cudaIpcCloseMemHandle(c->peer_base[side]);
        c->peer_base[side] = nullptr; c->peer_ipc[side] = false;
    }
}

void free_buffers(MeaoCtx *c)
{
    drop_graph(c);
    disconnect_peers(c);
    c->band_flags = nullptr;
    if (c->arena) cudaFree(c->arena);
    c->arena = nullptr; c->arena_bytes = 0;
    c->depth_stage[0] = c->depth_stage[1] = nullptr; c->ao_stage[0] = c->ao_stage[1] = nullptr;
    c->compute_done_valid = false;
}

int make_map(MeaoCtx *c, CUtensorMap *m, CUtensorMapDataType dt, int elem, void *base, int w, int h, int pitch_elems, int bw, int bh)
{
    cuuint64_t dims[2] = {(cuuint64_t)w, (cuuint64_t)h};
    cuuint64_t strides[1] = {(cuuint64_t)pitch_elems * elem};
    cuuint32_t box[2] = {(cuuint32_t)bw, (cuuint32_t)bh};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = c->encode(m, dt, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -1;
}

// rows of the low level (after clamping) that an upsample producing hi rows [a,b) reads
Range ups_lo_rows(Range hi, int loh)
{
    if (hi.hi <= hi.lo) return Range{0, 0};
    const int ymin = (hi.lo + 1) >> 1, ymax = hi.hi >> 1;      // Y = (py+1)>>1 for py in [a, b-1]
    return clampr(Range{ymin - 3, ymax + 3}, loh);             // quad rows Y-1..Y, blur radius 2
}
// rows of LowDepth<k> that a render producing rows [a,b) of level k reads (slice texel +-4 => +-16 rows, slice aligned)
Range ren_low_rows(Range out, int lh)
{
    if (out.hi <= out.lo) return Range{0, 0};
    return clampr(Range{4 * ((out.lo >> 2) - 4), 4 * (((out.hi - 1) >> 2) + 4) + 4}, lh);
}

struct BandNeeds { Range need_c[5]; Range need_low[5]; Range own_low[5]; };

BandNeeds compute_needs(const MeaoCtx *c, int b0, int b1)
{
    BandNeeds n;
    n.need_c[0] = Range{b0, b1};
    for (int k = 1; k <= 4; k++) n.need_c[k] = ups_lo_rows(n.need_c[k - 1], c->lh[k]);
    for (int k = 1; k <= 4; k++) {
        Range r = ren_low_rows(n.need_c[k], c->lh[k]);
        // the upsample also reads LowDepth<k> on need_c[k] (as lo depth) -- a subset of r
        if (n.need_c[k].lo < r.lo) r.lo = n.need_c[k].lo;
        if (n.need_c[k].hi > r.hi) r.hi = n.need_c[k].hi;
        n.need_low[k] = r;
        n.own_low[k] = Range{b0 >> k, (b1 + (1 << k) - 1) >> k};
    }
    n.need_low[0] = n.own_low[0] = Range{b0, b1};
    return n;
}

// A band's LowDepth rows beyond its own come from its neighbours, so its halo may reach into the band above (starting at row prev0,
// -1: none) and the band below (ending at row next1, -1: none) but not past them.
int check_halo_reach(MeaoCtx *c, const BandNeeds &n, int prev0, int next1)
{
    for (int k = 1; k <= 4; k++) {
        if (n.need_low[k].lo < n.own_low[k].lo && (prev0 < 0 || n.need_low[k].lo < (prev0 >> k)))
            return fail(c, MEAO_ERR_UNSUPPORTED, "halo of level %d reaches beyond the band above", k);
        if (n.need_low[k].hi > n.own_low[k].hi && (next1 < 0 || n.need_low[k].hi > ((next1 + (1 << k) - 1) >> k)))
            return fail(c, MEAO_ERR_UNSUPPORTED, "halo of level %d reaches beyond the band below", k);
    }
    return 0;
}

int setup_band(MeaoCtx *c)
{
    BandNeeds n = compute_needs(c, c->band0, c->band1);
    for (int k = 0; k <= 4; k++) { c->need_c[k] = n.need_c[k]; c->need_low[k] = n.need_low[k]; c->own_low[k] = n.own_low[k]; }
    return check_halo_reach(c, n, c->prev0, c->next1);
}

// The size the arena is laid out for: the reservation, or the current size
inline int arena_w(const MeaoCtx *c) { return c->res_w > 0 ? c->res_w : c->W; }
inline int arena_h(const MeaoCtx *c) { return c->res_w > 0 ? c->res_h : c->H; }

// Places the buffers of the current size (c->W x c->H) in the arena, where a fresh context of that size has them, with its camera
// tables in slot `slot`; encodes the TMA maps and resets the band to the whole frame.  Host work only: no allocation, no CUDA call.
int place_size(MeaoCtx *c, int slot)
{
    c->band0 = 0; c->band1 = c->H; c->prev0 = -1; c->next1 = -1;
    c->slot = slot;
    place_frame(*c, arena_layout(c->W, c->H, c->layers), (char *)c->arena, slot);
    if (!c->arena) return setup_band(c);
    c->tma_ok = c->encode && encode_maps(*c, [c](CUtensorMap &m, const MapSpec &sp) {
        return make_map(c, &m, sp.elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, sp.elem, sp.base, sp.w, sp.h,
                        sp.pitch_elems, sp.bw, sp.bh) == 0;
    });
    if (!c->tma_ok) memset(&c->maps, 0, sizeof c->maps);
    return setup_band(c);
}

// A new arena for arena_w x arena_h at the layer count, laid out by arena_layout; the current size (if any) is placed in it and
// re-planned by the next ensure_ready.  keep_old: allocate before freeing the old arena, so that MEAO_ERR_NOMEM leaves the context as
// it was (meao_reserve); otherwise the old arena goes first, as a resize always did.
int allocate(MeaoCtx *c, bool keep_old = false)
{
    const ArenaLayout a = arena_layout(arena_w(c), arena_h(c), c->layers);
    if (!c->plan_only) {
        if (!keep_old) free_buffers(c);
        void *arena = nullptr;
        cudaError_t e = cudaMalloc(&arena, a.bytes);
        if (e != cudaSuccess) return fail(c, e == cudaErrorMemoryAllocation ? MEAO_ERR_NOMEM : MEAO_ERR_CUDA,
                                          "cudaMalloc(%zu) failed: %s", a.bytes, cudaGetErrorString(e));
        if (keep_old) free_buffers(c);
        c->arena = arena;
        c->arena_bytes = a.bytes;
        c->arena_allocations++;
        CUDA_TRY(c, cudaMemsetAsync(c->arena, 0, a.bytes, c->stream));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
        char *b = (char *)c->arena;
        c->band_flags = (BandFlags *)b;
        {
            BandFlags init{}; init.epoch = 1;
            CUDA_TRY(c, cudaMemcpy(c->band_flags, &init, sizeof init, cudaMemcpyHostToDevice));
            if (c->host_error) *c->host_error = 0;
        }
        for (int i = 0; i < 2; i++) { c->depth_stage[i] = (float *)(b + a.depth_stage[i]); c->ao_stage[i] = (uint8_t *)(b + a.ao_stage[i]); }
    }
    c->plan_dirty = true;                           // the camera tables are written by the first ensure_ready
    for (auto &s : c->size_slots) s.valid = false;
    if (c->W <= 0) return 0;
    return place_size(c, 0);
}

// A frame-constant change (include/meao.h) since the current size was planned: its constants are planned again on the host, and its
// camera tables are written by the next frame on that frame's stream (write_tables) -- no synchronise, no graph dropped; the graphs
// re-target at their next launch (launch_cached).  A pending structural re-plan (plan_dirty) covers the constants itself.
void refresh_constants(MeaoCtx *c)
{
    if (c->plan_dirty || c->W <= 0 || c->plan_gen == c->consts_gen) return;
    build_plan(c);
    c->table_pending = !c->plan_only;
}

// Reserved contexts: make w x h the current size without touching the device.  The current size is parked in its slot; a size parked
// earlier is swapped back in as it was (plan, maps, camera tables); a new size takes a free slot or the least recently used one, and
// is planned on the host -- its camera tables are written by its first frame, on that frame's stream (write_tables).
// HAZARD: a parked size keeps the constants it was parked with.  Frame constants may have changed since, so a size swapped back in
// re-plans its constants here (refresh_constants) before any frame or getter can read them, and its graphs re-target at their first
// replay; it must never replay with the constants it was parked with.
int switch_size(MeaoCtx *c, int w, int h)
{
    SizeState &cur = *c;
    if (c->W > 0) c->size_slots[c->slot] = MeaoCtx::SizeSlot{true, c->size_clock, cur};
    int slot = -1;
    for (int i = 0; i < kSizeSlots; i++) {
        MeaoCtx::SizeSlot &s = c->size_slots[i];
        if (s.valid && s.s.W == w && s.s.H == h) {
            cur = s.s;
            s.last_use = ++c->size_clock;
            refresh_constants(c);
            return 0;
        }
        if (slot < 0 || (c->size_slots[slot].valid && (!s.valid || s.last_use < c->size_slots[slot].last_use))) slot = i;
    }
    c->W = w; c->H = h;
    int rc = place_size(c, slot);
    if (rc) return rc;
    if (!c->plan_dirty) {                           // else ensure_ready re-plans (and drops every other slot)
        build_plan(c);
        c->cam_table_stale = false;
        c->table_pending = !c->plan_only;
    }
    c->size_slots[slot] = MeaoCtx::SizeSlot{true, ++c->size_clock, cur};
    return 0;
}

// Write the per-layer camera tables to the arena.  Called by ensure_ready after a structural re-plan, once every frame that may read the
// old tables has finished (a device synchronise: frames may be in flight on any caller stream).
int upload_camera_tables(MeaoCtx *c)
{
    std::vector<LayerZ> zb;
    std::vector<LayerRender> ren;
    camera_tables(*c, zb, ren);
    CUDA_TRY(c, cudaDeviceSynchronize());
    CUDA_TRY(c, cudaMemcpy(c->layer_zb, zb.data(), zb.size() * sizeof(LayerZ), cudaMemcpyHostToDevice));
    CUDA_TRY(c, cudaMemcpy(c->layer_ren, ren.data(), ren.size() * sizeof(LayerRender), cudaMemcpyHostToDevice));
    c->cam_table_stale = false;
    c->table_pending = false;
    return 0;
}

// The tables of a size newly planned by switch_size, or re-planned after a frame-constant change (refresh_constants), written in
// stream order before the first frame that reads them, on that frame's stream.  The slot may have held another size's tables, or
// this size's older ones: frames of one context run in the order they are issued (include/meao.h), so every earlier frame that
// read it has completed before this copy lands.  The source is pageable, so the runtime stages it and
// the vectors may go when the call returns.
int write_tables(MeaoCtx *c, cudaStream_t s)
{
    if (!c->table_pending) return 0;
    std::vector<LayerZ> zb;
    std::vector<LayerRender> ren;
    camera_tables(*c, zb, ren);
    CUDA_TRY(c, cudaMemcpyAsync(c->layer_zb, zb.data(), zb.size() * sizeof(LayerZ), cudaMemcpyHostToDevice, s));
    CUDA_TRY(c, cudaMemcpyAsync(c->layer_ren, ren.data(), ren.size() * sizeof(LayerRender), cudaMemcpyHostToDevice, s));
    c->table_pending = false;
    return 0;
}

// A re-plan after a structural plan input changed: the parked sizes were planned with the old inputs, so they go (with the captured
// graphs), and the tables are uploaded after a device synchronise (upload_camera_tables).
void replan(MeaoCtx *c)
{
    build_plan(c);
    c->cam_table_stale = true;
    c->graphs_stale = true;
    for (int i = 0; i < kSizeSlots; i++) if (i != c->slot) c->size_slots[i].valid = false;
}

int ensure_ready(MeaoCtx *c)
{
    if (!c) return MEAO_ERR_INVALID;
    if (c->W <= 0) return fail(c, MEAO_ERR_INVALID, "meao_resize has not been called");
    if (c->plan_only) return fail(c, MEAO_ERR_CUDA, "plan-only context (device < 0): no CUDA device bound, and libmeao has no CPU fallback");
    CUDA_TRY(c, cudaSetDevice(c->device));
    if (c->plan_dirty) replan(c);
    refresh_constants(c);
    if (c->graphs_stale) drop_graph(c);
    if (c->cam_table_stale) { int rc = upload_camera_tables(c); if (rc) return rc; }
    return 0;
}

// ensure_ready for an entry point that issues work on stream s which may read the camera tables: every frame form, band phase and
// stage call, so that each sees the tables of the constants set before it was issued
int frame_ready(MeaoCtx *c, cudaStream_t s)
{
    int rc = ensure_ready(c);
    return rc ? rc : write_tables(c, s);
}

struct NvtxRange { explicit NvtxRange(const char *n) { nvtxRangePushA(n); } ~NvtxRange() { nvtxRangePop(); } };

// MEAO_REN_TILE = 0 / 1 / 2 forces a render tile variant for every level (a tuning aid); -1: the planner's rule
int forced_render_tile()
{
    const char *force = getenv("MEAO_REN_TILE");
    return (force && force[0] >= '0' && force[0] < '0' + kRenderTileVariants) ? force[0] - '0' : -1;
}

// ---- the recorders: frame_record.h's schedule, argument blocks and launcher choice -------------------------------------------

// One launch of the frame schedule on stream s, inside an NVTX range, counted.  io: the frame's depth and AO (FrameIO).  A prepare
// goes through record_downsample, which checks the depth kind first.
int record_launch(MeaoCtx *c, const FrameLaunch &l, const FrameIO &io, cudaStream_t s)
{
    static const char *nvtx[4] = {"meao::prepare_depth", "meao::render_ao", "meao::render_ao_wide", "meao::blur_upsample"};
    if (l.stage == kStageUpsample && l.level == 1) c->last_out = io.aio ? const_cast<void *>(io.aio->ao_array) : io.ao;
    NvtxRange nv(nvtx[l.stage]);
    CUDA_TRY(c, launch_entry(*c, l, io, forced_render_tile(), s));
    c->launches++;
    return 0;
}

// The FrameIO of a pointer frame: its depth and AO at the pitches of vp (nullptr: tight).  fused: the prepare writes LowDepth1..4
// only and the final upsample reads and linearises the same depth (what meao_render records).
FrameIO frame_io(MeaoCtx *c, const void *depth, int kind, void *ao_out, bool fused, const ViewPitch *vp = nullptr)
{
    FrameIO io;
    io.kind = kind; io.depth = depth_in(*c, depth, kind, vp); io.low_only = io.fused = fused; io.ao = ao_out; io.vp = vp;
    return io;
}

// PushDownsampleCommands, AO.cs:604-658: the prepare_depth of every entry point, the first launch of the frame schedule.  io.low_only:
// LowDepth1..4 only, for a frame whose final upsample reads the same depth; otherwise LinearDepth as well.
int record_downsample(MeaoCtx *c, const FrameIO &io, cudaStream_t s)
{
    if (io.kind < MEAO_DEPTH_RAW_F32 || io.kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", io.kind);
    c->last_kind = io.kind;
    return record_launch(c, FrameLaunch{kStagePrepare, 0, 0, -1, kPdlNever}, io, s);
}
// One entry of the frame schedule: the prepare through record_downsample, every other launch through record_launch
int record_entry(MeaoCtx *c, const FrameLaunch &l, const FrameIO &io, cudaStream_t s)
{
    return l.stage == kStagePrepare ? record_downsample(c, io, s) : record_launch(c, l, io, s);
}

// The stage API's recorders, one launch each: the prepare_depth of a pointer depth (tight rows), a render level, an upsample level.
int record_downsample(MeaoCtx *c, const void *depth, int kind, cudaStream_t s, bool low_only = false)
{
    FrameIO io = frame_io(c, depth, kind, nullptr, false);
    io.low_only = low_only;
    return record_downsample(c, io, s);
}
// PushRenderCommands, AO.cs:660-748.  wide = false: the call AmbientOcclusion.cs makes (tiled source, kernel main_interleaved);
// wide = true: the same recorder for the non-tiled source LowDepth<k> (kernel main) -> HighQuality<k>.
int record_render(MeaoCtx *c, int k, int kind, cudaStream_t s, bool wide = false)
{
    return record_launch(c, FrameLaunch{wide ? kStageRenderWide : kStageRender, k, 0, -1, kPdlNever}, frame_io(c, nullptr, kind, nullptr, false), s);
}
// PushUpsampleCommands with the wiring of AO.cs:528-531; the final level stores into ao_out (nullptr: the result buffer).
int record_upsample(MeaoCtx *c, int lo, void *ao_out, cudaStream_t s)
{
    return record_launch(c, FrameLaunch{kStageUpsample, lo, 0, -1, kPdlNever}, frame_io(c, nullptr, c->last_kind, ao_out, false), s);
}

// RAII: launches issued while one of these is alive (and `on`) carry the programmatic-dependent-launch attribute.
struct PdlScope { bool prev; explicit PdlScope(bool on) : prev(g_launch_pdl) { g_launch_pdl = on; } ~PdlScope() { g_launch_pdl = prev; } };

// The frame schedule from entry `first` on, recorded as a DAG on the caller's stream s and the forked streams (for graph capture):
// an event is recorded after every launch a later one waits for.  first = 1: the caller has recorded the prepare, or a band's halo or
// exchange kernel in its place; what waits for the prepare then waits for stream s as it stands here, so renders 2-4 still follow the
// halo rows.  pdl: the level of frame_schedule's PDL classes.  after_exchange: the launch before this DAG is the neighbour-exchange
// kernel, which spins on remote flags -- nothing may be scheduled "early" behind it (a grid parked in griddepcontrol.wait holds SM
// resources that the neighbour band's kernels may need: see DESIGN.md 4), so the first launch goes without PDL.
int record_frame_dag(MeaoCtx *c, const FrameIO &io, cudaStream_t s, size_t first, int pdl, bool after_exchange = false)
{
    const std::vector<FrameLaunch> sched = frame_schedule(c->plan.variants);
    const cudaStream_t st[4] = {s, c->branch[0], c->branch[1], c->branch[2]};
    std::vector<int> ev(sched.size(), -1);          // the event (of c->ev) recorded after launch i, if one waits for it: at most 4
    int nev = 0;
    for (const FrameLaunch &l : sched)
        if (l.wait >= 0 && ev[l.wait] < 0) ev[l.wait] = nev++;
    for (size_t i = 0; i < first; i++)
        if (ev[i] >= 0) CUDA_TRY(c, cudaEventRecord(c->ev[ev[i]], st[sched[i].branch]));
    for (size_t i = first; i < sched.size(); i++) {
        const FrameLaunch &l = sched[i];
        if (l.wait >= 0) CUDA_TRY(c, cudaStreamWaitEvent(st[l.branch], c->ev[ev[l.wait]], 0));
        {
            PdlScope p(pdl_on(l, pdl) && !(after_exchange && i == first));
            int rc = record_entry(c, l, io, st[l.branch]);
            if (rc) return rc;
        }
        if (ev[i] >= 0) CUDA_TRY(c, cudaEventRecord(c->ev[ev[i]], st[l.branch]));
    }
    return 0;
}

// The frame schedule from entry `first` on, serially on stream s (MEAO_FLAG_NO_GRAPH, meao_render_band_finish).  profile: an event
// pair around every launch (meao_profile_frame), each launched profile_repeats times.
int record_frame(MeaoCtx *c, const FrameIO &io, cudaStream_t s, size_t first, bool profile)
{
    const std::vector<FrameLaunch> sched = frame_schedule(c->plan.variants);
    std::vector<cudaEvent_t> ev;
    auto mark = [&]() { if (profile) { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, s); ev.push_back(e); } };
    const int reps = profile ? c->profile_repeats : 1;         // every kernel is idempotent (out of place), so repeating it is harmless
    mark();
    for (size_t i = first; i < sched.size(); i++) {
        for (int r = 0; r < reps; r++) { int rc = record_entry(c, sched[i], io, s); if (rc) return rc; }
        mark();
    }
    if (profile) {
        CUDA_TRY(c, cudaStreamSynchronize(s));
        c->last_profile.clear();
        for (size_t i = 0; i + 1 < ev.size(); i++) {
            float ms = 0; cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
            c->last_profile.push_back({launch_name(sched[first + i]), ms / (float)reps});
        }
        for (auto e : ev) cudaEventDestroy(e);
    }
    return 0;
}

// Before a debug read of buffer `id` on stream s: when the last frame stored its AO elsewhere (the caller's buffer or array), the
// context's own AO texture is regenerated from the still resident Combined1 / LowDepth1 / LinearDepth with the same kernel.  A debug
// read is not a frame: the launch count stays.
int own_ao(MeaoCtx *c, int id, cudaStream_t s)
{
    if (id != MEAO_BUF_AMBIENT_OCCLUSION || !c->last_out) return 0;
    const int64_t before = c->launches;
    const int rc = record_upsample(c, 1, nullptr, s);
    c->launches = before;
    return rc;
}

std::mutex g_event_mutex;
// arrays: meao_bind_event_arrays.  Otherwise a pointer frame at the pitches `pitch`, or, with tight (meao_bind_event), at the tight pitches
// of the context when the event runs -- a meao_resize between binding and rendering keeps meaning what it meant before.
struct EventBinding { MeaoCtx *ctx; const void *depth; int kind; void *out; void *stream; bool arrays; bool tight; ViewPitch pitch; };
std::map<int, EventBinding> g_events;

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int meao_abi_version(void) { return MEAO_ABI_VERSION; }

void meao_default_params(MeaoParams *p)
{
    if (!p) return;
    p->noise_filter_tolerance = 0.0f;   // AO.cs:20
    p->blur_tolerance = -4.6f;          // AO.cs:28
    p->upsample_tolerance = -12.0f;     // AO.cs:36
    p->thickness_modifier = 1.0f;       // AO.cs:44
    p->intensity = 1.0f;                // AO.cs:52
    p->debug = 0;                       // AO.cs:60
    p->ambient_only = 1;                // AO.cs:68
}

int meao_create(const MeaoDeviceCfg *cfg, MeaoCtx **out)
{
    if (!out) return fail(nullptr, MEAO_ERR_INVALID, "out_ctx is NULL");
    *out = nullptr;
    if (cfg && cfg->device < 0) {       // host-side planner only: constants, geometry, band/halo ranges
        MeaoCtx *c = new MeaoCtx();
        c->device = -1; c->plan_only = true; c->flags = cfg->flags;
        meao_default_params(&c->params);
        c->camera = MeaoCamera{0.3f, 1000.0f, 1.0f, 1};
        *out = c;
        return MEAO_OK;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, MEAO_ERR_CUDA, "no CUDA device available (%s); libmeao has no CPU fallback",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    const int dev = cfg ? cfg->device : 0;
    if (dev < 0 || dev >= ndev) return fail(nullptr, MEAO_ERR_INVALID, "device %d out of range (0..%d)", dev, ndev - 1);
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return fail(nullptr, MEAO_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, MEAO_ERR_CUDA, "device %d is sm_%d%d; libmeao is built for sm_90a (H100) only", dev, prop.major, prop.minor);
    e = cudaSetDevice(dev);
    if (e != cudaSuccess) return fail(nullptr, MEAO_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    MeaoCtx *c = new MeaoCtx();
    c->device = dev;
    c->sm_count = prop.multiProcessorCount;
    c->flags = cfg ? cfg->flags : 0;
    meao_default_params(&c->params);
    c->camera = MeaoCamera{0.3f, 1000.0f, 1.0f, 1};
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    for (int i = 0; i < 3 && e == cudaSuccess; i++) e = cudaStreamCreateWithFlags(&c->branch[i], cudaStreamNonBlocking);
    for (int i = 0; i < 5 && e == cudaSuccess; i++) e = cudaEventCreateWithFlags(&c->ev[i], cudaEventDisableTiming);
    for (int i = 0; i < 2 && e == cudaSuccess; i++) e = cudaStreamCreateWithFlags(&c->slot_stream[i], cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; i++) e = cudaEventCreateWithFlags(&c->slot_done[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->compute_done, cudaEventDisableTiming);
    if (e != cudaSuccess) { delete c; return fail(nullptr, MEAO_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
    if (cudaHostAlloc((void **)&c->host_error, 64, cudaHostAllocMapped) == cudaSuccess) {
        *c->host_error = 0;
        if (cudaHostGetDevicePointer((void **)&c->host_error_dev, c->host_error, 0) != cudaSuccess) c->host_error_dev = nullptr;
    } else c->host_error = nullptr;
    cudaGetLastError();
    {   // load every kernel of the library on this device NOW (kernels.h "eager loading"): a lazy load later could wait for a
        // spinning exchange kernel that in turn waits for the very launch that triggered the load
        static std::mutex preload_mutex;
        static std::map<int, bool> preloaded;
        std::lock_guard<std::mutex> g(preload_mutex);
        if (!preloaded[dev]) {
            cudaError_t pe = cudaSuccess;
            for (const KernelUnit *u : kKernelUnits) u->walk(&pe);
            if (pe != cudaSuccess) { cudaGetLastError(); meao_destroy(c); return fail(nullptr, MEAO_ERR_CUDA, "loading the kernels failed: %s", cudaGetErrorString(pe)); }
            preloaded[dev] = true;
        }
    }
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const char *no_tma = getenv("MEAO_DISABLE_TMA");     // debugging aid: force the gather path in every tile
    if (!(no_tma && no_tma[0] == '1') &&
        cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
        c->encode = (PFN_encodeTiled)fn;
    cudaGetLastError();
    *out = c;
    return MEAO_OK;
}

void meao_destroy(MeaoCtx *c)
{
    if (!c) return;
    {
        std::lock_guard<std::mutex> g(g_event_mutex);
        for (auto it = g_events.begin(); it != g_events.end();) { if (it->second.ctx == c) it = g_events.erase(it); else ++it; }
    }
    if (c->plan_only) { delete c; return; }
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    free_buffers(c);
    if (c->stream) cudaStreamDestroy(c->stream);
    for (auto b : c->branch) if (b) cudaStreamDestroy(b);
    for (auto e : c->ev) if (e) cudaEventDestroy(e);
    for (auto b : c->slot_stream) if (b) { cudaStreamSynchronize(b); cudaStreamDestroy(b); }
    for (auto e : c->slot_done) if (e) cudaEventDestroy(e);
    if (c->compute_done) cudaEventDestroy(c->compute_done);
    if (c->host_error) cudaFreeHost(c->host_error);
    delete c;
}

const char *meao_last_error(const MeaoCtx *c) { return c ? c->error.c_str() : g_create_error.c_str(); }

int meao_set_params(MeaoCtx *c, const MeaoParams *p)
{
    if (!c || !p) return MEAO_ERR_INVALID;
    // CheckPropertiesChanged, AO.cs:104-113 (ambient_only is not part of the change detection there either)
    bool changed = c->params.noise_filter_tolerance != p->noise_filter_tolerance || c->params.blur_tolerance != p->blur_tolerance ||
                   c->params.upsample_tolerance != p->upsample_tolerance || c->params.thickness_modifier != p->thickness_modifier ||
                   c->params.intensity != p->intensity || c->params.debug != p->debug;
    if (!(p->thickness_modifier > 0.0f)) return fail(c, MEAO_ERR_INVALID, "thickness_modifier must be > 0");
    c->params = *p;
    if (changed) c->consts_gen++;                   // frame constants: the next frame takes them without a re-plan
    return changed ? 1 : 0;
}

int meao_get_params(const MeaoCtx *c, MeaoParams *out)
{
    if (!c || !out) return MEAO_ERR_INVALID;
    *out = c->params;
    return MEAO_OK;
}

int meao_set_variants(MeaoCtx *c, const MeaoVariants *v)
{
    if (!c || !v) return MEAO_ERR_INVALID;
    if (v->high_quality_mask < 0 || v->high_quality_mask > 15) return fail(c, MEAO_ERR_INVALID, "high_quality_mask %d not in 0..15", v->high_quality_mask);
    if (v->single_scale && v->high_quality_mask) return fail(c, MEAO_ERR_INVALID, "single_scale excludes high_quality_mask");
    MeaoVariants n{v->single_pass_stereo ? 1 : 0, v->sample_exhaustively ? 1 : 0, v->high_quality_mask, v->single_scale ? 1 : 0};
    const bool changed = memcmp(&c->variants, &n, sizeof n) != 0;
    c->variants = n;
    if (changed) c->plan_dirty = true;          // re-plan + drop the captured graphs (ensure_ready)
    return changed ? 1 : 0;
}

int meao_get_variants(const MeaoCtx *c, MeaoVariants *out)
{
    if (!c || !out) return MEAO_ERR_INVALID;
    *out = c->variants;
    return MEAO_OK;
}

int meao_set_camera(MeaoCtx *c, const MeaoCamera *cam)
{
    if (!c || !cam) return MEAO_ERR_INVALID;
    if (!(cam->near_clip > 0) || !(cam->far_clip > cam->near_clip) || !(cam->tan_half_fov_h > 0))
        return fail(c, MEAO_ERR_INVALID, "bad camera (near %g far %g tanHalfFovH %g)", cam->near_clip, cam->far_clip, cam->tan_half_fov_h);
    if (memcmp(&c->camera, cam, sizeof *cam) != 0) {
        const int old_z = c->camera.reversed_z;
        c->camera = *cam;
        if (c->layer_cams.empty()) note_camera_change(c, old_z, cam->reversed_z);   // with a layer-camera table it takes effect when the table is cleared
    }
    return MEAO_OK;
}

int meao_set_layer_cameras(MeaoCtx *c, const MeaoCamera *cams, int32_t count)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!cams && count == 0) {
        if (c->layer_cams.empty()) return 0;
        const int old_z = ctx_reversed_z(c);
        c->layer_cams.clear();
        note_camera_change(c, old_z, c->camera.reversed_z);
        return 1;
    }
    if (!cams) return fail(c, MEAO_ERR_INVALID, "cameras is NULL with count %d (NULL clears the table only with count 0)", count);
    if (count != c->layers) return fail(c, MEAO_ERR_INVALID, "count %d differs from the context's %d layers (meao_set_layers)", count, c->layers);
    for (int l = 0; l < count; l++) {
        const MeaoCamera &k = cams[l];
        if (!(k.near_clip > 0)) return fail(c, MEAO_ERR_INVALID, "layer %d: bad camera near_clip %g (must be > 0)", l, k.near_clip);
        if (!(k.far_clip > k.near_clip))
            return fail(c, MEAO_ERR_INVALID, "layer %d: bad camera far_clip %g (must be > near_clip %g)", l, k.far_clip, k.near_clip);
        if (!(k.tan_half_fov_h > 0)) return fail(c, MEAO_ERR_INVALID, "layer %d: bad camera tan_half_fov_h %g (must be > 0)", l, k.tan_half_fov_h);
        if ((k.reversed_z != 0) != (cams[0].reversed_z != 0))
            return fail(c, MEAO_ERR_INVALID, "layer %d: camera reversed_z %d differs from layer 0's %d (one Z direction for all layers)", l,
                        k.reversed_z, cams[0].reversed_z);
    }
    if ((int)c->layer_cams.size() == count && memcmp(c->layer_cams.data(), cams, (size_t)count * sizeof(MeaoCamera)) == 0) return 0;
    const int old_z = ctx_reversed_z(c);
    c->layer_cams.assign(cams, cams + count);
    note_camera_change(c, old_z, cams[0].reversed_z);
    return 1;
}

int meao_get_layer_cameras(const MeaoCtx *c, MeaoCamera *out, int32_t capacity)
{
    if (!c) return MEAO_ERR_INVALID;
    const int n = (int)c->layer_cams.size();
    if (n && (!out || capacity < n)) return MEAO_ERR_INVALID;
    if (n) memcpy(out, c->layer_cams.data(), (size_t)n * sizeof(MeaoCamera));
    return n;
}

int meao_resize(MeaoCtx *c, int32_t w, int32_t h)
{
    if (!c) return MEAO_ERR_INVALID;
    if (w <= 0 || h <= 0 || w > 32768 || h > 32768) return fail(c, MEAO_ERR_INVALID, "bad size %dx%d", w, h);
    if (c->res_w > 0 && (w > c->res_w || h > c->res_h))      // never a silent re-allocation for a dynamic-resolution host
        return fail(c, MEAO_ERR_INVALID, "size %dx%d lies outside the reservation %dx%d (meao_reserve)", w, h, c->res_w, c->res_h);
    if (w == c->W && h == c->H && (c->arena || c->plan_only)) return 0;       // RTHandle.CheckBaseDimensions, AO.cs:145-148
    if (c->res_w > 0 && (c->arena || c->plan_only)) {
        const int rc = switch_size(c, w, h);        // no allocation, no synchronise, the other sizes' graphs stay
        return rc ? rc : 1;
    }
    if (!c->plan_only) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    c->W = w; c->H = h;
    int rc = allocate(c);
    if (rc) { c->W = c->H = 0; return rc; }
    return 1;
}

int meao_reserve(MeaoCtx *c, int32_t max_w, int32_t max_h)
{
    if (!c) return MEAO_ERR_INVALID;
    const bool clear = max_w == 0 && max_h == 0;
    if (!clear && (max_w <= 0 || max_h <= 0 || max_w > 32768 || max_h > 32768))
        return fail(c, MEAO_ERR_INVALID, "bad reservation %dx%d (each dimension in 1..32768, or 0x0 to clear)", max_w, max_h);
    if (c->W > 0 && (c->band0 != 0 || c->band1 != c->H || c->prev0 >= 0 || c->next1 >= 0))
        return fail(c, MEAO_ERR_UNSUPPORTED, "meao_reserve: this context has a row band (meao_set_row_band); row bands need an unreserved context");
    if (!clear && c->W > 0 && max_w < c->W)
        return fail(c, MEAO_ERR_INVALID, "reservation width %d is below the current width %d", max_w, c->W);
    if (!clear && c->H > 0 && max_h < c->H)
        return fail(c, MEAO_ERR_INVALID, "reservation height %d is below the current height %d", max_h, c->H);
    if (max_w == c->res_w && max_h == c->res_h) return 0;
    const int old_w = c->res_w, old_h = c->res_h;
    c->res_w = max_w; c->res_h = max_h;
    if (c->plan_only) return 1;                     // recorded; nothing to allocate
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (clear && c->W <= 0) { free_buffers(c); return 1; }
    const int rc = allocate(c, true);               // like a size change today, but the old arena stays until the new one exists
    if (rc) { c->res_w = old_w; c->res_h = old_h; return rc; }
    return 1;
}

int meao_reservation(const MeaoCtx *c, MeaoReservation *out)
{
    if (!c || !out) return MEAO_ERR_INVALID;
    memset(out, 0, sizeof *out);
    out->width = c->res_w; out->height = c->res_h;
    if (arena_w(c) > 0) out->arena_bytes = c->plan_only ? (int64_t)arena_layout(arena_w(c), arena_h(c), c->layers).bytes : (int64_t)c->arena_bytes;
    if (c->W > 0) out->arena_bytes_needed = (int64_t)arena_layout(c->W, c->H, c->layers).bytes;
    out->arena_allocations = c->arena_allocations;
    out->graphs_held = (int64_t)(c->graphs.size() + c->retired.size());
    out->graph_instantiations = c->graph_instantiations;
    return MEAO_OK;
}

int meao_set_layers(MeaoCtx *c, int32_t layers)
{
    if (!c) return MEAO_ERR_INVALID;
    if (layers < 1 || layers > kMaxLayers)
        return fail(c, MEAO_ERR_INVALID, "layers %d not in 1..%d (the layer is a grid dimension of the layered kernels)", layers, kMaxLayers);
    if (layers == c->layers) return 0;
    const int old = c->layers;
    std::vector<MeaoCamera> old_cams;
    old_cams.swap(c->layer_cams);                   // a table has one camera per layer: a new layer count clears it
    c->layers = layers;
    c->plan_dirty = true;
    if (c->W <= 0 && !c->arena) return 1;           // applied by the first meao_resize (a reserved arena is laid out again now)
    if (!c->plan_only) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    }
    int rc = allocate(c);                           // like a size change: new arena, whole-frame band, no neighbours, no graphs
    if (rc) {
        const std::string err = c->error;
        c->layers = old;
        c->layer_cams.swap(old_cams);
        if (allocate(c)) { c->W = c->H = 0; }        // the previous arena could not be restored either: the context needs meao_resize
        c->error = err;
        return rc;
    }
    return 1;
}

int meao_set_row_band(MeaoCtx *c, int32_t row0, int32_t row1, int32_t prev_row0, int32_t next_row1)
{
    if (!c || c->W <= 0) return MEAO_ERR_INVALID;
    BAND_GUARD(c, "meao_set_row_band");
    if (row0 < 0 || row1 > c->H || row0 >= row1 || (row0 % 16) || ((row1 % 16) && row1 != c->H))
        return fail(c, MEAO_ERR_INVALID, "band [%d,%d) must be 16-row aligned inside [0,%d)", row0, row1, c->H);
    if ((prev_row0 >= 0 && (prev_row0 % 16 || prev_row0 >= row0)) || (next_row1 >= 0 && (next_row1 <= row1 || next_row1 > c->H)))
        return fail(c, MEAO_ERR_INVALID, "bad neighbour extents");
    if ((row0 > 0) != (prev_row0 >= 0) || (row1 < c->H) != (next_row1 >= 0))
        return fail(c, MEAO_ERR_INVALID, "neighbour extents must be given exactly where the band is interior");
    // validated before anything changes: the context keeps its old band when the new one is refused
    int rc = check_halo_reach(c, compute_needs(c, row0, row1), prev_row0, next_row1);
    if (rc) return rc;
    if (!c->plan_only) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        drop_graph(c);
        disconnect_peers(c);        // the halo ranges change: the host exports / connects again
    }
    c->band0 = row0; c->band1 = row1; c->prev0 = prev_row0; c->next1 = next_row1;
    return setup_band(c);
}

static void halo_ranges(MeaoCtx *c, int side, bool send, Range out[5])
{
    // send up:   rows of my own range that the band above needs  = [own.lo, above.need.hi)
    // recv up:   [need.lo, own.lo)
    for (int k = 1; k <= 4; k++) out[k] = Range{0, 0};
    if (side == 0 && c->prev0 < 0) return;
    if (side == 1 && c->next1 < 0) return;
    if (!send) {
        for (int k = 1; k <= 4; k++) {
            if (side == 0) out[k] = Range{c->need_low[k].lo, c->own_low[k].lo};
            else out[k] = Range{c->own_low[k].hi, c->need_low[k].hi};
            if (out[k].hi < out[k].lo) out[k].hi = out[k].lo;
        }
        return;
    }
    BandNeeds nb = (side == 0) ? compute_needs(c, c->prev0, c->band0) : compute_needs(c, c->band1, c->next1);
    for (int k = 1; k <= 4; k++) {
        if (side == 0) out[k] = Range{c->own_low[k].lo, nb.need_low[k].hi};
        else out[k] = Range{nb.need_low[k].lo, c->own_low[k].hi};
        if (out[k].hi < out[k].lo) out[k].hi = out[k].lo;
    }
}

static int64_t halo_size(MeaoCtx *c, int side, bool send)
{
    if (!c || c->W <= 0 || (side != 0 && side != 1)) return MEAO_ERR_INVALID;
    BAND_GUARD(c, send ? "meao_halo_bytes" : "meao_halo_recv_bytes");
    Range r[5]; halo_ranges(c, side, send, r);
    int64_t bytes = 0;
    for (int k = 1; k <= 4; k++) bytes += (int64_t)(r[k].hi - r[k].lo) * c->lw[k] * 4;
    return bytes;
}
int64_t meao_halo_bytes(MeaoCtx *c, int32_t side) { return halo_size(c, side, true); }
int meao_halo_rows(MeaoCtx *c, int32_t side, int32_t send, int32_t out8[8])
{
    if (!c || c->W <= 0 || (side != 0 && side != 1) || !out8) return MEAO_ERR_INVALID;
    BAND_GUARD(c, "meao_halo_rows");
    Range r[5]; halo_ranges(c, side, send != 0, r);
    for (int k = 1; k <= 4; k++) { out8[2 * (k - 1)] = r[k].lo; out8[2 * (k - 1) + 1] = r[k].hi; }
    return MEAO_OK;
}
int meao_band_rows(MeaoCtx *c, int32_t out30[30])
{
    if (!c || c->W <= 0 || !out30) return MEAO_ERR_INVALID;
    for (int k = 0; k <= 4; k++) {
        out30[2 * k] = c->need_c[k].lo; out30[2 * k + 1] = c->need_c[k].hi;
        out30[10 + 2 * k] = c->need_low[k].lo; out30[10 + 2 * k + 1] = c->need_low[k].hi;
        out30[20 + 2 * k] = c->own_low[k].lo; out30[20 + 2 * k + 1] = c->own_low[k].hi;
    }
    return MEAO_OK;
}
int64_t meao_halo_recv_bytes(MeaoCtx *c, int32_t side) { return halo_size(c, side, false); }

static int halo_copy(MeaoCtx *c, int side, void *packed, bool pack, void *stream)
{
    BAND_GUARD(c, pack ? "meao_halo_pack" : "meao_halo_unpack");
    int rc = ensure_ready(c); if (rc) return rc;
    if (side != 0 && side != 1) return fail(c, MEAO_ERR_INVALID, "side must be 0 or 1");
    cudaStream_t s = (cudaStream_t)stream;
    Range r[5]; halo_ranges(c, side, pack, r);
    HaloArgs a{};
    halo_segments(*c, r, (float *)packed, pack, a);
    for (int i = 0; i < a.nseg; i++) {                  // copies, not halo_copy_kernel: no kernel launch
        const HaloSeg &g = a.seg[i];
        CUDA_TRY(c, cudaMemcpy2DAsync(g.dst, (size_t)g.dst_pitch * sizeof(float), g.src, (size_t)g.src_pitch * sizeof(float),
                                      (size_t)g.width * sizeof(float), g.rows, cudaMemcpyDeviceToDevice, s));
    }
    return MEAO_OK;
}
int meao_halo_pack(MeaoCtx *c, int32_t side, void *packed, void *stream) { return halo_copy(c, side, packed, true, stream); }
int meao_halo_unpack(MeaoCtx *c, int32_t side, const void *packed, void *stream) { return halo_copy(c, side, (void *)packed, false, stream); }

int meao_render_band_prepare(MeaoCtx *c, const void *depth, int32_t kind, void *stream)
{
    BAND_GUARD(c, "meao_render_band_prepare");
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (!depth) return fail(c, MEAO_ERR_INVALID, "depth is NULL");
    return record_downsample(c, depth, kind, (cudaStream_t)stream);
}

int meao_render_band_finish(MeaoCtx *c, void *ao_out, void *stream)
{
    BAND_GUARD(c, "meao_render_band_finish");
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    return record_frame(c, frame_io(c, nullptr, c->last_kind, ao_out, false), (cudaStream_t)stream, 1, false);
}

static int halo_kernel(MeaoCtx *c, void *up, void *down, bool pack, cudaStream_t s)
{
    HaloArgs a{};
    void *bufs[2] = {up, down};
    for (int side = 0; side < 2; side++) {
        if (!bufs[side]) continue;
        Range r[5]; halo_ranges(c, side, pack, r);
        halo_segments(*c, r, (float *)bufs[side], pack, a);
    }
    CUDA_TRY(c, launch_halo_copy(a, s));
    if (a.nseg) c->launches++;
    return 0;
}

// ---- graph cache ----------------------------------------------------------------------------------------------------
// record(stream, pdl) issues the launches; it is captured into a graph, with the highest programmatic-dependent-launch
// level the runtime accepts (tried once per context: 2, then 1, then 0 = plain edges).  *launches: the kernels it recorded.
static int capture_graph(MeaoCtx *c, const std::function<int(cudaStream_t, int)> &record, cudaGraph_t *out, int *launches)
{
    const char *env = getenv("MEAO_PDL");                           // tuning / debugging aid: cap the level (0 disables)
    const int cap = (env && env[0] >= '0' && env[0] <= '2') ? env[0] - '0' : 2;
    for (int level = (c->pdl_level >= 0 ? c->pdl_level : cap); level >= 0; level--) {
        cudaGraph_t g = nullptr;
        CUDA_TRY(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
        const int64_t before = c->launches;
        const int rc = record(c->stream, level);
        *launches = (int)(c->launches - before);
        c->launches = before;
        const cudaError_t e = cudaStreamEndCapture(c->stream, &g);
        if (rc == 0 && e == cudaSuccess) { c->pdl_level = level; *out = g; return 0; }
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        if (level == 0) {
            if (rc) return rc;
            return fail(c, MEAO_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(e));
        }
        // a capture that failed with PDL edges is retried one level lower (mixed programmatic + event dependencies may be refused)
    }
    return fail(c, MEAO_ERR_CUDA, "graph capture failed");
}

// The graph cache holds at most kMaxGraphs executable graphs; at most kMaxRetired more wait for their `done` event, so a context never
// holds more than kMaxGraphs + kMaxRetired (include/meao.h MeaoReservation.graphs_held), whatever sequence of sizes and buffers it sees.
constexpr size_t kMaxGraphs = 64, kMaxRetired = 8;
static_assert(MEAO_SIZE_SLOTS == kSizeSlots && MEAO_MAX_GRAPHS_HELD == kMaxGraphs + kMaxRetired, "include/meao.h states these bounds");

// Destroys the retired executable graphs whose `done` event has completed; with wait, first waits for the oldest (an event wait on
// the host, not a device synchronise).
static void reclaim_retired(MeaoCtx *c, bool wait)
{
    if (wait && !c->retired.empty()) cudaEventSynchronize(c->retired.front().done);
    for (auto it = c->retired.begin(); it != c->retired.end();) {
        const cudaError_t e = cudaEventQuery(it->done);
        if (e == cudaErrorNotReady) { cudaGetLastError(); ++it; continue; }
        cudaGetLastError();
        cudaGraphExecDestroy(it->exec);
        cudaEventDestroy(it->done);
        it = c->retired.erase(it);
    }
}

// Re-targets the executable graph *ge to the freshly captured g with cudaGraphExecUpdate: new kernel arguments and pointers, no device
// synchronise, launches already enqueued are unaffected.  When the update is refused (another topology), *ge is retired instead -- its
// `done` event is recorded on s now and again after the frame that replaces it (*retiring) -- and *ge becomes nullptr: the caller
// instantiates g.
static int retarget(MeaoCtx *c, cudaGraphExec_t *ge, cudaGraph_t g, cudaStream_t s, bool *retiring)
{
    cudaGraphExecUpdateResultInfo info;
    if (cudaGraphExecUpdate(*ge, g, &info) == cudaSuccess) return 0;
    cudaGetLastError();
    cudaEvent_t done = nullptr;
    if (cudaEventCreateWithFlags(&done, cudaEventDisableTiming) != cudaSuccess) return fail(c, MEAO_ERR_CUDA, "cudaEventCreate failed");
    c->retired.push_back(MeaoCtx::Retired{*ge, done});
    cudaEventRecord(done, s);                       // recorded again after the new launch; this covers a launch that fails
    *retiring = true;
    *ge = nullptr;
    return 0;
}

// Replays the graph of `key`, captured from record(stream, pdl) on first use; a replay counts the launches its capture recorded.  A
// graph captured before the frame constants last changed (its gen) is captured again and re-targeted in place before it is launched:
// lazily, so a change costs one capture + update per graph actually replayed, not one per cached graph.
static int launch_cached(MeaoCtx *c, const MeaoCtx::GraphKey &key_in, cudaStream_t s, const std::function<int(cudaStream_t, int)> &record)
{
    if (c->flags & MEAO_FLAG_NO_GRAPH) return record(s, 0);
    MeaoCtx::GraphKey key = key_in;
    key.size[0] = c->W; key.size[1] = c->H; key.size[2] = c->slot;
    auto it = c->graphs.find(key);
    bool retiring = false;
    if (it == c->graphs.end() || it->second.gen != c->plan_gen) {
        if (!c->retired.empty()) reclaim_retired(c, c->retired.size() >= kMaxRetired);
        cudaGraph_t g = nullptr;
        int launches = 0;
        int rc = capture_graph(c, record, &g, &launches);
        if (rc) return rc;
        cudaGraphExec_t ge = nullptr;
        auto victim = it;
        if (victim == c->graphs.end() && c->graphs.size() >= kMaxGraphs) {
            // a caller that rotates more buffers (or visits more frame sizes) than the cache holds: re-target the least recently used
            // executable graph (same topology, new kernel arguments) instead of synchronising the device and instantiating again
            victim = c->graphs.begin();
            for (auto j = c->graphs.begin(); j != c->graphs.end(); ++j) if (j->second.last_use < victim->second.last_use) victim = j;
        }
        if (victim != c->graphs.end()) {
            ge = victim->second.exec;
            if ((rc = retarget(c, &ge, g, s, &retiring))) { cudaGraphDestroy(g); return rc; }
            c->graphs.erase(victim);
        }
        if (!ge) {
            cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
            if (e != cudaSuccess && c->pdl_level > 0) {             // be conservative: fall back to plain edges once and for all
                cudaGetLastError();
                cudaGraphDestroy(g); g = nullptr;
                c->pdl_level = 0;
                if ((rc = capture_graph(c, record, &g, &launches))) return rc;
                e = cudaGraphInstantiate(&ge, g, 0);
            }
            if (e != cudaSuccess) { if (g) cudaGraphDestroy(g); return fail(c, MEAO_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e)); }
            c->graph_instantiations++;
        }
        cudaGraphDestroy(g);
        it = c->graphs.emplace(key, MeaoCtx::GraphEntry{ge, 0, launches, c->plan_gen}).first;
    }
    it->second.last_use = ++c->graph_clock;
    CUDA_TRY(c, cudaGraphLaunch(it->second.exec, s));
    if (retiring) CUDA_TRY(c, cudaEventRecord(c->retired.back().done, s));    // after the frame that replaced it
    c->launches += it->second.launches;
    return 0;
}

int meao_band_phase_a(MeaoCtx *c, const void *depth, int32_t kind, void *send_up, void *send_down, void *stream)
{
    BAND_GUARD(c, "meao_band_phase_a");
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (!depth) return fail(c, MEAO_ERR_INVALID, "depth is NULL");
    c->last_kind = kind;
    const MeaoCtx::GraphKey key{{depth, send_up, send_down, nullptr}, 100 + kind};
    return launch_cached(c, key, (cudaStream_t)stream, [&](cudaStream_t s, int pdl) {
        int r = record_downsample(c, depth, kind, s);
        if (r) return r;
        PdlScope p(pdl >= 1);
        return halo_kernel(c, send_up, send_down, true, s);
    });
}

int meao_band_phase_b(MeaoCtx *c, const void *recv_up, const void *recv_down, void *ao_out, void *stream)
{
    BAND_GUARD(c, "meao_band_phase_b");
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (!ao_out) return fail(c, MEAO_ERR_INVALID, "ao_out is NULL");
    const int kind = c->last_kind;
    const MeaoCtx::GraphKey key{{recv_up, recv_down, ao_out, nullptr}, 200 + kind};
    c->last_out = ao_out;
    return launch_cached(c, key, (cudaStream_t)stream, [&](cudaStream_t s, int pdl) {
        int r = halo_kernel(c, (void *)recv_up, (void *)recv_down, false, s);
        if (r) return r;
        return record_frame_dag(c, frame_io(c, nullptr, kind, ao_out, false), s, 1, pdl);
    });
}

// ---- native neighbour exchange (include/meao.h) -----------------------------------------------------------------------
namespace {
struct PeerHandlePod {              // what MeaoPeerHandle carries (<= MEAO_PEER_HANDLE_BYTES)
    uint32_t magic;                 // 'MEAO'
    int32_t device;
    int64_t pid;
    int32_t W, H;
    uint64_t arena_bytes;
    uint64_t arena_ptr;             // valid in the exporting process only
    cudaIpcMemHandle_t ipc;         // valid in every other process on this node
};
static_assert(sizeof(PeerHandlePod) <= MEAO_PEER_HANDLE_BYTES, "MeaoPeerHandle too small");
constexpr uint32_t kPeerMagic = 0x4d45414fu;
}  // namespace

int meao_band_export(MeaoCtx *c, MeaoPeerHandle *out)
{
    BAND_GUARD(c, "meao_band_export");
    int rc = ensure_ready(c); if (rc) return rc;
    if (!out) return fail(c, MEAO_ERR_INVALID, "out is NULL");
    PeerHandlePod h{};
    h.magic = kPeerMagic; h.device = c->device; h.pid = (int64_t)getpid(); h.W = c->W; h.H = c->H;
    h.arena_bytes = c->arena_bytes; h.arena_ptr = (uint64_t)(uintptr_t)c->arena;
    const cudaError_t e = cudaIpcGetMemHandle(&h.ipc, c->arena);
    if (e != cudaSuccess) { cudaGetLastError(); memset(&h.ipc, 0, sizeof h.ipc); }     // in-process peers still work without IPC
    memset(out, 0, sizeof *out);
    memcpy(out->bytes, &h, sizeof h);
    return MEAO_OK;
}

int meao_band_connect(MeaoCtx *c, int32_t side, const MeaoPeerHandle *peer)
{
    BAND_GUARD(c, "meao_band_connect");
    int rc = ensure_ready(c); if (rc) return rc;
    if (side != 0 && side != 1) return fail(c, MEAO_ERR_INVALID, "side must be 0 (up) or 1 (down)");
    drop_graph(c);                                  // captured band steps carry the old peer pointers
    if (c->peer_base[side] && c->peer_ipc[side]) cudaIpcCloseMemHandle(c->peer_base[side]);
    c->peer_base[side] = nullptr; c->peer_ipc[side] = false;
    if (!peer) return MEAO_OK;
    if ((side == 0 && c->prev0 < 0) || (side == 1 && c->next1 < 0)) return fail(c, MEAO_ERR_INVALID, "this band has no neighbour on side %d", side);
    {   // The epoch counters of neighbouring bands advance in lock step from 1.  A context that has already stepped can only be
        // (re)connected as a whole: with the other side still attached its epoch cannot restart, and the new neighbour starts at 1.
        BandFlags f{};
        CUDA_TRY(c, cudaMemcpy(&f, c->band_flags, sizeof f, cudaMemcpyDeviceToHost));
        if (f.epoch != 1 || f.error != 0) {
            if (c->peer_base[side ^ 1])
                return fail(c, MEAO_ERR_INVALID, "this band has stepped (epoch %u): disconnect BOTH sides, then connect them again -- every band of the frame restarts at epoch 1", f.epoch);
            BandFlags init{}; init.epoch = 1;
            CUDA_TRY(c, cudaMemcpy(c->band_flags, &init, sizeof init, cudaMemcpyHostToDevice));
            if (c->host_error) *c->host_error = 0;
        }
    }
    PeerHandlePod h;
    memcpy(&h, peer->bytes, sizeof h);
    if (h.magic != kPeerMagic) return fail(c, MEAO_ERR_INVALID, "not a MeaoPeerHandle");
    if (h.W != c->W || h.H != c->H || h.arena_bytes != c->arena_bytes)
        return fail(c, MEAO_ERR_INVALID, "neighbour frame %dx%d (arena %llu B) differs from this context's %dx%d (%zu B)", h.W, h.H,
                    (unsigned long long)h.arena_bytes, c->W, c->H, c->arena_bytes);
    if (h.pid == (int64_t)getpid()) {
        if (h.device != c->device) {
            int can = 0;
            CUDA_TRY(c, cudaDeviceCanAccessPeer(&can, c->device, h.device));
            if (!can) return fail(c, MEAO_ERR_UNSUPPORTED, "device %d cannot access device %d", c->device, h.device);
            const cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(c, MEAO_ERR_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
            cudaGetLastError();
        }
        c->peer_base[side] = (void *)(uintptr_t)h.arena_ptr;
    } else {
        void *p = nullptr;
        const cudaError_t e = cudaIpcOpenMemHandle(&p, h.ipc, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(c, MEAO_ERR_CUDA, "cudaIpcOpenMemHandle: %s", cudaGetErrorString(e)); }
        c->peer_base[side] = p; c->peer_ipc[side] = true;
    }
    const char *t = getenv("MEAO_BAND_TIMEOUT_MS");
    if (t && atof(t) > 0) c->band_timeout_ns = (unsigned long long)(atof(t) * 1e6);
    return MEAO_OK;
}

// prepare_depth on the band has run: push my border rows into the neighbours' LowDepth1..4, signal, wait for theirs
static int record_exchange(MeaoCtx *c, cudaStream_t s)
{
    NvtxRange nv("meao::band_exchange");
    XchgArgs a{};
    a.local = c->band_flags;
    a.host_error = c->host_error_dev;
    a.timeout_ns = c->band_timeout_ns;
    for (int side = 0; side < 2; side++) {
        a.peer[side] = (BandFlags *)c->peer_base[side];                 // BandFlags sit at offset 0 of every arena
        if (!c->peer_base[side]) continue;
        Range r[5]; halo_ranges(c, side, true, r);
        exchange_segments(*c, (const char *)c->arena, (char *)c->peer_base[side], side, r, a);
    }
    if (a.nseg == 0) return 0;
    CUDA_TRY(c, launch_band_exchange(a, s));
    c->launches++;
    return 0;
}

int meao_band_step(MeaoCtx *c, const void *depth, int32_t kind, void *ao_out, void *stream)
{
    BAND_GUARD(c, "meao_band_step");
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (!depth || !ao_out) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    if ((c->prev0 >= 0 && !c->peer_base[0]) || (c->next1 >= 0 && !c->peer_base[1]))
        return fail(c, MEAO_ERR_INVALID, "meao_band_step: connect every neighbour first (meao_band_export / meao_band_connect)");
    // a time-out of an earlier step is sticky; the kernel mirrors it into a mapped host word, so this costs no CUDA call
    if (c->host_error && *(volatile uint32_t *)c->host_error != 0)
        return fail(c, MEAO_ERR_PEER, "neighbour exchange timed out earlier (error %u): see meao_band_status", *(volatile uint32_t *)c->host_error);
    NvtxRange nv("meao::band_step");
    c->last_kind = kind; c->last_out = ao_out;
    const MeaoCtx::GraphKey key{{depth, ao_out, c->peer_base[0], c->peer_base[1]}, 300 + kind};
    const bool has_peer = c->peer_base[0] || c->peer_base[1];
    return launch_cached(c, key, (cudaStream_t)stream, [&](cudaStream_t s, int pdl) {
        int r = record_downsample(c, depth, kind, s, true);
        if (r) return r;
        { PdlScope p(pdl >= 1); if ((r = record_exchange(c, s))) return r; }
        return record_frame_dag(c, frame_io(c, depth, kind, ao_out, true), s, 1, pdl, has_peer);
    });
}

int meao_band_step_host(MeaoCtx *c, const void *depth_host, int32_t kind, uint8_t *ao_host)
{
    BAND_GUARD(c, "meao_band_step_host");
    int rc = ensure_ready(c); if (rc) return rc;
    if (!depth_host || !ao_host) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    const size_t rows = (size_t)(c->band1 - c->band0);
    cudaStream_t s = c->slot_stream[0];
    CUDA_TRY(c, cudaMemcpyAsync(c->depth_stage[0], depth_host, rows * c->W * depth_esize(kind), cudaMemcpyHostToDevice, s));
    if ((rc = meao_band_step(c, c->depth_stage[0], kind, c->ao_stage[0], s))) return rc;
    CUDA_TRY(c, cudaMemcpyAsync(ao_host, c->ao_stage[0], rows * c->W, cudaMemcpyDeviceToHost, s));
    return MEAO_OK;
}

int meao_band_status(MeaoCtx *c, int32_t out4[4])
{
    if (!c || !out4 || c->plan_only || !c->band_flags) return MEAO_ERR_INVALID;
    CUDA_TRY(c, cudaSetDevice(c->device));
    BandFlags f{};
    // a dedicated non-blocking stream: never waits for (or delays) the frames in flight
    CUDA_TRY(c, cudaMemcpyAsync(&f, c->band_flags, sizeof f, cudaMemcpyDeviceToHost, c->slot_stream[1]));
    CUDA_TRY(c, cudaStreamSynchronize(c->slot_stream[1]));
    out4[0] = (int32_t)f.epoch; out4[1] = (int32_t)f.error; out4[2] = c->peer_base[0] ? 1 : 0; out4[3] = c->peer_base[1] ? 1 : 0;
    return MEAO_OK;
}

namespace {
// Every check of meao_render_pitched / meao_bind_event_pitched, on the host before anything is launched.  On success the layer pitches
// of a single-layer context (unused) are replaced by the tight values, so that equivalent views share one cached graph.
int check_views(MeaoCtx *c, const void *depth, int kind, const void *ao_out, ViewPitch *p)
{
    if (!depth || !ao_out) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    if (c->need_low[1].lo < c->own_low[1].lo || c->need_low[1].hi > c->own_low[1].hi)
        return fail(c, MEAO_ERR_INVALID, "interior row band: use meao_render_band_prepare / halo exchange / meao_render_band_finish");
    const int64_t es = depth_esize(kind), rows = c->band1 - c->band0, L = c->layers, W = c->W;
    const struct { const char *name; int64_t v; } all[4] = {{"depth_row_pitch", p->depth_row}, {"depth_layer_pitch", p->depth_layer},
                                                             {"ao_row_pitch", p->ao_row}, {"ao_layer_pitch", p->ao_layer}};
    for (const auto &f : all)
        if (f.v < 0) return fail(c, MEAO_ERR_INVALID, "%s %lld is negative (bottom-up views are not supported)", f.name, (long long)f.v);
    if (p->depth_row > INT32_MAX) return fail(c, MEAO_ERR_INVALID, "depth_row_pitch %lld exceeds INT32_MAX", (long long)p->depth_row);
    if (p->ao_row > INT32_MAX) return fail(c, MEAO_ERR_INVALID, "ao_row_pitch %lld exceeds INT32_MAX", (long long)p->ao_row);
    if (p->depth_row < W * es || p->depth_row % es)
        return fail(c, MEAO_ERR_INVALID, "depth_row_pitch %lld: must be at least width x %lld = %lld bytes and a multiple of %lld",
                    (long long)p->depth_row, (long long)es, (long long)(W * es), (long long)es);
    if (p->ao_row < W) return fail(c, MEAO_ERR_INVALID, "ao_row_pitch %lld is below the width %lld", (long long)p->ao_row, (long long)W);
    if ((uintptr_t)depth % es) return fail(c, MEAO_ERR_INVALID, "depth_dev %p is not aligned to its %lld-byte element", depth, (long long)es);
    if (L > 1) {
        // layers must not overlap.  The extents below are then at most L x layer pitch: at most 2^16 x 2^63, which __int128 holds
        const int64_t dmin = (rows - 1) * p->depth_row + W * es, amin = (rows - 1) * p->ao_row + W;
        if (p->depth_layer < dmin)
            return fail(c, MEAO_ERR_INVALID, "depth_layer_pitch %lld is below (rows - 1) x row pitch + width x %lld = %lld: layers would overlap",
                        (long long)p->depth_layer, (long long)es, (long long)dmin);
        // the kernels address the depth in elements: a layer pitch between two elements would read every layer after the first
        // from misaligned bytes that start outside the view
        if (p->depth_layer % es)
            return fail(c, MEAO_ERR_INVALID, "depth_layer_pitch %lld is not a multiple of the %lld-byte element", (long long)p->depth_layer,
                        (long long)es);
        if (p->ao_layer < amin)
            return fail(c, MEAO_ERR_INVALID, "ao_layer_pitch %lld is below (rows - 1) x row pitch + width = %lld: layers would overlap",
                        (long long)p->ao_layer, (long long)amin);
    } else {
        const ViewPitch t = tight_pitch(*c, kind);
        p->depth_layer = t.depth_layer; p->ao_layer = t.ao_layer;
    }
    // The depth is read through the non-coherent path (ld.global.nc), so an AO view that shares bytes with it is undefined.  The test
    // is conservative: it compares the byte ranges from each view's first to its last element, so two views that interleave without
    // touching a common byte are refused as well.
    using i128 = __int128;
    const i128 d0 = (i128)(uintptr_t)depth, a0 = (i128)(uintptr_t)ao_out;
    const i128 d1 = d0 + (i128)(L - 1) * p->depth_layer + (i128)(rows - 1) * p->depth_row + W * es;
    const i128 a1 = a0 + (i128)(L - 1) * p->ao_layer + (i128)(rows - 1) * p->ao_row + W;
    if (d0 < a1 && a0 < d1) return fail(c, MEAO_ERR_INVALID, "the byte extents of the depth view and the AO view (ao_out_dev) intersect");
    return 0;
}
}  // namespace

namespace {
// The frame of meao_render / meao_render_pitched on a context that ensure_ready has prepared.
int render_views(MeaoCtx *c, const void *depth, int kind, void *ao_out, ViewPitch p, void *stream)
{
    int rc;
    if ((rc = check_views(c, depth, kind, ao_out, &p))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (c->flags & MEAO_FLAG_NO_GRAPH) return record_frame(c, frame_io(c, depth, kind, ao_out, true, &p), s, 0, false);

    // plan-once / replay: one captured graph per (depth, out, kind, pitches), like the reference's command buffer
    // that is re-recorded only when something changed (AO.cs:334-347)
    NvtxRange nv("meao::frame");
    const MeaoCtx::GraphKey key{{depth, ao_out, nullptr, nullptr}, kind, {p.depth_row, p.depth_layer, p.ao_row, p.ao_layer}};
    c->last_kind = kind; c->last_out = ao_out;
    return launch_cached(c, key, s, [&](cudaStream_t cs, int pdl) {
        return record_frame_dag(c, frame_io(c, depth, kind, ao_out, true, &p), cs, 0, pdl);
    });
}
}  // namespace

int meao_render(MeaoCtx *c, const void *depth, int32_t kind, void *ao_out, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    return render_views(c, depth, kind, ao_out, tight_pitch(*c, kind), stream);      // meao_render_pitched at the tight pitches
}

int meao_render_pitched(MeaoCtx *c, const void *depth, int64_t depth_row_pitch, int64_t depth_layer_pitch, int32_t kind,
                        void *ao_out, int64_t ao_row_pitch, int64_t ao_layer_pitch, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    return render_views(c, depth, kind, ao_out, ViewPitch{depth_row_pitch, depth_layer_pitch, ao_row_pitch, ao_layer_pitch}, stream);
}

// ---- CUDA arrays (include/meao.h "CUDA arrays") ------------------------------------------------------------------------
namespace {
constexpr int kArrayGraphKind = 400;        // GraphKey.kind of an array frame: 400 + depth kind

// What a cudaArray_t is, checked against the context on the host before anything is launched.  elem_bits / is_float: the one
// channel the role needs.  Returns 0 and the layer addressing, or fails with a message naming the field.
int check_array(MeaoCtx *c, const void *arr, const char *role, int elem_bits, bool is_float, int *surf_kind)
{
    cudaChannelFormatDesc d{};
    cudaExtent e{};
    unsigned int flags = 0;
    const cudaError_t err = cudaArrayGetInfo(&d, &e, &flags, (cudaArray_t)arr);
    if (err != cudaSuccess) { cudaGetLastError(); return fail(c, MEAO_ERR_INVALID, "%s: not a CUDA array (cudaArrayGetInfo: %s)", role, cudaGetErrorString(err)); }
    const bool one_channel = d.x == elem_bits && d.y == 0 && d.z == 0 && d.w == 0;
    bool kind_ok;
    if (is_float) kind_ok = d.f == cudaChannelFormatKindFloat;
    else kind_ok = d.f == cudaChannelFormatKindUnsigned ||
                   (elem_bits == 8 && d.f == cudaChannelFormatKindUnsignedNormalized8X1) ||
                   (elem_bits == 16 && d.f == cudaChannelFormatKindUnsignedNormalized16X1);
    if (!one_channel || !kind_ok)
        return fail(c, MEAO_ERR_INVALID, "%s: channel format (%d,%d,%d,%d bits, kind %d) is not one %d-bit %s channel", role, d.x, d.y, d.z, d.w, (int)d.f,
                    elem_bits, is_float ? "float" : "unsigned (normalised or not)");
    if ((int)e.width != c->W || (int)e.height != c->H || e.width != (size_t)c->W || e.height != (size_t)c->H)
        return fail(c, MEAO_ERR_INVALID, "%s: extent %zux%zu differs from the context's %dx%d", role, e.width, e.height, c->W, c->H);
    if (!(flags & cudaArraySurfaceLoadStore))
        return fail(c, MEAO_ERR_INVALID, "%s: flags 0x%x lack cudaArraySurfaceLoadStore (register the resource with cudaGraphicsRegisterFlagsSurfaceLoadStore)", role, flags);
    int layers;
    if (flags & cudaArrayCubemap) {
        if (flags & cudaArrayLayered) return fail(c, MEAO_ERR_UNSUPPORTED, "%s: cube-map arrays (cudaArrayCubemap | cudaArrayLayered) are not supported", role);
        layers = 6; *surf_kind = kSurfCube;
    } else if (flags & cudaArrayLayered) {
        layers = e.depth > 0 ? (int)e.depth : 1; *surf_kind = kSurfLayered;
    } else {
        if (e.depth > 1) return fail(c, MEAO_ERR_INVALID, "%s: depth %zu: a 3-D array is not a 2-D or layered image", role, e.depth);
        layers = 1; *surf_kind = kSurf2D;
    }
    if (layers != c->layers)
        return fail(c, MEAO_ERR_INVALID, "%s: layer count %d differs from the context's %d (meao_set_layers)", role, layers, c->layers);
    return 0;
}

int surface_of(MeaoCtx *c, const void *arr, cudaSurfaceObject_t *out)
{
    auto it = c->surfaces.find(arr);
    if (it != c->surfaces.end()) { *out = it->second; return 0; }
    cudaResourceDesc rd{};
    rd.resType = cudaResourceTypeArray;
    rd.res.array.array = (cudaArray_t)arr;
    cudaSurfaceObject_t so = 0;
    CUDA_TRY(c, cudaCreateSurfaceObject(&so, &rd));
    c->surfaces.emplace(arr, so);
    *out = so;
    return 0;
}

// every check of meao_render_arrays / meao_bind_event_arrays; on success `io` holds the surfaces of a frame (made on first use)
int prepare_arrays(MeaoCtx *c, const void *depth_array, int kind, const void *ao_array, ArrayIO *io)
{
    if (!depth_array || !ao_array) return fail(c, MEAO_ERR_INVALID, "depth_array / ao_array is NULL");
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    if (kind == MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_UNSUPPORTED, "depth_kind RAW_D24S8: CUDA arrays have no depth-stencil format");
    if (c->band0 != 0 || c->band1 != c->H) return fail(c, MEAO_ERR_UNSUPPORTED, "CUDA-array frames need a whole-frame context (no row band)");
    int rc;
    const bool d16 = kind == MEAO_DEPTH_RAW_D16_UNORM;
    if ((rc = check_array(c, depth_array, "depth_array", d16 ? 16 : 32, !d16, &io->depth_surf))) return rc;
    if ((rc = check_array(c, ao_array, "ao_array", 8, false, &io->ao_surf))) return rc;
    if ((rc = surface_of(c, depth_array, &io->depth))) return rc;
    if ((rc = surface_of(c, ao_array, &io->ao))) return rc;
    io->ao_array = ao_array;
    return 0;
}
}  // namespace

int meao_render_arrays(MeaoCtx *c, const void *depth_array, int32_t kind, void *ao_array, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    ArrayIO io;
    if ((rc = prepare_arrays(c, depth_array, kind, ao_array, &io))) return rc;
    // the frame graph of meao_render with its first and last node reading / writing the arrays
    NvtxRange nv("meao::frame_arrays");
    const MeaoCtx::GraphKey key{{depth_array, ao_array, nullptr, nullptr}, kArrayGraphKind + kind};
    c->last_kind = kind; c->last_out = ao_array;
    return launch_cached(c, key, (cudaStream_t)stream, [&](cudaStream_t cs, int pdl) {
        FrameIO fio = frame_io(c, nullptr, kind, nullptr, false);
        fio.aio = &io;
        return record_frame_dag(c, fio, cs, 0, pdl);
    });
}

int meao_release_array(MeaoCtx *c, const void *array)
{
    if (!c) return MEAO_ERR_INVALID;
    if (c->plan_only) return fail(c, MEAO_ERR_CUDA, "plan-only context (device < 0): no CUDA device bound, and libmeao has no CPU fallback");
    if (!array) return fail(c, MEAO_ERR_INVALID, "array is NULL");
    {   // a plugin event bound to the array would re-create its surface after the array is freed
        std::lock_guard<std::mutex> g(g_event_mutex);
        for (auto it = g_events.begin(); it != g_events.end();) {
            if (it->second.ctx == c && it->second.arrays && (it->second.depth == array || it->second.out == array)) it = g_events.erase(it); else ++it;
        }
    }
    bool used = c->surfaces.count(array) != 0;
    for (auto &kv : c->graphs) used |= kv.first.kind >= kArrayGraphKind && (kv.first.p[0] == array || kv.first.p[1] == array);
    if (!used) return MEAO_OK;
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaDeviceSynchronize());       // frames that use the array may be in flight on any stream
    for (auto it = c->graphs.begin(); it != c->graphs.end();) {
        if (it->first.kind >= kArrayGraphKind && (it->first.p[0] == array || it->first.p[1] == array)) {
            cudaGraphExecDestroy(it->second.exec);
            it = c->graphs.erase(it);
        } else ++it;
    }
    for (auto &r : c->retired) { cudaGraphExecDestroy(r.exec); cudaEventDestroy(r.done); }     // a retired graph may be an array frame: none is in flight any more
    c->retired.clear();
    auto s = c->surfaces.find(array);
    if (s != c->surfaces.end()) { cudaDestroySurfaceObject(s->second); c->surfaces.erase(s); }
    return MEAO_OK;
}

int meao_render_host_async(MeaoCtx *c, const void *depth_host, int32_t kind, uint8_t *ao_host, int32_t slot)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if (!depth_host || !ao_host) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    if (slot != 0 && slot != 1) return fail(c, MEAO_ERR_INVALID, "slot must be 0 or 1");
    const size_t rows = (size_t)(c->band1 - c->band0) * c->layers;      // layered: L images of H rows (no band)
    cudaStream_t s = c->slot_stream[slot];
    CUDA_TRY(c, cudaMemcpyAsync(c->depth_stage[slot], depth_host, rows * c->W * depth_esize(kind), cudaMemcpyHostToDevice, s));
    // the two slots share the context's intermediates: kernels of consecutive frames are serialised, copies are not
    if (c->compute_done_valid) CUDA_TRY(c, cudaStreamWaitEvent(s, c->compute_done, 0));
    if ((rc = meao_render(c, c->depth_stage[slot], kind, c->ao_stage[slot], s))) return rc;
    CUDA_TRY(c, cudaEventRecord(c->compute_done, s));
    c->compute_done_valid = true;
    CUDA_TRY(c, cudaMemcpyAsync(ao_host, c->ao_stage[slot], rows * c->W, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(c, cudaEventRecord(c->slot_done[slot], s));
    return MEAO_OK;
}

int meao_host_wait(MeaoCtx *c, int32_t slot)
{
    if (!c || (slot != 0 && slot != 1)) return MEAO_ERR_INVALID;
    if (c->plan_only) return MEAO_OK;
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaStreamSynchronize(c->slot_stream[slot]));
    return MEAO_OK;
}

int meao_render_host(MeaoCtx *c, const void *depth_host, int32_t kind, uint8_t *ao_host)
{
    int rc = meao_render_host_async(c, depth_host, kind, ao_host, 0);
    if (rc) return rc;
    return meao_host_wait(c, 0);
}

int meao_synchronize(MeaoCtx *c)
{
    if (!c) return MEAO_ERR_INVALID;
    if (c->plan_only) return MEAO_OK;
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    for (auto st : c->slot_stream) CUDA_TRY(c, cudaStreamSynchronize(st));
    return MEAO_OK;
}

void *meao_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void meao_host_free(void *p) { if (p) cudaFreeHost(p); }

int meao_stage_downsample(MeaoCtx *c, const void *depth, int32_t kind, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (!depth) return fail(c, MEAO_ERR_INVALID, "depth is NULL");
    return record_downsample(c, depth, kind, (cudaStream_t)stream);
}

int meao_stage_render(MeaoCtx *c, int32_t level, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (level < 1 || level > 4) return fail(c, MEAO_ERR_INVALID, "render level %d not in 1..4", level);
    return record_render(c, level, c->last_kind, (cudaStream_t)stream);
}

int meao_stage_render_wide(MeaoCtx *c, int32_t level, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (level < 1 || level > 4) return fail(c, MEAO_ERR_INVALID, "render level %d not in 1..4", level);
    return record_render(c, level, c->last_kind, (cudaStream_t)stream, true);
}

int meao_stage_upsample(MeaoCtx *c, int32_t lo_level, void *ao_out, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    if (lo_level < 1 || lo_level > 4) return fail(c, MEAO_ERR_INVALID, "upsample lo level %d not in 1..4", lo_level);
    return record_upsample(c, lo_level, lo_level == 1 ? ao_out : nullptr, (cudaStream_t)stream);
}

int meao_buffer_desc(const MeaoCtx *c, int32_t id, MeaoBufferDesc *out)
{
    if (!c || !out || c->W <= 0) return MEAO_ERR_INVALID;
    BufferRef b;
    if (!buffer_ref(*c, id, b)) return MEAO_ERR_INVALID;
    out->width = c->lw[b.level]; out->height = c->lh[b.level]; out->slices = b.slices; out->elem_bytes = b.elem;
    return MEAO_OK;
}

int meao_get_buffer(MeaoCtx *c, int32_t id, void *host_out, size_t host_bytes)
{
    int rc = frame_ready(c, c->stream); if (rc) return rc;
    BufferRef b;
    if (!host_out || !buffer_ref(*c, id, b)) return fail(c, MEAO_ERR_INVALID, "bad buffer id %d", id);
    const size_t wb = (size_t)c->lw[b.level] * b.elem, one = wb * c->lh[b.level] * b.slices, need = one * c->layers;     // [L][reference layout]
    if (host_bytes < need) return fail(c, MEAO_ERR_INVALID, "buffer %d needs %zu bytes, got %zu", id, need, host_bytes);
    CUDA_TRY(c, cudaDeviceSynchronize());     // debug path: frames may be in flight on any caller stream
    if (b.slices == 16) {
        __half *tmp = nullptr;
        CUDA_TRY(c, cudaMalloc(&tmp, need));
        cudaError_t e = cudaSuccess;
        for (int l = 0; l < c->layers && e == cudaSuccess; l++)
            e = launch_tiled_atlas(*c, b.level - 2, l, c->last_kind, (__half *)((char *)tmp + l * one), c->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(host_out, tmp, need, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        cudaFree(tmp);
        if (e != cudaSuccess) return fail(c, MEAO_ERR_CUDA, "tiled view: %s", cudaGetErrorString(e));
        return MEAO_OK;
    }
    if ((rc = own_ao(c, id, c->stream))) return rc;
    CUDA_TRY(c, cudaMemcpy2DAsync(host_out, wb, b.base, b.pitch, wb, (size_t)c->lh[b.level] * c->layers, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return MEAO_OK;
}

int meao_debug_view(MeaoCtx *c, int32_t id, void *out, void *stream)
{
    int rc = frame_ready(c, (cudaStream_t)stream); if (rc) return rc;
    BufferRef b;
    if (!out || !buffer_ref(*c, id, b)) return fail(c, MEAO_ERR_INVALID, "bad buffer id %d / out is NULL", id);
    if (c->band0 != 0 || c->band1 != c->H) return fail(c, MEAO_ERR_UNSUPPORTED, "debug views need a whole-frame context (no row band)");
    cudaStream_t s = (cudaStream_t)stream;
    if ((rc = own_ao(c, id, s))) return rc;
    for (int l = 0; l < c->layers; l++) {                           // layered: L images, each from its own layer of the source
        DebugViewArgs a;
        debug_view_args(*c, id, l, c->last_kind, (uint8_t *)out + (size_t)l * c->W * c->H, a);
        CUDA_TRY(c, launch_debug_view(a, s));
        c->launches++;
    }
    return MEAO_OK;
}

int meao_set_buffer(MeaoCtx *c, int32_t id, const void *host_in, size_t host_bytes)
{
    int rc = ensure_ready(c); if (rc) return rc;
    BufferRef b;
    if (!host_in || !buffer_ref(*c, id, b) || b.slices != 1)
        return fail(c, MEAO_ERR_INVALID, "buffer id %d cannot be set", id);
    const size_t wb = (size_t)c->lw[b.level] * b.elem, need = wb * c->lh[b.level] * c->layers;      // [L][h][w]
    if (host_bytes < need) return fail(c, MEAO_ERR_INVALID, "buffer %d needs %zu bytes, got %zu", id, need, host_bytes);
    CUDA_TRY(c, cudaDeviceSynchronize());
    CUDA_TRY(c, cudaMemcpy2DAsync(b.base, b.pitch, host_in, wb, wb, (size_t)c->lh[b.level] * c->layers, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    return MEAO_OK;
}

// The constant getters work without a device context being current: they only need the plan.
static int plan_only(MeaoCtx *c)
{
    if (!c || c->W <= 0) return MEAO_ERR_INVALID;
    if (c->plan_dirty) replan(c);           // the captured graphs are dropped by the next ensure_ready, on c->device
    refresh_constants(c);                   // the tables are written by the next frame, on its stream
    return 0;
}

int meao_render_constants(MeaoCtx *c, int32_t level, float out[28])
{
    if (plan_only(c) || !out || level < 1 || level > 4) return MEAO_ERR_INVALID;
    memcpy(out, c->plan.inv_thickness[level], 48);
    memcpy(out + 12, c->plan.sample_weight[level], 48);
    out[24] = c->plan.inv_slice_dim[level][0]; out[25] = c->plan.inv_slice_dim[level][1];
    out[26] = c->plan.reject_fadeoff; out[27] = c->plan.intensity;
    return MEAO_OK;
}

int meao_render_constants_wide(MeaoCtx *c, int32_t level, float out[28])
{
    if (plan_only(c) || !out || level < 1 || level > 4) return MEAO_ERR_INVALID;
    memcpy(out, c->plan.inv_thickness_wide[level], 48);
    memcpy(out + 12, c->plan.sample_weight[level], 48);
    out[24] = c->plan.inv_slice_dim_wide[level][0]; out[25] = c->plan.inv_slice_dim_wide[level][1];
    out[26] = c->plan.reject_fadeoff; out[27] = c->plan.intensity;
    return MEAO_OK;
}

int meao_upsample_constants(MeaoCtx *c, int32_t lo, float out[8])
{
    if (plan_only(c) || !out || lo < 1 || lo > 4) return MEAO_ERR_INVALID;
    out[0] = c->plan.inv_low[lo][0]; out[1] = c->plan.inv_low[lo][1];
    out[2] = c->plan.inv_high[lo][0]; out[3] = c->plan.inv_high[lo][1];
    out[4] = c->plan.noise_filter_strength[lo]; out[5] = c->plan.step_size[lo];
    out[6] = c->plan.blur_tolerance[lo]; out[7] = c->plan.upsample_tolerance[lo];
    return MEAO_OK;
}

int meao_zbuffer_params(MeaoCtx *c, float out[4])
{
    if (plan_only(c) || !out) return MEAO_ERR_INVALID;
    memcpy(out, c->plan.zb, 16);
    return MEAO_OK;
}

int meao_render_constants_layer(MeaoCtx *c, int32_t layer, int32_t level, int32_t wide, float out[28])
{
    if (plan_only(c) || !out || level < 1 || level > 4 || layer < 0 || layer >= c->layers) return MEAO_ERR_INVALID;
    int rc = wide ? meao_render_constants_wide(c, level, out) : meao_render_constants(c, level, out);
    if (rc) return rc;
    const CamConsts &cc = c->layer_consts[layer];
    memcpy(out, wide ? cc.inv_thickness_wide[level] : cc.inv_thickness[level], 48);
    return MEAO_OK;
}

int meao_zbuffer_params_layer(MeaoCtx *c, int32_t layer, float out[4])
{
    if (plan_only(c) || !out || layer < 0 || layer >= c->layers) return MEAO_ERR_INVALID;
    const CamConsts &cc = c->layer_consts[layer];
    out[0] = cc.zb[0]; out[1] = cc.zb[1]; out[2] = out[3] = 0.0f;
    return MEAO_OK;
}

static int composite_args(MeaoCtx *c, const void *ao, const void *color, int fmt)
{
    if (!ao || !color) return fail(c, MEAO_ERR_INVALID, "ao / colour target is NULL");
    if (fmt != MEAO_FMT_RGBA8_UNORM && fmt != MEAO_FMT_RGBA16_FLOAT) return fail(c, MEAO_ERR_INVALID, "bad colour format %d", fmt);
    if (((uintptr_t)ao & 3) || ((uintptr_t)color & 15)) return fail(c, MEAO_ERR_INVALID, "composite needs a 4-byte aligned AO and a 16-byte aligned colour pointer");
    return 0;
}

int meao_composite_framebuffer(MeaoCtx *c, const void *ao, void *color, int32_t fmt, void *stream)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if ((rc = composite_args(c, ao, color, fmt))) return rc;
    const long long npix = (long long)c->W * (c->band1 - c->band0) * c->layers;
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, color, npix, fmt == MEAO_FMT_RGBA16_FLOAT, 1, 1, 0, (cudaStream_t)stream));
    c->launches++;
    return MEAO_OK;
}

int meao_composite_gbuffer(MeaoCtx *c, const void *ao, void *g0, void *g3, int32_t fmt3, void *stream)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if ((rc = composite_args(c, ao, g0, MEAO_FMT_RGBA8_UNORM)) || (rc = composite_args(c, ao, g3, fmt3))) return rc;
    const long long npix = (long long)c->W * (c->band1 - c->band0) * c->layers;
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, g0, npix, 0, 0, 1, 1, (cudaStream_t)stream));                               // gbuffer0.a
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, g3, npix, fmt3 == MEAO_FMT_RGBA16_FLOAT, 1, 0, 1, (cudaStream_t)stream));   // gbuffer3.rgb
    c->launches += 2;
    return MEAO_OK;
}

int meao_composite_debug(MeaoCtx *c, const void *view, void *color, int32_t fmt, void *stream)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if ((rc = composite_args(c, view, color, fmt))) return rc;
    const long long npix = (long long)c->W * (c->band1 - c->band0) * c->layers;
    CUDA_TRY(c, launch_debug_composite((const uint8_t *)view, color, npix, fmt == MEAO_FMT_RGBA16_FLOAT, (cudaStream_t)stream));
    c->launches++;
    return MEAO_OK;
}

int meao_bind_event(MeaoCtx *c, int32_t event_id, const void *depth, int32_t kind, void *ao_out, void *stream)
{
    if (!c) return MEAO_ERR_INVALID;
    std::lock_guard<std::mutex> g(g_event_mutex);
    if (!depth && !ao_out) { g_events.erase(event_id); return MEAO_OK; }
    g_events[event_id] = EventBinding{c, depth, kind, ao_out, stream, false, true, ViewPitch{}};
    return MEAO_OK;
}

int meao_bind_event_pitched(MeaoCtx *c, int32_t event_id, const void *depth, int64_t depth_row_pitch, int64_t depth_layer_pitch, int32_t kind,
                            void *ao_out, int64_t ao_row_pitch, int64_t ao_layer_pitch, void *stream)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!depth && !ao_out) {
        std::lock_guard<std::mutex> g(g_event_mutex);
        g_events.erase(event_id);
        return MEAO_OK;
    }
    // checked now: the plugin event cannot report an error
    int rc = ensure_ready(c); if (rc) return rc;
    ViewPitch p{depth_row_pitch, depth_layer_pitch, ao_row_pitch, ao_layer_pitch};
    if ((rc = check_views(c, depth, kind, ao_out, &p))) return rc;
    std::lock_guard<std::mutex> g(g_event_mutex);
    g_events[event_id] = EventBinding{c, depth, kind, ao_out, stream, false, false, p};
    return MEAO_OK;
}

int meao_bind_event_arrays(MeaoCtx *c, int32_t event_id, const void *depth_array, int32_t kind, void *ao_array, void *stream)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!depth_array && !ao_array) {
        std::lock_guard<std::mutex> g(g_event_mutex);
        g_events.erase(event_id);
        return MEAO_OK;
    }
    // checked now: the plugin event cannot report an error
    int rc = ensure_ready(c); if (rc) return rc;
    ArrayIO io;
    if ((rc = prepare_arrays(c, depth_array, kind, ao_array, &io))) return rc;
    std::lock_guard<std::mutex> g(g_event_mutex);
    g_events[event_id] = EventBinding{c, depth_array, kind, ao_array, stream, true, false, ViewPitch{}};
    return MEAO_OK;
}

void meao_render_event(int event_id)
{
    EventBinding b;
    {
        std::lock_guard<std::mutex> g(g_event_mutex);
        auto it = g_events.find(event_id);
        if (it == g_events.end()) return;
        b = it->second;
    }
    if (b.arrays) meao_render_arrays(b.ctx, b.depth, b.kind, b.out, b.stream);
    else if (b.tight) meao_render(b.ctx, b.depth, b.kind, b.out, b.stream);      // meao_render_pitched at the tight pitches of now
    else meao_render_pitched(b.ctx, b.depth, b.pitch.depth_row, b.pitch.depth_layer, b.kind, b.out, b.pitch.ao_row, b.pitch.ao_layer, b.stream);
}

MeaoRenderEventFunc meao_get_render_event_func(void) { return meao_render_event; }

int64_t meao_launch_count(const MeaoCtx *c) { return c ? c->launches : 0; }
int meao_pdl_level(const MeaoCtx *c) { return c ? c->pdl_level : -1; }
int meao_kernels_per_frame(const MeaoCtx *c)
{
    return (int)frame_schedule(c ? c->variants : MeaoVariants{}).size();        // as set: the plan may not be rebuilt yet
}

int64_t meao_algorithmic_bytes(const MeaoCtx *c, int32_t stage)
{
    if (!c || c->W <= 0) return MEAO_ERR_INVALID;
    auto px = [&](int l) { return (int64_t)c->lw[l] * c->lh[l] * c->layers; };      // every layer moves the same bytes
    // SURVEY.md 8(d): every buffer of the reference data-flow read once per consuming stage, written once
    const int64_t ds1 = 6 * px(0) + 4 * px(1) + 4 * px(2) + 32 * px(3) + 32 * px(4);
    const int64_t ds2 = 4 * px(2) + 4 * px(3) + 4 * px(4) + 32 * px(5) + 32 * px(6);
    int64_t ren = 0, ups = 0, ups_final = 0;
    for (int k = 1; k <= 4; k++) ren += 32 * px(k + 2) + px(k);
    for (int lo = 4; lo >= 1; lo--) {
        const int hi = lo - 1;
        const int64_t b = 5 * px(lo) + (hi == 0 ? 2 : 5) * px(hi) + px(hi);
        ups += b;
        if (lo == 1) ups_final = b;
    }
    switch (stage) {
        case 0: return ds1 + ds2 + ren + ups;
        case 1: return ds1;
        case 2: return ds2;
        case 3: return ren;
        case 4: return ups;
        case 5: return ups_final;
        default: return MEAO_ERR_INVALID;
    }
}

int meao_selftest_div(MeaoCtx *c, uint64_t n, uint32_t seed, uint64_t *mismatches)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if (!mismatches) return fail(c, MEAO_ERR_INVALID, "mismatches is NULL");
    unsigned long long *d = nullptr;
    CUDA_TRY(c, cudaMalloc(&d, sizeof *d));
    cudaError_t e = cudaMemsetAsync(d, 0, sizeof *d, c->stream);
    if (e == cudaSuccess) e = launch_selftest_div(n, seed, d, c->sm_count, c->stream);
    unsigned long long h = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h, d, sizeof h, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    cudaFree(d);
    if (e != cudaSuccess) return fail(c, MEAO_ERR_CUDA, "selftest: %s", cudaGetErrorString(e));
    *mismatches = h;
    return MEAO_OK;
}

int meao_set_profile_repeats(MeaoCtx *c, int32_t n)
{
    if (!c || n < 1 || n > 1000) return MEAO_ERR_INVALID;
    c->profile_repeats = n;
    return MEAO_OK;
}

int meao_profile_frame(MeaoCtx *c, const void *depth, int32_t kind, void *ao_out, float *ms_out, const char **names_out, int32_t capacity)
{
    int rc = frame_ready(c, c->stream); if (rc) return rc;
    if (!depth || !ao_out) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    CUDA_TRY(c, cudaDeviceSynchronize());
    if ((rc = record_frame(c, frame_io(c, depth, kind, ao_out, true), c->stream, 0, true))) return rc;
    const int n = (int)c->last_profile.size();
    for (int i = 0; i < n && i < capacity; i++) {
        if (ms_out) ms_out[i] = c->last_profile[i].second;
        if (names_out) names_out[i] = c->last_profile[i].first.c_str();
    }
    return n;
}

}  // extern "C"
