// meao_api.cu -- context, planner and C ABI of libmeao.so (see include/meao.h).
//
// Host-side mirror of the parts of AmbientOcclusion.cs that own the hot path:
//   RTHandle geometry/formats (AO.cs:124-282), the CPU constant math of the three Push*Commands
//   recorders (AO.cs:561-593, 660-734, 750-771), the record order of RebuildCommandBuffers
//   (AO.cs:511-531) and the re-plan triggers of LateUpdate (AO.cs:329-350).
// "Plan once, replay per frame" maps to: constants + TMA descriptors are rebuilt only when a
// parameter, the camera or the size changes; a frame is then ten kernel launches (or one CUDA
// graph launch) on one stream.
#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
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

// Everything of a context that depends on the frame size and the layer count: what the recorders read (frame_record.h FrameState)
// plus the band's neighbours and row ranges and the state of the per-layer camera table slot.  A reserved context (meao_reserve,
// meao_reserve_layers) keeps one of these per recently used (W, H, L) (MeaoCtx::size_slots) and swaps it in on a resize or a layer
// change to it, so a return to a planned (W, H, L) is host bookkeeping only.
struct SizeState : FrameState {
    int prev0 = -1, next1 = -1;             // the neighbour bands' extents (meao_set_row_band)
    Range need_low[5];                      // rows of LowDepth<k> required by this band
    Range own_low[5];                       // rows of LowDepth<k> this band produces
    bool cam_table_stale = true;            // a structural re-plan changed layer_consts (ensure_ready uploads them after a device synchronise)
    int slot = 0;                           // the arena slot of this size's camera tables (FrameState::layer_zb / layer_ren)
    bool table_pending = false;             // the slot's tables are not written yet: the next frame writes them on its own stream
    uint64_t plan_gen = 0;                  // the frame-constant generation (MeaoCtx::consts_gen) this size's plan was built at
    // a host camera changed while a device camera buffer was bound (note_camera_change), or a host thickness_modifier / intensity while a
    // device parameter buffer was (meao_set_params): the change moved no generation, so this size's plan still holds the older host
    // values, which the constant getters describe -- they plan it again first
    bool host_consts_stale = false;
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
    // meao_set_layer_viewports: one viewport per layer, or empty (the tight layer layout).  views_pending: the arena's copy
    // (FrameState::layer_views) is older than the table; the next frame writes it on its own stream (write_tables).  views_max[i]: the
    // layer with the largest value of field i (depth_x .. ao_slice), for the per-frame fit tests of arrays.  views_last[r][0] / [1]: the
    // layer whose rectangle ends last in (y, x) / (slice, y, x) order, for role r (0 depth, 1 AO) -- with every row inside its row pitch
    // the one whose last byte lies furthest into its slice / into the view (check_view_pitches).  views_checked: the sizes at which the
    // AO rectangles were found disjoint, none larger than another (a rectangle at a smaller size lies inside the larger one at the same
    // origin), cleared with the table.
    std::vector<MeaoLayerViewport> views;
    bool views_pending = false;
    int views_max[6] = {0, 0, 0, 0, 0, 0};
    int views_last[2][2] = {{0, 0}, {0, 0}};
    std::vector<std::pair<int, int>> views_checked;
    MeaoVariants variants = {0, 0, 0, 0};
    int hierarchy_depth = 4;                // meao_set_hierarchy_depth (a structural input: the schedule's levels, frame_record.h effective_depth)
    int projection = MEAO_PROJECTION_PERSPECTIVE;  // meao_set_projection (a structural input: it selects the orthographic kernels)
    // meao_set_layer_projections: one MeaoProjection per layer, or empty (every layer has `projection`).  A structural input like the
    // context's projection: a table that mixes both selects the mixed kernels (frame_record.h launch_entry_mixed).  layer_proj_ortho: its
    // orthographic entries.
    std::vector<int32_t> layer_proj;
    int layer_proj_ortho = 0;
    // meao_bind_device_cameras: the bound buffer (cams.cams, nullptr: none) and its capacity in cameras.  A structural input: the frames
    // run the camera stage (frame_record.h frame_schedule) and take the layered kernels at every layer count.  cams.status: the kernel's
    // status words, a small allocation of their own made at bind time (nullptr on a plan-only context).
    DeviceCameras cams;
    int cams_capacity = 0;
    // meao_bind_device_params: the bound buffer (dev_params.params, nullptr: none).  A structural input: the frames run the parameter
    // stage (frame_record.h frame_schedule) and take the *_params_layered renders at every layer count.  dev_params.derived / .status: the
    // derived slot and the kernel's status words, one small allocation made at bind time (nullptr on a plan-only context).
    RenderParamArgs dev_params{};
    bool plan_dirty = true;                 // a structural input changed: the next frame re-plans (replan)
    // Frame constants (include/meao.h): bumped by every change of MeaoParams or of a camera that keeps the Z direction.  A size whose
    // plan_gen is older re-plans its constants on the host (refresh_constants); a graph captured at an older one re-targets (launch_cached).
    uint64_t consts_gen = 0;
    // meao_frame_generation: bumped by every change a frame recorded into a caller's graph depends on (include/meao.h)
    int64_t frame_gen = 0;

    // meao_reserve: the arena is laid out for res_w x res_h (0 x 0: for the current size) and every size inside it keeps its plan;
    // meao_reserve_layers: and for res_layers layers (0: the current count), with every layer count up to it keeping its plan too
    int res_w = 0, res_h = 0, res_layers = 0;
    struct SizeSlot { bool valid = false; uint64_t last_use = 0; SizeState s; };
    SizeSlot size_slots[kSizeSlots];        // slot i: the parked state of a planned (W, H, L) whose camera tables live in arena slot i
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
    // size: the frame size, camera table slot and layer count the graph was captured at (launch_cached fills it in) -- a reserved
    // context keeps the graphs of every (W, H, L) it has visited, a size re-planned into another slot never replays a graph that reads
    // the old slot, and a slot re-used by another layer count never replays a graph launched with the other count's grid.
    // table: the layer-viewport table an array frame reads (nullptr: none; a pointer frame carries it in p[2]), so that on a context
    // whose table may come and go without a re-plan (meao_reserve_layers) a frame never replays a graph recorded with the other choice.
    // list / list_hash: a batch's whole list (kBatchArrayGraphKind+: the depth arrays, then the AO arrays; kBatchGraphKind+: depth, depth
    // row pitch, AO, AO row pitch per layer), compared by its hash first and in full on a tie, so a graph replays only its own list.
    struct GraphKey { const void *p[4]; int kind; int64_t pitch[4] = {0, 0, 0, 0}; int size[4] = {0, 0, 0, 0}; uint64_t list_hash = 0;
        std::vector<uintptr_t> list = {};
        const void *table = nullptr;
        uint64_t proj = 0;                  // FrameState::proj_key: the layers' projections the graph was recorded with
        const void *cams = nullptr;         // the device camera buffer the graph's camera stage reads (nullptr: none)
        const void *params = nullptr;       // the device parameter buffer the graph's parameter stage reads (nullptr: none)
        bool operator<(const GraphKey &o) const {
        for (int i = 0; i < 4; i++) if (p[i] != o.p[i]) return p[i] < o.p[i];
        if (kind != o.kind) return kind < o.kind;
        if (proj != o.proj) return proj < o.proj;
        if (cams != o.cams) return cams < o.cams;
        if (params != o.params) return params < o.params;
        for (int i = 0; i < 4; i++) if (pitch[i] != o.pitch[i]) return pitch[i] < o.pitch[i];
        for (int i = 0; i < 4; i++) if (size[i] != o.size[i]) return size[i] < o.size[i];
        if (table != o.table) return table < o.table;
        if (list_hash != o.list_hash) return list_hash < o.list_hash;
        return list < o.list; } };
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
    if (c->res_w <= 0)
        return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands need an unreserved context (this one reserves %d layers, meao_reserve_layers)", what,
                    c->res_layers);
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands need an unreserved context (this one reserves %dx%d, meao_reserve)", what, c->res_w, c->res_h);
}
// Row bands and an orthographic projection exclude each other too: the band paths have no orthographic kernels.
int refuse_ortho_band(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands and the halo exchange are not supported under an orthographic projection "
                "(meao_set_projection)", what);
}
// An orthographic layer of a projection table (meao_set_layer_projections) carries the same restriction.
int refuse_ortho_layer_band(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands and the halo exchange are not supported with an orthographic layer "
                "(meao_set_layer_projections)", what);
}
// And a bound device camera buffer too: the band paths run the single-image kernels, which read the camera from their arguments.
int refuse_device_cameras_band(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands and the halo exchange are not supported while a device camera buffer is bound "
                "(meao_bind_device_cameras)", what);
}
// And a bound device parameter buffer: the band paths run the single-image kernels, which read reject_fadeoff and intensity from their
// arguments.
int refuse_device_params_band(MeaoCtx *c, const char *what)
{
    return fail(c, MEAO_ERR_UNSUPPORTED, "%s: row bands and the halo exchange are not supported while a device parameter buffer is bound "
                "(meao_bind_device_params)", what);
}
#define BAND_GUARD(c, what) do { if ((c) && (c)->layers > 1) return refuse_layered((c), (what)); \
    if ((c) && ((c)->res_w > 0 || (c)->res_layers > 0)) return refuse_reserved((c), (what)); \
    if ((c) && (c)->projection != MEAO_PROJECTION_PERSPECTIVE) return refuse_ortho_band((c), (what)); \
    if ((c) && (c)->layer_proj_ortho > 0) return refuse_ortho_layer_band((c), (what)); \
    if ((c) && (c)->cams.cams) return refuse_device_cameras_band((c), (what)); \
    if ((c) && (c)->dev_params.params) return refuse_device_params_band((c), (what)); } while (0)
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

// The projection of layer l: its entry of the projection table while one is set, else the context's (meao_set_layer_projections)
inline int layer_projection(const MeaoCtx *c, int l) { return c->layer_proj.empty() ? c->projection : c->layer_proj[l]; }

// Z direction of the context's cameras (meao_set_layer_cameras requires one for all layers)
inline int ctx_reversed_z(const MeaoCtx *c) { return c->layer_cams.empty() ? c->camera.reversed_z : c->layer_cams[0].reversed_z; }

// A change of the cameras in effect.  Their near and far planes and fields of view are frame constants; their Z direction selects
// kernel instantiations (prepare_slot), so a change of it re-plans like any structural input.  While a device camera buffer is bound the
// planes and fields of view are the buffer's: a host change that keeps the Z direction is only recorded, for after the unbind.
void note_camera_change(MeaoCtx *c, int old_reversed_z, int new_reversed_z)
{
    if (c->cams.cams && old_reversed_z == new_reversed_z) {
        c->host_consts_stale = true;
        for (auto &slot : c->size_slots) slot.s.host_consts_stale = true;
        return;
    }
    c->frame_gen++;
    if (old_reversed_z != new_reversed_z) c->plan_dirty = true;
    else c->consts_gen++;
}

// The camera-dependent constants of camera `cam` (the part of build_plan that reads the camera).
// Under an orthographic projection (include/meao.h meao_set_projection) ZBufferParams holds the affine linearisation {1 - n/f, n/f}
// (reversed: {n/f - 1, 1}), the inv_thickness tables hold it_i = (far / ThicknessMultiplier) / SampleThickness[i] -- a sphere of constant
// size, in units of LinearDepth (eye depth / far) -- and the padding value is the linearisation of raw depth 0.  `projection`: that of
// the camera's layer (layer_projection).
void camera_consts(const MeaoCtx *c, const MeaoCamera &cam, int projection, CamConsts &p)
{
    const bool ortho = projection == MEAO_PROJECTION_ORTHOGRAPHIC;
    if (!ortho) {
        // AO.cs:561-568
        const float fpn = cam.far_clip / cam.near_clip;
        if (cam.reversed_z) { p.zb[0] = fpn - 1; p.zb[1] = 1; } else { p.zb[0] = 1 - fpn; p.zb[1] = fpn; }
    } else {
        const float r = cam.near_clip / cam.far_clip;
        if (cam.reversed_z) { p.zb[0] = r - 1; p.zb[1] = 1; } else { p.zb[0] = 1 - r; p.zb[1] = r; }
    }

    float thick[12];
    sample_thickness(thick);
    for (int k = 1; k <= 4; k++) {
        const int src_w = c->lw[k + 2];
        const float ScreenspaceDiameter = 10;                                                        // AO.cs:669
        float ThicknessMultiplier = 2 * cam.tan_half_fov_h * ScreenspaceDiameter / src_w;           // AO.cs:678
        if (c->variants.single_pass_stereo) ThicknessMultiplier *= 2;                                // AO.cs:680
        float InverseRangeFactor = ortho ? cam.far_clip / ThicknessMultiplier : 1 / ThicknessMultiplier;   // AO.cs:683
        for (int i = 0; i < 12; i++) p.inv_thickness[k][i] = InverseRangeFactor / thick[i];          // AO.cs:687-688
        {   // the same recorder fed a non-tiled source (LowDepth<k>): kernel "main"
            float tm = 2 * cam.tan_half_fov_h * ScreenspaceDiameter / c->lw[k];                     // AO.cs:678
            tm *= 2;                                                                                 // AO.cs:679 (!source.isTiled)
            if (c->variants.single_pass_stereo) tm *= 2;                                             // AO.cs:680
            const float irf = ortho ? cam.far_clip / tm : 1 / tm;                                    // AO.cs:683
            for (int i = 0; i < 12; i++) p.inv_thickness_wide[k][i] = irf / thick[i];
        }
        // value of the atlas padding texels (SURVEY.md P3): Downsample1 writes Linearize(OOB load = 0),
        // Downsample2 writes 0 (its OOB load of DS4x)
        float pad = 0.0f;
        if (k <= 2) {
            // raw depth 0 through Linearize (DS1:40-45); linear ingest: 0
            if (ortho) pad = cam.reversed_z ? 1e5f : std::fmaf(p.zb[0], 0.0f, p.zb[1]);
            else pad = cam.reversed_z ? 1e5f : 1.0f / std::fmaf(p.zb[0], 0.0f, p.zb[1]);
        }
        p.pad[k] = pad;   // the depth-kind dependent part (linear ingest -> 0) is applied at launch
    }
}

// Rebuild the per-dispatch constants (the CPU half of RebuildCommandBuffers, AO.cs:496-540).
void build_plan(MeaoCtx *c)
{
    Plan &p = c->plan;
    // every layer's camera constants, with its camera and its projection: one entry per run of layers that share both computed, copied to
    // the others of the run
    const int L = c->layers;
    c->layer_consts.resize(L);
    auto cam = [c](int l) -> const MeaoCamera & { return c->layer_cams.empty() ? c->camera : c->layer_cams[l]; };
    for (int l = 0; l < L; l++) {
        if (l > 0 && layer_projection(c, l) == layer_projection(c, l - 1) && memcmp(&cam(l), &cam(l - 1), sizeof(MeaoCamera)) == 0)
            c->layer_consts[l] = c->layer_consts[l - 1];
        else camera_consts(c, cam(l), layer_projection(c, l), c->layer_consts[l]);
    }
    // the Plan's own camera constants: the first layer's
    const CamConsts &cc = c->layer_consts[0];
    p.zb[0] = cc.zb[0]; p.zb[1] = cc.zb[1];
    p.zb[2] = p.zb[3] = 0;
    p.variants = PlanVariants(c->variants, c->hierarchy_depth);
    p.reversed_z = ctx_reversed_z(c);
    plan_projections(*c, [c](int l) { return layer_projection(c, l) == MEAO_PROJECTION_ORTHOGRAPHIC; });
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
    c->host_consts_stale = false;
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
    c->frame_gen++;                     // a recorded frame would touch freed memory
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
// The layer count the arena is laid out for: the layer reservation, or the current count
inline int arena_layers(const MeaoCtx *c) { return c->res_layers > 0 ? c->res_layers : c->layers; }

// Places the buffers of the current size and layer count (c->W x c->H x c->layers) in the arena, where a fresh context of that size has
// them (with a layer reservation: the tables where one of the reserved count has them), with its camera tables in slot `slot`; encodes
// the TMA maps and resets the band to the whole frame.  Host work only: no allocation, no CUDA call.
int place_size(MeaoCtx *c, int slot)
{
    c->band0 = 0; c->band1 = c->H; c->prev0 = -1; c->next1 = -1;
    c->slot = slot;
    place_frame(*c, arena_layout(c->W, c->H, c->layers, arena_layers(c)), (char *)c->arena, slot);
    if (!c->arena) return setup_band(c);
    c->tma_ok = c->encode && encode_maps(*c, [c](CUtensorMap &m, const MapSpec &sp) {
        return make_map(c, &m, sp.elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, sp.elem, sp.base, sp.w, sp.h,
                        sp.pitch_elems, sp.bw, sp.bh) == 0;
    });
    if (!c->tma_ok) memset(&c->maps, 0, sizeof c->maps);
    return setup_band(c);
}

// A new arena for arena_w x arena_h x arena_layers, laid out by arena_layout; the current size (if any) is placed in it and
// re-planned by the next ensure_ready.  keep_old: allocate before freeing the old arena, so that MEAO_ERR_NOMEM leaves the context as
// it was (meao_reserve); otherwise the old arena goes first, as a resize always did.
int allocate(MeaoCtx *c, bool keep_old = false)
{
    const ArenaLayout a = arena_layout(arena_w(c), arena_h(c), arena_layers(c));
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
    c->frame_gen++;
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

// Reserved contexts: make w x h x layers the current size and layer count without touching the device.  The current one is parked in
// its slot; a (W, H, L) parked earlier is swapped back in as it was (plan, maps, camera tables); a new one takes a free slot or the
// least recently used one, and is planned on the host -- its camera tables are written by its first frame, on that frame's stream
// (write_tables).
// HAZARD: a parked size keeps the constants it was parked with.  Frame constants may have changed since, so a size swapped back in
// re-plans its constants here (refresh_constants) before any frame or getter can read them, and its graphs re-target at their first
// replay; it must never replay with the constants it was parked with.
int switch_size(MeaoCtx *c, int w, int h, int layers)
{
    c->frame_gen++;
    SizeState &cur = *c;
    if (c->W > 0) c->size_slots[c->slot] = MeaoCtx::SizeSlot{true, c->size_clock, cur};
    int slot = -1;
    for (int i = 0; i < kSizeSlots; i++) {
        MeaoCtx::SizeSlot &s = c->size_slots[i];
        if (s.valid && s.s.W == w && s.s.H == h && s.s.layers == layers) {
            cur = s.s;
            s.last_use = ++c->size_clock;
            refresh_constants(c);
            return 0;
        }
        if (slot < 0 || (c->size_slots[slot].valid && (!s.valid || s.last_use < c->size_slots[slot].last_use))) slot = i;
    }
    c->W = w; c->H = h; c->layers = layers;
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
    if (!c->views.empty()) CUDA_TRY(c, cudaMemcpy(c->layer_views, c->views.data(), c->views.size() * sizeof(LayerView), cudaMemcpyHostToDevice));
    c->cam_table_stale = false;
    c->table_pending = false;
    c->views_pending = false;
    return 0;
}

// The tables of a size newly planned by switch_size, or re-planned after a frame-constant change (refresh_constants), written in
// stream order before the first frame that reads them, on that frame's stream.  The slot may have held another size's tables, or
// this size's older ones: frames of one context run in the order they are issued (include/meao.h), so every earlier frame that
// read it has completed before this copy lands.  The source is pageable, so the runtime stages it and
// the vectors may go when the call returns.
int write_tables(MeaoCtx *c, cudaStream_t s)
{
    if (c->views_pending) {         // a changed layer-viewport table (one for every size): the same stream-order rule
        CUDA_TRY(c, cudaMemcpyAsync(c->layer_views, c->views.data(), c->views.size() * sizeof(LayerView), cudaMemcpyHostToDevice, s));
        c->views_pending = false;
    }
    if (!c->table_pending) return 0;
    // a bound device camera buffer: every frame's camera stage derives the tables, and the later calls of a staged frame read the ones
    // meao_stage_downsample derived -- the host cameras' tables must not land over them
    if (c->cams.cams) { c->table_pending = false; return 0; }
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

// ---- frames inside a caller's graph (include/meao.h) ------------------------------------------------------------------------
// *active: the caller's stream s is being captured (cudaStreamBeginCapture, torch.cuda.graph), so the call records its launches into
// that capture.  The legacy NULL stream is never captured; a query on cudaStreamLegacy while another stream captures may fail with
// cudaErrorStreamCaptureImplicit, which means the same.  An invalidated capture is refused: nothing can be recorded into it.
int stream_capturing(MeaoCtx *c, cudaStream_t s, bool *active)
{
    *active = false;
    if (!s) return 0;
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamGetCaptureInfo(s, &st);
    if (e == cudaErrorStreamCaptureImplicit) { cudaGetLastError(); return 0; }
    if (e == cudaErrorStreamCaptureInvalidated) { cudaGetLastError(); st = cudaStreamCaptureStatusInvalidated; }
    else if (e != cudaSuccess) return fail(c, MEAO_ERR_CUDA, "cudaStreamGetCaptureInfo failed: %s", cudaGetErrorString(e));
    if (st == cudaStreamCaptureStatusInvalidated)
        return fail(c, MEAO_ERR_CUDA, "the stream's capture has been invalidated by an earlier error: nothing recorded");
    *active = st == cudaStreamCaptureStatusActive;
    return 0;
}

// Inside a caller's capture a call may issue nothing but kernel launches: a re-plan synchronises the device and uploads the camera
// tables with blocking copies, and a table write is a pageable copy from a temporary.  Refused before any of them, so the caller's
// capture stays valid.
int refuse_unsettled(MeaoCtx *c)
{
    const char *why = nullptr;
    if (c->plan_dirty || c->graphs_stale || c->cam_table_stale) why = "a structural change is pending (a re-plan synchronises the device)";
    else if (c->table_pending || c->plan_gen != c->consts_gen) why = "the camera tables of new frame constants or of a new size are not written yet";
    else if (c->views_pending) why = "a changed layer-viewport table is not written yet";
    if (!why) return 0;
    return fail(c, MEAO_ERR_INVALID, "cannot record into the stream's capture: %s; issue one frame outside the capture first", why);
}

// A capture that holds a graph-path frame of this context is still open: the forked streams that frame joined to it stay in it until
// the caller ends the capture.
bool in_open_capture(MeaoCtx *c)
{
    for (cudaStream_t b : c->branch) {
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(b, &st) != cudaSuccess) { cudaGetLastError(); continue; }
        if (st != cudaStreamCaptureStatusNone) return true;
    }
    return false;
}

// capturing: the call issues work on the caller's stream s; *capturing tells whether s is being captured, and a context that is not
// settled (refuse_unsettled) is refused then.
int ensure_ready(MeaoCtx *c, cudaStream_t s = nullptr, bool *capturing = nullptr)
{
    if (!c) return MEAO_ERR_INVALID;
    if (c->W <= 0) return fail(c, MEAO_ERR_INVALID, "meao_resize has not been called");
    if (c->plan_only) return fail(c, MEAO_ERR_CUDA, "plan-only context (device < 0): no CUDA device bound, and libmeao has no CPU fallback");
    CUDA_TRY(c, cudaSetDevice(c->device));
    if (capturing) {
        int rc = stream_capturing(c, s, capturing);
        if (!rc && *capturing) rc = refuse_unsettled(c);
        if (rc) return rc;
    }
    if (c->plan_dirty) replan(c);
    refresh_constants(c);
    if (c->graphs_stale) drop_graph(c);
    if (c->cam_table_stale) { int rc = upload_camera_tables(c); if (rc) return rc; }
    return 0;
}

// ensure_ready for an entry point that issues work on stream s which may read the camera tables: every frame form, band phase and
// stage call, so that each sees the tables of the constants set before it was issued.  *capturing (optional): s is being captured.
int frame_ready(MeaoCtx *c, cudaStream_t s, bool *capturing = nullptr)
{
    if (c && c->cams.cams && c->layers > c->cams_capacity)
        return fail(c, MEAO_ERR_INVALID, "the frame has %d layers and the bound device camera buffer holds %d cameras (meao_bind_device_cameras)",
                    c->layers, c->cams_capacity);
    bool cap = false;
    int rc = ensure_ready(c, s, capturing ? capturing : &cap);
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
    static const char *nvtx[6] = {"meao::prepare_depth", "meao::render_ao", "meao::render_ao_wide", "meao::blur_upsample", "meao::camera_tables",
                                  "meao::render_params"};
    if (l.stage == kStageUpsample && l.level == 1 && !io.batch) c->last_out = io.aio ? const_cast<void *>(io.aio->ao_array) : io.ao;
    NvtxRange nv(nvtx[l.stage]);
    const bool render = l.stage == kStageRender || l.stage == kStageRenderWide;
    if (l.stage == kStageCamera) CUDA_TRY(c, io.cams ? launch_cameras(*c, *io.cams, s) : cudaErrorInvalidValue);
    else if (l.stage == kStageParams) CUDA_TRY(c, io.params ? launch_render_params(*io.params, s) : cudaErrorInvalidValue);
    else if (io.params && render) CUDA_TRY(c, launch_render_params_entry(*c, l, io, forced_render_tile(), s));
    else if (io.batch) CUDA_TRY(c, launch_entry_batch(*c, l, io, forced_render_tile(), s));
    else if (!c->layer_ortho.empty()) CUDA_TRY(c, launch_entry_mixed(*c, l, io, forced_render_tile(), s));
    else CUDA_TRY(c, c->plan.orthographic ? launch_entry_ortho(*c, l, io, forced_render_tile(), s) : launch_entry_views(*c, l, io, forced_render_tile(), s));
    c->launches++;
    return 0;
}

// The FrameIO of a pointer frame: its depth and AO at the pitches of vp (nullptr: tight).  fused: the prepare writes LowDepth1..4
// only and the final upsample reads and linearises the same depth (what meao_render records).
FrameIO frame_io(MeaoCtx *c, const void *depth, int kind, void *ao_out, bool fused, const ViewPitch *vp = nullptr)
{
    FrameIO io;
    io.kind = kind; io.depth = depth_in(*c, depth, kind, vp); io.low_only = io.fused = fused; io.ao = ao_out; io.vp = vp;
    io.cams = c->cams.cams ? &c->cams : nullptr;
    io.params = c->dev_params.params ? &c->dev_params : nullptr;
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
// The camera stage alone (a bound device camera buffer), ahead of a stage call's prepare and of the AO regeneration
int record_cameras(MeaoCtx *c, cudaStream_t s)
{
    if (!c->cams.cams) return 0;
    return record_launch(c, FrameLaunch{kStageCamera, 0, 0, -1, kPdlNever}, frame_io(c, nullptr, c->last_kind, nullptr, false), s);
}
// The parameter stage alone (a bound device parameter buffer), ahead of a stage call's prepare
int record_params(MeaoCtx *c, cudaStream_t s)
{
    if (!c->dev_params.params) return 0;
    return record_launch(c, FrameLaunch{kStageParams, 0, 0, -1, kPdlNever}, frame_io(c, nullptr, c->last_kind, nullptr, false), s);
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
    const std::vector<FrameLaunch> sched = frame_schedule(c->plan.variants, c->cams.cams != nullptr, c->dev_params.params != nullptr);
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
    const std::vector<FrameLaunch> sched = frame_schedule(c->plan.variants, c->cams.cams != nullptr, c->dev_params.params != nullptr);
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
    int rc = record_cameras(c, s);
    if (!rc) rc = record_upsample(c, 1, nullptr, s);
    c->launches = before;
    return rc;
}

std::mutex g_event_mutex;
// arrays: meao_bind_event_arrays(_at), at the viewport origins `org` (depth x, y, AO x, y), checked again at the size of the frame
// each time the event runs; exact: meao_bind_event_arrays (W x H arrays).  Otherwise a pointer frame at the pitches `pitch`, or, with
// tight (meao_bind_event), at the tight pitches of the context when the event runs -- a meao_resize between binding and rendering keeps
// meaning what it meant before.
// batch (meao_bind_event_arrays_batch): copies of the lists, depth arrays then AO arrays (depth / out unused).
struct EventBinding { MeaoCtx *ctx; const void *depth; int kind; void *out; void *stream; bool arrays; bool tight; ViewPitch pitch;
                      int org[4] = {0, 0, 0, 0}; bool exact = false; std::vector<const void *> batch = {}; };
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
            for (const KernelUnit *u : kViewKernelUnits) u->walk(&pe);
            for (const KernelUnit *u : kOrthoKernelUnits) u->walk(&pe);
            for (const KernelUnit *u : kBatchKernelUnits) u->walk(&pe);
            for (const KernelUnit *u : kMixedKernelUnits) u->walk(&pe);
            for (const KernelUnit *u : kCameraKernelUnits) u->walk(&pe);
            for (const KernelUnit *u : kParamKernelUnits) u->walk(&pe);
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
    if (c->cams.status) cudaFree(c->cams.status);
    if (c->dev_params.derived) cudaFree(c->dev_params.derived);
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
    // a bound device parameter buffer decides thickness_modifier and intensity: a change of those two alone is only recorded, for after the
    // unbind, and the constant getters plan the host values again first
    const bool render_only = c->dev_params.params && c->params.noise_filter_tolerance == p->noise_filter_tolerance &&
                             c->params.blur_tolerance == p->blur_tolerance && c->params.upsample_tolerance == p->upsample_tolerance &&
                             c->params.debug == p->debug;
    c->params = *p;
    if (changed && render_only) {
        c->host_consts_stale = true;
        for (auto &slot : c->size_slots) slot.s.host_consts_stale = true;
    } else if (changed) { c->consts_gen++; c->frame_gen++; }   // frame constants: the next frame takes them without a re-plan
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
    if (changed) { c->plan_dirty = true; c->frame_gen++; }      // re-plan + drop the captured graphs (ensure_ready)
    return changed ? 1 : 0;
}

int meao_get_variants(const MeaoCtx *c, MeaoVariants *out)
{
    if (!c || !out) return MEAO_ERR_INVALID;
    *out = c->variants;
    return MEAO_OK;
}

int meao_set_hierarchy_depth(MeaoCtx *c, int32_t levels)
{
    if (!c) return MEAO_ERR_INVALID;
    if (levels < 1 || levels > 4) return fail(c, MEAO_ERR_INVALID, "hierarchy depth (levels) %d not in 1..4", levels);
    if (levels == c->hierarchy_depth) return 0;
    c->hierarchy_depth = levels;
    c->plan_dirty = true;           // another schedule: re-plan + drop the captured graphs (ensure_ready)
    c->frame_gen++;
    return 1;
}

int meao_get_hierarchy_depth(const MeaoCtx *c) { return c ? c->hierarchy_depth : MEAO_ERR_INVALID; }

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

int meao_set_projection(MeaoCtx *c, int32_t projection)
{
    if (!c) return MEAO_ERR_INVALID;
    if (projection != MEAO_PROJECTION_PERSPECTIVE && projection != MEAO_PROJECTION_ORTHOGRAPHIC)
        return fail(c, MEAO_ERR_INVALID, "projection %d is neither MEAO_PROJECTION_PERSPECTIVE (0) nor MEAO_PROJECTION_ORTHOGRAPHIC (1)", projection);
    if (projection == c->projection) return 0;
    if (projection == MEAO_PROJECTION_ORTHOGRAPHIC) {
        if (!c->views.empty())
            return fail(c, MEAO_ERR_UNSUPPORTED, "an orthographic projection is not supported with a layer-viewport table (meao_set_layer_viewports)");
        if ((c->W > 0 && (c->band0 != 0 || c->band1 != c->H)) || c->peer_base[0] || c->peer_base[1])
            return fail(c, MEAO_ERR_UNSUPPORTED, "an orthographic projection is not supported with a row band or a neighbour connection "
                        "(meao_set_row_band, meao_band_connect)");
    }
    c->projection = projection;
    c->plan_dirty = true;           // other kernels and other constants: re-plan + drop the captured graphs (ensure_ready)
    c->frame_gen++;
    return 1;
}

int meao_get_projection(const MeaoCtx *c) { return c ? c->projection : MEAO_ERR_INVALID; }

int meao_set_layer_projections(MeaoCtx *c, const int32_t *projections, int32_t count)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!projections && count == 0) {
        if (c->layer_proj.empty()) return 0;
        c->layer_proj.clear();
        c->layer_proj_ortho = 0;
        c->plan_dirty = true;       // the context's projection again: re-plan + drop the captured graphs (ensure_ready)
        c->frame_gen++;
        return 1;
    }
    if (!projections) return fail(c, MEAO_ERR_INVALID, "projections is NULL with count %d (NULL clears the table only with count 0)", count);
    if (count != c->layers) return fail(c, MEAO_ERR_INVALID, "count %d differs from the context's %d layers (meao_set_layers)", count, c->layers);
    int ortho = 0;
    for (int l = 0; l < count; l++) {
        if (projections[l] != MEAO_PROJECTION_PERSPECTIVE && projections[l] != MEAO_PROJECTION_ORTHOGRAPHIC)
            return fail(c, MEAO_ERR_INVALID, "layer %d: projection %d is neither MEAO_PROJECTION_PERSPECTIVE (0) nor MEAO_PROJECTION_ORTHOGRAPHIC (1)",
                        l, projections[l]);
        if (projections[l] == MEAO_PROJECTION_ORTHOGRAPHIC) ortho++;
    }
    if (ortho) {        // an orthographic layer carries the restrictions of an orthographic context (meao_set_projection)
        const int l = (int)(std::find(projections, projections + count, (int32_t)MEAO_PROJECTION_ORTHOGRAPHIC) - projections);
        if (!c->views.empty())
            return fail(c, MEAO_ERR_UNSUPPORTED, "layer %d: projection: an orthographic layer is not supported with a layer-viewport table "
                        "(meao_set_layer_viewports)", l);
        if ((c->W > 0 && (c->band0 != 0 || c->band1 != c->H)) || c->peer_base[0] || c->peer_base[1])
            return fail(c, MEAO_ERR_UNSUPPORTED, "layer %d: projection: an orthographic layer is not supported with a row band or a neighbour "
                        "connection (meao_set_row_band, meao_band_connect)", l);
    }
    if ((int)c->layer_proj.size() == count && std::equal(projections, projections + count, c->layer_proj.begin())) return 0;
    c->layer_proj.assign(projections, projections + count);
    c->layer_proj_ortho = ortho;
    c->plan_dirty = true;           // other kernels and other constants: re-plan + drop the captured graphs (ensure_ready)
    c->frame_gen++;
    return 1;
}

int meao_get_layer_projections(const MeaoCtx *c, int32_t *out, int32_t capacity)
{
    if (!c) return MEAO_ERR_INVALID;
    const int n = (int)c->layer_proj.size();
    if (n && (!out || capacity < n)) return MEAO_ERR_INVALID;
    if (n) std::copy(c->layer_proj.begin(), c->layer_proj.end(), out);
    return n;
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

static_assert(sizeof(LayerView) == sizeof(MeaoLayerViewport) && offsetof(LayerView, ao_slice) == offsetof(MeaoLayerViewport, ao_slice),
              "the arena's layer-viewport table is the public table, field for field");
namespace {
const char *const kViewField[6] = {"depth_x", "depth_y", "depth_slice", "ao_x", "ao_y", "ao_slice"};
inline int view_field(const MeaoLayerViewport &v, int i) { return (&v.depth_x)[i]; }
}  // namespace

int meao_set_layer_viewports(MeaoCtx *c, const MeaoLayerViewport *views, int32_t count)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!views && count == 0) {
        if (c->views.empty()) return 0;
        c->views.clear();
        c->views_pending = false;
        // back to the kernels without a table: a structural change, except under a layer reservation, whose table offset is one for
        // every (W, H, L) and whose graph keys carry the table a frame reads
        if (!c->res_layers) c->plan_dirty = true;
        c->frame_gen++;
        return 1;
    }
    if (!views) return fail(c, MEAO_ERR_INVALID, "views is NULL with count %d (NULL clears the table only with count 0)", count);
    if (c->projection != MEAO_PROJECTION_PERSPECTIVE)
        return fail(c, MEAO_ERR_UNSUPPORTED, "a layer-viewport table is not supported under an orthographic projection (meao_set_projection)");
    if (c->layer_proj_ortho > 0)
        return fail(c, MEAO_ERR_UNSUPPORTED, "a layer-viewport table is not supported with an orthographic layer (meao_set_layer_projections)");
    if (count != c->layers) return fail(c, MEAO_ERR_INVALID, "count %d differs from the context's %d layers (meao_set_layers)", count, c->layers);
    for (int l = 0; l < count; l++)
        for (int i = 0; i < 6; i++)
            if (view_field(views[l], i) < 0)
                return fail(c, MEAO_ERR_INVALID, "layer %d: %s = %d is negative", l, kViewField[i], view_field(views[l], i));
    if ((int)c->views.size() == count && memcmp(c->views.data(), views, (size_t)count * sizeof(MeaoLayerViewport)) == 0) return 0;
    if (c->views.empty() && !c->res_layers) c->plan_dirty = true;   // the table kernels replace the array kernels: a structural change
    else c->views_pending = !c->plan_only;          // a frame constant: written by the next frame on its stream
    c->views.assign(views, views + count);
    for (int i = 0; i < 6; i++) {
        int m = 0;
        for (int l = 1; l < count; l++) if (view_field(views[l], i) > view_field(views[m], i)) m = l;
        c->views_max[i] = m;
    }
    for (int r = 0; r < 2; r++) {
        const int f = 3 * r;        // depth_x or ao_x; then y, slice
        auto yx = [&](int l) { return std::make_pair(view_field(views[l], f + 1), view_field(views[l], f)); };
        auto syx = [&](int l) { return std::make_tuple(view_field(views[l], f + 2), view_field(views[l], f + 1), view_field(views[l], f)); };
        int a = 0, b = 0;
        for (int l = 1; l < count; l++) {
            if (yx(l) > yx(a)) a = l;
            if (syx(l) > syx(b)) b = l;
        }
        c->views_last[r][0] = a; c->views_last[r][1] = b;
    }
    c->views_checked.clear();
    c->frame_gen++;
    return 1;
}

int meao_get_layer_viewports(const MeaoCtx *c, MeaoLayerViewport *out, int32_t capacity)
{
    if (!c) return MEAO_ERR_INVALID;
    const int n = (int)c->views.size();
    if (n && (!out || capacity < n)) return MEAO_ERR_INVALID;
    if (n) memcpy(out, c->views.data(), (size_t)n * sizeof(MeaoLayerViewport));
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
        const int rc = switch_size(c, w, h, c->layers);     // no allocation, no synchronise, the other sizes' graphs stay
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
    if (c->plan_only) { c->frame_gen++; return 1; }     // recorded; nothing to allocate
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
    if (arena_w(c) > 0) out->arena_bytes = c->plan_only ? (int64_t)arena_layout(arena_w(c), arena_h(c), arena_layers(c)).bytes : (int64_t)c->arena_bytes;
    if (c->W > 0) out->arena_bytes_needed = (int64_t)arena_layout(c->W, c->H, c->layers).bytes;
    out->arena_allocations = c->arena_allocations;
    out->graphs_held = (int64_t)(c->graphs.size() + c->retired.size());
    out->graph_instantiations = c->graph_instantiations;
    return MEAO_OK;
}

// meao_set_layers inside a layer reservation: host bookkeeping.  The tables are cleared -- the layer cameras as a camera change
// (note_camera_change), the viewport table as meao_set_layer_viewports clears it -- and the new count is swapped in like a size
// (switch_size); the arena, the graphs and every other planned (W, H, L) stay.
static int switch_layers(MeaoCtx *c, int layers)
{
    c->frame_gen++;
    if (!c->layer_cams.empty()) {
        const int old_z = ctx_reversed_z(c);
        c->layer_cams.clear();
        note_camera_change(c, old_z, c->camera.reversed_z);
    }
    if (!c->layer_proj.empty()) {
        // the projection table too, as host bookkeeping: every planned (W, H, L) plans its constants and projections again when it is
        // next swapped in (refresh_constants), and the graph keys carry the projections a frame was recorded with (GraphKey::proj)
        c->layer_proj.clear();
        c->layer_proj_ortho = 0;
        c->consts_gen++;
    }
    c->views.clear();
    c->views_pending = false;
    c->views_checked.clear();
    if (c->W <= 0) { c->layers = layers; return 1; }    // placed by the first meao_resize
    const int rc = switch_size(c, c->W, c->H, layers);
    return rc ? rc : 1;
}

int meao_set_layers(MeaoCtx *c, int32_t layers)
{
    if (!c) return MEAO_ERR_INVALID;
    if (layers < 1 || layers > kMaxLayers)
        return fail(c, MEAO_ERR_INVALID, "layers %d not in 1..%d (the layer is a grid dimension of the layered kernels)", layers, kMaxLayers);
    if (c->res_layers > 0 && layers > c->res_layers)    // never a silent re-allocation for a host that reserved its layer count
        return fail(c, MEAO_ERR_INVALID, "layers %d lies above the layer reservation %d (meao_reserve_layers)", layers, c->res_layers);
    if (layers == c->layers) return 0;
    if (c->res_layers > 0) return switch_layers(c, layers);
    const int old = c->layers;
    c->frame_gen++;
    std::vector<MeaoCamera> old_cams;
    old_cams.swap(c->layer_cams);                   // a table has one camera per layer: a new layer count clears it
    std::vector<MeaoLayerViewport> old_views;       // and so does a viewport table
    old_views.swap(c->views);
    std::vector<int32_t> old_proj;                  // and a projection table
    old_proj.swap(c->layer_proj);
    const int old_proj_ortho = c->layer_proj_ortho;
    c->layer_proj_ortho = 0;
    const bool old_views_pending = c->views_pending;
    c->views_pending = false;
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
        c->views.swap(old_views);
        c->views_pending = old_views_pending;
        c->layer_proj.swap(old_proj);
        c->layer_proj_ortho = old_proj_ortho;
        if (allocate(c)) { c->W = c->H = 0; }        // the previous arena could not be restored either: the context needs meao_resize
        c->error = err;
        return rc;
    }
    return 1;
}

int meao_reserve_layers(MeaoCtx *c, int32_t max_layers)
{
    if (!c) return MEAO_ERR_INVALID;
    const bool clear = max_layers == 0;
    if (!clear && (max_layers < 1 || max_layers > kMaxLayers))
        return fail(c, MEAO_ERR_INVALID, "bad max_layers %d (in 1..%d, or 0 to clear)", max_layers, kMaxLayers);
    if (c->W > 0 && (c->band0 != 0 || c->band1 != c->H || c->prev0 >= 0 || c->next1 >= 0))
        return fail(c, MEAO_ERR_UNSUPPORTED, "meao_reserve_layers: this context has a row band (meao_set_row_band); row bands need an unreserved context");
    if (!clear && max_layers < c->layers)
        return fail(c, MEAO_ERR_INVALID, "max_layers %d is below the current layer count %d", max_layers, c->layers);
    if (max_layers == c->res_layers) return 0;
    const int old = c->res_layers;
    c->res_layers = max_layers;
    if (c->plan_only) { c->frame_gen++; return 1; }     // recorded; nothing to allocate
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    if (arena_w(c) <= 0) { c->frame_gen++; return 1; }  // no size yet: laid out by the first meao_resize
    const int rc = allocate(c, true);               // like meao_reserve: the old arena stays until the new one exists
    if (rc) { c->res_layers = old; return rc; }
    return 1;
}

int meao_layer_reservation(const MeaoCtx *c) { return c ? c->res_layers : MEAO_ERR_INVALID; }

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
    c->frame_gen++;
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
    cudaStream_t s = (cudaStream_t)stream;
    bool capturing;
    int rc = ensure_ready(c, s, &capturing); if (rc) return rc;
    if (side != 0 && side != 1) return fail(c, MEAO_ERR_INVALID, "side must be 0 or 1");
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
// capturing: s is being captured by the caller, whose graph then holds the launches themselves -- no graph of the context is captured,
// instantiated, launched or evicted.  PDL at the level an instantiation of this context has accepted (0 before the first): a level
// is never tried inside the caller's capture, where a refused attempt would invalidate it.
static int launch_cached(MeaoCtx *c, const MeaoCtx::GraphKey &key_in, cudaStream_t s, bool capturing,
                         const std::function<int(cudaStream_t, int)> &record)
{
    if (c->flags & MEAO_FLAG_NO_GRAPH) return record(s, 0);
    if (capturing) return record(s, c->pdl_level >= 0 ? c->pdl_level : 0);
    MeaoCtx::GraphKey key = key_in;
    key.size[0] = c->W; key.size[1] = c->H; key.size[2] = c->slot; key.size[3] = c->layers;
    key.proj = c->proj_key;
    key.cams = c->cams.cams;
    key.params = c->dev_params.params;
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
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if (!depth) return fail(c, MEAO_ERR_INVALID, "depth is NULL");
    c->last_kind = kind;
    const MeaoCtx::GraphKey key{{depth, send_up, send_down, nullptr}, 100 + kind};
    return launch_cached(c, key, (cudaStream_t)stream, capturing, [&](cudaStream_t s, int pdl) {
        int r = record_downsample(c, depth, kind, s);
        if (r) return r;
        PdlScope p(pdl >= 1);
        return halo_kernel(c, send_up, send_down, true, s);
    });
}

int meao_band_phase_b(MeaoCtx *c, const void *recv_up, const void *recv_down, void *ao_out, void *stream)
{
    BAND_GUARD(c, "meao_band_phase_b");
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if (!ao_out) return fail(c, MEAO_ERR_INVALID, "ao_out is NULL");
    const int kind = c->last_kind;
    const MeaoCtx::GraphKey key{{recv_up, recv_down, ao_out, nullptr}, 200 + kind};
    c->last_out = ao_out;
    return launch_cached(c, key, (cudaStream_t)stream, capturing, [&](cudaStream_t s, int pdl) {
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
    c->frame_gen++;
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
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
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
    return launch_cached(c, key, (cudaStream_t)stream, capturing, [&](cudaStream_t s, int pdl) {
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
int check_ao_disjoint(MeaoCtx *c);

// The layer-viewport table against the caller's pitched views (check_views, table set): the checks check_view_fit makes for arrays.
// Every row of every rectangle fits its row pitch; when some slice is > 0, every rectangle fits inside its slice (so slices never
// share a byte) and the depth layer pitch is a whole number of elements; no two AO rectangles share a byte (check_ao_disjoint: with
// rows inside the row pitch and rectangles inside their slices, two share a byte exactly when they share a texel).  Constant time
// (views_max, views_last), except check_ao_disjoint's once per (table, size).  Both the slice test and the extents are exact: once every
// row fits its row pitch, a rectangle further down (or in a later slice) ends further in than any rectangle above it, whatever the x.
int check_view_pitches(MeaoCtx *c, const void *depth, int64_t es, const void *ao_out, const ViewPitch &p)
{
    if (c->band0 != 0 || c->band1 != c->H) return fail(c, MEAO_ERR_UNSUPPORTED, "a layer-viewport table needs a whole-frame context (no row band)");
    const int64_t W = c->W, H = c->H;
    const struct { const char *role; int f0; int64_t es, row, layer; } views[2] = {{"depth", 0, es, p.depth_row, p.depth_layer},
                                                                                    {"ao", 3, 1, p.ao_row, p.ao_layer}};
    int64_t extent[2];
    for (int i = 0; i < 2; i++) {
        const auto &v = views[i];
        const int lx = c->views_max[v.f0], ls = c->views_max[v.f0 + 2];
        const int64_t x = view_field(c->views[lx], v.f0), sl = view_field(c->views[ls], v.f0 + 2);
        if ((x + W) * v.es > v.row)
            return fail(c, MEAO_ERR_INVALID, "layer %d: %s_x = %lld: a row of the %lldx%lld rectangle overflows %s_row_pitch %lld", lx, v.role,
                        (long long)x, (long long)W, (long long)H, v.role, (long long)v.row);
        // where a rectangle's last byte lies in its slice.  Slices at most 2^31 at a pitch of at most 2^63, rows at most 2^31 at a pitch
        // of at most 2^31: every product below stays inside __int128
        auto in_slice = [&](int l) {
            const MeaoLayerViewport &e = c->views[l];
            return (__int128)(view_field(e, v.f0 + 1) + H - 1) * v.row + (view_field(e, v.f0) + W) * v.es;
        };
        if (sl > 0) {
            const int ly = c->views_last[i][0];
            if (in_slice(ly) > v.layer)
                return fail(c, MEAO_ERR_INVALID, "layer %d: %s_x, %s_y = %d, %d: the %lldx%lld rectangle overflows %s_layer_pitch %lld (its slice)",
                            ly, v.role, v.role, view_field(c->views[ly], v.f0), view_field(c->views[ly], v.f0 + 1), (long long)W, (long long)H,
                            v.role, (long long)v.layer);
            if (v.layer % v.es)
                return fail(c, MEAO_ERR_INVALID, "layer %d: %s_slice = %lld: %s_layer_pitch %lld is not a multiple of the %lld-byte element", ls,
                            v.role, (long long)sl, v.role, (long long)v.layer, (long long)v.es);
        }
        const int le = c->views_last[i][1];
        const __int128 end = (__int128)view_field(c->views[le], v.f0 + 2) * v.layer + in_slice(le);
        if (end > INT64_MAX) return fail(c, MEAO_ERR_INVALID, "layer %d: %s_slice = %d: the view ends beyond 2^63 bytes", le, v.role,
                                         view_field(c->views[le], v.f0 + 2));
        extent[i] = (int64_t)end;
    }
    int rc = check_ao_disjoint(c);
    if (rc) return rc;
    // the existing extent test, from each view's base to the end of its last rectangle
    const __int128 d0 = (__int128)(uintptr_t)depth, a0 = (__int128)(uintptr_t)ao_out;
    if (d0 < a0 + extent[1] && a0 < d0 + extent[0])
        return fail(c, MEAO_ERR_INVALID, "the byte extents of the depth view and the AO view (ao_out_dev) intersect");
    return 0;
}

// Every check of meao_render_pitched / meao_bind_event_pitched, on the host before anything is launched.  On success the layer pitches
// of a single-layer context (unused) are replaced by the tight values, so that equivalent views share one cached graph.
int check_views(MeaoCtx *c, const void *depth, int kind, const void *ao_out, ViewPitch *p, bool table = true)
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
    if (table && !c->views.empty()) return check_view_pitches(c, depth, es, ao_out, *p);
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
// table: honour the layer-viewport table when one is set; false for the host-buffer calls, whose staging buffers hold the tight layout.
int render_views(MeaoCtx *c, const void *depth, int kind, void *ao_out, ViewPitch p, void *stream, bool capturing, bool table = true)
{
    int rc;
    if ((rc = check_views(c, depth, kind, ao_out, &p, table))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    // a layer-viewport table: the rectangles of the arena's table; checked against these views by check_views
    const LayerView *views = (!table || c->views.empty()) ? nullptr : c->layer_views;
    auto io = [&]() { FrameIO fio = frame_io(c, depth, kind, ao_out, true, &p); fio.views = views; return fio; };
    if (c->flags & MEAO_FLAG_NO_GRAPH) return record_frame(c, io(), s, 0, false);

    // plan-once / replay: one captured graph per (depth, out, kind, pitches), like the reference's command buffer
    // that is re-recorded only when something changed (AO.cs:334-347).  p[2]: the table a frame reads (nullptr: none), so a frame that
    // ignores a set table never replays one recorded through it, nor the reverse
    NvtxRange nv("meao::frame");
    const MeaoCtx::GraphKey key{{depth, ao_out, views, nullptr}, kind, {p.depth_row, p.depth_layer, p.ao_row, p.ao_layer}};
    c->last_kind = kind; c->last_out = ao_out;
    return launch_cached(c, key, s, capturing, [&](cudaStream_t cs, int pdl) {
        return record_frame_dag(c, io(), cs, 0, pdl);
    });
}
}  // namespace

int meao_render(MeaoCtx *c, const void *depth, int32_t kind, void *ao_out, void *stream)
{
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    return render_views(c, depth, kind, ao_out, tight_pitch(*c, kind), stream, capturing);      // meao_render_pitched at the tight pitches
}

int meao_render_pitched(MeaoCtx *c, const void *depth, int64_t depth_row_pitch, int64_t depth_layer_pitch, int32_t kind,
                        void *ao_out, int64_t ao_row_pitch, int64_t ao_layer_pitch, void *stream)
{
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    return render_views(c, depth, kind, ao_out, ViewPitch{depth_row_pitch, depth_layer_pitch, ao_row_pitch, ao_layer_pitch}, stream, capturing);
}

// ---- CUDA arrays (include/meao.h "CUDA arrays") ------------------------------------------------------------------------
namespace {
constexpr int kArrayGraphKind = 400;        // GraphKey.kind of an array frame: 400 + depth kind
// GraphKey.kind of a batch over CUDA arrays / over device buffers (meao_render_arrays_batch / meao_render_batch): + depth kind
constexpr int kBatchArrayGraphKind = 500, kBatchGraphKind = 600;

// The graph of `k` launches with `array`: an array frame's p[0] / p[1], or an entry of an array batch's list
bool graph_names_array(const MeaoCtx::GraphKey &k, const void *array)
{
    if (k.kind >= kBatchArrayGraphKind && k.kind < kBatchGraphKind) return std::count(k.list.begin(), k.list.end(), (uintptr_t)array) != 0;
    return k.kind >= kArrayGraphKind && k.kind < kBatchArrayGraphKind && (k.p[0] == array || k.p[1] == array);
}

// What a cudaArray_t is, checked against the context on the host before anything is launched.  role: "depth" or "ao", the prefix of
// the fields named in a refusal (<role>_array, <role>_x, <role>_y).  elem_bits / is_float: the one channel the role needs.  exact: the
// extent must be the context's W x H (meao_render_arrays); otherwise the W x H viewport at (x, y) must lie inside it.  Returns 0 and
// the layer addressing, or fails with a message naming the field.  ext / layers_out (a layer-viewport table is set): no extent, origin
// or layer-count test here; the array's extent and layer count are returned for check_view_fit instead.
int check_array(MeaoCtx *c, const void *arr, const char *role, int elem_bits, bool is_float, int x, int y, bool exact, int *surf_kind,
                cudaExtent *ext = nullptr, int *layers_out = nullptr)
{
    cudaChannelFormatDesc d{};
    cudaExtent e{};
    unsigned int flags = 0;
    const cudaError_t err = cudaArrayGetInfo(&d, &e, &flags, (cudaArray_t)arr);
    if (err != cudaSuccess) { cudaGetLastError(); return fail(c, MEAO_ERR_INVALID, "%s_array: not a CUDA array (cudaArrayGetInfo: %s)", role, cudaGetErrorString(err)); }
    const bool one_channel = d.x == elem_bits && d.y == 0 && d.z == 0 && d.w == 0;
    bool kind_ok;
    if (is_float) kind_ok = d.f == cudaChannelFormatKindFloat;
    else kind_ok = d.f == cudaChannelFormatKindUnsigned ||
                   (elem_bits == 8 && d.f == cudaChannelFormatKindUnsignedNormalized8X1) ||
                   (elem_bits == 16 && d.f == cudaChannelFormatKindUnsignedNormalized16X1);
    if (!one_channel || !kind_ok)
        return fail(c, MEAO_ERR_INVALID, "%s_array: channel format (%d,%d,%d,%d bits, kind %d) is not one %d-bit %s channel", role, d.x, d.y, d.z, d.w, (int)d.f,
                    elem_bits, is_float ? "float" : "unsigned (normalised or not)");
    if (ext) {
        *ext = e;
    } else if (exact) {
        if ((int)e.width != c->W || (int)e.height != c->H || e.width != (size_t)c->W || e.height != (size_t)c->H)
            return fail(c, MEAO_ERR_INVALID, "%s_array: extent %zux%zu differs from the context's %dx%d", role, e.width, e.height, c->W, c->H);
    } else {
        if (x < 0) return fail(c, MEAO_ERR_INVALID, "%s_x = %d: the viewport origin is negative", role, x);
        if (y < 0) return fail(c, MEAO_ERR_INVALID, "%s_y = %d: the viewport origin is negative", role, y);
        if ((size_t)x + (size_t)c->W > e.width)
            return fail(c, MEAO_ERR_INVALID, "%s_x = %d: the %dx%d viewport overflows %s_array's width %zu", role, x, c->W, c->H, role, e.width);
        if ((size_t)y + (size_t)c->H > e.height)
            return fail(c, MEAO_ERR_INVALID, "%s_y = %d: the %dx%d viewport overflows %s_array's height %zu", role, y, c->W, c->H, role, e.height);
    }
    if (!(flags & cudaArraySurfaceLoadStore))
        return fail(c, MEAO_ERR_INVALID, "%s_array: flags 0x%x lack cudaArraySurfaceLoadStore (register the resource with cudaGraphicsRegisterFlagsSurfaceLoadStore)", role, flags);
    int layers;
    if (flags & cudaArrayCubemap) {
        if (flags & cudaArrayLayered) return fail(c, MEAO_ERR_UNSUPPORTED, "%s_array: cube-map arrays (cudaArrayCubemap | cudaArrayLayered) are not supported", role);
        layers = 6; *surf_kind = kSurfCube;
    } else if (flags & cudaArrayLayered) {
        layers = e.depth > 0 ? (int)e.depth : 1; *surf_kind = kSurfLayered;
    } else {
        if (e.depth > 1) return fail(c, MEAO_ERR_INVALID, "%s_array: depth %zu: a 3-D array is not a 2-D or layered image", role, e.depth);
        layers = 1; *surf_kind = kSurf2D;
    }
    if (layers_out) { *layers_out = layers; return 0; }
    if (layers != c->layers)
        return fail(c, MEAO_ERR_INVALID, "%s_array: layer count %d differs from the context's %d (meao_set_layers)", role, layers, c->layers);
    return 0;
}

// The layer-viewport table against one array at the current W x H: every rectangle inside the array's extent and every slice below
// its layer count.  f0: the table's first field of the role (0: depth_x, 3: ao_x).  Constant time: views_max holds, per field, the layer
// with the largest value.
int check_view_fit(MeaoCtx *c, const char *role, const cudaExtent &e, int layers, int f0)
{
    const int lx = c->views_max[f0], ly = c->views_max[f0 + 1], ls = c->views_max[f0 + 2];
    const int x = view_field(c->views[lx], f0), y = view_field(c->views[ly], f0 + 1), sl = view_field(c->views[ls], f0 + 2);
    if ((size_t)x + (size_t)c->W > e.width)
        return fail(c, MEAO_ERR_INVALID, "layer %d: %s_x = %d: the %dx%d rectangle overflows %s_array's width %zu", lx, role, x, c->W, c->H, role, e.width);
    if ((size_t)y + (size_t)c->H > e.height)
        return fail(c, MEAO_ERR_INVALID, "layer %d: %s_y = %d: the %dx%d rectangle overflows %s_array's height %zu", ly, role, y, c->W, c->H, role, e.height);
    if (sl >= layers)
        return fail(c, MEAO_ERR_INVALID, "layer %d: %s_slice = %d: %s_array has %d layer(s)", ls, role, sl, role, layers);
    return 0;
}

// No two layers' AO rectangles on one slice share a texel, at the current W x H; once per (table, size), and not at all at a size no
// larger in either dimension than one that passed.  Every rectangle is W x H, so
// two overlap exactly when their origins are less than W apart in x and less than H apart in y.  The origins are binned into W x H
// cells: an overlapping pair lies in the same or in neighbouring cells, and disjoint rectangles leave at most one origin per cell, so
// the test takes L map lookups and insertions rather than L^2 comparisons.
int check_ao_disjoint(MeaoCtx *c)
{
    const int W = c->W, H = c->H;
    for (const auto &wh : c->views_checked)
        if (W <= wh.first && H <= wh.second) return 0;
    std::map<std::array<int, 3>, int> cells;
    for (int l = 0; l < (int)c->views.size(); l++) {
        const MeaoLayerViewport &v = c->views[l];
        const int cx = v.ao_x / W, cy = v.ao_y / H;
        for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
                auto it = cells.find({v.ao_slice, cx + dx, cy + dy});
                if (it == cells.end()) continue;
                const MeaoLayerViewport &o = c->views[it->second];
                if (std::abs(v.ao_x - o.ao_x) < W && std::abs(v.ao_y - o.ao_y) < H)
                    return fail(c, MEAO_ERR_INVALID, "layer %d: ao_x, ao_y = %d, %d: its %dx%d AO rectangle shares texels with layer %d's at %d, %d "
                                                     "(ao_slice %d)", l, v.ao_x, v.ao_y, W, H, it->second, o.ao_x, o.ao_y, v.ao_slice);
            }
        cells.emplace(std::array<int, 3>{v.ao_slice, cx, cy}, l);
    }
    // keep only the sizes no other passed size holds
    auto held = [&](const std::pair<int, int> &wh) { return wh.first <= W && wh.second <= H; };
    c->views_checked.erase(std::remove_if(c->views_checked.begin(), c->views_checked.end(), held), c->views_checked.end());
    c->views_checked.emplace_back(W, H);
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

// every check of meao_render_arrays(_at) / meao_bind_event_arrays(_at); on success `io` holds the surfaces of a frame (made on first use)
// and its viewport origins.  exact: both arrays must be W x H, the origins are (0, 0) (the entry points without _at).
int prepare_arrays(MeaoCtx *c, const void *depth_array, int dx, int dy, int kind, const void *ao_array, int ax, int ay, bool exact, ArrayIO *io)
{
    if (!depth_array || !ao_array) return fail(c, MEAO_ERR_INVALID, "depth_array / ao_array is NULL");
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    if (kind == MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_UNSUPPORTED, "depth_kind RAW_D24S8: CUDA arrays have no depth-stencil format");
    if (c->band0 != 0 || c->band1 != c->H) return fail(c, MEAO_ERR_UNSUPPORTED, "CUDA-array frames need a whole-frame context (no row band)");
    int rc;
    const bool d16 = kind == MEAO_DEPTH_RAW_D16_UNORM;
    if (!c->views.empty()) {        // the table says where every layer goes (meao_set_layer_viewports)
        if (!exact)
            return fail(c, MEAO_ERR_INVALID, "a layer-viewport table is set (meao_set_layer_viewports): it places every layer, so the origins of "
                                             "meao_render_arrays_at / meao_bind_event_arrays_at are refused; use meao_render_arrays");
        cudaExtent de{}, ae{};
        int dn = 0, an = 0;
        if ((rc = check_array(c, depth_array, "depth", d16 ? 16 : 32, !d16, 0, 0, false, &io->depth_surf, &de, &dn))) return rc;
        if ((rc = check_array(c, ao_array, "ao", 8, false, 0, 0, false, &io->ao_surf, &ae, &an))) return rc;
        if ((rc = check_view_fit(c, "depth", de, dn, 0)) || (rc = check_view_fit(c, "ao", ae, an, 3)) || (rc = check_ao_disjoint(c))) return rc;
    } else {
        if ((rc = check_array(c, depth_array, "depth", d16 ? 16 : 32, !d16, dx, dy, exact, &io->depth_surf))) return rc;
        if ((rc = check_array(c, ao_array, "ao", 8, false, ax, ay, exact, &io->ao_surf))) return rc;
    }
    if ((rc = surface_of(c, depth_array, &io->depth))) return rc;
    if ((rc = surface_of(c, ao_array, &io->ao))) return rc;
    io->ao_array = ao_array;
    io->depth_x = dx; io->depth_y = dy; io->ao_x = ax; io->ao_y = ay;
    return 0;
}

// GraphKey.p[2] / p[3] of an array frame: a viewport origin, so that a frame at other origins never replays a graph recorded for these
// ((0, 0) is nullptr: meao_render_arrays's key)
const void *origin_key(int x, int y) { return (const void *)(uintptr_t)(((uint64_t)(uint32_t)x << 32) | (uint32_t)y); }

// meao_render_arrays (exact) and meao_render_arrays_at: one path
int render_arrays(MeaoCtx *c, const void *depth_array, int dx, int dy, int kind, void *ao_array, int ax, int ay, bool exact, void *stream)
{
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    // a surface object is made on an array's first frame, which therefore cannot be recorded into a caller's capture
    if (capturing && (!c->surfaces.count(depth_array) || !c->surfaces.count(ao_array)))
        return fail(c, MEAO_ERR_INVALID, "cannot record into the stream's capture: an array this context has not rendered with needs a surface "
                                         "object first; issue one frame with these arrays outside the capture first");
    ArrayIO io;
    if ((rc = prepare_arrays(c, depth_array, dx, dy, kind, ao_array, ax, ay, exact, &io))) return rc;
    // the frame graph of meao_render with its first and last node reading / writing the arrays
    NvtxRange nv("meao::frame_arrays");
    MeaoCtx::GraphKey key{{depth_array, ao_array, origin_key(dx, dy), origin_key(ax, ay)}, kArrayGraphKind + kind};
    key.table = c->views.empty() ? nullptr : c->layer_views;
    c->last_kind = kind; c->last_out = ao_array;
    return launch_cached(c, key, (cudaStream_t)stream, capturing, [&](cudaStream_t cs, int pdl) {
        FrameIO fio = frame_io(c, nullptr, kind, nullptr, false);
        fio.aio = &io;
        if (!c->views.empty()) fio.views = c->layer_views;
        return record_frame_dag(c, fio, cs, 0, pdl);
    });
}
}  // namespace

int meao_render_arrays(MeaoCtx *c, const void *depth_array, int32_t kind, void *ao_array, void *stream)
{
    return render_arrays(c, depth_array, 0, 0, kind, ao_array, 0, 0, true, stream);
}

int meao_render_arrays_at(MeaoCtx *c, const void *depth_array, int32_t depth_x, int32_t depth_y, int32_t kind, void *ao_array, int32_t ao_x,
                          int32_t ao_y, void *stream)
{
    return render_arrays(c, depth_array, depth_x, depth_y, kind, ao_array, ao_x, ao_y, false, stream);
}

int meao_release_array(MeaoCtx *c, const void *array)
{
    if (!c) return MEAO_ERR_INVALID;
    if (c->plan_only) return fail(c, MEAO_ERR_CUDA, "plan-only context (device < 0): no CUDA device bound, and libmeao has no CPU fallback");
    if (!array) return fail(c, MEAO_ERR_INVALID, "array is NULL");
    {   // a plugin event bound to the array would re-create its surface after the array is freed
        std::lock_guard<std::mutex> g(g_event_mutex);
        for (auto it = g_events.begin(); it != g_events.end();) {
            const EventBinding &b = it->second;
            const bool names = b.arrays && (b.depth == array || b.out == array || std::count(b.batch.begin(), b.batch.end(), array));
            if (b.ctx == c && names) it = g_events.erase(it); else ++it;
        }
    }
    bool used = c->surfaces.count(array) != 0;
    for (auto &kv : c->graphs) used |= graph_names_array(kv.first, array);
    if (!used) return MEAO_OK;
    c->frame_gen++;
    CUDA_TRY(c, cudaSetDevice(c->device));
    CUDA_TRY(c, cudaDeviceSynchronize());       // frames that use the array may be in flight on any stream
    for (auto it = c->graphs.begin(); it != c->graphs.end();) {
        if (graph_names_array(it->first, array)) {
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

// ---- batches (include/meao.h "Batches") ------------------------------------------------------------------------------------
namespace {
static_assert(MEAO_MAX_BATCH == kMaxBatch, "include/meao.h states the batch bound");

// a refusal about one entry: the message names its layer first
int layer_fail(MeaoCtx *c, int rc, int l)
{
    c->error = "layer " + std::to_string(l) + ": " + c->error;
    return rc;
}

// The checks of a batch before its entries: the count, the depth kind and the forms a batch does not combine with.
int check_batch(MeaoCtx *c, int count, int kind, bool arrays)
{
    if (count < 1 || count > MEAO_MAX_BATCH)
        return fail(c, MEAO_ERR_INVALID, "count %d: a batch holds 1 .. MEAO_MAX_BATCH (%d) layers", count, MEAO_MAX_BATCH);
    if (count != c->layers)
        return fail(c, MEAO_ERR_INVALID, "count %d differs from the context's layer count %d (meao_set_layers)", count, c->layers);
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    if (arrays && kind == MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_UNSUPPORTED, "depth_kind RAW_D24S8: CUDA arrays have no depth-stencil format");
    if (!c->views.empty())
        return fail(c, MEAO_ERR_INVALID, "a layer-viewport table is set (meao_set_layer_viewports): a batch places every layer in resources of "
                                         "its own; clear the table first");
    if (c->projection != MEAO_PROJECTION_PERSPECTIVE)
        return fail(c, MEAO_ERR_UNSUPPORTED, "batches are perspective-only: this context has an orthographic projection (meao_set_projection)");
    if (c->layer_proj_ortho > 0)
        return fail(c, MEAO_ERR_UNSUPPORTED, "batches are perspective-only: this context has an orthographic layer (meao_set_layer_projections)");
    if (c->band0 != 0 || c->band1 != c->H) return fail(c, MEAO_ERR_UNSUPPORTED, "batches need a whole-frame context (no row band)");
    return 0;
}

// One array of an array batch: check_array's format and flag tests, a 2-D array or a layered array of depth 1, at least W x H.
int check_batch_array(MeaoCtx *c, int l, const void *arr, const char *role, bool d16, int *surf_kind)
{
    if (!arr) return fail(c, MEAO_ERR_INVALID, "layer %d: %s_arrays[%d] is NULL", l, role, l);
    const bool depth = role[0] == 'd';
    cudaExtent e{};
    int n = 0;
    const int rc = check_array(c, arr, role, depth ? (d16 ? 16 : 32) : 8, depth && !d16, 0, 0, false, surf_kind, &e, &n);
    if (rc) return layer_fail(c, rc, l);
    if (*surf_kind == kSurfCube || n != 1)
        return fail(c, MEAO_ERR_INVALID, "layer %d: %s_arrays[%d] has %d layers: a batch entry is a 2-D array or a layered array of depth 1",
                    l, role, l, n);
    if (e.width < (size_t)c->W || e.height < (size_t)c->H)
        return fail(c, MEAO_ERR_INVALID, "layer %d: %s_arrays[%d]: extent %zux%zu is smaller than the context's %dx%d", l, role, l, e.width,
                    e.height, c->W, c->H);
    return 0;
}

// Every check of an array batch after check_batch; on success `io` holds each layer's surfaces (made on first use).  capturing: the
// frame records into a caller's capture, where no surface object can be made.
int prepare_batch_arrays(MeaoCtx *c, const void *const *depth_arrays, int kind, const void *const *ao_arrays, int count, bool capturing,
                         BatchIO *io)
{
    if (!depth_arrays || !ao_arrays) return fail(c, MEAO_ERR_INVALID, "depth_arrays / ao_arrays is NULL");
    const bool d16 = kind == MEAO_DEPTH_RAW_D16_UNORM;
    int rc;
    for (int l = 0; l < count; l++) {
        if ((rc = check_batch_array(c, l, depth_arrays[l], "depth", d16, &io->depth.e[l].kind))) return rc;
        if ((rc = check_batch_array(c, l, ao_arrays[l], "ao", d16, &io->ao.e[l].kind))) return rc;
    }
    // no two layers write one AO array: sorted handles, so O(L log L)
    std::vector<std::pair<const void *, int>> ao(count);
    for (int l = 0; l < count; l++) ao[l] = {ao_arrays[l], l};
    std::sort(ao.begin(), ao.end());
    for (int i = 1; i < count; i++)
        if (ao[i].first == ao[i - 1].first)
            return fail(c, MEAO_ERR_INVALID, "layer %d: ao_arrays[%d] is layer %d's AO array too", ao[i].second, ao[i].second, ao[i - 1].second);
    if (capturing)      // a surface object is made on an array's first frame, which therefore cannot be recorded into a capture
        for (int l = 0; l < count; l++)
            if (!c->surfaces.count(depth_arrays[l]) || !c->surfaces.count(ao_arrays[l]))
                return fail(c, MEAO_ERR_INVALID, "layer %d: cannot record into the stream's capture: an array this context has not rendered with "
                                                 "needs a surface object first; issue one frame with these arrays outside the capture first", l);
    for (int l = 0; l < count; l++) {
        if ((rc = surface_of(c, depth_arrays[l], &io->depth.e[l].surf))) return rc;
        if ((rc = surface_of(c, ao_arrays[l], &io->ao.e[l].surf))) return rc;
    }
    io->arrays = true;
    return 0;
}

// Every check of a pointer batch after check_batch: per layer those of meao_render_pitched (pitch bounds and multiples, the depth's
// alignment to its element); no two AO extents intersect, and no AO extent intersects any depth extent (depth entries may repeat).  An
// extent runs from a layer's first byte to its last, (H - 1) x row pitch + W x element size.  The AO extents are sorted and then
// disjoint, so their ends are sorted too: a depth extent meets one exactly when the last AO extent that starts before its end ends after
// its start.  O(L log L).  On success `io` holds each layer's bases and pitches (rows in elements for the depth).
int prepare_batch_pointers(MeaoCtx *c, const void *const *depth, const int64_t *depth_row_pitch, int kind, void *const *ao,
                           const int64_t *ao_row_pitch, int count, BatchIO *io)
{
    if (!depth || !depth_row_pitch || !ao || !ao_row_pitch) return fail(c, MEAO_ERR_INVALID, "depth / depth_row_pitch / ao / ao_row_pitch is NULL");
    const int64_t es = depth_esize(kind), W = c->W, H = c->H;
    struct Extent { __int128 lo, hi; int l; bool operator<(const Extent &o) const { return lo < o.lo; } };
    std::vector<Extent> dx(count), ax(count);
    for (int l = 0; l < count; l++) {
        if (!depth[l]) return fail(c, MEAO_ERR_INVALID, "layer %d: depth[%d] is NULL", l, l);
        if (!ao[l]) return fail(c, MEAO_ERR_INVALID, "layer %d: ao[%d] is NULL", l, l);
        const int64_t dr = depth_row_pitch[l] ? depth_row_pitch[l] : W * es, ar = ao_row_pitch[l] ? ao_row_pitch[l] : W;
        if (dr < 0 || dr > INT32_MAX || dr < W * es || dr % es)
            return fail(c, MEAO_ERR_INVALID, "layer %d: depth_row_pitch[%d] = %lld: must be at least width x %lld = %lld bytes, at most INT32_MAX "
                        "and a multiple of %lld", l, l, (long long)depth_row_pitch[l], (long long)es, (long long)(W * es), (long long)es);
        if (ar < 0 || ar > INT32_MAX || ar < W)
            return fail(c, MEAO_ERR_INVALID, "layer %d: ao_row_pitch[%d] = %lld: must be at least the width %lld and at most INT32_MAX", l, l,
                        (long long)ao_row_pitch[l], (long long)W);
        if ((uintptr_t)depth[l] % es)
            return fail(c, MEAO_ERR_INVALID, "layer %d: depth[%d] %p is not aligned to its %lld-byte element", l, l, depth[l], (long long)es);
        io->ptr.e[l] = BatchPtr{depth[l], (uint8_t *)ao[l], (int)(dr / es), (int)ar};
        const __int128 d0 = (__int128)(uintptr_t)depth[l], a0 = (__int128)(uintptr_t)ao[l];
        dx[l] = Extent{d0, d0 + (__int128)(H - 1) * dr + W * es, l};
        ax[l] = Extent{a0, a0 + (__int128)(H - 1) * ar + W, l};
    }
    std::sort(ax.begin(), ax.end());
    for (int i = 1; i < count; i++)
        if (ax[i].lo < ax[i - 1].hi)
            return fail(c, MEAO_ERR_INVALID, "layer %d: the byte extent of ao[%d] intersects layer %d's AO extent", ax[i].l, ax[i].l, ax[i - 1].l);
    for (const Extent &d : dx) {
        auto it = std::lower_bound(ax.begin(), ax.end(), Extent{d.hi, 0, 0});     // the first AO extent that starts at or after d's end
        if (it != ax.begin() && std::prev(it)->hi > d.lo)
            return fail(c, MEAO_ERR_INVALID, "layer %d: the byte extent of ao[%d] intersects layer %d's depth extent (depth[%d])", std::prev(it)->l,
                        std::prev(it)->l, d.l, d.l);
    }
    io->arrays = false;
    return 0;
}

// FNV-1a over a batch's list (GraphKey.list_hash)
uint64_t list_hash(const std::vector<uintptr_t> &v)
{
    uint64_t h = 1469598103934665603ull;
    for (uintptr_t w : v)
        for (int b = 0; b < 8; b++) { h ^= (w >> (8 * b)) & 0xffu; h *= 1099511628211ull; }
    return h;
}

// A checked batch on a context that frame_ready has prepared: the frame graph of meao_render_arrays / meao_render with its first and last
// node reading and writing each layer's own resources.  The list is a kernel parameter of those two nodes, so it is baked into the graph
// (GraphKey.list) and into a caller's capture.
int render_batch(MeaoCtx *c, const BatchIO &io, int kind, std::vector<uintptr_t> list, void *last_out, cudaStream_t s, bool capturing)
{
    NvtxRange nv("meao::frame_batch");
    MeaoCtx::GraphKey key{{nullptr, nullptr, nullptr, nullptr}, (io.arrays ? kBatchArrayGraphKind : kBatchGraphKind) + kind};
    key.list_hash = list_hash(list);
    key.list = std::move(list);
    c->last_kind = kind; c->last_out = last_out;
    return launch_cached(c, key, s, capturing, [&](cudaStream_t cs, int pdl) {
        FrameIO fio = frame_io(c, nullptr, kind, nullptr, !io.arrays);      // pointers: the fused frame (low-only prepare)
        fio.batch = &io;
        return record_frame_dag(c, fio, cs, 0, pdl);
    });
}
}  // namespace

int meao_render_arrays_batch(MeaoCtx *c, const void *const *depth_arrays, int32_t kind, void *const *ao_arrays, int32_t count, void *stream)
{
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if ((rc = check_batch(c, count, kind, true))) return rc;
    std::unique_ptr<BatchIO> io(new BatchIO);
    if ((rc = prepare_batch_arrays(c, depth_arrays, kind, ao_arrays, count, capturing, io.get()))) return rc;
    std::vector<uintptr_t> list(2 * (size_t)count);
    for (int l = 0; l < count; l++) { list[l] = (uintptr_t)depth_arrays[l]; list[count + l] = (uintptr_t)ao_arrays[l]; }
    return render_batch(c, *io, kind, std::move(list), ao_arrays[0], (cudaStream_t)stream, capturing);
}

int meao_render_batch(MeaoCtx *c, const void *const *depth, const int64_t *depth_row_pitch, int32_t kind, void *const *ao,
                      const int64_t *ao_row_pitch, int32_t count, void *stream)
{
    bool capturing;
    int rc = frame_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if ((rc = check_batch(c, count, kind, false))) return rc;
    std::unique_ptr<BatchIO> io(new BatchIO);
    if ((rc = prepare_batch_pointers(c, depth, depth_row_pitch, kind, ao, ao_row_pitch, count, io.get()))) return rc;
    std::vector<uintptr_t> list(4 * (size_t)count);
    for (int l = 0; l < count; l++) {
        const BatchPtr &e = io->ptr.e[l];
        list[4 * l] = (uintptr_t)e.depth; list[4 * l + 1] = (uintptr_t)e.depth_pitch;
        list[4 * l + 2] = (uintptr_t)e.ao; list[4 * l + 3] = (uintptr_t)e.ao_pitch;
    }
    return render_batch(c, *io, kind, std::move(list), ao[0], (cudaStream_t)stream, capturing);
}

int meao_render_host_async(MeaoCtx *c, const void *depth_host, int32_t kind, uint8_t *ao_host, int32_t slot)
{
    int rc = ensure_ready(c); if (rc) return rc;
    if (c->cams.cams && c->layers > c->cams_capacity) return frame_ready(c, c->stream);     // refused before the staging copy
    if (!depth_host || !ao_host) return fail(c, MEAO_ERR_INVALID, "depth / ao_out is NULL");
    if (slot != 0 && slot != 1) return fail(c, MEAO_ERR_INVALID, "slot must be 0 or 1");
    const size_t rows = (size_t)(c->band1 - c->band0) * c->layers;      // layered: L images of H rows (no band)
    cudaStream_t s = c->slot_stream[slot];
    CUDA_TRY(c, cudaMemcpyAsync(c->depth_stage[slot], depth_host, rows * c->W * depth_esize(kind), cudaMemcpyHostToDevice, s));
    // the two slots share the context's intermediates: kernels of consecutive frames are serialised, copies are not
    if (c->compute_done_valid) CUDA_TRY(c, cudaStreamWaitEvent(s, c->compute_done, 0));
    // meao_render of the staging buffers, which hold the tight layout whether or not a layer-viewport table is set
    bool capturing;
    if ((rc = frame_ready(c, s, &capturing))) return rc;
    if ((rc = render_views(c, c->depth_stage[slot], kind, c->ao_stage[slot], tight_pitch(*c, kind), s, capturing, false))) return rc;
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
    if (kind < MEAO_DEPTH_RAW_F32 || kind > MEAO_DEPTH_RAW_D24S8) return fail(c, MEAO_ERR_INVALID, "bad depth kind %d", kind);
    if ((rc = record_cameras(c, (cudaStream_t)stream))) return rc;      // the later stage calls read the tables it derives
    if ((rc = record_params(c, (cudaStream_t)stream))) return rc;       // and the slot it derives
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
    if (lo_level > effective_depth(c->plan.variants))
        return fail(c, MEAO_ERR_INVALID, "upsample lo level %d is above the frame's hierarchy depth %d (meao_set_hierarchy_depth, single_scale)",
                    lo_level, effective_depth(c->plan.variants));
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
        const int k = b.level - 2;
        // a bound device camera buffer: each layer's padding value is the one its last frame derived, read back from the table slot
        std::vector<float> pads;
        if (c->cams.cams) {
            pads.resize(c->layers);
            CUDA_TRY(c, cudaMemcpy2D(pads.data(), sizeof(float), &c->layer_ren[(size_t)2 * (k - 1) * c->layers].pad, sizeof(LayerRender),
                                     sizeof(float), c->layers, cudaMemcpyDeviceToHost));
        }
        __half *tmp = nullptr;
        CUDA_TRY(c, cudaMalloc(&tmp, need));
        cudaError_t e = cudaSuccess;
        for (int l = 0; l < c->layers && e == cudaSuccess; l++)
            e = launch_tiled_atlas(*c, k, l, c->last_kind, (__half *)((char *)tmp + l * one), c->stream, pads.empty() ? nullptr : &pads[l]);
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
    if (b.slices == 16 && c->cams.cams)
        return fail(c, MEAO_ERR_UNSUPPORTED, "debug view %d: the TiledDepth views take the atlas padding from the host cameras, and a device "
                                             "camera buffer is bound (meao_bind_device_cameras); meao_get_buffer reads them", id);
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
    // a host camera changed while a device camera buffer is bound, or a host thickness_modifier / intensity while a device parameter
    // buffer is, without moving the generation: the getters describe the host values, so the plan takes them now (the frames derive
    // theirs on the device and never read these)
    if (c->host_consts_stale) build_plan(c);
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
    bool capturing;
    int rc = ensure_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if ((rc = composite_args(c, ao, color, fmt))) return rc;
    const long long npix = (long long)c->W * (c->band1 - c->band0) * c->layers;
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, color, npix, fmt == MEAO_FMT_RGBA16_FLOAT, 1, 1, 0, (cudaStream_t)stream));
    c->launches++;
    return MEAO_OK;
}

int meao_composite_gbuffer(MeaoCtx *c, const void *ao, void *g0, void *g3, int32_t fmt3, void *stream)
{
    bool capturing;
    int rc = ensure_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
    if ((rc = composite_args(c, ao, g0, MEAO_FMT_RGBA8_UNORM)) || (rc = composite_args(c, ao, g3, fmt3))) return rc;
    const long long npix = (long long)c->W * (c->band1 - c->band0) * c->layers;
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, g0, npix, 0, 0, 1, 1, (cudaStream_t)stream));                               // gbuffer0.a
    CUDA_TRY(c, launch_composite((const uint8_t *)ao, g3, npix, fmt3 == MEAO_FMT_RGBA16_FLOAT, 1, 0, 1, (cudaStream_t)stream));   // gbuffer3.rgb
    c->launches += 2;
    return MEAO_OK;
}

int meao_composite_debug(MeaoCtx *c, const void *view, void *color, int32_t fmt, void *stream)
{
    bool capturing;
    int rc = ensure_ready(c, (cudaStream_t)stream, &capturing); if (rc) return rc;
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

namespace {
int bind_event_arrays(MeaoCtx *c, int32_t event_id, const void *depth_array, int dx, int dy, int kind, void *ao_array, int ax, int ay, bool exact,
                      void *stream)
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
    if ((rc = prepare_arrays(c, depth_array, dx, dy, kind, ao_array, ax, ay, exact, &io))) return rc;
    std::lock_guard<std::mutex> g(g_event_mutex);
    g_events[event_id] = EventBinding{c, depth_array, kind, ao_array, stream, true, false, ViewPitch{}, {dx, dy, ax, ay}, exact};
    return MEAO_OK;
}
}  // namespace

int meao_bind_event_arrays(MeaoCtx *c, int32_t event_id, const void *depth_array, int32_t kind, void *ao_array, void *stream)
{
    return bind_event_arrays(c, event_id, depth_array, 0, 0, kind, ao_array, 0, 0, true, stream);
}

int meao_bind_event_arrays_at(MeaoCtx *c, int32_t event_id, const void *depth_array, int32_t depth_x, int32_t depth_y, int32_t kind,
                              void *ao_array, int32_t ao_x, int32_t ao_y, void *stream)
{
    return bind_event_arrays(c, event_id, depth_array, depth_x, depth_y, kind, ao_array, ao_x, ao_y, false, stream);
}

int meao_bind_event_arrays_batch(MeaoCtx *c, int32_t event_id, const void *const *depth_arrays, int32_t kind, void *const *ao_arrays,
                                 int32_t count, void *stream)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!depth_arrays && !ao_arrays) {
        std::lock_guard<std::mutex> g(g_event_mutex);
        g_events.erase(event_id);
        return MEAO_OK;
    }
    // checked now: the plugin event cannot report an error.  The surfaces are made now too, so the event may run inside a capture
    int rc = ensure_ready(c); if (rc) return rc;
    if ((rc = check_batch(c, count, kind, true))) return rc;
    std::unique_ptr<BatchIO> io(new BatchIO);
    if ((rc = prepare_batch_arrays(c, depth_arrays, kind, ao_arrays, count, false, io.get()))) return rc;
    std::vector<const void *> list(depth_arrays, depth_arrays + count);
    list.insert(list.end(), ao_arrays, ao_arrays + count);
    std::lock_guard<std::mutex> g(g_event_mutex);
    g_events[event_id] = EventBinding{c, nullptr, kind, nullptr, stream, true, false, ViewPitch{}, {0, 0, 0, 0}, true, std::move(list)};
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
    if (!b.batch.empty()) {
        const size_t n = b.batch.size() / 2;
        meao_render_arrays_batch(b.ctx, b.batch.data(), b.kind, const_cast<void *const *>(b.batch.data() + n), (int32_t)n, b.stream);
    } else if (b.arrays) render_arrays(b.ctx, b.depth, b.org[0], b.org[1], b.kind, b.out, b.org[2], b.org[3], b.exact, b.stream);
    else if (b.tight) meao_render(b.ctx, b.depth, b.kind, b.out, b.stream);      // meao_render_pitched at the tight pitches of now
    else meao_render_pitched(b.ctx, b.depth, b.pitch.depth_row, b.pitch.depth_layer, b.kind, b.out, b.pitch.ao_row, b.pitch.ao_layer, b.stream);
}

MeaoRenderEventFunc meao_get_render_event_func(void) { return meao_render_event; }

int meao_bind_device_cameras(MeaoCtx *c, const float *cameras_dev, int32_t capacity)
{
    if (!c) return MEAO_ERR_INVALID;
    if (!c->plan_only && in_open_capture(c))
        return fail(c, MEAO_ERR_UNSUPPORTED, "meao_bind_device_cameras synchronises the device: not while a capture that holds a frame of this context is open");
    if (!cameras_dev && capacity == 0) {
        if (!c->cams.cams) return 0;
        if (!c->plan_only) {
            CUDA_TRY(c, cudaSetDevice(c->device));
            CUDA_TRY(c, cudaDeviceSynchronize());       // frames in flight may still write the status words
            CUDA_TRY(c, cudaFree(c->cams.status));
        }
        c->cams = DeviceCameras{};
        c->cams_capacity = 0;
        c->plan_dirty = true;           // the host cameras and the single-image kernels again: re-plan + drop the captured graphs
        c->frame_gen++;
        return 1;
    }
    if (!cameras_dev) return fail(c, MEAO_ERR_INVALID, "cameras_dev is NULL with capacity %d (NULL unbinds only with capacity 0)", capacity);
    if (capacity < 1 || capacity > kMaxLayers) return fail(c, MEAO_ERR_INVALID, "capacity %d not in 1..%d", capacity, kMaxLayers);
    if ((uintptr_t)cameras_dev % alignof(float)) return fail(c, MEAO_ERR_INVALID, "cameras_dev %p is not aligned to a float", (const void *)cameras_dev);
    if ((c->W > 0 && (c->band0 != 0 || c->band1 != c->H)) || c->peer_base[0] || c->peer_base[1])
        return fail(c, MEAO_ERR_UNSUPPORTED, "a device camera buffer is not supported with a row band or a neighbour connection "
                                             "(meao_set_row_band, meao_band_connect)");
    if (cameras_dev == c->cams.cams && capacity == c->cams_capacity) return 0;
    if (!c->plan_only) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, cameras_dev) != cudaSuccess || (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) ||
            at.device != c->device) {
            cudaGetLastError();
            return fail(c, MEAO_ERR_INVALID, "cameras_dev %p is not device memory of device %d", (const void *)cameras_dev, c->device);
        }
        CUDA_TRY(c, cudaDeviceSynchronize());           // frames in flight may still read the old buffer and write the status words
        if (!c->cams.status) CUDA_TRY(c, cudaMalloc(&c->cams.status, kCameraStatusWords * sizeof(uint32_t)));
        CUDA_TRY(c, cudaMemset(c->cams.status, 0, kCameraStatusWords * sizeof(uint32_t)));     // kernels.h CameraTableArgs
    }
    sample_thickness(c->cams.thick);
    c->cams.cams = cameras_dev;
    c->cams_capacity = capacity;
    c->plan_dirty = true;               // the camera stage and the layered kernels at every layer count: re-plan + drop the captured graphs
    c->frame_gen++;
    return 1;
}

int meao_device_camera_status(const MeaoCtx *cc, int32_t out4[4])
{
    MeaoCtx *c = const_cast<MeaoCtx *>(cc);
    if (!c || !out4) return MEAO_ERR_INVALID;
    if (!c->cams.cams) return fail(c, MEAO_ERR_INVALID, "no device camera buffer is bound (meao_bind_device_cameras)");
    uint32_t w[4] = {0, 0, 0, 0};
    if (c->cams.status) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        // a dedicated non-blocking stream, like meao_band_status: never waits for (or delays) the frames in flight
        CUDA_TRY(c, cudaMemcpyAsync(w, c->cams.status, sizeof w, cudaMemcpyDeviceToHost, c->slot_stream[1]));
        CUDA_TRY(c, cudaStreamSynchronize(c->slot_stream[1]));
    }
    out4[0] = (int32_t)w[0]; out4[1] = (int32_t)w[1]; out4[2] = (int32_t)w[2]; out4[3] = 0;
    return MEAO_OK;
}

int meao_bind_device_params(MeaoCtx *c, const float *params_dev)
{
    if (!c) return MEAO_ERR_INVALID;
    if ((uintptr_t)params_dev % alignof(float)) return fail(c, MEAO_ERR_INVALID, "params_dev %p is not aligned to a float", (const void *)params_dev);
    if (!c->plan_only && in_open_capture(c))
        return fail(c, MEAO_ERR_UNSUPPORTED, "meao_bind_device_params synchronises the device: not while a capture that holds a frame of this context is open");
    if (!params_dev) {
        if (!c->dev_params.params) return 0;
        if (!c->plan_only) {
            CUDA_TRY(c, cudaSetDevice(c->device));
            CUDA_TRY(c, cudaDeviceSynchronize());       // frames in flight may still write the slot and the status words
            CUDA_TRY(c, cudaFree(c->dev_params.derived));
        }
        c->dev_params = RenderParamArgs{};
        c->plan_dirty = true;           // the host parameters and the renders of the plan again: re-plan + drop the captured graphs
        c->frame_gen++;
        return 1;
    }
    if ((c->W > 0 && (c->band0 != 0 || c->band1 != c->H)) || c->peer_base[0] || c->peer_base[1])
        return fail(c, MEAO_ERR_UNSUPPORTED, "a device parameter buffer is not supported with a row band or a neighbour connection "
                                             "(meao_set_row_band, meao_band_connect)");
    if (params_dev == c->dev_params.params) return 0;
    if (!c->plan_only) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, params_dev) != cudaSuccess || (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) ||
            at.device != c->device) {
            cudaGetLastError();
            return fail(c, MEAO_ERR_INVALID, "params_dev %p is not device memory of device %d", (const void *)params_dev, c->device);
        }
        CUDA_TRY(c, cudaDeviceSynchronize());           // frames in flight may still read the old buffer and write the slot
        if (!c->dev_params.derived) {
            void *mem = nullptr;
            CUDA_TRY(c, cudaMalloc(&mem, 2 * sizeof(float) + kParamStatusWords * sizeof(uint32_t)));
            c->dev_params.derived = static_cast<float *>(mem);
            c->dev_params.status = reinterpret_cast<uint32_t *>(c->dev_params.derived + 2);
        }
        // the slot starts at the host parameters (build_plan's arithmetic), which an invalid first block leaves in place; the status at zero
        struct { float derived[2]; uint32_t status[kParamStatusWords]; } init = {{-1 / c->params.thickness_modifier, c->params.intensity}, {0, 0}};
        CUDA_TRY(c, cudaMemcpy(c->dev_params.derived, &init, sizeof init, cudaMemcpyHostToDevice));
    }
    c->dev_params.params = params_dev;
    c->plan_dirty = true;               // the parameter stage and the *_params_layered renders: re-plan + drop the captured graphs
    c->frame_gen++;
    return 1;
}

int meao_device_param_status(const MeaoCtx *cc, int32_t out4[4])
{
    MeaoCtx *c = const_cast<MeaoCtx *>(cc);
    if (!c || !out4) return MEAO_ERR_INVALID;
    if (!c->dev_params.params) return fail(c, MEAO_ERR_INVALID, "no device parameter buffer is bound (meao_bind_device_params)");
    uint32_t w[kParamStatusWords] = {0, 0};
    if (c->dev_params.status) {
        CUDA_TRY(c, cudaSetDevice(c->device));
        // a dedicated non-blocking stream, like meao_device_camera_status: never waits for (or delays) the frames in flight
        CUDA_TRY(c, cudaMemcpyAsync(w, c->dev_params.status, sizeof w, cudaMemcpyDeviceToHost, c->slot_stream[1]));
        CUDA_TRY(c, cudaStreamSynchronize(c->slot_stream[1]));
    }
    out4[0] = (int32_t)w[0]; out4[1] = (int32_t)w[1]; out4[2] = 0; out4[3] = 0;
    return MEAO_OK;
}

int64_t meao_launch_count(const MeaoCtx *c) { return c ? c->launches : 0; }
int64_t meao_frame_generation(const MeaoCtx *c) { return c ? c->frame_gen : MEAO_ERR_INVALID; }
int meao_pdl_level(const MeaoCtx *c) { return c ? c->pdl_level : -1; }
int meao_kernels_per_frame(const MeaoCtx *c)
{
    if (!c) return (int)frame_schedule(PlanVariants()).size();
    return (int)frame_schedule(PlanVariants(c->variants, c->hierarchy_depth), c->cams.cams != nullptr, c->dev_params.params != nullptr).size();     // as set: the plan may not be rebuilt yet
}

int64_t meao_algorithmic_bytes(const MeaoCtx *c, int32_t stage)
{
    if (!c || c->W <= 0) return MEAO_ERR_INVALID;
    auto px = [&](int l) { return (int64_t)c->lw[l] * c->lh[l] * c->layers; };      // every layer moves the same bytes
    // SURVEY.md 8(d): every buffer of the reference data-flow read once per consuming stage, written once; the renders and upsamples of
    // the levels the frame runs (its hierarchy depth, as set)
    const int n = effective_depth(PlanVariants(c->variants, c->hierarchy_depth));
    const int64_t ds1 = 6 * px(0) + 4 * px(1) + 4 * px(2) + 32 * px(3) + 32 * px(4);
    const int64_t ds2 = 4 * px(2) + 4 * px(3) + 4 * px(4) + 32 * px(5) + 32 * px(6);
    int64_t ren = 0, ups = 0, ups_final = 0;
    for (int k = 1; k <= n; k++) ren += 32 * px(k + 2) + px(k);
    for (int lo = n; lo >= 1; lo--) {
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
    if (c && !c->plan_only && in_open_capture(c))
        return fail(c, MEAO_ERR_UNSUPPORTED, "meao_profile_frame synchronises the device: not while a capture that holds a frame of this context is open");
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
