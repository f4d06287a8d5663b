/*
 * meao.h -- C ABI of libmeao.so: the H100-native multi-scale SSAO pipeline that stands in for
 * the compute path of keijiro/MiniEngineAO's AmbientOcclusion component.
 *
 * The reference has no FFI seam: its boundary is the set of CommandBuffer calls
 * AmbientOcclusion.cs makes against four ComputeShader assets.  Each entry point below names
 * the reference interface it replaces (paths relative to Assets/MiniEngineAO/ of the reference project).
 * The C# P/Invoke binding a maintainer would add is host/AmbientOcclusionNative.cs and is
 * described in INTEGRATION.md.
 *
 * Conventions: plain C types only; every call returns 0 on success or a negative MeaoStatus;
 * meao_last_error() gives the text.  A context is owned by one thread at a time (the reference
 * records on Unity's main thread and replays on one render thread); distinct contexts are
 * independent.  The caller owns the depth input and the AO output memory; the context owns the
 * 16 intermediate buffers (LinearDepth, LowDepth1-4, Occlusion1-4, Combined1-3; the four
 * TiledDepth atlases are virtual, see DESIGN.md).
 * There is NO CPU fallback: every compute entry point fails with MEAO_ERR_CUDA when no
 * sm_90 (H100) device is usable.
 */
#ifndef MEAO_H
#define MEAO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define MEAO_ABI_VERSION 3   /* 2: + MeaoVariants, meao_stage_render_wide, meao_debug_view, meao_composite_debug, buffer ids 18..21
                              * 3: + MeaoVariants.single_scale, native peer halo exchange (meao_band_export / _connect / _step / _status),
                              *      meao_bind_event takes the stream
                              *    + meao_set_layers (layered frames; additive, so the version stays 3)
                              *    + meao_render_arrays / meao_bind_event_arrays / meao_release_array (CUDA-array I/O; additive)
                              *    + meao_render_pitched / meao_bind_event_pitched (depth and AO with their own row and layer pitch; additive)
                              *    + meao_reserve / meao_reservation (dynamic resolution; additive)
                              *    + meao_frame_generation (frames inside a caller's CUDA graph; additive)
                              *    + meao_render_arrays_at / meao_bind_event_arrays_at (viewports of larger CUDA arrays; additive)
                              *    + MeaoLayerViewport, meao_set_layer_viewports / meao_get_layer_viewports (each layer at its own
                              *      viewport of shared CUDA arrays: split-screen, side-by-side stereo, cube atlases; additive)
                              *    + MeaoProjection, meao_set_projection / meao_get_projection (orthographic cameras; additive)
                              *    + MEAO_MAX_BATCH, meao_render_arrays_batch / meao_render_batch / meao_bind_event_arrays_batch (each
                              *      layer with its own depth and AO resources: several cameras, each with its own targets; additive)
                              *    + meao_reserve_layers / meao_layer_reservation (dynamic view counts: a layer change inside the
                              *      reservation is host bookkeeping; additive)
                              *    + meao_set_layer_projections / meao_get_layer_projections (perspective and orthographic layers in one
                              *      layered frame; additive)
                              *    + meao_bind_device_cameras / meao_device_camera_status (cameras read from device memory at every
                              *      launch and graph replay; additive)
                              *    + meao_set_hierarchy_depth / meao_get_hierarchy_depth (render and upsample only the finest 1-4 levels;
                              *      additive, MeaoVariants unchanged)
                              *    + meao_bind_device_params / meao_device_param_status (thickness_modifier and intensity read from
                              *      device memory at every launch and graph replay; additive) */

typedef struct MeaoCtx MeaoCtx;

typedef enum {
    MEAO_OK = 0,
    MEAO_ERR_INVALID = -1,      /* bad argument / call order */
    MEAO_ERR_CUDA = -2,         /* CUDA runtime or driver error, or no usable device */
    MEAO_ERR_UNSUPPORTED = -3,  /* e.g. halo deeper than the neighbouring band */
    MEAO_ERR_NOMEM = -4,
    MEAO_ERR_PEER = -5          /* native halo exchange: a neighbour did not arrive within the time-out (meao_band_status) */
} MeaoStatus;

/* AmbientOcclusion.cs:20-68 -- the serialized parameter surface, same names, ranges, defaults. */
typedef struct {
    float noise_filter_tolerance;   /* Range(-8, 0)    default 0      AO.cs:20-26 */
    float blur_tolerance;           /* Range(-8, -1)   default -4.6   AO.cs:28-34 */
    float upsample_tolerance;       /* Range(-12, -1)  default -12    AO.cs:36-42 */
    float thickness_modifier;       /* Range(1, 10)    default 1      AO.cs:44-50 */
    float intensity;                /* Range(0, 2)     default 1      AO.cs:52-58 */
    int32_t debug;                  /* Range(0, 17)    default 0      AO.cs:60    (carried; selects nothing on the compute path) */
    int32_t ambient_only;           /* default 1       AO.cs:62-68   (carried; composite is out of scope) */
} MeaoParams;

/* Camera inputs of the CPU-side constant math: AO.cs:561-573.  Their meaning under an orthographic projection: meao_set_projection. */
typedef struct {
    float near_clip;        /* camera.nearClipPlane                         AO.cs:563 */
    float far_clip;         /* camera.farClipPlane                          AO.cs:563 */
    float tan_half_fov_h;   /* 1 / camera.projectionMatrix[0,0]             AO.cs:570-573 (orthographic: the view volume's half-width) */
    int32_t reversed_z;     /* SystemInfo.usesReversedZBuffer (D3D11/12: 1) AO.cs:564, Downsample1.compute:41-45 */
} MeaoCamera;

typedef struct {
    int32_t device;         /* CUDA device ordinal; < 0 = host-side PLANNING context only (constants, geometry,
                               band / halo row ranges) -- every compute call on it fails with MEAO_ERR_CUDA */
    uint32_t flags;         /* MEAO_FLAG_* */
} MeaoDeviceCfg;

#define MEAO_FLAG_NONE        0u
#define MEAO_FLAG_NO_GRAPH    1u   /* launch the kernels on the stream instead of replaying the captured CUDA graph */

typedef enum {
    MEAO_DEPTH_RAW_F32 = 0,     /* camera depth, linearised by Downsample1.compute:37-48 (reference behaviour) */
    MEAO_DEPTH_LINEAR_F32 = 1,  /* already-linear depth (Linearize becomes the identity; not in the reference): eye depth / far_clip, the
                                   values LinearDepth holds.  Perspective AO does not depend on the scale; orthographic AO does */
    /* native depth-buffer formats (what Blit.shader pass 0 :48-64 samples; SURVEY.md 8f.1): the UNORM code is
     * converted with the D3D rule (float)code * (1 / (2^n - 1)) and then linearised like RAW_F32 */
    MEAO_DEPTH_RAW_D16_UNORM = 2,   /* uint16 codes, 2 bytes / pixel */
    MEAO_DEPTH_RAW_D24S8 = 3        /* uint32 words, depth in the low 24 bits (D24_UNORM_S8_UINT), stencil ignored */
} MeaoDepthKind;

/* Debug buffer ids, numbering of AmbientOcclusion.cs:787-808. */
typedef enum {
    MEAO_BUF_LINEAR_DEPTH = 1,                                  /* L0, f16 */
    MEAO_BUF_LOW_DEPTH1 = 2, MEAO_BUF_LOW_DEPTH2 = 3,           /* L1..L4, f32 */
    MEAO_BUF_LOW_DEPTH3 = 4, MEAO_BUF_LOW_DEPTH4 = 5,
    MEAO_BUF_TILED_DEPTH1 = 6, MEAO_BUF_TILED_DEPTH2 = 7,       /* L3..L6 x 16 slices, f16 */
    MEAO_BUF_TILED_DEPTH3 = 8, MEAO_BUF_TILED_DEPTH4 = 9,
    MEAO_BUF_OCCLUSION1 = 10, MEAO_BUF_OCCLUSION2 = 11,         /* L1..L4, unorm8 */
    MEAO_BUF_OCCLUSION3 = 12, MEAO_BUF_OCCLUSION4 = 13,
    MEAO_BUF_COMBINED1 = 14, MEAO_BUF_COMBINED2 = 15, MEAO_BUF_COMBINED3 = 16,   /* L1..L3, unorm8 */
    MEAO_BUF_AMBIENT_OCCLUSION = 17,                            /* L0, unorm8 */
    /* extension ids (not in AO.cs:787-808): output of Render.compute kernel "main" (MeaoVariants.high_quality_mask) */
    MEAO_BUF_HIGH_QUALITY1 = 18, MEAO_BUF_HIGH_QUALITY2 = 19,   /* L1..L4, unorm8 */
    MEAO_BUF_HIGH_QUALITY3 = 20, MEAO_BUF_HIGH_QUALITY4 = 21
} MeaoBufferId;

typedef struct {
    int32_t width, height, slices;  /* reference texture dimensions (AO.cs:276-281; slices = 16 when tiled, AO.cs:154) */
    int32_t elem_bytes;             /* 1 = unorm8, 2 = f16 bits, 4 = f32  (AO.cs:262-273) */
} MeaoBufferDesc;

/* Shader / host variants that the reference SHIPS but never selects (SURVEY.md 8f.2, 8f.4).  All zero = exactly what
 * AmbientOcclusion.cs records; every field is a plan input like MeaoParams (a change re-plans, AO.cs:334-347). */
typedef struct {
    int32_t single_pass_stereo;   /* singlePassStereoEnabled (AO.cs:392-401): ThicknessMultiplier *= 2 (AO.cs:680).  The caller passes the
                                     DOUBLE-WIDE eye pair to meao_resize, as LateUpdate / RebuildCommandBuffers do (AO.cs:338-341, 501-504). */
    int32_t sample_exhaustively;  /* Render.compute:144-159 "#define SAMPLE_EXHAUSTIVELY": 68 taps instead of the 36-tap checker, and the
                                     weight zeroing of AO.cs:709-715 ("FIXME: should we support SAMPLE_EXHAUSTIVELY mode?") is skipped */
    int32_t high_quality_mask;    /* bit k-1 (k = 1..4): level k ALSO runs Render.compute kernel "main" (WIDE_SAMPLING, :22,27-29,46-50,79-82:
                                     non-tiled source LowDepth<k>, so PushRenderCommands takes the "!source.isTiled" branch AO.cs:679) into
                                     HighQuality<k>, and the upsample whose LOW level is k runs Upsample.compute kernel "main_premin" /
                                     "main_premin_blendout" (:23,25,32-34,58-60) with LoResAO2 = HighQuality<k>.  E.g. 8 = coarsest level
                                     only, 15 = every level (the quality ladder of the upstream MiniEngine sample, which is not vendored). */
    int32_t single_scale;         /* BASELINE.json configs[0] "single-scale AO": the frame is Downsample1 -> Render level 1 -> the FINAL-style
                                     Upsample (kernel "main", AO.cs:531's dispatch with LoResAO1 = Occlusion1 instead of Combined1): three of
                                     the ten dispatches of AO.cs:511-531, no coarser level contributes.  Requires high_quality_mask == 0.
                                     It is the frame of hierarchy depth 1 (meao_set_hierarchy_depth): while set, the depth in effect is 1. */
} MeaoVariants;

/* ---- lifetime ------------------------------------------------------------------------------ */
/* replaces: component construction + DoLazyInitialization (AO.cs:440-494). */
int meao_create(const MeaoDeviceCfg *cfg, MeaoCtx **out_ctx);
/* replaces: OnDestroy (AO.cs:357-381). */
void meao_destroy(MeaoCtx *ctx);
const char *meao_last_error(const MeaoCtx *ctx);   /* ctx may be NULL: error of the last failed meao_create on this thread */
int meao_abi_version(void);

/* ---- parameters (plan inputs) ----------------------------------------------------------------
 * The plan inputs fall into two classes.
 * FRAME CONSTANTS take effect at the next frame issued on the context, with no device or stream synchronise, no re-plan, no graph
 * dropped or instantiated, no CUDA array released and no planned size forgotten (meao_reserve): the five floats of MeaoParams (and
 * `debug`, which selects nothing), the near_clip, far_clip and tan_half_fov_h of a MeaoCamera, and the whole meao_set_layer_cameras
 * table, clearing it included.  The host plans the new constants at once (the constant getters below return them), the next frame
 * writes the per-layer camera tables on its own stream before its kernels, and each captured graph is re-targeted to the new kernel
 * arguments (cudaGraphExecUpdate) at its next launch.  Under the ordering contract (meao_reserve) frame n sees the constants set
 * before it was issued, and frame n-1, still in flight, keeps its own.  A host may therefore animate the camera and the
 * parameters every frame.
 * STRUCTURAL INPUTS re-plan with a device synchronise and drop the captured graphs: MeaoVariants, meao_set_hierarchy_depth, meao_set_layers without a layer
 * reservation, a resize without a reservation, meao_reserve, row bands, a change of the cameras' reversed_z (it selects kernel instantiations; it is a
 * platform property) and meao_set_projection.
 * A refused camera, table or parameter block leaves the context exactly as it was. */
/* replaces: the property setters AO.cs:22-66 (CheckPropertiesChanged, AO.cs:104-113): returns 1 if a value changed, 0 if not. */
int meao_set_params(MeaoCtx *ctx, const MeaoParams *params);
int meao_get_params(const MeaoCtx *ctx, MeaoParams *out);
void meao_default_params(MeaoParams *out);          /* AO.cs:20-68 defaults */
/* Selects the undispatched shader variants above (a structural input); returns 1 if a value changed, 0 if not. */
int meao_set_variants(MeaoCtx *ctx, const MeaoVariants *variants);
int meao_get_variants(const MeaoCtx *ctx, MeaoVariants *out);
/* ---- hierarchy depth: how many levels of the AO pyramid a frame renders and upsamples (upstream MiniEngine's "Hierarchy Depth").
 * levels = n in 1..4, default 4 (the reference's frame).  A frame of depth n:
 *   - prepares as at depth 4: LowDepth1..4 (and LinearDepth) are always written;
 *   - renders levels 1..n, and the wide render of every high_quality_mask bit k <= n.  Mask bits above n launch nothing: they are kept,
 *     not refused, so that meao_set_variants and this setter may be called in either order;
 *   - runs n upsamples, lo levels n, n-1, ..., 1.  The first reads Occlusion<n> (and HighQuality<n> when bit n is set) where the depth-4
 *     frame's lo-level-4 upsample reads Occlusion4; every later one reads the Combined<lo> the one before wrote.  At n = 1 the first
 *     upsample is the final one, on Occlusion1: the single_scale frame.  With single_scale = 0 and n = 1 a high_quality_mask bit 0 is
 *     allowed (the premin final upsample on Occlusion1 and HighQuality1).
 * The depth in effect is MeaoVariants.single_scale ? 1 : levels; meao_get_hierarchy_depth returns `levels` as set.
 * The kernels are the depth-4 frame's: fewer levels, fewer launches.  meao_kernels_per_frame = 1 + n + (mask bits <= n) + n (+1 with
 * a bound device camera buffer), meao_algorithmic_bytes counts the renders and upsamples of levels 1..n, and meao_profile_frame lists
 * the launches of the schedule.  The stage API refuses meao_stage_upsample(lo_level > n) with MEAO_ERR_INVALID; lo_level = n reads
 * Occlusion<n>.  meao_stage_render is unchanged.
 * The debug buffers of stages a frame of depth n does not run -- Occlusion<k> and HighQuality<k> for k > n, Combined<k> for k >= n --
 * have unspecified contents; reading them is not refused.
 * Every frame form, reservation, capture and row band takes it; a band's halo rows are those of the depth-4 frame.
 * A structural input, like MeaoVariants: a change re-plans behind a device synchronise, drops the captured graphs and moves
 * meao_frame_generation, so a host that toggles it every frame pays a re-plan per toggle.  Under a size or layer reservation the arena
 * stays; the other planned (W, H, L) are forgotten.  Plan-only contexts accept it.
 * Returns 1 on a change, 0 for the value already set; any value outside 1..4 returns MEAO_ERR_INVALID, names the field in
 * meao_last_error and changes nothing. */
int meao_set_hierarchy_depth(MeaoCtx *ctx, int32_t levels);
int meao_get_hierarchy_depth(const MeaoCtx *ctx);
/* replaces: CalculateZBufferParams / CalculateTanHalfFovHeight inputs (AO.cs:561-573).  A frame constant, except reversed_z;
 * returns MEAO_OK. */
int meao_set_camera(MeaoCtx *ctx, const MeaoCamera *camera);

/* ---- projection ----------------------------------------------------------------------------------
 * The projection model of the context's cameras, one for all layers; a layered frame whose layers differ sets a projection per layer
 * with meao_set_layer_projections below.
 * PERSPECTIVE (the default) is what the reference does.  ORTHOGRAPHIC (isometric and top-down views, CAD viewers, editor views):
 *   - raw depth is affine in eye depth: with r = near_clip / far_clip, lin = fma(1 - r, d, r), reversed Z lin = fma(r - 1, d, 1) -- eye
 *     depth / far_clip, LinearDepth's convention; d == 1 (reversed: d == 0) is sky, 1e5, as for perspective.  meao_zbuffer_params
 *     returns {1 - r, r, 0, 0} (reversed: {r - 1, 1, 0, 0}), and the atlas padding of render levels 1-2 is r (reversed: 1e5).
 *     MEAO_DEPTH_LINEAR_F32 input must follow the same convention, eye depth / far_clip: the sphere's thickness is absolute.
 *   - the sampling sphere has a constant world size instead of growing with the centre depth: with the reference's ThicknessMultiplier
 *     TM (AO.cs:671-683, from tan_half_fov_h and the source width), sample i has invRange = it_i = (far_clip / TM) / SampleThickness[i]
 *     and frontDepth = centre x it_i - 0.5.  meao_render_constants return it_i in the gInvThicknessTable slots.
 *   - tan_half_fov_h = 1 / projectionMatrix[0,0] (CalculateTanHalfFovHeight, AO.cs:570-573) is the half-width of the view volume in world
 *     units (Unity: orthographicSize x aspect).  near_clip must be > 0 as for perspective, although Unity allows near <= 0 for an
 *     orthographic camera: a linear depth of 0 would reach the upsample's 1 / depth.
 *   - the planes and the half-width stay frame constants: an orthographic zoom takes effect at the next frame without a re-plan.
 *   - the upsample and blur are the perspective ones (they work on the stored linear depth through 1 / depth, DESIGN.md 2.14).
 * A change of projection is a structural input: it re-plans with a device synchronise, drops the captured graphs, moves
 * meao_frame_generation and returns 1; the same value returns 0.  Not supported under ORTHOGRAPHIC, refused with MEAO_ERR_UNSUPPORTED in
 * either order (setting the projection while one is set, or setting one under an orthographic projection), before anything changes:
 * a layer-viewport table (meao_set_layer_viewports) and row bands with their halo and native-exchange calls.  An unknown value is
 * MEAO_ERR_INVALID and changes nothing.  Both calls work on plan-only contexts. */
typedef enum {
    MEAO_PROJECTION_PERSPECTIVE = 0,
    MEAO_PROJECTION_ORTHOGRAPHIC = 1
} MeaoProjection;
int meao_set_projection(MeaoCtx *ctx, int32_t projection);
int meao_get_projection(const MeaoCtx *ctx);     /* MeaoProjection, or MEAO_ERR_INVALID for a NULL context */
/* ---- per-layer projections ------------------------------------------------------------------------
 * One MeaoProjection per layer of a layered frame (meao_set_layers): an editor's perspective pane beside its top, front and side
 * orthographic panes, a bird's-eye-view camera beside perspective sensor cameras, an isometric view beside a perspective one -- in one
 * frame, one set of intermediates and one graph instead of a context per projection.
 *   - count must equal the layer count; projections == NULL with count == 0 clears the table.  Every entry must be
 *     MEAO_PROJECTION_PERSPECTIVE or MEAO_PROJECTION_ORTHOGRAPHIC.  A refusal returns MEAO_ERR_INVALID, names the layer and the field in
 *     meao_last_error and changes nothing.
 *   - While a table is set it alone decides each layer's projection.  meao_set_projection still records the context's projection, which
 *     takes effect again when the table is cleared (as meao_set_camera relates to meao_set_layer_cameras).  A change of the layer count
 *     clears the table, as it clears the layer-camera and layer-viewport tables.
 *   - A layer's projection decides how its camera (the table's or the context's) is read, exactly as meao_set_projection describes for a
 *     whole context: under ORTHOGRAPHIC tan_half_fov_h is the view volume's half-width and MEAO_DEPTH_LINEAR_F32 input is eye depth /
 *     far_clip.  meao_zbuffer_params_layer and meao_render_constants_layer return each layer's constants for its own projection, and the
 *     layer's atlas padding follows it.  Every layer of a frame equals a single-layer frame of its depth with that projection and camera.
 *   - A set returns 1 if the table changed, 0 if not.  A change is a structural input like meao_set_projection: it re-plans with a device
 *     synchronise, drops the captured graphs and moves meao_frame_generation.  Inside a layer reservation (meao_reserve_layers) the clearing
 *     done by meao_set_layers stays host bookkeeping like the other tables': no synchronise, allocation or graph destruction.  Setting
 *     the table again for the new count is a change, hence structural: a host that changes the layer count of a frame that keeps mixing
 *     projections pays one re-plan with a device synchronise per count change, even inside the reservation.
 *   - A table with an ORTHOGRAPHIC entry carries the restrictions of an orthographic context, each refused with MEAO_ERR_UNSUPPORTED
 *     before anything changes, in either order: a layer-viewport table, batches (meao_render_arrays_batch, meao_render_batch and their
 *     event) and row bands.  The context-level refusals of meao_set_projection stay as they are.
 *   - Every other frame form of a layered context takes the table: pointers, pitched views, host buffers, CUDA arrays and their _at
 *     viewports, the bound events, MEAO_FLAG_NO_GRAPH, recording into a caller's capture, reservations, per-layer cameras, every
 *     MeaoVariants and both Z directions.  Plan-only contexts accept the table.
 *   - A table whose layers are all alike records the frame of a context with that projection; one that mixes both runs layered kernels
 *     that pick each layer's projection per CTA (DESIGN.md 2.17).
 * The getter follows meao_get_layer_cameras: it returns the entry count (0: no table), or MEAO_ERR_INVALID if the table does not fit in
 * capacity. */
int meao_set_layer_projections(MeaoCtx *ctx, const int32_t *projections, int32_t count);
int meao_get_layer_projections(const MeaoCtx *ctx, int32_t *out, int32_t capacity);
/* Cameras from device memory: a frame recorded into a graph (the context's own or a caller's capture, torch.cuda.graph) follows a moving
 * camera without a capture or an instantiation per camera change, and a camera that already lives on the GPU (a pose network's output,
 * a GPU-side camera animation) is never copied to the host.
 *   - cameras_dev: device memory of the context's device holding `capacity` cameras of 3 floats each, {near_clip, far_clip,
 *     tan_half_fov_h}, each with the meaning of MeaoCamera under its layer's projection.  A contiguous [n, 3] float32 CUDA tensor fits.
 *     Layer l of every frame uses entry l.  A frame with more layers than capacity is refused with MEAO_ERR_INVALID and launches nothing,
 *     so one buffer of max_layers cameras serves every layer count of a reservation (meao_reserve_layers).
 *   - cameras_dev == NULL with capacity == 0 unbinds.  capacity must be in 1..65535.  Returns 1 when the binding changed, 0 when the same
 *     one is set again.  Binding, unbinding and a new pointer or capacity are structural inputs: a re-plan with a device synchronise, the
 *     captured graphs dropped, meao_frame_generation moved.  Plan-only contexts record the binding and allocate nothing.
 *   - The buffer's CONTENTS are not tracked: they are read by the frame's first kernel, in stream order, at every launch and every replay.
 *     Writing new cameras moves no generation and needs no capture.  The host-buffer calls (meao_render_host, _async) run on the context's
 *     own streams, so the buffer must be complete before such a call is made.  The caller keeps the buffer alive while it is bound.
 *   - While a buffer is bound it alone decides every layer's near and far planes and field of view.  meao_set_camera and
 *     meao_set_layer_cameras still record their values, which apply again once the buffer is unbound; a change that keeps the Z direction
 *     neither moves meao_frame_generation nor marks tables pending, so it never makes a recording into a caller's capture refuse.
 *     reversed_z and the projections (meao_set_projection, meao_set_layer_projections) stay structural, host-side inputs.
 *   - The constant getters (meao_zbuffer_params, meao_render_constants and their _layer forms) keep describing the HOST cameras.
 *   - Every frame form runs the derivation first: pointers, pitched views, host buffers, CUDA arrays and _at, layer-viewport tables,
 *     batches, orthographic and mixed projection tables, the bound events, MEAO_FLAG_NO_GRAPH and recording into a caller's capture.
 *     meao_stage_downsample runs it too, and the later stage calls use the tables it derived.  meao_kernels_per_frame counts it (+1).  A
 *     single-layer frame takes the layered kernels with one layer, which read the derived tables; each layer is bit-identical to a frame
 *     of a context whose host cameras are the buffer's.
 *   - Refused with MEAO_ERR_UNSUPPORTED before anything changes, in either order: row bands and their halo and exchange calls; and while
 *     bound, meao_debug_view of the TiledDepth ids 6-9, whose atlas padding is a host value.  meao_get_buffer of ids 6-9 reads each
 *     layer's padding back from the derived tables.
 * meao_device_camera_status: {frames that met an invalid camera since the bind, the lowest such layer of the latest of them, its field (1
 * near_clip, 2 far_clip, 3 tan_half_fov_h), 0}.  An entry is invalid when it fails meao_set_camera's tests (!(near > 0), !(far > near),
 * !(tan_half_fov_h > 0); NaN fails): its layer's tables are not written, so its AO is unspecified, and every other layer is exact.  A
 * stream-less read like meao_band_status, without a device synchronise; all zeros on a plan-only context; MEAO_ERR_INVALID when nothing
 * is bound. */
int meao_bind_device_cameras(MeaoCtx *ctx, const float *cameras_dev, int32_t capacity);
int meao_device_camera_status(const MeaoCtx *ctx, int32_t out4[4]);
/* Thickness and intensity from device memory: a frame recorded into a graph (the context's own or a caller's capture, torch.cuda.graph,
 * the torch operator under torch.compile) follows an AO fade, a quality slider or a tuning loop without a capture or an instantiation per
 * change.
 *   - params_dev: device memory of the context's device holding 2 floats, {thickness_modifier, intensity}, with the meaning of the
 *     MeaoParams fields.  A contiguous float32 CUDA tensor of shape [2] fits.  It must be 4-byte aligned (else MEAO_ERR_INVALID, nothing
 *     changes).
 *   - params_dev == NULL unbinds.  Returns 1 when the binding changed, 0 when the same pointer is bound again.  Binding, unbinding and a
 *     new pointer are structural inputs: a re-plan with a device synchronise, the captured graphs dropped, meao_frame_generation moved.
 *     Plan-only contexts record the binding and allocate nothing.
 *   - The buffer's CONTENTS are not tracked: a stage ahead of the renders reads them, in stream order, at every launch and every replay,
 *     and derives the renders' reject_fadeoff (-1 / thickness_modifier, bit for bit the host's) and intensity.  Writing new values moves no
 *     generation and needs no capture.  The host-buffer calls (meao_render_host, _async) run on the context's own streams, so the buffer
 *     must be complete before such a call is made.  The caller keeps the buffer alive while it is bound.
 *   - A block is valid when it passes meao_set_params's test, thickness_modifier > 0 (NaN fails); intensity is taken as the host takes it.
 *     An invalid block leaves the derived values as they were -- the last valid block's, or the host parameters at bind time -- so the
 *     frame's AO is that of a host-parameter frame with those values.
 *   - While a buffer is bound it alone decides thickness_modifier and intensity.  meao_set_params still records them, and they apply
 *     again once the buffer is unbound: a change of those two fields alone returns 1 but moves no meao_frame_generation and marks nothing
 *     pending.  A change of a tolerance (or of debug) behaves as without a binding: the three tolerances stay host frame constants.
 *     meao_render_constants and its _layer and _wide forms keep describing the HOST values.
 *   - Every frame form runs the stage: pointers, pitched views, host buffers, CUDA arrays and _at, layer-viewport tables, both batch
 *     calls, orthographic and mixed projections, device cameras (both may be bound), the bound events, MEAO_FLAG_NO_GRAPH, recording into a
 *     caller's capture, both reservations and every hierarchy depth.  meao_stage_downsample runs it too, and the later meao_stage_render /
 *     _render_wide use the values it derived.  A single-layer frame takes the layered render kernels with one layer; every frame is
 *     bit-identical to a frame of a context whose host parameters are the buffer's.  meao_kernels_per_frame counts the stage (+1), and
 *     meao_profile_frame names it "render_params".
 *   - Refused with MEAO_ERR_UNSUPPORTED before anything changes, in either order: row bands and their halo and exchange calls.
 * meao_device_param_status: {frames that met an invalid block since the bind, the field of the latest (1 thickness_modifier), 0, 0}.  The
 * count is of the stage's launches: a frame launches it once, and meao_profile_frame, which launches every kernel profile_repeats times
 * (meao_set_profile_repeats), adds profile_repeats for a profiled frame that meets an invalid block.  A stream-less read like
 * meao_device_camera_status, without a device synchronise; all zeros on a plan-only context; MEAO_ERR_INVALID when nothing is bound. */
int meao_bind_device_params(MeaoCtx *ctx, const float *params_dev);
int meao_device_param_status(const MeaoCtx *ctx, int32_t out4[4]);
/* replaces: RTHandle.SetBaseDimensions + AllocateNow + the rebuild it triggers (AO.cs:338-341, 501-506).
 * Allocates the intermediates for width x height.  Returns 1 if dimensions changed, 0 if not.
 * A size change RESETS the row band to the whole frame and drops the neighbour connections (meao_set_row_band,
 * meao_band_connect): a band host must set its band again after every call that returned 1. */
int meao_resize(MeaoCtx *ctx, int32_t width, int32_t height);
/* ---- dynamic resolution ------------------------------------------------------------------------------------------------------
 * meao_reserve lays the intermediates out ONCE for max_width x max_height at the context's layer count, so that meao_resize to any
 * size inside the reservation is host bookkeeping: no allocation, free or memset, no stream or device synchronise, no graph
 * destruction.  Every planned size keeps its plan, TMA maps and captured graphs: a return to a size used recently (the last 8,
 * MEAO_SIZE_SLOTS) is a plain graph replay; a new size is planned on the host, its per-layer camera tables are written in stream order
 * by its first frame, and its graph is captured and, once the graph cache is full, re-targets the least recently used executable graph.
 * At most MEAO_MAX_GRAPHS_HELD executable graphs are alive at any time (MeaoReservation.graphs_held), whatever sizes a host visits.
 *   - Returns 1 when the reservation changed (the arena was re-allocated: a synchronising plan change like a resize without one), 0
 *     when the same reservation is set again.  Bounds as meao_resize (1..32768).  (0, 0) clears the reservation: the arena is then
 *     re-allocated at the current size.
 *   - Refused with MEAO_ERR_INVALID if the reservation is below the current size (meao_last_error names the dimension);
 *     MEAO_ERR_NOMEM leaves the previous reservation and arena in place.
 *   - meao_resize on a reserved context returns 1 when the size changed, as always; a size outside the reservation is refused with
 *     MEAO_ERR_INVALID and changes nothing -- a dynamic-resolution host never gets a silent re-allocation.
 *   - meao_set_layers re-allocates at the reservation x the new layer count, unless the count lies inside a layer reservation
 *     (meao_reserve_layers).  A change of MeaoVariants or of the cameras' reversed_z
 *     re-plans with a device synchronise, as without a reservation, and forgets the other planned sizes; the arena stays.  A change
 *     of a frame constant (MeaoParams, a camera's planes and field of view, the layer-camera table) keeps every planned size: a size
 *     parked with older constants is planned again on the host when it is swapped back in, and its graphs are re-targeted at their
 *     first replay.
 *   - Row bands and reservations exclude each other: meao_reserve on a context with a row band, and meao_set_row_band, the halo calls
 *     and the native exchange on a reserved context, return MEAO_ERR_UNSUPPORTED.
 *   - After a size change the intermediates (meao_get_buffer, meao_debug_view) describe the new size; their contents are unspecified
 *     until the first frame at that size (a fresh arena is zeroed; a reserved one holds whatever earlier sizes left there).
 *   - Works on plan-only contexts (device < 0): the reservation is recorded and nothing is allocated.
 * ORDERING CONTRACT (every context, reserved or not): the frames of one context run in the order they are issued -- they share the
 * context's intermediates (and, reserved, its camera table slots).  Frames issued on one stream are ordered by it; a host that
 * issues consecutive frames of one context on different streams orders them itself (an event, as meao_render_host_async does). */
#define MEAO_SIZE_SLOTS 8
#define MEAO_MAX_GRAPHS_HELD 72
int meao_reserve(MeaoCtx *ctx, int32_t max_width, int32_t max_height);
/* ---- dynamic view counts -----------------------------------------------------------------------------------------------------
 * meao_reserve_layers lays the intermediates out for max_layers layers (at the size reservation, or without one at the current size),
 * so that meao_set_layers to any count in 1..max_layers is host bookkeeping: no allocation, free or memset, no stream or device
 * synchronise, no graph destruction -- for hosts whose view count changes at run time (split-screen players joining and leaving,
 * mirrors and portals coming into view, the visible faces of a cube map, the short last batch of an epoch).
 *   - Returns 1 when the reservation changed (the arena is re-allocated once, with a synchronise, like meao_reserve), 0 when the same
 *     one is set again; 0 clears it (the arena is then re-allocated at the current count).  max_layers must be in 1..65535 and not
 *     below the current layer count, else MEAO_ERR_INVALID naming the field, and nothing changes; MEAO_ERR_NOMEM leaves the previous
 *     reservation and arena in place.  Works on plan-only contexts (device < 0): the reservation is recorded, nothing is allocated.
 *   - MeaoReservation.arena_bytes reports the arena laid out for max_layers; arena_bytes_needed is the current (W, H, L)'s layout.
 *   - meao_set_layers(L), 1 <= L <= max_layers, still returns 1 when L changed, moves meao_frame_generation and clears the
 *     layer-camera and layer-viewport tables, but allocates, frees, memsets, synchronises and destroys nothing.  An L above the
 *     reservation is refused with MEAO_ERR_INVALID and changes nothing: a host never gets a silent re-allocation.
 *   - Planned (W, H, L) triples share the MEAO_SIZE_SLOTS slots of meao_reserve, least recently used out: a return to a recently used
 *     one is a plain graph replay; a new one is planned on the host and its camera tables are written in stream order by its first
 *     frame (which is therefore refused inside a caller's capture, with the "issue one frame outside the capture first" message).
 *   - Setting a layer-viewport table where there was none, or clearing one, is a frame constant too on such a context: no re-plan, no
 *     synchronise; the next frame writes the table on its own stream.
 *   - MeaoVariants, a change of reversed_z and meao_set_projection stay structural: they re-plan with a device synchronise and forget
 *     the other planned (W, H, L); the arena stays.
 *   - Row bands and a layer reservation exclude each other (MEAO_ERR_UNSUPPORTED both ways, before anything changes).
 *   - After a layer change meao_get_buffer and meao_debug_view describe L layers; their contents are unspecified until the first frame
 *     at that L (a reserved arena holds whatever earlier frames left). */
int meao_reserve_layers(MeaoCtx *ctx, int32_t max_layers);
int meao_layer_reservation(const MeaoCtx *ctx);   /* the reserved maximum layer count, 0 = none; MEAO_ERR_INVALID for a NULL context */
typedef struct {
    int32_t width, height;              /* the reservation; 0 x 0 = none */
    int64_t arena_bytes;                /* bytes of the arena (plan-only contexts: what it would allocate) */
    int64_t arena_bytes_needed;         /* bytes the current size's layout needs (<= arena_bytes) */
    int64_t arena_allocations;          /* arenas allocated since meao_create */
    int64_t graphs_held;                /* executable graphs alive, retired ones waiting for their last launch included */
    int64_t graph_instantiations;       /* cudaGraphInstantiate calls since meao_create */
} MeaoReservation;
int meao_reservation(const MeaoCtx *ctx, MeaoReservation *out);
/* Layered frames: every frame holds `layers` independent views of width x height (texture-array stereo: 2 eye slices; cube-map
 * AO: 6 faces; a batch of frames of one camera), rendered by ONE launch per stage.  Each layer's result is bit-identical to
 * rendering that layer alone; one MeaoParams / MeaoCamera / MeaoVariants applies to all layers unless meao_set_layer_cameras gives
 * each layer its own camera.  Layout rule: every image argument
 * holds the L images stacked at a stride of one tight image -- depth is L*width*height elements of the depth kind, the AO output
 * L*width*height bytes -- for meao_render, meao_render_host(_async), meao_bind_event, meao_profile_frame, the meao_stage_* calls,
 * meao_debug_view (L images) and the meao_composite_* calls (L*width*height pixels).  meao_get_buffer / meao_set_buffer use
 * [L][reference layout] (host_bytes = L x the single size; MeaoBufferDesc stays per layer).  meao_kernels_per_frame is unchanged
 * (one layered launch is one kernel); meao_algorithmic_bytes scales by L.
 * A plan input like meao_resize: default 1 (every entry point behaves as without layers); returns 1 if the value changed, 0 if
 * not.  A change re-allocates the intermediates, drops the captured graphs, resets the row band to the whole frame and drops the
 * neighbour connections -- except inside a layer reservation (meao_reserve_layers), where it is host bookkeeping.  layers must be in 1..65535 (the layer is a grid dimension of the layered kernels), else
 * MEAO_ERR_INVALID; MEAO_ERR_NOMEM if the intermediates do not fit (the context keeps its previous layer count).
 * Row bands and layers exclude each other: with layers > 1, meao_set_row_band, the halo calls (meao_halo_*, meao_render_band_*,
 * meao_band_phase_a / _b) and the native exchange (meao_band_export / _connect / _step / _step_host) return MEAO_ERR_UNSUPPORTED.
 * A change of the layer count also CLEARS the per-layer camera table (meao_set_layer_cameras): set it again after every call that
 * returned 1. */
int meao_set_layers(MeaoCtx *ctx, int32_t layers);
/* Per-layer cameras for layered frames (split-screen viewports, mirrors and portals, batches of frames from several cameras): layer
 * l is rendered with cameras[l] -- its near and far planes and field of view -- and is bit-identical to a single-layer meao_render
 * of that layer's depth with meao_set_camera(cameras[l]), for the AO and every debug buffer.  MeaoParams, MeaoVariants and the
 * size stay shared.  count must equal meao_set_layers; cameras == NULL with count == 0 clears the table, and every layer then uses
 * the meao_set_camera camera again.  Each entry is validated like meao_set_camera, and all entries must have the same reversed_z
 * (a platform property).  A refusal returns MEAO_ERR_INVALID, names the layer and field in meao_last_error, and changes nothing.
 * A frame constant like meao_set_camera's planes and field of view: returns 1 if a value changed (the next frame takes the new table
 * without a re-plan), 0 if the same table is set again -- so a host may call it every frame.  A table (or clearing one) that
 * changes the Z direction in effect is a structural change and re-plans.  While a table is set it alone defines every layer's
 * camera; meao_set_camera still records the shared camera, which takes effect when the table is cleared.  A change of the layer
 * count clears the table.  Works on plan-only contexts (device < 0); with layers == 1 a table of one camera behaves exactly like
 * meao_set_camera. */
int meao_set_layer_cameras(MeaoCtx *ctx, const MeaoCamera *cameras, int32_t count);
/* Copies the table into out (capacity entries; MEAO_ERR_INVALID if it does not fit) and returns its entry count (0 = no table). */
int meao_get_layer_cameras(const MeaoCtx *ctx, MeaoCamera *out, int32_t capacity);
/* Per-layer viewports for layered frames: where each layer of the frame lives in the caller's arrays or buffers, so that several views
 * share one render target (2- and 4-player split-screen in one 2-D texture, a side-by-side stereo pair, the six faces of a cube into
 * the cells of one 2-D atlas).  Layer l of a meao_render_arrays frame reads the depth texels [depth_x, depth_x + W) x [depth_y,
 * depth_y + H) of the depth array's layer depth_slice and writes its AO into [ao_x, ao_x + W) x [ao_y, ao_y + H) of the AO array's layer
 * ao_slice, W x H being the context's current size; it is bit-identical to a single-layer meao_render_arrays_at (meao_render_pitched)
 * frame of that rectangle with that layer's camera.  No texel outside the rectangles is read or written.  With meao_set_layer_cameras each view also has its
 * own camera.
 * count must equal meao_set_layers; views == NULL with count == 0 clears the table.  Every coordinate must be >= 0; a refusal
 * returns MEAO_ERR_INVALID, names the layer and field in meao_last_error and leaves the previous table in place.  A change of the
 * layer count clears the table.
 * A frame constant: changing the entries of a set table returns 1 and the next frame takes the new table without a re-plan, a device
 * synchronise or a graph instantiation; setting the same table again returns 0.  Setting a table where there was none, or clearing
 * one, switches kernels: it returns 1 and re-plans like a structural change (inside a layer reservation, meao_reserve_layers, it is a
 * frame constant as well).  meao_frame_generation moves with every change.  A frame
 * whose new table is not written yet is refused inside a caller's capture, like new camera tables.  Works on plan-only contexts.
 * Checked at every frame, against the current W x H (a reserved context may change size under a set table).  CUDA arrays: every
 * rectangle fits its array (x + W <= width, y + H <= height) and every slice is below the array's layer count (1 for a 2-D array, n for a layered one,
 * 6 for a cube map) -- the context's layer count no longer has to equal the arrays'; and no two layers' AO rectangles on one slice
 * share a texel (depth rectangles may overlap: the depth is only read).  That test is linear in the layer count and runs once per
 * (table, size), and not at all at a size no larger in either dimension than one that passed.  A refusal returns MEAO_ERR_INVALID naming the layer and field and launches nothing; so does a bound event.
 * Pointer frames (meao_render_pitched, and meao_render at its tight pitches): slice s of a view starts s x layer pitch bytes in, and
 * the rectangle's rows are the view's rows.  Every row of a rectangle must fit its row pitch ((x + W) x element size <= row pitch);
 * when some slice is > 0, every rectangle must fit inside its slice (and the depth layer pitch be a whole number of elements); the
 * depth and AO views' byte extents, from each base to the end of its last rectangle, must not intersect.  A layer whose
 * rectangle starts misaligned for the vector accesses (16 bytes for the depth, 8 for the AO, with rows of such pitches) takes the
 * element-wise path for its own pixels, with the same result.
 * Which calls honour it: meao_render_arrays, meao_render_pitched, meao_render, and the events that render through them
 * (meao_bind_event_arrays, meao_bind_event_pitched, meao_bind_event).  meao_render_arrays_at (and its event) names one origin for
 * every layer and is refused with MEAO_ERR_INVALID while a table is set.  The host-buffer calls (meao_render_host(_async)), the
 * stage API, meao_profile_frame, meao_debug_view and the composites keep the tight layer layout and ignore the table.  Row bands and
 * tables exclude each other (MEAO_ERR_UNSUPPORTED). */
typedef struct {
    int32_t depth_x, depth_y, depth_slice;  /* layer l reads depth [x, x+W) x [y, y+H) of slice depth_slice */
    int32_t ao_x, ao_y, ao_slice;           /* and writes its AO into [x, x+W) x [y, y+H) of slice ao_slice */
} MeaoLayerViewport;
int meao_set_layer_viewports(MeaoCtx *ctx, const MeaoLayerViewport *views, int32_t count);
/* Copies the table into out (capacity entries; MEAO_ERR_INVALID if it does not fit) and returns its entry count (0 = no table). */
int meao_get_layer_viewports(const MeaoCtx *ctx, MeaoLayerViewport *out, int32_t capacity);

/* ---- the frame ------------------------------------------------------------------------------- */
/* replaces: replay of the "SSAO" command buffer, steps 1-10 of RebuildCommandBuffers (AO.cs:511-531):
 * Downsample1+2, Render x4, Upsample x4.  depth: device pointer, width*height f32, rows contiguous
 * (row pitch = width*4).  ao_out: device pointer, width*height bytes (R8, AO.cs:475).
 * stream: a cudaStream_t, used as given (NULL = the CUDA legacy default stream).  Asynchronous.  Re-plans first after a structural
 * change (LateUpdate, AO.cs:329-350); takes changed frame constants without one. */
int meao_render(MeaoCtx *ctx, const void *depth_dev, int32_t depth_kind, void *ao_out_dev, void *stream);
/* ---- pitched views -----------------------------------------------------------------------------------------------------------
 * meao_render with the depth and the AO as views inside larger allocations, every pitch in BYTES: a cudaMallocPitch / cudaMalloc3D
 * image, a D3D12 / Vulkan buffer shared through external memory (rows keep the API's pitch, e.g. D3D12's 256-byte footprint rows),
 * or the top-left width x height corner of a render target sized for a larger resolution (a sub-rectangle: the same view with a base
 * offset).  Row r of layer l of the depth starts at depth_dev + l*depth_layer_pitch + r*depth_row_pitch, the AO likewise; r counts
 * the rows meao_render reads (the band's rows with a row band, depth_row0 as there).  meao_render IS this call with the tight
 * pitches (width*esize, rows*width*esize, width, rows*width; esize = 4 for RAW_F32 / LINEAR_F32 / RAW_D24S8, 2 for RAW_D16_UNORM).
 * Everything else is meao_render's: whole frames, layered contexts and top / bottom row bands; graphs are captured and replayed per
 * (depth, ao_out, kind, the four pitches); meao_get_buffer / meao_debug_view of the AO (id 17) regenerate the context's own copy;
 * MEAO_FLAG_NO_GRAPH is honoured; the AO is bit-identical to meao_render on a tight copy of the same view.  Bytes outside the views
 * are neither read nor written.  Refused with MEAO_ERR_INVALID (meao_last_error names the field; nothing is launched), besides
 * meao_render's own refusals (NULL pointers, bad kind, interior row band):
 *   - a negative pitch (bottom-up views are not supported), or a row pitch above INT32_MAX;
 *   - depth_row_pitch below width*esize or not a multiple of esize; ao_row_pitch below width; depth_dev not aligned to esize;
 *   - with layers > 1: a layer pitch below (rows - 1)*row pitch + width*esize (width for the AO): the layers would overlap; a depth
 *     layer pitch that is not a multiple of esize.  With one layer the layer pitches are not used;
 *   - depth and AO byte extents (first to last byte of each view) that intersect: the depth is read through the non-coherent cache,
 *     so aliasing is undefined.  The test is conservative -- interleaved views that share no byte are refused as well.
 * Speed: 128-bit depth loads need depth_dev 16-byte aligned and the row (layered: and layer) pitch a multiple of 16 bytes; 64-bit AO
 * stores need ao_out_dev 8-byte aligned and the AO pitches multiples of 8.  Otherwise the affected pixels take the scalar path, with
 * the same result.  Tight-only, unchanged: the stage API, meao_render_band_prepare / _finish, meao_band_phase_a / _b,
 * meao_band_step(_host), the host-buffer calls, meao_profile_frame, the composites and the debug-view outputs. */
int meao_render_pitched(MeaoCtx *ctx,
                        const void *depth_dev, int64_t depth_row_pitch, int64_t depth_layer_pitch, int32_t depth_kind,
                        void *ao_out_dev, int64_t ao_row_pitch, int64_t ao_layer_pitch, void *stream);
/* Same with HOST buffers: H2D copy of depth, the ten passes, D2H copy of the AO texture, then a
 * stream synchronise.  Use meao_host_alloc for pinned memory. */
int meao_render_host(MeaoCtx *ctx, const void *depth_host, int32_t depth_kind, uint8_t *ao_out_host);
/* ---- CUDA arrays -------------------------------------------------------------------------------------------------------------
 * The frame of meao_render with the depth read from, and the AO written into, CUDA arrays -- what graphics interop hands out for a
 * shared texture (D3D11 / D3D12 / GL: cudaGraphicsSubResourceGetMappedArray; Vulkan: cudaExternalMemoryGetMappedMipmappedArray, then
 * level 0 through cudaGetMipmappedArrayLevel).  No copy to or from linear memory: the first and the last kernel of the frame access
 * the arrays through surface objects.  Registering and mapping the resource stays with the host (it is graphics-API specific).
 * depth_array / ao_array: cudaArray_t, passed as void *.  Checked on the host before anything is launched:
 *   - depth_kind RAW_F32 / LINEAR_F32: one 32-bit float channel; RAW_D16_UNORM: one 16-bit unsigned channel (normalised or not);
 *     RAW_D24S8 returns MEAO_ERR_UNSUPPORTED (no CUDA array holds a depth-stencil format).  ao_array: one 8-bit unsigned channel
 *     (normalised or not; the R8 texture of AO.cs:475).
 *   - width x height must be the context's; both arrays need cudaArraySurfaceLoadStore (interop: register the resource with
 *     cudaGraphicsRegisterFlagsSurfaceLoadStore).
 *   - layers: a 2-D array (or a cudaArrayLayered array of depth 1) has 1, a cudaArrayLayered array of depth n has n, a
 *     cudaArrayCubemap array 6 (face f = layer f); each must equal meao_set_layers.  The two arrays may be of different shapes.
 *     Cube-map arrays (cudaArrayCubemap | cudaArrayLayered) return MEAO_ERR_UNSUPPORTED.
 *   - a context with a row band (meao_set_row_band) returns MEAO_ERR_UNSUPPORTED.
 * A refused call returns MEAO_ERR_INVALID / MEAO_ERR_UNSUPPORTED with meao_last_error naming the field, and launches nothing.
 * The result is bit-identical to meao_render on the same depth; graphs are captured and replayed per (depth_array, ao_array, kind)
 * like meao_render's, and meao_get_buffer / meao_debug_view of the AO (id 17) regenerate the context's own copy as after a pointer
 * frame.  meao_kernels_per_frame is unchanged.
 * RELEASE CONTRACT: the context caches a surface object per array and the graphs that use it; both describe the array's MEMORY.
 * Before freeing, unmapping or re-registering an array this context has rendered with (or bound with meao_bind_event_arrays), call
 * meao_release_array(ctx, array): it synchronises the device, drops that array's graphs, surface object and event bindings.  A new
 * array may come back with the same handle, and without the release the next frame would replay into freed memory.
 * meao_destroy and every structural plan change (meao_resize without a reservation, meao_reserve, meao_set_layers, meao_set_variants,
 * a reversed_z change, meao_set_projection, meao_set_row_band) release all arrays; a frame-constant change (MeaoParams, the cameras' planes and fields of
 * view) releases none.  Releasing an array this context never used returns MEAO_OK. */
int meao_render_arrays(MeaoCtx *ctx, const void *depth_array, int32_t depth_kind, void *ao_array, void *stream);
/* Viewports: meao_render_arrays with the frame read from, and written into, a W x H rectangle of larger arrays -- render targets
 * allocated (and registered) once at the largest size of a dynamic-resolution engine, or one player's half of a split-screen texture.
 * The frame reads the context's current W x H (meao_resize, reserved or not) from the depth array's texels [depth_x, depth_x + W) x
 * [depth_y, depth_y + H) and writes the AO into [ao_x, ao_x + W) x [ao_y, ao_y + H) of the AO array, in every layer or cube face.
 * No texel outside the two rectangles is read or written.  The arrays may have different extents and origins (say an exact-size depth
 * copy and a maximum-size AO target).  The checks are meao_render_arrays's, except the exact extent: instead each origin must be >= 0
 * and the viewport must fit, x + W <= width and y + H <= height; a refusal returns MEAO_ERR_INVALID naming the array and the field
 * (depth_x, depth_y, ao_x, ao_y) and launches nothing.  Everything else is meao_render_arrays's contract: layered and cube-map
 * contexts, per-layer cameras, MEAO_FLAG_NO_GRAPH, the release contract, regeneration of id 17, recording into a caller's capture after
 * one frame outside it.  The origins are arguments like the arrays: a graph is cached per (arrays, origins, kind), they do not move
 * meao_frame_generation, and a frame recorded into a caller's graph replays at the origins it was recorded with.
 * meao_render_arrays(ctx, d, kind, a, s) is meao_render_arrays_at(ctx, d, 0, 0, kind, a, 0, 0, s) on arrays of exactly W x H. */
int meao_render_arrays_at(MeaoCtx *ctx, const void *depth_array, int32_t depth_x, int32_t depth_y, int32_t depth_kind,
                          void *ao_array, int32_t ao_x, int32_t ao_y, void *stream);
int meao_release_array(MeaoCtx *ctx, const void *array);
/* ---- Batches: each layer with its own depth and AO --------------------------------------------------------------------------
 * A layered frame (meao_set_layers L) whose layer l reads its own depth and writes its own AO: cameras that each render into their own
 * targets (a Camera's own render textures, separate split-screen targets, one buffer per sensor, a list of tensors) in one frame of 9
 * launches instead of L contexts or a copy into and out of one stacked allocation.  Only the frame's first and last kernel touch the
 * caller's memory; they take the whole list as a kernel parameter.
 *   - Bit-identical per layer: layer l is bit-identical, on the AO and on every debug buffer, to a single-layer frame of that layer's
 *     depth with that layer's camera (meao_set_layer_cameras, or the context's camera for every layer).
 *   - count must equal the layer count, and be at most MEAO_MAX_BATCH.
 *   - Arrays (meao_render_arrays_batch): each entry is a 2-D array, or a cudaArrayLayered array of depth 1, with the formats and the
 *     cudaArraySurfaceLoadStore flag meao_render_arrays requires (RAW_D24S8: MEAO_ERR_UNSUPPORTED).  Each must be AT LEAST W x H; the
 *     frame sits at its top-left corner, so a dynamic-resolution host (meao_reserve) keeps per-camera targets at their maximum size.
 *     No texel outside W x H is read or written.  No two layers may share an AO array; depth arrays may repeat.
 *   - Pointers (meao_render_batch): layer l reads depth[l], rows depth_row_pitch[l] bytes apart, and writes ao[l], rows ao_row_pitch[l]
 *     bytes apart (0 = tight: W x element size, W).  Per layer the checks of meao_render_pitched: pitches at least a row, at most
 *     INT32_MAX, the depth pitch a multiple of the element size, depth[l] aligned to its element.  No two AO byte extents may
 *     intersect, nor an AO extent any depth extent (an extent: first to last byte of a layer's view); depth entries may repeat.  The
 *     check sorts the extents: O(L log L).  Each layer's vector loads and stores depend on its own base and pitch (16 bytes for the
 *     depth, 8 for the AO); a misaligned layer takes the element-wise path for its own pixels only, with the same result.
 *   - Refusals: MEAO_ERR_INVALID with the layer and field named in meao_last_error, and nothing launched, for a count that differs from
 *     the layer count or exceeds MEAO_MAX_BATCH, a NULL list or entry, a shared AO array, intersecting extents, and every per-entry
 *     check above.  A set layer-viewport table (meao_set_layer_viewports) is refused with MEAO_ERR_INVALID; an orthographic projection
 *     and a row band with MEAO_ERR_UNSUPPORTED.
 *   - Everything else is the layered frame's contract: per-layer cameras, the variants, MEAO_FLAG_NO_GRAPH, reservations, live frame
 *     constants, and after a frame the regeneration of id 17 by meao_get_buffer / meao_debug_view.  meao_kernels_per_frame is unchanged.
 *   - Graphs: one per (list, kind, size), the list compared in full; a host that rotates more lists than the cache holds re-targets
 *     the least recently used graph like any other frame.  Capturable into a caller's graph: the list is baked into the recorded frame,
 *     so a list, like an array or an origin, does not move meao_frame_generation.  An array batch is refused inside a capture for an
 *     array this context has not rendered with yet (its surface object is made then).
 *   - Release contract: meao_release_array(a) drops every cached graph and event binding whose list names a. */
#define MEAO_MAX_BATCH 256
/* Layer l of the frame reads depth_arrays[l] and writes ao_arrays[l]; count must equal meao_set_layers. */
int meao_render_arrays_batch(MeaoCtx *ctx, const void *const *depth_arrays, int32_t depth_kind, void *const *ao_arrays, int32_t count,
                             void *stream);
/* Layer l reads depth[l] (row pitch depth_row_pitch[l] bytes, 0 = tight) and writes ao[l] (ao_row_pitch[l], 0 = tight). */
int meao_render_batch(MeaoCtx *ctx, const void *const *depth, const int64_t *depth_row_pitch, int32_t depth_kind, void *const *ao,
                      const int64_t *ao_row_pitch, int32_t count, void *stream);
/* Pipelined form of meao_render_host for frame streams: enqueues H2D + kernels + D2H of one frame on staging slot
 * `slot` (0 or 1) and returns; meao_host_wait(slot) blocks until that frame's AO is in ao_out_host.  Alternating the
 * two slots overlaps the H2D copy of frame i+1 with the kernels and the D2H copy of frame i (the kernels of
 * consecutive frames stay serialised: they share the context's intermediates).  Host buffers must be pinned
 * (meao_host_alloc) for the copies to be asynchronous, and must stay valid until the matching wait. */
int meao_render_host_async(MeaoCtx *ctx, const void *depth_host, int32_t depth_kind, uint8_t *ao_out_host, int32_t slot);
int meao_host_wait(MeaoCtx *ctx, int32_t slot);
int meao_synchronize(MeaoCtx *ctx);
void *meao_host_alloc(size_t bytes);                /* cudaHostAlloc; NULL on failure */
void meao_host_free(void *p);

/* ---- per-stage entry points (stage parity; mirror the three Push*Commands recorders) ----------- */
/* replaces: PushDownsampleCommands (AO.cs:604-658) -> LinearDepth, LowDepth1..4 (+ virtual TiledDepth1..4) */
int meao_stage_downsample(MeaoCtx *ctx, const void *depth_dev, int32_t depth_kind, void *stream);
/* replaces: PushRenderCommands (AO.cs:660-748) for TiledDepth<level> -> Occlusion<level>, level 1..4 */
int meao_stage_render(MeaoCtx *ctx, int32_t level, void *stream);
/* PushRenderCommands (AO.cs:660-748) for a NON-tiled source: LowDepth<level> -> HighQuality<level> with Render.compute kernel
 * "main" (FindKernel would name it instead of "main_interleaved", AO.cs:728; thread-group size 16x16 from AO.cs:739-747). */
int meao_stage_render_wide(MeaoCtx *ctx, int32_t level, void *stream);
/* replaces: PushUpsampleCommands (AO.cs:750-785) with the wiring of AO.cs:528-531; lo_level 4..1.
 * lo_level == 1 writes the final AO into ao_out_dev (or the context's own result buffer if NULL).
 * Uses the main_premin variants for the levels selected in MeaoVariants.high_quality_mask. */
int meao_stage_upsample(MeaoCtx *ctx, int32_t lo_level, void *ao_out_dev, void *stream);

/* ---- buffers (debug views, AO.cs:787-820) ------------------------------------------------------ */
int meao_buffer_desc(const MeaoCtx *ctx, int32_t buffer_id, MeaoBufferDesc *out);
/* Copies buffer <id> to host in the REFERENCE layout (tightly packed rows; tiled = [16][h][w]) and
 * native storage type (f16 bits / f32 / unorm8 codes).  Synchronises the context stream.
 * The TiledDepth views are synthesised from LowDepth<k> exactly as Downsample1/2 would have
 * written them (including the padding texels, SURVEY.md P3). */
int meao_get_buffer(MeaoCtx *ctx, int32_t buffer_id, void *host_out, size_t host_bytes);
/* Test hook: overwrite an intermediate (ids 1-5, 10-21) from host data in the same format. */
int meao_set_buffer(MeaoCtx *ctx, int32_t buffer_id, const void *host_in, size_t host_bytes);
/* replaces: PushDebugBlitCommands (AO.cs:787-820) + the debug composite, Blit.shader pass 3 (:116-134): writes the
 * width x height R8 image that _result holds after the debug blit of buffer <buffer_id> (1..17, the `debug` property
 * AO.cs:60; 18..21 for the HighQuality extension) into out_r8_dev (tight rows).  Non-tiled sources: cmd.Blit(rt, _result),
 * a point-sampled stretch (texel = floor(uv * size) at the pixel centre); TiledDepth1..4: Blit.shader pass 4 "Detile"
 * (:136-156), a 4 x 4 mosaic of the 16 slices; 17: the AO texture itself.  Asynchronous on `stream`. */
int meao_debug_view(MeaoCtx *ctx, int32_t buffer_id, void *out_r8_dev, void *stream);

/* ---- CPU-side constants, exposed so they can be checked against the reference math ------------- */
/* out[0..11] gInvThicknessTable, out[12..23] gSampleWeightTable, out[24..25] gInvSliceDimension,
 * out[26] gRejectFadeoff, out[27] gIntensity            (AO.cs:678-734) */
int meao_render_constants(MeaoCtx *ctx, int32_t level, float out28[28]);
/* same layout for the non-tiled dispatch of meao_stage_render_wide (source = LowDepth<level>, AO.cs:679 applied) */
int meao_render_constants_wide(MeaoCtx *ctx, int32_t level, float out28[28]);
/* out[0..1] InvLowResolution, out[2..3] InvHighResolution, out[4] NoiseFilterStrength, out[5] StepSize,
 * out[6] kBlurTolerance, out[7] kUpsampleTolerance       (AO.cs:760-771) */
int meao_upsample_constants(MeaoCtx *ctx, int32_t lo_level, float out8[8]);
/* out[0..3] ZBufferParams (AO.cs:561-568) */
int meao_zbuffer_params(MeaoCtx *ctx, float out4[4]);
/* The same per layer (0 .. layers-1) of a layered context: its own camera's values under meao_set_layer_cameras, the shared ones
 * without a table.  The getters above return layer 0's.  wide: the layout of meao_render_constants_wide. */
int meao_render_constants_layer(MeaoCtx *ctx, int32_t layer, int32_t level, int32_t wide, float out28[28]);
int meao_zbuffer_params_layer(MeaoCtx *ctx, int32_t layer, float out4[4]);

/* ---- row-band partitioning of one frame over several GPUs (new capability, SURVEY.md 8e) -------- */
/* This context computes output rows [row0, row1) of the width x height frame set by meao_resize
 * (global coordinates everywhere; image-edge semantics only at the true top/bottom).
 * row0/row1 must be multiples of 16 except row1 == height.  prev_row0 / next_row1 give the extent
 * of the bands above and below (-1 = none).  depth passed to render/stage_downsample is then the
 * BAND's rows only (row1-row0 rows), and ao_out receives the band's rows only. */
int meao_set_row_band(MeaoCtx *ctx, int32_t row0, int32_t row1, int32_t prev_row0, int32_t next_row1);
/* Border rows of LowDepth1..4 that a neighbour needs.  side: 0 = towards row 0 (up), 1 = down.
 * meao_halo_bytes: size of the packed message this context SENDS to that side (== what the
 * neighbour's unpack of the opposite side expects). */
int64_t meao_halo_bytes(MeaoCtx *ctx, int32_t side);
int64_t meao_halo_recv_bytes(MeaoCtx *ctx, int32_t side);
/* Row ranges behind those sizes: out8 = {lo1,hi1, lo2,hi2, lo3,hi3, lo4,hi4} rows of LowDepth1..4 that
 * are sent (send != 0) / received (send == 0) on that side; the packed message is those rows, level 1
 * first, each row lw[k] tightly packed f32. */
int meao_halo_rows(MeaoCtx *ctx, int32_t side, int32_t send, int32_t out8[8]);
/* out30 = for k = 0..4: rows of level k to produce [2k,2k+1]; rows of LowDepth<k> read [10+2k..];
 * rows of LowDepth<k> this band owns [20+2k..]. */
int meao_band_rows(MeaoCtx *ctx, int32_t out30[30]);
int meao_halo_pack(MeaoCtx *ctx, int32_t side, void *packed_dev, void *stream);
int meao_halo_unpack(MeaoCtx *ctx, int32_t side, const void *packed_dev, void *stream);
/* Split of meao_render around the exchange: phase A = downsample own rows; (exchange); phase B =
 * render + upsample. */
int meao_render_band_prepare(MeaoCtx *ctx, const void *depth_band_dev, int32_t depth_kind, void *stream);
int meao_render_band_finish(MeaoCtx *ctx, void *ao_band_out_dev, void *stream);

/* The same split with the halo pack / unpack fused in and each half replayed as ONE CUDA graph:
 *   phase A = prepare_depth on the band + pack of both outgoing halos (send_* may be NULL at the frame edge);
 *   phase B = unpack of both incoming halos + Render x4 + Upsample x4.
 * A band step is then: phase A, one neighbour send/recv per side (NCCL or peer copy), phase B. */
int meao_band_phase_a(MeaoCtx *ctx, const void *depth_band_dev, int32_t depth_kind, void *send_up_dev, void *send_down_dev, void *stream);
int meao_band_phase_b(MeaoCtx *ctx, const void *recv_up_dev, const void *recv_down_dev, void *ao_band_out_dev, void *stream);

/* ---- native neighbour exchange (ABI 3): the halo rows travel by PEER STORES over NVLink, inside the frame's one CUDA graph ----
 * Every band context keeps its LowDepth1..4 in full-frame global coordinates, so a band's border rows have the SAME byte offset
 * in every context's arena: the exchange kernel (csrc/band_exchange.cu) writes them straight into the neighbour's LowDepth
 * buffers through a peer mapping -- no pack, no staging, no unpack, no NCCL call -- then raises an epoch flag in the neighbour's
 * memory (st.release.sys) and waits for the neighbour's own flag (ld.acquire.sys).  A step of a connected band is ONE graph
 * launch: prepare_depth -> exchange -> Render x4 + Upsample x4 (DAG), no host code between the phases.
 *   1. meao_resize + meao_set_row_band on every band context (one per GPU; same or different processes)
 *   2. meao_band_export -> an opaque POD handle; move it to the neighbours any way the host likes (memcpy in-process;
 *      torch.distributed / MPI / a pipe between processes -- it contains a cudaIpcMemHandle_t)
 *   3. meao_band_connect(ctx, side, &neighbour_handle) for each existing neighbour (side 0 = up, 1 = down)
 *   4. per frame, on every band in lock step: meao_band_step (asynchronous on `stream`)
 * All bands must run the same number of steps.  A wait that exceeds the time-out (default 2 s, env MEAO_BAND_TIMEOUT_MS)
 * sets a sticky error instead of hanging the GPU: the remaining kernels of that step still run (on stale halo rows),
 * meao_band_status reports it and the next meao_band_step fails with MEAO_ERR_PEER.
 * meao_resize and meao_set_row_band DISCONNECT (the arena / the halo ranges change): export + connect again afterwards.
 * Scheduling contract.  The exchange kernel spins on flags its NEIGHBOUR raises, so the neighbour's kernels must be able to run
 * while it waits.  With one band per GPU that is automatic as long as every host issues the steps of its band contexts in the same
 * order (frame streams over several contexts per GPU are fine: bench.py runs 12).  When NEIGHBOURING bands share one GPU (tests,
 * single-GPU development) every band's streams need their own hardware queue: set CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts
 * and keep to <= 3 bands per GPU -- otherwise a band's kernels (or its first graph instantiation) can end up waiting behind the
 * spinning kernel that waits for them, which the time-out then reports as error 1 / 2 (DESIGN.md section 4). */
#define MEAO_PEER_HANDLE_BYTES 128
typedef struct { unsigned char bytes[MEAO_PEER_HANDLE_BYTES]; } MeaoPeerHandle;
int meao_band_export(MeaoCtx *ctx, MeaoPeerHandle *out);
/* peer == NULL disconnects that side.  Same process: direct pointer (+ cudaDeviceEnablePeerAccess across devices);
 * another process: cudaIpcOpenMemHandle.  Fails with MEAO_ERR_INVALID if the neighbour's frame size differs.
 * The bands' epoch counters run in lock step from 1, so a band that has already stepped can only be reconnected as a whole:
 * disconnect both of its sides (and do the same on every other band of the frame), then connect again -- the first connect of a
 * fully disconnected band restarts its epoch and clears a sticky time-out error. */
int meao_band_connect(MeaoCtx *ctx, int32_t side, const MeaoPeerHandle *peer);
int meao_band_step(MeaoCtx *ctx, const void *depth_band_dev, int32_t depth_kind, void *ao_band_out_dev, void *stream);
/* The same with HOST buffers (the band's rows only): H2D copy, the step, D2H copy, all enqueued on the context's staging slot 0 --
 * asynchronous, because the neighbours' steps must be enqueued too before anyone waits; then meao_host_wait(ctx, 0) on every band.
 * The host buffers MUST be pinned (meao_host_alloc): a pageable copy blocks the calling thread until it has completed, which it
 * cannot before the neighbour -- not yet enqueued by that same thread -- has taken part in the exchange.
 * This is what lets a single-threaded C / C# host drive all GPUs of a box (tests/c_abi/smoke.c "bands"). */
int meao_band_step_host(MeaoCtx *ctx, const void *depth_band_host, int32_t depth_kind, uint8_t *ao_band_out_host);
/* out4 = { epoch of the next exchange (1 + completed exchanges), sticky error (0 ok, 1 = time-out waiting for a neighbour's
 * ack, 2 = time-out waiting for a neighbour's rows), connected-up, connected-down }.  Synchronises nothing: reads the
 * flags with a stream-less copy, so call it after the stream has drained for a definitive answer. */
int meao_band_status(MeaoCtx *ctx, int32_t out4[4]);

/* ---- composite: the consumer end of the pipe (SURVEY.md 8f.1) ------------------------------------------- */
typedef enum {
    MEAO_FMT_RGBA8_UNORM = 0,   /* ARGB32-class LDR target, 4 bytes / pixel */
    MEAO_FMT_RGBA16_FLOAT = 1   /* ARGBHalf HDR target, 8 bytes / pixel */
} MeaoColorFormat;
/* replaces: PushCompositeCommands, frame-buffer branch (AO.cs:835-838) = Blit.shader pass 2 (:84-101),
 * "Blend Zero SrcAlpha" with src = ao.rrrr:   color.rgba *= ao.   ao_dev: width*height R8 codes (tight rows, what
 * meao_render wrote); color_dev: width*height pixels, tight rows, updated in place.  16-byte aligned pointers. */
int meao_composite_framebuffer(MeaoCtx *ctx, const void *ao_dev, void *color_dev, int32_t color_format, void *stream);
/* replaces: PushCompositeCommands, ambient-only deferred branch (AO.cs:830-834) = Blit.shader pass 1 (:66-92),
 * "Blend Zero OneMinusSrcColor, Zero OneMinusSrcAlpha" with src0 = (0,0,0,1-ao), src1 = (1-ao,1-ao,1-ao,0):
 *   gbuffer0.a *= 1-(1-ao)  (RGBA8, occlusion channel),  gbuffer3.rgb *= 1-(1-ao)  (ambient/emission target). */
int meao_composite_gbuffer(MeaoCtx *ctx, const void *ao_dev, void *gbuffer0_rgba8_dev, void *gbuffer3_dev, int32_t gbuffer3_format, void *stream);
/* replaces: PushCompositeCommands, debug branch (AO.cs:826-829) = Blit.shader pass 3 "Debug" (:116-134), no blending:
 *   color.rgba = view.rrrr   where view_r8_dev is the width*height R8 image written by meao_debug_view (or the AO texture). */
int meao_composite_debug(MeaoCtx *ctx, const void *view_r8_dev, void *color_dev, int32_t color_format, void *stream);

/* ---- command-buffer hook (Unity native-plugin style) -------------------------------------------- */
/* replaces: camera.AddCommandBuffer(..., _renderCommand) (AO.cs:412-429): a host engine issues
 * CommandBuffer.IssuePluginEvent(meao_get_render_event_func(), event_id). */
typedef void (*MeaoRenderEventFunc)(int event_id);
/* stream: the cudaStream_t the plugin event renders on (ABI 3; NULL = the CUDA legacy default stream, as before). */
int meao_bind_event(MeaoCtx *ctx, int32_t event_id, const void *depth_dev, int32_t depth_kind, void *ao_out_dev, void *stream);
/* The array twin of meao_bind_event: the event renders meao_render_arrays(ctx, depth_array, depth_kind, ao_array, stream).  The arrays
 * are checked now (the event cannot report an error), with the statuses of meao_render_arrays; both NULL unbinds.  An id holds one
 * binding: binding it again, with either call, replaces it.  meao_release_array also removes the bindings that name the array. */
int meao_bind_event_arrays(MeaoCtx *ctx, int32_t event_id, const void *depth_array, int32_t depth_kind, void *ao_array, void *stream);
/* The viewport twin: the event renders meao_render_arrays_at with these origins.  Checked now at the current size, and again at the
 * size of the frame each time the event runs, so one binding to maximum-size arrays serves every size of a reservation; a viewport that
 * no longer fits launches nothing and leaves the reason in meao_last_error. */
int meao_bind_event_arrays_at(MeaoCtx *ctx, int32_t event_id, const void *depth_array, int32_t depth_x, int32_t depth_y,
                              int32_t depth_kind, void *ao_array, int32_t ao_x, int32_t ao_y, void *stream);
/* The pitched twin of meao_bind_event: the event renders meao_render_pitched with these views.  The views are checked now, with the
 * refusals of meao_render_pitched; both pointers NULL unbinds.  meao_bind_event binds the tight views of the context as it is when the
 * event runs. */
int meao_bind_event_pitched(MeaoCtx *ctx, int32_t event_id,
                            const void *depth_dev, int64_t depth_row_pitch, int64_t depth_layer_pitch, int32_t depth_kind,
                            void *ao_out_dev, int64_t ao_row_pitch, int64_t ao_layer_pitch, void *stream);
/* The plugin-event twin of meao_render_arrays_batch: copies the lists and checks them now (with its refusals, and makes the surface
 * objects, so the event may run inside a capture); both NULL unbinds.  meao_release_array removes the bindings whose lists name the
 * array. */
int meao_bind_event_arrays_batch(MeaoCtx *ctx, int32_t event_id, const void *const *depth_arrays, int32_t depth_kind,
                                 void *const *ao_arrays, int32_t count, void *stream);
void meao_render_event(int event_id);
MeaoRenderEventFunc meao_get_render_event_func(void);

/* ---- frames inside a caller's graph ------------------------------------------------------------------------------------------
 * When the stream an entry point is given is being captured (cudaStreamBeginCapture in any mode, torch.cuda.graph, the graph trees of
 * torch.compile(mode="reduce-overhead"), which reach a frame through the torch.library operator meao::ambient_occlusion of
 * miniengineao_b200/torch_ops.py), the call records its kernel launches straight into that capture: the caller's graph then
 * holds the frame, and every replay of it runs the frame.  No graph of the context is captured, instantiated or launched, and the
 * graph cache is neither used nor changed.  A graph-path frame forks to the context's own streams and joins back inside the caller's
 * capture (cross-stream dependencies of the caller's graph); a MEAO_FLAG_NO_GRAPH frame records its launches serially.  The launches
 * carry programmatic dependent launch at the level an instantiation of this context has accepted (meao_pdl_level; none before the
 * first), so a frame recorded into a caller's graph matches the context's own.  The capture status query is the only cost a frame
 * outside a capture pays for this.
 * Capturable: meao_render, meao_render_pitched, meao_render_arrays(_at), meao_render_arrays_batch, meao_render_batch, meao_render_event
 * (any binding), the meao_stage_* calls,
 * meao_render_band_prepare / _finish, meao_band_phase_a / _b, meao_band_step, meao_halo_pack / _unpack, meao_debug_view and the three
 * meao_composite_* calls.
 * SETTLED CONTEXTS ONLY: inside a capture a call may issue nothing but kernel launches.  It is refused with MEAO_ERR_INVALID, records
 * nothing and leaves the caller's capture valid (meao_last_error says why: "issue one frame outside the capture first") when
 *   - a structural change is pending (a re-plan synchronises the device; meao_set_projection is one),
 *   - the per-layer camera tables are still to be written: after a frame-constant change, or on the first frame at a size,
 *   - a changed layer-viewport table (meao_set_layer_viewports) is still to be written,
 *   - or, for meao_render_arrays(_at) and meao_render_arrays_batch, the context has not rendered with one of the arrays yet (its
 *     surface object is made then).
 * One frame of the same form issued outside the capture settles the context; torch's warm-up before torch.cuda.graph does that.
 * A capture that has been invalidated returns MEAO_ERR_CUDA and records nothing.
 * NOT capturable: the host-buffer calls (meao_render_host, _host_async, meao_host_wait, meao_band_step_host; they run on the
 * context's own streams), meao_get_buffer, meao_set_buffer, meao_release_array, meao_synchronize, meao_band_connect, meao_band_status,
 * meao_profile_frame and every structural setter (they may allocate or synchronise).  meao_profile_frame returns MEAO_ERR_UNSUPPORTED
 * while a capture that holds a graph-path frame of this context is open; the others must not be called while one is.  While such a
 * capture is open, issue this context's frames into that capture only.
 * REPLAY CONTRACT: a recorded frame replays with the plan, size, buffers, arrays and frame constants it was recorded with -- the
 * constants are baked into the caller's graph, as every kernel argument of a CUDA graph is (frame constants are live for frames the
 * context issues itself, not inside a caller's graph).  meao_frame_generation changes whenever anything a recorded frame depends on
 * changes: a frame constant, a switch of size or size slot (meao_resize), a structural re-plan, an arena re-allocation, a
 * meao_release_array that released something, meao_band_connect or meao_set_row_band.  It does not change for a setter that changes
 * nothing, for a refused call, for frames or for replays.  A host may replay a recorded frame only while meao_frame_generation equals
 * the value it read right after recording; otherwise it re-captures (after one frame outside the capture).  Replaying after a
 * re-allocation, a resize without a reservation or a release would read and write freed memory.
 * Counting: meao_launch_count counts a recorded frame's kernels once, when it is recorded (replays of the caller's graph are
 * invisible to the library); MeaoReservation.graph_instantiations does not move.  Works on plan-only contexts. */
int64_t meao_frame_generation(const MeaoCtx *ctx);   /* >= 0; MEAO_ERR_INVALID for NULL */

/* ---- introspection ------------------------------------------------------------------------------ */
int64_t meao_launch_count(const MeaoCtx *ctx);       /* kernels launched (or replayed via graph) so far */
/* Programmatic-dependent-launch level of the captured frame graphs: -1 = nothing captured yet, 0 = plain edges, 1 = PDL on the
 * kernels whose only predecessor is the kernel before them in their stream, 2 = also where a cross-branch event joins.  The runtime
 * decides what it accepts at the first capture; env MEAO_PDL=0|1|2 caps it. */
int meao_pdl_level(const MeaoCtx *ctx);
int meao_kernels_per_frame(const MeaoCtx *ctx);      /* kernel nodes in one frame: 9 + one per bit of high_quality_mask (3 with single_scale);
                                                       at hierarchy depth n, 1 + 2 n + the mask bits <= n (+1 with device cameras,
                                                       +1 with device parameters) */
/* Algorithmic bytes of the reference data-flow (SURVEY.md 8d): stage 0 = whole frame, 1 = Downsample1,
 * 2 = Downsample2, 3 = Render x4, 4 = Upsample x4, 5 = final Upsample (L1->L0) only. */
int64_t meao_algorithmic_bytes(const MeaoCtx *ctx, int32_t stage);
/* Device time (ms) of the individual kernels of the last meao_profile_frame() call, which runs one
 * frame with a cudaEvent pair around every kernel.  names/ms arrays of length >= meao_kernels_per_frame(). */
int meao_profile_frame(MeaoCtx *ctx, const void *depth_dev, int32_t depth_kind, void *ao_out_dev,
                       float *ms_out, const char **names_out, int32_t capacity);
/* Launches per kernel inside meao_profile_frame's event pairs (default 1).  With n > 1 every kernel is launched n times back to back
 * (all of them are idempotent: out of place, inputs untouched) and the reported time is the mean -- the event pair's own overhead and
 * the launch gap are amortised, which is what a roofline figure of ONE kernel wants. */
int meao_set_profile_repeats(MeaoCtx *ctx, int32_t n);

/* Device self test: compares the guarded fast division / reciprocal the kernels use (MUFU.RCP + FMA
 * refinement, csrc/common.cuh) with the IEEE operators on n random operand pairs; *mismatches must be 0. */
int meao_selftest_div(MeaoCtx *ctx, uint64_t n, uint32_t seed, uint64_t *mismatches);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MEAO_H */
