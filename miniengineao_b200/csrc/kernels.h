// kernels.h -- argument blocks and host-side launchers of the three libmeao pipeline stages.
//
// All intermediate buffers live in HBM in NATURAL (row-major, non-deinterleaved) layout with
// global frame coordinates; rows are pitched to 128 bytes.  The four 16-slice TiledDepth atlases
// of the reference (Downsample1.compute:71,78, Downsample2.compute:41,49) are never materialised:
// the render kernel reads LowDepth<k> and applies the f16 rounding, the slice-space clamp and the
// atlas padding values itself (see render_ao.cu).
#pragma once

#ifdef MEAO_EMULATE              // tests/emu only (see common.cuh)
#include "cuda_emu.h"
#include "cuda_emu_surface.h"     // cudaSurfaceObject_t and the surface calls of the CUDA-array kernels
#else
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#endif
#include <stdint.h>

// Kernel launch.  `k` is the kernel name IN PARENTHESES (they protect the commas of template arguments from the
// preprocessor).  CUDA build: cudaLaunchKernelEx, with the programmatic-dependent-launch attribute when the recorder asked
// for it (meao::g_launch_pdl, set by meao_api.cu around the launches whose predecessor IN THE SAME STREAM is one of our
// kernels): the dependent grid may then be scheduled while its predecessor drains, runs its prologue and blocks in
// pdl_wait() (griddepcontrol.wait) until the predecessor has completed and flushed -- see common.cuh.  Emulated build: the kernel's
// address is reported to the runtime before the launch, for its ledger of the kernels launched (tests/emu/emu_runtime.cpp).  The hook
// is weak, so an emulator runtime without a ledger still links and launches as before.
#define MEAO_UNPAREN(...) __VA_ARGS__
#ifdef MEAO_EMULATE
namespace meao_emu { __attribute__((weak)) void note_launch(const void *kernel); }
#define MEAO_LAUNCH(k, grid, block, smem, stream, ...) \
    ((meao_emu::note_launch ? meao_emu::note_launch(reinterpret_cast<const void *>(MEAO_UNPAREN k)) : (void)0), \
     meao_emu::launch((grid), (block), (smem), [&]() { MEAO_UNPAREN k(__VA_ARGS__); }))
#else
namespace meao {
inline thread_local bool g_launch_pdl = false;
template <class... KArgs, class... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args &&...args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = g_launch_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
}  // namespace meao
#define MEAO_LAUNCH(k, grid, block, smem, stream, ...) (void)meao::launch_ex(MEAO_UNPAREN k, (grid), (block), (smem), (stream), __VA_ARGS__)
#endif

// Kernel tables.  Every translation unit holds its __global__ instantiations in one static table of typed function pointers
// (kKernels), laid out by the slot functions below; its launchers check their arguments, size the grid and launch
// kKernels[...][slot].  The MEAO_*_SLOTS macros list one kernel template's instantiations in slot order, so each order is written
// once, next to its slot function.  A slot a unit's form does not have holds nullptr: the macros' second argument is MEAO_SLOT, or
// MEAO_NO_SLOT for the slots named in the macro's comment.
#define MEAO_SLOT(...) __VA_ARGS__
#define MEAO_NO_SLOT(...) nullptr

namespace meao {

template <class... P> using Kernel = void (*)(P...);

// ---- stage 1: prepare_depth = Downsample1.compute + Downsample2.compute fused ----------------
struct PrepareArgs {
    const void *depth;      // input rows [depth_row0, ...) of the frame, row pitch = depth_pitch elements (f32 / u16 / u32)
    int in_format;          // 0 = f32, 1 = D16_UNORM codes (u16), 2 = D24_UNORM_S8_UINT words (u32, depth in the low 24 bits)
    int W, H;               // full-frame size
    int depth_row0;         // global row of depth[0]
    int row0, row1;         // global L0 rows to process; row0 % 16 == 0
    __half *lin;            // LinearDepth, L0, f16
    int lin_pitch;          // elements
    float *low[4];          // LowDepth1..4, f32
    int low_pitch[4];       // elements
    float zbx, zby;         // ZBufferParams.xy (AmbientOcclusion.cs:561-568)
    int raw;                // 1: Linearize (DS1:37-48); 0: depth is already linear
    int reversed_z;         // UNITY_REVERSED_Z (DS1:41-45)
    int vec_ok;             // depth pointer 16B aligned and rows (layered: and layers) stay 16B aligned: the depth_pitch (and
                            //    depth_layer_pitch) bytes are multiples of 16 -- for a tight frame W % 4 == 0 (f32/u32), W % 8 == 0 (u16)
    // appended last so that every field above keeps its parameter offset.  0 means tight (resolved by the launchers, so zero-filled
    // argument blocks keep their meaning): depth_pitch = W, depth_layer_pitch = depth_pitch x H.
    int depth_pitch;        // elements from one depth row to the next
    long long depth_layer_pitch;    // layered: elements from one layer of `depth` to the next
};
// `a` with its zero pitches replaced by the tight values (what the prepare launchers pass to the kernels)
inline PrepareArgs resolve_pitches(PrepareArgs a)
{
    if (!a.depth_pitch) a.depth_pitch = a.W;
    if (!a.depth_layer_pitch) a.depth_layer_pitch = (long long)a.depth_pitch * a.H;
    return a;
}
// Raw depth format slot: 0 f32 (also any other code), 1 D16, 2 D24S8 -- PrepareArgs.in_format's codes, the IN_* of depth_in.cuh
constexpr int kDepthFormatSlots = 3;
inline int depth_format_slot(int in_format) { return in_format == 1 || in_format == 2 ? in_format : 0; }
// prepare_depth<RAW, REVERSED, IN>: linear input (read as f32), then raw f32 / D16 / D24S8, reversed Z first.  D24S8: the last two.
constexpr int kPrepareSlots = 7;
inline int prepare_slot(const PrepareArgs &a) { return a.raw ? 1 + 2 * depth_format_slot(a.in_format) + (a.reversed_z ? 0 : 1) : 0; }
#define MEAO_PREPARE_SLOTS(K, D24S8) {K<false, true, IN_F32>, K<true, true, IN_F32>, K<true, false, IN_F32>, K<true, true, IN_D16>, \
                                      K<true, false, IN_D16>, D24S8(K<true, true, IN_D24S8>), D24S8(K<true, false, IN_D24S8>)}
// low_only: write LowDepth1..4 only, loading the even rows alone (a.lin is not written); the frame's final upsample then
// linearises its own pixels and writes LinearDepth (launch_blur_upsample_lin)
cudaError_t launch_prepare_depth(const PrepareArgs &a, cudaStream_t s, bool low_only = false);

// ---- stage 2: render_ao = Render.compute main_interleaved, one mip level -----------------------
struct RenderArgs {
    const float *low;       // LowDepth<k>
    int lw, lh, lpitch;     // size of level k, pitch in elements
    uint8_t *occ;           // Occlusion<k>, unorm8
    int opitch;
    int sw, sh;             // size of the (virtual) TiledDepth<k> slice = level k+2
    float pad;              // value of atlas padding texels (already f16-rounded): Linearize(0) for k=1,2; 0 for k=3,4
    float inv_thickness[12];// gInvThicknessTable entries in CALL order: 7 used by Render.compute:162-168 (checker), 12 by :148-159 (exhaustive)
    float neg_front[12];    // -(invThickness - 0.5)  (Render.compute:85)
    float weight[12];       // gSampleWeightTable entries, same order
    float reject_fadeoff;   // gRejectFadeoff
    float intensity;        // gIntensity
    int row0, row1;         // output rows (level k) to produce
    int wide;               // 0: kernel main_interleaved (virtual f16 atlas of level k+2); 1: kernel main (WIDE_SAMPLING on f32 LowDepth<k>;
                            //    sw/sh/pad unused, low_map must carry the kRenderWideBox box)
    int exhaustive;         // SAMPLE_EXHAUSTIVELY (Render.compute:144-159)
    int tile_h;             // output rows per CTA, one of kRenderTileHs (32: big levels; 16 / 8: coarse levels -- 2x / 4x the CTAs and a half / a
                            //    quarter of the per-CTA latency: the coarse renders are latency-bound); low_map must carry the matching box
};
cudaError_t launch_render_ao(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, cudaStream_t s);
constexpr int kRenderTileVariants = 3;
constexpr int kRenderTileHs[kRenderTileVariants] = {32, 16, 8};
constexpr int kRenderBoxW = 96, kRenderWideBoxW = 80;               // TMA box widths of the render kernel (f32 elements): 64 + 2 x apron (16 / wide: 8)
constexpr int render_box_h(int tile_h, bool wide) { return tile_h + (wide ? 16 : 32); }
constexpr size_t render_smem_bytes(int tile_h, bool wide) { return (size_t)(wide ? kRenderWideBoxW : kRenderBoxW) * render_box_h(tile_h, wide) * sizeof(float); }
// render_ao<MODE, EXH, TH>: wide, then exhaustive, then the tile variant (kRenderTileHs); -1: a tile height without a kernel
constexpr int kRenderSlots = 4 * kRenderTileVariants;
inline int render_slot(const RenderArgs &a)
{
    for (int t = 0; t < kRenderTileVariants; t++)
        if (a.tile_h == kRenderTileHs[t]) return ((a.wide ? 2 : 0) + (a.exhaustive ? 1 : 0)) * kRenderTileVariants + t;
    return -1;
}
#define MEAO_RENDER_SLOTS(K) {K<0, false, 32>, K<0, false, 16>, K<0, false, 8>, K<0, true, 32>, K<0, true, 16>, K<0, true, 8>, \
                              K<1, false, 32>, K<1, false, 16>, K<1, false, 8>, K<1, true, 32>, K<1, true, 16>, K<1, true, 8>}
static_assert(kRenderTileHs[0] == 32 && kRenderTileHs[1] == 16 && kRenderTileHs[2] == 8, "MEAO_RENDER_SLOTS lists the tile heights");

// ---- stage 3: blur_upsample = Upsample.compute main / main_blendout, one level ----------------
struct UpsampleArgs {
    const float *lo_depth;  // LoResDB  (LowDepth<lo>)
    int low, loh, lo_dpitch;
    const uint8_t *lo_ao;   // LoResAO1 (Occlusion4 or Combined<lo>)
    int lo_apitch;
    const void *hi_depth;   // HiResDB  (LowDepth<hi> f32, or LinearDepth f16 when hi == 0)
    int hi_is_half;
    int hi_dpitch;
    const uint8_t *hi_ao;   // HiResAO (Occlusion<hi>) or nullptr => kernel "main" (Upsample.compute:223)
    int hi_apitch;
    uint8_t *out;           // AoResult
    int out_pitch;
    int out_row_origin;     // global row stored at out[0]
    int out_vec_ok;         // out is 8B aligned and out_pitch % 8 == 0
    int hiw, hih;
    float noise_filter_strength, step_size, blur_tolerance, upsample_tolerance;
    int fast_div_ok;        // upsample_fast_div_ok(upsample_tolerance, noise_filter_strength); 0: every pixel takes the IEEE path
    int row0, row1;         // output rows (hi level) to produce
    uint32_t *tile_ctr;     // [0] next tile, [1] CTAs that have run out of tiles: device words owned by (context, level), zero between launches
    int tiles_x, tiles_y;   // tile grid (filled by launch_blur_upsample)
};
// The tolerances for which the upsample's fast divisions are proven exact: 2^-55 <= tol < 2^60 and 2^-52 <= nfs < 2^58.
// Within them the final division needs no per-pixel range test (the proof is at bilateral2 in blur_upsample_device.inc).
inline bool upsample_fast_div_ok(float tol, float nfs)
{
    return tol >= 2.7755575615628914e-17f && tol < 1152921504606846976.0f && nfs >= 2.220446049250313e-16f && nfs < 288230376151711744.0f;
}
// main_premin / main_premin_blendout (COMBINE_LOWER_RESOLUTIONS): the same arguments plus LoResAO2 = HighQuality<lo>
struct UpsamplePreminArgs { UpsampleArgs base; const uint8_t *lo_ao2; int lo_a2pitch; };
// blur_upsample<BLEND, HI_HALF>: blend (a hi-res AO, kernel main_blendout), then hi-half (the hi-res depth is LinearDepth, f16).  The
// premin kernels take other parameters: a unit lists them apart, in the same order.  upsample_args blends exactly when the hi level is
// not L0, so only two slots have a kernel: the final level's {0, 1} and the coarse levels' {1, 0}.  MEAO_NO_SLOT: the coarse levels'.
constexpr int kUpsampleSlots = 4;
inline int upsample_slot(const UpsampleArgs &a) { return (a.hi_ao ? 2 : 0) + (a.hi_is_half ? 1 : 0); }
#define MEAO_UPSAMPLE_SLOTS(K, BLEND) {nullptr, K<false, true>, BLEND(K<true, false>), nullptr}
// lo_ao2 == nullptr: kernels main / main_blendout; otherwise the premin kernels (lo_ao2_map = its TMA descriptor).
// sm_count: SMs of the device (sizes the one-wave grid of the persistent tile loop)
cudaError_t launch_blur_upsample(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                 const UpsampleArgs &a, const uint8_t *lo_ao2, int lo_a2pitch, int sm_count, cudaStream_t s);
constexpr int kUpsDepthBoxW = 40, kUpsDepthBoxH = 22; // TMA boxes of the upsample kernel
constexpr int kUpsAoBoxW = 64, kUpsAoBoxH = 22;

// The final upsample of a whole frame (L1 -> L0), reading the caller's raw depth instead of LinearDepth: each thread loads the
// raw depth of its own eight pixels, linearises them with prepare_depth's arithmetic (depth_in.cuh), stores the f16 values to
// LinearDepth (a.hi_depth, which must be the LinearDepth arena buffer) and upsamples with them -- so LinearDepth is still produced
// every frame, and prepare_depth runs low_only.  A kernel parameter of its own: UpsampleArgs stays as it is (see
// blur_upsample_kernel.inc).  layers > 1: the layered kernels (depth: L images depth_layer_pitch elements apart, AO: L images
// ao_layer_pitch bytes apart; the AO row pitch is UpsampleArgs.out_pitch).
struct DepthIn {
    const void *depth;      // rows [depth_row0, ...) of the frame, row pitch = depth_pitch elements (PrepareArgs.depth)
    int in_format;          // PrepareArgs.in_format
    int depth_row0;         // global row of depth[0]
    float zbx, zby;         // ZBufferParams.xy
    int raw, reversed_z;    // as PrepareArgs
    int vec_ok;             // as PrepareArgs
    // appended last; 0 means tight (resolved by launch_blur_upsample_lin): hiw, depth_pitch x hih, hih x out_pitch
    int depth_pitch;        // elements from one depth row to the next
    long long depth_layer_pitch;    // layered: elements from one depth layer to the next
    long long ao_layer_pitch;       // layered: bytes from one layer of UpsampleArgs.out to the next
    // appended last: the layered kernels' per-layer ZBufferParams (LayerZ table below); nullptr: zbx / zby for every layer
    const struct LayerZ *layer_zb;
};
cudaError_t launch_blur_upsample_lin(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                     const UpsampleArgs &a, const uint8_t *lo_ao2, int lo_a2pitch, const DepthIn &din, int layers, int sm_count,
                                     cudaStream_t s);
// blur_upsample_lin<IN>: depth_format_slot(DepthIn.in_format).  The plain / premin and single-image / layered kernels take other
// parameters: the unit lists each apart, in this order.
#define MEAO_LIN_SLOTS(K) {K<IN_F32>, K<IN_D16>, K<IN_D24S8>}

// ---- layered frames (meao_set_layers): L same-size views through one launch per stage ------------------------------------
// Every image is L images of the same pitch stored back to back ([L][h][pitch]), so layer l of an image starts l x rows x pitch
// elements after layer 0; the caller's depth and AO advance by their own layer pitches (PrepareArgs / DepthIn).  The arguments are the single-image ones (row0 = 0,
// row1 = the level's height, out_row_origin = 0) describing layer 0; the TMA maps span all layers (height L x h), and the kernels
// fetch a box only when it lies inside one layer.  Separate kernels and translation units (*_layered.cu), so the single-image
// kernels keep their code.  kMaxLayers: the prepare_depth / render_ao grids carry the layer in gridDim.z (at most 65535).
constexpr int kMaxLayers = 65535;

// Per-layer cameras (meao_set_layer_cameras): the camera-dependent constants of every layer, in tables in the context's arena (any
// layer count up to kMaxLayers, so neither kernel parameters nor __constant__ memory).  The plan fills every entry alike when the
// layers share one camera; the layered and array kernels read entry blockIdx.z (the fused upsample: its tile's layer).
struct LayerZ { float zbx, zby; };              // ZBufferParams.xy of one layer
struct LayerRender {                            // the camera-dependent RenderArgs fields of one layer at one render launch (level, wide)
    float2 it_nf[12];                           // {inv_thickness[i], neg_front[i]} in CALL order (RenderArgs): one 8-byte read per sample group
    float pad;                                  // raw ingest's atlas padding value of the level, f16-rounded (RenderArgs.pad)
    float pad_[7];                              // to 128 bytes
};
static_assert(sizeof(LayerRender) == 128, "LayerRender is one 128-byte line");
// layer_zb / layer_cam: the per-layer camera tables below, entry l = layer l (nullptr: the argument block's constants for every layer);
// layer_pad: 1 = the entries' pad (raw ingest), 0 = RenderArgs.pad (linear ingest pads with 0)
cudaError_t launch_prepare_depth_layered(const PrepareArgs &a, int layers, cudaStream_t s, bool low_only = false, const struct LayerZ *layer_zb = nullptr);
cudaError_t launch_render_ao_layered(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, int layers, cudaStream_t s,
                                     const struct LayerRender *layer_cam = nullptr, int layer_pad = 0);
cudaError_t launch_blur_upsample_layered(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                         const UpsampleArgs &a, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count, cudaStream_t s);

// ---- CUDA arrays (meao_render_arrays): the depth read from, the AO written into a 2-D / layered / cube-map array --------------------
// The first and the last kernel of the frame in a form that reaches the array through a surface object (surface_io.cuh: kSurf2D /
// kSurfLayered / kSurfCube); the arguments are the layered ones (layers >= 1, whole frame), the intermediates stay in the arena and the
// other kernels are the existing ones.  prepare: in_format f32 or D16 (no CUDA array holds D24S8); upsample: the final level only
// (hi_depth = LinearDepth, no hi_ao; a.out is unused).  Separate kernels and translation units (*_array.cu).
enum { kSurf2D = 0, kSurfLayered = 1, kSurfCube = 2 };    // how a surface's layer coordinate is addressed (the array's shape)
cudaError_t launch_prepare_depth_array(const PrepareArgs &a, cudaSurfaceObject_t depth, int surf_kind, int layers, cudaStream_t s,
                                       const struct LayerZ *layer_zb = nullptr);
cudaError_t launch_blur_upsample_array(const CUtensorMap &lo_depth_map, const CUtensorMap &lo_ao_map, const CUtensorMap *lo_ao2_map, bool use_tma,
                                       const UpsampleArgs &a, const uint8_t *lo_ao2, int lo_a2pitch, int layers, int sm_count,
                                       cudaSurfaceObject_t out, int surf_kind, cudaStream_t s);

// ---- debug: synthesise a TiledDepth<k> view (reference layout [16][sh][sw], f16 bits) ----------
cudaError_t launch_synth_tiled(const float *low, int lw, int lh, int lpitch, int sw, int sh, float pad,
                               __half *out, cudaStream_t s);

// ---- debug views (PushDebugBlitCommands AO.cs:787-820, Blit.shader pass 4): buffer -> W x H R8 image ----------
struct DebugViewArgs {
    const void *src;        // non-tiled: the buffer itself; tiled: LowDepth<k> (the atlas is virtual)
    int elem;               // bytes per source element: 1 unorm8, 2 f16, 4 f32
    int sw, sh;             // source texture size (tiled: size of one slice)
    int spitch;             // source pitch in elements
    int tiled;              // 1: TiledDepth<k> view synthesised from LowDepth<k>
    int lw, lh;             // tiled: size of level k
    float pad;              // tiled: value of the atlas padding texels (f16-rounded)
    uint8_t *out;           // W x H R8 codes
    int out_pitch;
    int W, H;
};
cudaError_t launch_debug_view(const DebugViewArgs &a, cudaStream_t s);
// Blit.shader pass 3 (AO.cs:826-829): colour target (RGBA8 / RGBA16F, tight) = (r, r, r, r) of the R8 view
cudaError_t launch_debug_composite(const uint8_t *view, void *color, long long npix, int half, cudaStream_t s);

// ---- composite (Blit.shader passes 1 and 2): colour *= ao, 4 pixels per thread ------------------------
cudaError_t launch_composite(const uint8_t *ao, void *color, long long npix, int half, int rgb, int alpha, int one_minus, cudaStream_t s);

// ---- self test: div_fast / rcp_fast vs the IEEE operators on n random in-range operand pairs ------
cudaError_t launch_selftest_div(uint64_t n, uint32_t seed, unsigned long long *mismatch_dev, int sm_count, cudaStream_t s);

// ---- native neighbour exchange (include/meao.h "native neighbour exchange"): peer stores + epoch flags, one launch ------
// Flags live in every band context's arena (zeroed at allocation).  ready / ack are written by the NEIGHBOURS through
// their peer mapping; epoch / done / error are local.
struct BandFlags {
    uint32_t ready[2];      // [side]: epoch of the halo rows the neighbour on `side` has delivered into this arena
    uint32_t ack[2];        // [side]: epoch the neighbour on `side` is about to RECEIVE, i.e. everything it read before is consumed
    uint32_t epoch;         // epoch of this context's next exchange (first = 1)
    uint32_t done;          // CTA completion counter of the running exchange kernel
    uint32_t error;         // sticky: 0 ok, 1 timed out waiting for an ack, 2 timed out waiting for rows
    uint32_t pad_;
};
struct XchgSeg { const uint4 *src; uint4 *dst; uint32_t n16; int32_t side; };     // one flat 16-byte-granular copy into the neighbour on `side`
struct XchgArgs {
    XchgSeg seg[8];         // LowDepth1..4 border rows x 2 sides (whole pitched rows: contiguous, 128-byte aligned)
    int nseg;
    BandFlags *local;
    BandFlags *peer[2];     // neighbour's flags through the peer mapping; nullptr = no neighbour on that side
    uint32_t *host_error;   // mapped host word mirroring local->error (may be nullptr)
    unsigned long long timeout_ns;
};
cudaError_t launch_band_exchange(const XchgArgs &a, cudaStream_t s);

// ---- eager loading ------------------------------------------------------------------------------------------------------
// CUDA loads kernels lazily, on first launch, and that load can wait for kernels already RUNNING on the device.  A band's exchange
// kernel spins until its neighbour has run -- if the neighbour's first launch then has to load a kernel on the same device, the two
// wait for each other until the exchange times out (seen when the band tests ran first in a fresh process).  meao_create therefore
// touches every kernel of the library once per device (cudaFuncGetAttributes forces the load), walking every unit's kernel table.
// A kernel that is launched is in its unit's table (the launchers take it from there), so it is loaded too; the test suite checks
// that each table holds every kernel its unit compiles to.
struct KernelUnit {
    const char *file;                       // the translation unit (build.py SOURCES)
    int (*walk)(cudaError_t *load);         // walk_kernels over the unit's table: its kernel count; load != nullptr: loads them too
};
// The number of kernels in a (nested) table, nullptr slots skipped.  load != nullptr: loads each one while *load is cudaSuccess and
// keeps the first error there.
template <class... P> inline int walk_kernels(cudaError_t *load, Kernel<P...> k)
{
    if (!k) return 0;
#ifndef MEAO_EMULATE
    cudaFuncAttributes at;
    if (load && *load == cudaSuccess) *load = cudaFuncGetAttributes(&at, (const void *)k);
#endif
    return 1;
}
template <class T, size_t N> inline int walk_kernels(cudaError_t *load, const T (&t)[N])
{
    int n = 0;
    for (const T &e : t) n += walk_kernels(load, e);
    return n;
}
template <class T, class U, class... R> inline int walk_kernels(cudaError_t *load, const T &t, const U &u, const R &...r)
{
    return walk_kernels(load, t) + walk_kernels(load, u, r...);
}
// Every kernel unit, in build.py SOURCES order.  The CPU emulator builds all but the GPU self test.
extern const KernelUnit kPrepareDepthUnit, kRenderAoUnit, kBlurUpsampleUnit, kSelftestUnit, kHaloUnit, kBandExchangeUnit, kCompositeUnit,
    kDebugViewUnit, kPrepareDepthLayeredUnit, kRenderAoLayeredUnit, kBlurUpsampleLayeredUnit, kPrepareDepthArrayUnit, kBlurUpsampleArrayUnit,
    kBlurUpsampleLinUnit;
inline const KernelUnit *const kKernelUnits[] = {
    &kPrepareDepthUnit, &kRenderAoUnit, &kBlurUpsampleUnit,
#ifndef MEAO_EMULATE
    &kSelftestUnit,
#endif
    &kHaloUnit, &kBandExchangeUnit, &kCompositeUnit, &kDebugViewUnit, &kPrepareDepthLayeredUnit, &kRenderAoLayeredUnit,
    &kBlurUpsampleLayeredUnit, &kPrepareDepthArrayUnit, &kBlurUpsampleArrayUnit, &kBlurUpsampleLinUnit};

// ---- halo pack / unpack: row blocks of pitched buffers <-> contiguous staging, one launch ------
struct HaloSeg { const float *src; float *dst; int src_pitch, dst_pitch, width, rows; };
struct HaloArgs { HaloSeg seg[8]; int nseg; };
cudaError_t launch_halo_copy(const HaloArgs &a, cudaStream_t s);

}  // namespace meao
