// prepare_depth_mixed_layered.cu -- prepare_depth_ortho_layered.cu's kernels for a layered frame whose layers mix both projections
// (meao_set_layer_projections): prepare_depth_kernel.inc with MEAO_LAYERED 1 and MEAO_ORTHO 2, so each CTA reads its layer's bit of the
// LayerProjections parameter once and linearises with depth_in.cuh's perspective or affine linearize8.  Linear ingest stays with
// prepare_depth_layered.cu's kernels.  A translation unit of its own (build.py MIXED_SOURCES).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 2
#define MEAO_LAYERED 1
#define prepare_depth_layered_kernel prepare_depth_mixed_layered_kernel
#define prepare_depth_low_layered_kernel prepare_depth_low_mixed_layered_kernel
#include "prepare_depth_kernel.inc"
#undef prepare_depth_low_layered_kernel
#undef prepare_depth_layered_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [low_only][prepare_slot]; slot 0 (linear ingest) is prepare_depth_layered.cu's
const Kernel<PrepareArgs, const LayerZ *, LayerProjections> kKernels[2][kPrepareSlots] = {
    MEAO_PREPARE_SLOTS_RAW(prepare_depth_mixed_layered_kernel, MEAO_SLOT), MEAO_PREPARE_SLOTS_RAW(prepare_depth_low_mixed_layered_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_prepare_depth_mixed_layered(const PrepareArgs &a_in, int layers, cudaStream_t s, bool low_only, const LayerZ *layer_zb,
                                               const LayerProjections &proj)
{
    if (!a_in.raw) return launch_prepare_depth_layered(a_in, layers, s, low_only, layer_zb);
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    if (layers < 1 || layers > kMaxLayers || !layer_zb) return cudaErrorInvalidValue;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[low_only][prepare_slot(a)]), grid, kPrepThreads, 0, s, a, layer_zb, proj);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthMixedLayeredUnit = {"prepare_depth_mixed_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
