// prepare_depth_ortho_layered.cu -- prepare_depth_layered.cu's kernels for raw depth under an orthographic projection
// (meao_set_projection): prepare_depth_kernel.inc with MEAO_LAYERED 1 and MEAO_ORTHO 1 (depth_in.cuh's affine linearize8).  Linear
// ingest stays with prepare_depth_layered.cu's kernels.  A translation unit of its own (build.py ORTHO_SOURCES).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 1
#define MEAO_LAYERED 1
#define prepare_depth_layered_kernel prepare_depth_ortho_layered_kernel
#define prepare_depth_low_layered_kernel prepare_depth_low_ortho_layered_kernel
#include "prepare_depth_kernel.inc"
#undef prepare_depth_low_layered_kernel
#undef prepare_depth_layered_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [low_only][prepare_slot]; slot 0 (linear ingest) is prepare_depth_layered.cu's
const Kernel<PrepareArgs, const LayerZ *> kKernels[2][kPrepareSlots] = {MEAO_PREPARE_SLOTS_RAW(prepare_depth_ortho_layered_kernel, MEAO_SLOT),
                                                                        MEAO_PREPARE_SLOTS_RAW(prepare_depth_low_ortho_layered_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_prepare_depth_ortho_layered(const PrepareArgs &a_in, int layers, cudaStream_t s, bool low_only, const LayerZ *layer_zb)
{
    if (!a_in.raw) return launch_prepare_depth_layered(a_in, layers, s, low_only, layer_zb);
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[low_only][prepare_slot(a)]), grid, kPrepThreads, 0, s, a, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthOrthoLayeredUnit = {"prepare_depth_ortho_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
