// prepare_depth_array_mixed.cu -- prepare_depth_array_ortho.cu's kernels for a frame whose layers mix both projections
// (meao_set_layer_projections): prepare_depth_kernel.inc with MEAO_ARRAY 1 and MEAO_ORTHO 2, so each CTA reads its layer's bit of the
// LayerProjections parameter once and linearises with depth_in.cuh's perspective or affine linearize8.  Linear ingest stays with
// prepare_depth_array.cu's kernel.  A translation unit of its own (build.py MIXED_SOURCES).
#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_ORTHO 2
#define MEAO_LAYERED 1
#define MEAO_ARRAY 1
#define MEAO_PREP_ARRAY_MINB 5      // prepare_depth_array_ortho.cu's bound: its affine linearisation alone needs more than 40 registers
#define prepare_depth_array_kernel prepare_depth_array_mixed_kernel
#include "prepare_depth_kernel.inc"
#undef prepare_depth_array_kernel
#undef MEAO_ARRAY
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [prepare_slot]; slot 0 (linear ingest) is prepare_depth_array.cu's, and no CUDA array holds D24S8
const Kernel<PrepareArgs, cudaSurfaceObject_t, int, int, int, const LayerZ *, LayerProjections> kKernels[kPrepareSlots] =
    MEAO_PREPARE_SLOTS_RAW(prepare_depth_array_mixed_kernel, MEAO_NO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_array_mixed(const PrepareArgs &a_in, cudaSurfaceObject_t depth, int surf_kind, int depth_x, int depth_y,
                                             int layers, cudaStream_t s, const LayerZ *layer_zb, const LayerProjections &proj)
{
    if (!a_in.raw) return launch_prepare_depth_array(a_in, depth, surf_kind, depth_x, depth_y, layers, s, layer_zb);
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || !layer_zb || a_in.in_format == IN_D24S8 || depth_x < 0 || depth_y < 0) return cudaErrorInvalidValue;
    PrepareArgs a = a_in;
    a.depth = nullptr;
    a.vec_ok = 1;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, depth, surf_kind, depth_x, depth_y, layer_zb, proj);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthArrayMixedUnit = {"prepare_depth_array_mixed.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
