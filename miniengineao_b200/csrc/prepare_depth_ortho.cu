// prepare_depth_ortho.cu -- prepare_depth.cu's kernels for raw depth under an orthographic projection (meao_set_projection): the same
// body (prepare_depth_kernel.inc) with MEAO_ORTHO 1, whose linearize8 (depth_in.cuh) is the affine one.  Linear ingest does not depend
// on the projection and stays with prepare_depth.cu's kernels.  A translation unit of its own (build.py ORTHO_SOURCES) so that the
// perspective kernels compile to exactly the code they did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 1
#define MEAO_LAYERED 0
#define prepare_depth_kernel prepare_depth_ortho_kernel             // the names of the orthographic instantiations
#define prepare_depth_low_kernel prepare_depth_low_ortho_kernel
#include "prepare_depth_kernel.inc"
#undef prepare_depth_low_kernel
#undef prepare_depth_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [low_only][prepare_slot]; slot 0 (linear ingest) is prepare_depth.cu's
const Kernel<PrepareArgs> kKernels[2][kPrepareSlots] = {MEAO_PREPARE_SLOTS_RAW(prepare_depth_ortho_kernel, MEAO_SLOT),
                                                        MEAO_PREPARE_SLOTS_RAW(prepare_depth_low_ortho_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_prepare_depth_ortho(const PrepareArgs &a_in, cudaStream_t s, bool low_only)
{
    if (!a_in.raw) return launch_prepare_depth(a_in, s, low_only);
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH));
    MEAO_LAUNCH((kKernels[low_only][prepare_slot(a)]), grid, kPrepThreads, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthOrthoUnit = {"prepare_depth_ortho.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
