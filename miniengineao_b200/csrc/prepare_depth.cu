// prepare_depth.cu -- stage 1 of the SSAO pipe: depth linearise + point-sampled mip hierarchy.
//
// Replaces Downsample1.compute (Linearize :37-48, main :52-81) and Downsample2.compute (main
// :32-51) with ONE streaming pass:   raw depth (f32, L0)  ->  LinearDepth (f16, L0),
// LowDepth1..4 (f32; LowDepth<k>(i,j) = lin(2^k i, 2^k j), a pure point sample -- DS1:64-66,
// DS2:35).  The deinterleaved f16 atlases are not written (see kernels.h).
//
// Bound: HBM.  Algorithmic bytes per L0 pixel: 4 (read) + 2 + 4/4 + 4/16 + 4/64 + 4/256 = 7.33
// (the reference's Downsample1+2 move 8.24 B/px because they also write and re-read the atlases).
// There is no data reuse between threads, so no shared-memory staging: each thread streams
// 2 x 8 pixels with 128-bit loads (L1::no_allocate) and 128-bit stores.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 0
#include "prepare_depth_kernel.inc"
#undef MEAO_LAYERED

static_assert(IN_D16 == 1 && IN_D24S8 == 2, "depth_format_slot takes the IN_* codes");

// [low_only][prepare_slot]
const Kernel<PrepareArgs> kKernels[2][kPrepareSlots] = {MEAO_PREPARE_SLOTS(prepare_depth_kernel, MEAO_SLOT),
                                                        MEAO_PREPARE_SLOTS(prepare_depth_low_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_prepare_depth(const PrepareArgs &a_in, cudaStream_t s, bool low_only)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH));
    MEAO_LAUNCH((kKernels[low_only][prepare_slot(a)]), grid, kPrepThreads, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthUnit = {"prepare_depth.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
