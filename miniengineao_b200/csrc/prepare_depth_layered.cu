// prepare_depth_layered.cu -- stage 1 for a layered frame (meao_set_layers): L same-size depth images stacked at a stride of
// PrepareArgs.depth_layer_pitch (tight: one W x H image), ONE launch for all of them.  The kernel body is prepare_depth.cu's (prepare_depth_kernel.inc); the
// layer is blockIdx.z and selects the input image and the output images of every level (kernels.h "layered frames").
// A translation unit of its own so that prepare_depth.cu compiles to exactly the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#include "prepare_depth_kernel.inc"
#undef MEAO_LAYERED

// [low_only][prepare_slot]
const Kernel<PrepareArgs, const LayerZ *> kKernels[2][kPrepareSlots] = {MEAO_PREPARE_SLOTS(prepare_depth_layered_kernel, MEAO_SLOT),
                                                                        MEAO_PREPARE_SLOTS(prepare_depth_low_layered_kernel, MEAO_SLOT)};

}  // namespace

cudaError_t launch_prepare_depth_layered(const PrepareArgs &a_in, int layers, cudaStream_t s, bool low_only, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    const PrepareArgs a = resolve_pitches(a_in);
    if (layers < 1 || layers > kMaxLayers) return cudaErrorInvalidValue;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, low_only ? kPrepLowTileH : kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[low_only][prepare_slot(a)]), grid, kPrepThreads, 0, s, a, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthLayeredUnit = {"prepare_depth_layered.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
