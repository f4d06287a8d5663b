// prepare_depth_batch.cu -- stage 1 of a batch over device buffers (meao_render_batch): layer l reads the W x H frame from its own
// buffer at its own row pitch, ONE launch for all layers.  Only the low-only form: such a frame is always fused (its final upsample
// linearises the full-resolution depth, blur_upsample_lin_batch.cu).  The kernel body is prepare_depth_layered.cu's
// (prepare_depth_kernel.inc with MEAO_LAYERED 1 and MEAO_BATCH 1): only the base and pitch of each layer's depth, taken from entry
// blockIdx.z of the batch table (kernels.h BatchPointers, a kernel parameter), and its vector-load test differ.  A translation unit of
// its own so that prepare_depth_layered.cu compiles to exactly the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#define MEAO_BATCH 1
#include "prepare_depth_kernel.inc"
#undef MEAO_BATCH
#undef MEAO_LAYERED

// [prepare_slot]
const Kernel<PrepareArgs, BatchPointers, const LayerZ *> kKernels[kPrepareSlots] = MEAO_PREPARE_SLOTS(prepare_depth_low_batch_kernel, MEAO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_batch(const PrepareArgs &a_in, const BatchPointers &io, int layers, cudaStream_t s, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxBatch || a_in.depth_row0 != 0) return cudaErrorInvalidValue;
    PrepareArgs a = a_in;
    a.depth = nullptr;          // each layer's base, pitch and vector test come from its entry
    a.depth_pitch = 0; a.depth_layer_pitch = 0; a.vec_ok = 0;
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepLowTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, io, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthBatchUnit = {"prepare_depth_batch.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
