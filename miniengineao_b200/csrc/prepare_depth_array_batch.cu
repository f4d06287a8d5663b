// prepare_depth_array_batch.cu -- stage 1 of a batch over CUDA arrays (meao_render_arrays_batch): layer l reads the W x H frame at the
// top-left corner of its own 2-D array, ONE launch for all layers.  The kernel body is prepare_depth_array.cu's (prepare_depth_kernel.inc
// with MEAO_ARRAY 1 and MEAO_BATCH 1): only the surface of the loads differs, taken from entry blockIdx.z of the batch table (kernels.h
// BatchArrays), a kernel parameter.  A translation unit of its own so that prepare_depth_array.cu compiles to exactly the code it did
// before.
#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#define MEAO_ARRAY 1
#define MEAO_BATCH 1
#include "prepare_depth_kernel.inc"
#undef MEAO_BATCH
#undef MEAO_ARRAY
#undef MEAO_LAYERED

// [prepare_slot]; no CUDA array holds D24S8
const Kernel<PrepareArgs, BatchArrays, const LayerZ *> kKernels[kPrepareSlots] = MEAO_PREPARE_SLOTS(prepare_depth_array_batch_kernel, MEAO_NO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_array_batch(const PrepareArgs &a_in, const BatchArrays &depth, int layers, cudaStream_t s, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxBatch || a_in.in_format == IN_D24S8) return cudaErrorInvalidValue;
    PrepareArgs a = a_in;
    a.depth = nullptr;
    a.vec_ok = 1;               // the input is read element by element; the intermediates' pitched rows keep the vector stores aligned
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, depth, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthArrayBatchUnit = {"prepare_depth_array_batch.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
