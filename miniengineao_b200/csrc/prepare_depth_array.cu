// prepare_depth_array.cu -- stage 1 with the depth in a CUDA array (meao_render_arrays): a 2-D, layered or cube-map array of L
// layers, ONE launch for all of them.  The kernel body is prepare_depth.cu's (prepare_depth_kernel.inc, in its layered form: the
// layer is blockIdx.z); only the loads differ -- element-sized surface loads of the layer (surface_io.cuh) instead of load8.  The
// decoding, the linearisation and every store to the intermediates are the existing code.  A translation unit of its own so that
// prepare_depth.cu and prepare_depth_layered.cu compile to exactly the code they did before.
#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#define MEAO_ARRAY 1
#include "prepare_depth_kernel.inc"
#undef MEAO_ARRAY
#undef MEAO_LAYERED

// [prepare_slot]; no CUDA array holds D24S8
const Kernel<PrepareArgs, cudaSurfaceObject_t, int, const LayerZ *> kKernels[kPrepareSlots] =
    MEAO_PREPARE_SLOTS(prepare_depth_array_kernel, MEAO_NO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_array(const PrepareArgs &a_in, cudaSurfaceObject_t depth, int surf_kind, int layers, cudaStream_t s,
                                       const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || a_in.in_format == IN_D24S8) return cudaErrorInvalidValue;
    PrepareArgs a = a_in;
    a.depth = nullptr;
    a.vec_ok = 1;               // the input is read element by element; the intermediates' pitched rows keep the vector stores aligned
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, depth, surf_kind, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthArrayUnit = {"prepare_depth_array.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
