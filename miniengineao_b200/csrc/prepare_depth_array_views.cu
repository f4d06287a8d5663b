// prepare_depth_array_views.cu -- stage 1 of a layered CUDA-array frame with a layer-viewport table (meao_set_layer_viewports): layer l
// reads the W x H rectangle of its table entry (kernels.h LayerView) from the depth array's layer depth_slice, ONE launch for all
// layers.  The kernel body is prepare_depth_array.cu's (prepare_depth_kernel.inc with MEAO_ARRAY 1 and MEAO_VIEWS 1): only the origin
// and the layer of the surface loads differ.  A translation unit of its own so that prepare_depth_array.cu compiles to exactly the code
// it did before.
#include "common.cuh"
#include "kernels.h"
#include "surface_io.cuh"

namespace meao {

namespace {

#define MEAO_LAYERED 1
#define MEAO_ARRAY 1
#define MEAO_VIEWS 1
#include "prepare_depth_kernel.inc"
#undef MEAO_VIEWS
#undef MEAO_ARRAY
#undef MEAO_LAYERED

// [prepare_slot]; no CUDA array holds D24S8
const Kernel<PrepareArgs, cudaSurfaceObject_t, int, const LayerView *, const LayerZ *> kKernels[kPrepareSlots] =
    MEAO_PREPARE_SLOTS(prepare_depth_array_views_kernel, MEAO_NO_SLOT);

}  // namespace

cudaError_t launch_prepare_depth_array_views(const PrepareArgs &a_in, cudaSurfaceObject_t depth, int surf_kind, const LayerView *views, int layers,
                                             cudaStream_t s, const LayerZ *layer_zb)
{
    if (a_in.row1 <= a_in.row0) return cudaSuccess;
    if (layers < 1 || layers > kMaxLayers || a_in.in_format == IN_D24S8 || !views) return cudaErrorInvalidValue;
    PrepareArgs a = a_in;
    a.depth = nullptr;
    a.vec_ok = 1;               // the input is read element by element; the intermediates' pitched rows keep the vector stores aligned
    dim3 grid(ceil_div(a.W, kPrepTileW), ceil_div(a.row1 - a.row0, kPrepTileH), layers);
    MEAO_LAUNCH((kKernels[prepare_slot(a)]), grid, kPrepThreads, 0, s, a, depth, surf_kind, views, layer_zb);
    return cudaGetLastError();
}

const KernelUnit kPrepareDepthArrayViewsUnit = {"prepare_depth_array_views.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
