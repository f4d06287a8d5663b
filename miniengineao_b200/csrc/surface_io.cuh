// surface_io.cuh -- element-sized surface loads and stores of the CUDA-array kernels (prepare_depth_array.cu,
// blur_upsample_array.cu; meao_render_arrays in include/meao.h).
//
// A CUDA array is opaque, block-linear memory: the kernels reach it only through a surface object.  Every access here moves
// exactly one element (4 or 2 bytes per depth load, 1 byte per AO store): suld.b / sust.b address the lowest dimension in BYTES
// and the PTX ISA defines a transfer only for the size of the surface's element.  The callers guard every access in range
// (partial row ends included); every access also passes cudaBoundaryModeZero, so an out-of-range access would read 0 / be dropped
// instead of trapping the context (the default, cudaBoundaryModeTrap, turns an off-by-one into a context fault).
#pragma once

#include "common.cuh"
#include "kernels.h"

namespace meao {

// element x of row y of layer `layer`; kind (kSurf2D / kSurfLayered / kSurfCube, kernels.h) is a kernel argument: warp-uniform
template <class T>
__device__ __forceinline__ T surf_load(cudaSurfaceObject_t s, int kind, int x, int y, int layer)
{
    const int xb = x * (int)sizeof(T);
    if (kind == kSurf2D) return surf2Dread<T>(s, xb, y, cudaBoundaryModeZero);
    if (kind == kSurfLayered) return surf2DLayeredread<T>(s, xb, y, layer, cudaBoundaryModeZero);
    return surfCubemapread<T>(s, xb, y, layer, cudaBoundaryModeZero);
}

__device__ __forceinline__ void surf_store_u8(cudaSurfaceObject_t s, int kind, int x, int y, int layer, uint32_t code)
{
    const unsigned char v = (unsigned char)code;
    if (kind == kSurf2D) surf2Dwrite<unsigned char>(v, s, x, y, cudaBoundaryModeZero);
    else if (kind == kSurfLayered) surf2DLayeredwrite<unsigned char>(v, s, x, y, layer, cudaBoundaryModeZero);
    else surfCubemapwrite<unsigned char>(v, s, x, y, layer, cudaBoundaryModeZero);
}

}  // namespace meao
