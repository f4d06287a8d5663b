// cuda_emu_surface.h -- HOST stand-ins for the CUDA surface objects used by the CUDA-array kernels (miniengineao_b200/csrc/*_array.cu,
// surface_io.cuh).  TEST INFRASTRUCTURE ONLY, an extension of cuda_emu.h (see there); included with it by kernels.h under MEAO_EMULATE.
#pragma once

#include "cuda_emu.h"

typedef unsigned long long cudaSurfaceObject_t;
enum cudaSurfaceBoundaryMode { cudaBoundaryModeZero = 0, cudaBoundaryModeClamp = 1, cudaBoundaryModeTrap = 2 };

// ---- surface objects over a CUDA array (surf2D* / surf2DLayered* / surfCubemap*) ---------------------------------------------------
// An emulated array is `layers` images of w x h elements of `elem` bytes, rows pitch_bytes apart, layer l at l x h x pitch_bytes; the
// surface object is its address.  Like suld.b / sust.b, x is a BYTE offset, and the access must move exactly one element at an
// element boundary (anything else is undefined on the GPU: refused here).  The access form must match the array's shape (2-D, layered,
// cube).  Out of range: cudaBoundaryModeZero reads 0 / drops the store; the trap mode is refused (it faults the context on the GPU).
namespace meao_emu {
enum { SURF_2D = 0, SURF_LAYERED = 1, SURF_CUBE = 2 };
struct Surface { void *base; int elem, w, h, layers; size_t pitch_bytes; int shape; };
extern long long surface_accesses;   // emulated surface loads + stores so far (tests assert the surface path really ran)
inline char *surface_texel(cudaSurfaceObject_t obj, int shape, size_t size, int xb, int y, int layer, cudaSurfaceBoundaryMode mode)
{
    const Surface *s = reinterpret_cast<const Surface *>(obj);
    if (s->shape != shape) unsupported("surface access form does not match the array's shape");
    if ((int)size != s->elem) unsupported("surface access wider or narrower than the array's element (undefined for suld.b / sust.b)");
    if (xb % s->elem != 0) unsupported("surface byte offset not on an element boundary");
    surface_accesses++;
    const int x = xb / s->elem;
    if (x < 0 || y < 0 || layer < 0 || x >= s->w || y >= s->h || layer >= s->layers) {
        if (mode != cudaBoundaryModeZero) unsupported("out-of-range surface access in trap mode (a context fault on the GPU)");
        return nullptr;
    }
    return (char *)s->base + ((size_t)layer * s->h + y) * s->pitch_bytes + (size_t)x * s->elem;
}
template <class T> inline T surface_read(cudaSurfaceObject_t o, int shape, int xb, int y, int layer, cudaSurfaceBoundaryMode m)
{
    T v{};
    if (const char *p = surface_texel(o, shape, sizeof(T), xb, y, layer, m)) memcpy(&v, p, sizeof(T));
    return v;
}
template <class T> inline void surface_write(T v, cudaSurfaceObject_t o, int shape, int xb, int y, int layer, cudaSurfaceBoundaryMode m)
{
    if (char *p = surface_texel(o, shape, sizeof(T), xb, y, layer, m)) memcpy(p, &v, sizeof(T));
}
}
template <class T> inline T surf2Dread(cudaSurfaceObject_t o, int x, int y, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ return meao_emu::surface_read<T>(o, meao_emu::SURF_2D, x, y, 0, m); }
template <class T> inline T surf2DLayeredread(cudaSurfaceObject_t o, int x, int y, int layer, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ return meao_emu::surface_read<T>(o, meao_emu::SURF_LAYERED, x, y, layer, m); }
template <class T> inline T surfCubemapread(cudaSurfaceObject_t o, int x, int y, int face, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ return meao_emu::surface_read<T>(o, meao_emu::SURF_CUBE, x, y, face, m); }
template <class T> inline void surf2Dwrite(T v, cudaSurfaceObject_t o, int x, int y, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ meao_emu::surface_write<T>(v, o, meao_emu::SURF_2D, x, y, 0, m); }
template <class T> inline void surf2DLayeredwrite(T v, cudaSurfaceObject_t o, int x, int y, int layer, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ meao_emu::surface_write<T>(v, o, meao_emu::SURF_LAYERED, x, y, layer, m); }
template <class T> inline void surfCubemapwrite(T v, cudaSurfaceObject_t o, int x, int y, int face, cudaSurfaceBoundaryMode m = cudaBoundaryModeTrap)
{ meao_emu::surface_write<T>(v, o, meao_emu::SURF_CUBE, x, y, face, m); }
