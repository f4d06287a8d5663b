// debug_view.cu -- the debug views of the AmbientOcclusion component (SURVEY.md 8f.3).
//
// Replaces PushDebugBlitCommands (AmbientOcclusion.cs:787-820): cmd.Blit(rt, _result) for a non-tiled buffer
// (point-sampled stretch: the RTs are FilterMode.Point, AO.cs:206,228,236) or Blit.shader pass 4 "Detile"
// (:136-156) for a TiledDepth atlas, followed by the R8 store of the _result target (AO.cs:475).  The raster
// passes sample at the pixel centre uv = ((x + .5) / W, (y + .5) / H); texel indices are evaluated in exact
// integer arithmetic (floor((2x+1) * sw / (2W))), which is what an exact rasteriser + point sampler yields.
//
// The TiledDepth atlases are virtual here (DESIGN.md 1): slice s, texel (tx, ty) is natural pixel
// (4 tx + (s & 3), 4 ty + (s >> 2)) of LowDepth<k> rounded to f16, or the padding value outside the level.
// Bound: HBM (1 B written per pixel, <= 4 B read per source texel); not on the frame path.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

__global__ void __launch_bounds__(256) debug_view_kernel(const DebugViewArgs a)
{
#ifdef MEAO_DEVICE_OK
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= a.W) return;
    // 32-bit unsigned arithmetic is exact here: W, H <= 32768 (meao_resize), so (2x+1) * sw < 2^31 and r * sw < 2^29
    const uint32_t W2 = 2u * (uint32_t)a.W, H2 = 2u * (uint32_t)a.H;
    float v;
    if (a.tiled) {
        // Blit.shader:150-152: uv4 = uv * 4; slice = floor(uv4.x) + floor(uv4.y) * 4; sample the slice at frac(uv4)
        const uint32_t nx = 8u * x + 4u, ny = 8u * y + 4u;                  // 4 * uv = n / (2 * size)
        const uint32_t qx = nx / W2, qy = ny / H2;
        const uint32_t rx = nx - W2 * qx, ry = ny - H2 * qy;                // frac = r / (2 * size)
        const int tx = (int)(rx * (uint32_t)a.sw / W2), ty = (int)(ry * (uint32_t)a.sh / H2);
        const int px = 4 * tx + (int)qx, py = 4 * ty + (int)qy;             // inverse of DS1:69,71 with slice = qx | qy << 2
        v = a.pad;
        if (px < a.lw && py < a.lh) v = f16_round(reinterpret_cast<const float *>(a.src)[(size_t)py * a.spitch + px]);
    } else {
        // cmd.Blit(rt, _result), AO.cs:817
        const int tx = (int)((2u * x + 1u) * (uint32_t)a.sw / W2), ty = (int)((2u * y + 1u) * (uint32_t)a.sh / H2);
        const size_t i = (size_t)ty * a.spitch + tx;
        if (a.elem == 1) { a.out[(size_t)y * a.out_pitch + x] = reinterpret_cast<const uint8_t *>(a.src)[i]; return; }   // R8 -> R8: store(load(k)) == k
        v = (a.elem == 2) ? __half2float(reinterpret_cast<const __half *>(a.src)[i]) : reinterpret_cast<const float *>(a.src)[i];
    }
    a.out[(size_t)y * a.out_pitch + x] = (uint8_t)unorm8_code(v);
#endif
}

// Blit.shader pass 3 "Debug" (:116-134), recorded by PushCompositeCommands when _debug > 0 (AO.cs:826-829):
// cmd.Blit(_result, CameraTarget, material, 3) with no blending -- the target becomes (r, r, r, r), r = the R8 view.
// 4 pixels per thread: one 32-bit load of codes, one 128-bit (RGBA8) or two 128-bit (RGBA16F) stores.
template <bool HALF>
__global__ void __launch_bounds__(256) debug_composite_kernel(const uint8_t *__restrict__ view, void *__restrict__ color, long long npix)
{
#ifdef MEAO_DEVICE_OK
    const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i4 >= npix) return;
    const int n = (npix - i4 >= 4) ? 4 : (int)(npix - i4);
    uint32_t k[4] = {0, 0, 0, 0};
    if (n == 4) { const uint32_t q = *reinterpret_cast<const uint32_t *>(view + i4); k[0] = q & 0xffu; k[1] = (q >> 8) & 0xffu; k[2] = (q >> 16) & 0xffu; k[3] = q >> 24; }
    else for (int e = 0; e < n; e++) k[e] = view[i4 + e];
    if (HALF) {
        __half *dst = reinterpret_cast<__half *>(color) + i4 * 4;
        for (int e = 0; e < n; e++) {
            const __half h = __float2half_rn(unorm8_load(k[e]));          // R8 sample -> float -> RGBA16F store (RTNE)
            dst[4 * e] = h; dst[4 * e + 1] = h; dst[4 * e + 2] = h; dst[4 * e + 3] = h;
        }
    } else {
        uint32_t *dst = reinterpret_cast<uint32_t *>(color) + i4;
        for (int e = 0; e < n; e++) dst[e] = k[e] * 0x01010101u;          // store(load(k)) == k on every channel
    }
#endif
}

const struct {
    Kernel<DebugViewArgs> view;
    Kernel<const uint8_t *, void *, long long> composite[2];       // [half]
} kKernels = {debug_view_kernel, {debug_composite_kernel<false>, debug_composite_kernel<true>}};

}  // namespace

cudaError_t launch_debug_composite(const uint8_t *view, void *color, long long npix, int half, cudaStream_t s)
{
    const int blocks = (int)((npix + 4 * 256 - 1) / (4 * 256));
    if (blocks <= 0) return cudaSuccess;
    MEAO_LAUNCH((kKernels.composite[half ? 1 : 0]), blocks, 256, 0, s, view, color, npix);
    return cudaGetLastError();
}

cudaError_t launch_debug_view(const DebugViewArgs &a, cudaStream_t s)
{
    dim3 grid(ceil_div(a.W, 256), a.H);
    MEAO_LAUNCH((debug_view_kernel), grid, 256, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kDebugViewUnit = {"debug_view.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels.view, kKernels.composite); }};

}  // namespace meao
