// composite.cu -- the consumer end of the pipe (SURVEY.md 8f.1): multiply the AO texture into the colour
// targets.  Replaces the two raster composite passes of Blit.shader, whose arithmetic is fixed-function
// output-merger blending:
//   pass 2 (Blit.shader:84-101, recorded at AmbientOcclusion.cs:837)   Blend Zero SrcAlpha, src = ao.rrrr
//        =>  dst.rgba *= ao
//   pass 1 (Blit.shader:66-92, recorded at AmbientOcclusion.cs:832-833) Blend Zero OneMinusSrcColor, Zero OneMinusSrcAlpha,
//        src0 = (0,0,0,1-ao), src1 = (1-ao,1-ao,1-ao,0)
//        =>  gbuffer0.a *= 1-(1-ao);  gbuffer3.rgb *= 1-(1-ao)      (everything else is multiplied by 1)
// Conventions (D3D11 output merger, unpinned like the rest): blend in fp32; ao = k * (1/255) (point-sampled R8 at
// the pixel centre); RGBA8 targets load k * (1/255) and store (uint)(saturate(x) * 255 + 0.5); RGBA16F targets
// load exactly and store RTNE.
// Bound: HBM -- 8 (RGBA8) or 16 (RGBA16F) + 1 bytes per pixel of pure streaming; 4 pixels per thread, 128-bit accesses.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

constexpr int kCompThreads = 256;

__device__ __forceinline__ uint32_t scale_rgba8(uint32_t px, float f, bool rgb, bool alpha)
{
    uint32_t out = 0;
#pragma unroll
    for (int ch = 0; ch < 4; ch++) {
        const uint32_t k = (px >> (8 * ch)) & 0xffu;
        const bool on = (ch < 3) ? rgb : alpha;
        const uint32_t r = on ? unorm8_code(__fmul_rn(unorm8_load(k), f)) : k;
        out |= r << (8 * ch);
    }
    return out;
}

__device__ __forceinline__ uint2 scale_rgba16f(uint2 px, float f, bool rgb, bool alpha)
{
    __half2 lo = *reinterpret_cast<__half2 *>(&px.x), hi = *reinterpret_cast<__half2 *>(&px.y);   // (r,g) (b,a)
    float2 a = __half22float2(lo), b = __half22float2(hi);
    if (rgb) { a.x = __fmul_rn(a.x, f); a.y = __fmul_rn(a.y, f); b.x = __fmul_rn(b.x, f); }
    if (alpha) b.y = __fmul_rn(b.y, f);
    lo = __floats2half2_rn(a.x, a.y); hi = __floats2half2_rn(b.x, b.y);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t *>(&lo); o.y = *reinterpret_cast<uint32_t *>(&hi);
    return o;
}

// one_minus: factor = 1 - (1 - ao) (pass 1) instead of ao (pass 2)
template <bool HALF>
__global__ void __launch_bounds__(kCompThreads)
composite_kernel(const uint8_t *__restrict__ ao, void *__restrict__ color, long long npix, int rgb, int alpha, int one_minus)
{
#ifdef MEAO_DEVICE_OK
    const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i4 >= npix) return;
    if (i4 + 4 <= npix) {
        const uint32_t a4 = __ldg(reinterpret_cast<const uint32_t *>(ao + i4));
        float f[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float t = unorm8_load((a4 >> (8 * e)) & 0xffu);
            f[e] = one_minus ? __fadd_rn(1.0f, -__fadd_rn(1.0f, -t)) : t;
        }
        if (HALF) {
            uint4 *p = reinterpret_cast<uint4 *>(color) + (i4 >> 1);
            uint4 q0 = p[0], q1 = p[1];
            uint2 r0 = scale_rgba16f(make_uint2(q0.x, q0.y), f[0], rgb, alpha), r1 = scale_rgba16f(make_uint2(q0.z, q0.w), f[1], rgb, alpha);
            uint2 r2 = scale_rgba16f(make_uint2(q1.x, q1.y), f[2], rgb, alpha), r3 = scale_rgba16f(make_uint2(q1.z, q1.w), f[3], rgb, alpha);
            p[0] = make_uint4(r0.x, r0.y, r1.x, r1.y);
            p[1] = make_uint4(r2.x, r2.y, r3.x, r3.y);
        } else {
            uint4 *p = reinterpret_cast<uint4 *>(color) + (i4 >> 2);
            uint4 q = *p;
            q.x = scale_rgba8(q.x, f[0], rgb, alpha); q.y = scale_rgba8(q.y, f[1], rgb, alpha);
            q.z = scale_rgba8(q.z, f[2], rgb, alpha); q.w = scale_rgba8(q.w, f[3], rgb, alpha);
            *p = q;
        }
    } else {
        for (long long i = i4; i < npix; i++) {
            const float t = unorm8_load(ao[i]);
            const float f = one_minus ? __fadd_rn(1.0f, -__fadd_rn(1.0f, -t)) : t;
            if (HALF) { uint2 *p = reinterpret_cast<uint2 *>(color) + i; *p = scale_rgba16f(*p, f, rgb, alpha); }
            else { uint32_t *p = reinterpret_cast<uint32_t *>(color) + i; *p = scale_rgba8(*p, f, rgb, alpha); }
        }
    }
#endif
}

const Kernel<const uint8_t *, void *, long long, int, int, int> kKernels[2] = {composite_kernel<false>, composite_kernel<true>};    // [half]

}  // namespace

cudaError_t launch_composite(const uint8_t *ao, void *color, long long npix, int half, int rgb, int alpha, int one_minus, cudaStream_t s)
{
    if (npix <= 0) return cudaSuccess;
    const long long groups = (npix + 3) / 4;
    const unsigned blocks = (unsigned)((groups + kCompThreads - 1) / kCompThreads);
    MEAO_LAUNCH((kKernels[half ? 1 : 0]), blocks, kCompThreads, 0, s, ao, color, npix, rgb, alpha, one_minus);
    return cudaGetLastError();
}

const KernelUnit kCompositeUnit = {"composite.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
