// selftest.cu -- device-side brute-force check that the guarded fast division / reciprocal of
// common.cuh return exactly what the IEEE operators `a / b` and `1 / x` return (meao_selftest_div).
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

__device__ __forceinline__ uint32_t pcg(uint32_t &s)
{
    s = s * 747796405u + 2891336453u;
    uint32_t w = ((s >> ((s >> 28u) + 4u)) ^ s) * 277803737u;
    return (w >> 22u) ^ w;
}
// random positive normal float with biased exponent in [67, 186]  ==  [2^-60, 2^60)
__device__ __forceinline__ float rand_safe(uint32_t &s)
{
    const uint32_t m = pcg(s) & 0x7fffffu;
    const uint32_t e = 67u + pcg(s) % 120u;
    return __uint_as_float((e << 23) | m);
}

__global__ void selftest_div_kernel(uint64_t n_per_thread, uint32_t seed, unsigned long long *mismatch)
{
#ifdef MEAO_DEVICE_OK
    uint32_t s = seed ^ (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
    unsigned long long bad = 0;
    for (uint64_t i = 0; i < n_per_thread; i++) {
        const float b = rand_safe(s);
        float a;
        switch (pcg(s) & 7u) {
            case 0: a = 1.0f; break;
            case 1: a = 3.0f; break;
            case 2: a = 9.0f; break;
            case 3: a = 0.0f; break;
            case 4: a = b * (1.0f + (float)(pcg(s) & 0xffu) * 1.1920929e-7f); break;   // quotient near 1
            default: a = rand_safe(s); break;
        }
        if (__float_as_uint(div_fast(a, b)) != __float_as_uint(a / b)) bad++;
        if (__float_as_uint(rcp_fast(b)) != __float_as_uint(1.0f / b)) bad++;
        if (__float_as_uint(rcp_ieee(b)) != __float_as_uint(1.0f / b)) bad++;
        // guard rejects what it must: specials never take the fast path
        const float sp[6] = {0.0f, __uint_as_float(0x7f800000u), __uint_as_float(0x7fc00000u), 1e-40f, -1.0f, __uint_as_float(0x5d800000u)};
        if (in_safe_range(sp[i % 6])) bad++;
    }
    if (bad) atomicAdd(mismatch, bad);
#endif
}

const Kernel<uint64_t, uint32_t, unsigned long long *> kKernels[] = {selftest_div_kernel};

}  // namespace

cudaError_t launch_selftest_div(uint64_t n, uint32_t seed, unsigned long long *mismatch_dev, int sm_count, cudaStream_t s)
{
    const int blocks = sm_count * 8, threads = 256;
    const uint64_t per = (n + (uint64_t)blocks * threads - 1) / ((uint64_t)blocks * threads);
    MEAO_LAUNCH((selftest_div_kernel), blocks, threads, 0, s, per, seed, mismatch_dev);
    return cudaGetLastError();
}

const KernelUnit kSelftestUnit = {"selftest.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
