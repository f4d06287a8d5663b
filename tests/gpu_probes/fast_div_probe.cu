// fast_div_probe.cu -- exhaustive check of the building blocks of the kernels' guarded fast division (csrc/common.cuh and
// csrc/blur_upsample_device.inc, included exactly as the kernels include them) against float64 statements of what they promise.
// Built and run by tests/test_fast_div_exhaustive_gpu.py; it is not part of libmeao.
//
//   part 1  every one of the 2^32 bit patterns: in_safe_range(x) == (x not NaN and 2^-60 <= x < 2^60); in_safe_range_neg(x) ==
//           in_safe_range(-x); for every negative or NaN s, neg_order(s) < 0xdd800000 (the bilateral pair guard) exactly when s is
//           finite and s > -2^60
//   part 2  every x with in_safe_range(x): rcp_fast(x), both lanes of rcp2_fast_neg and 1.0f / x == RN(1 / x)
//   part 3  every in-range b: div_fast(a, b) and both lanes of div2_fast_neg == RN(a / b) for a in {1, 3, 9}; plus a seeded sample
//           of in-range pairs (a, b) whose quotient is in range
//   part 4  bilateral2<BLEND> against unorm8_code(bilateral<BLEND>(...)) on a seeded sample of adversarial operands, wherever its
//           pair guard passes; the guard must also fail on some of them (the generator reaches the fallback)
//
// RN(a / b) is computed as (float)((double)a / (double)b): with 53 >= 2 * 24 + 2 bits the double rounding cannot change the result.
// With -DMEAO_EMULATE the file is a host program (g++, tests/emu/cuda_emu.h defines __device__ away) that runs part 1 only.
// Output: one "RESULT <check> checked=<n> mismatches=<m>" line per check, "COUNT <what> <n>" lines and "WALL <part> <ms>" lines.
#include <algorithm>
#include <array>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace meao {
namespace {
#include "blur_upsample_device.inc"
}  // namespace
}  // namespace meao

using namespace meao;

namespace probe {

constexpr double kLo = 0x1p-60, kHi = 0x1p60;

__device__ inline bool ref_in_range(float x)
{
    const double d = x;
    return d == d && d >= kLo && d < kHi;
}
__device__ inline bool is_nan_bits(uint32_t u) { return (u & 0x7fffffffu) > 0x7f800000u; }

// part 1 for one bit pattern; adds to c[0..4]: in_safe_range mismatches, in_safe_range_neg mismatches, pair-guard mismatches,
// in-range patterns, patterns the pair guard was checked on
__device__ inline void part1_one(uint32_t u, unsigned long long *c)
{
    const float x = __uint_as_float(u);
    const bool in = in_safe_range(x);
    c[0] += in != ref_in_range(x);
    c[1] += in_safe_range_neg(x) != in_safe_range(__uint_as_float(u ^ 0x80000000u));
    c[3] += in;
    if ((u & 0x80000000u) || is_nan_bits(u)) {
        const bool guard = neg_order(x) < (int)0xdd800000u;
        const double d = x;
        const bool want = !is_nan_bits(u) && (u & 0x7fffffffu) != 0x7f800000u && d > -kHi;
        c[2] += guard != want;
        c[4] += 1;
    }
}

void report(const char *name, unsigned long long checked, unsigned long long bad)
{
    printf("RESULT %s checked=%llu mismatches=%llu\n", name, checked, bad);
}

}  // namespace probe
using namespace probe;

#ifdef MEAO_EMULATE
// ---- host build: part 1 on every CPU thread ------------------------------------------------------------------------------------
int main()
{
    const auto t0 = std::chrono::steady_clock::now();
    const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
    std::vector<std::array<unsigned long long, 5>> acc(nt);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; t++)
        th.emplace_back([t, nt, &acc] {
            unsigned long long c[5] = {0, 0, 0, 0, 0};
            const uint64_t lo = (1ull << 32) * t / nt, hi = (1ull << 32) * (t + 1) / nt;
            for (uint64_t u = lo; u < hi; u++) part1_one((uint32_t)u, c);
            for (int i = 0; i < 5; i++) acc[t][i] = c[i];
        });
    for (auto &x : th) x.join();
    unsigned long long c[5] = {0, 0, 0, 0, 0};
    for (auto &a : acc)
        for (int i = 0; i < 5; i++) c[i] += a[i];
    report("in_safe_range", 1ull << 32, c[0]);
    report("in_safe_range_neg", 1ull << 32, c[1]);
    report("pair_guard", c[4], c[2]);
    printf("COUNT in_range %llu\n", c[3]);
    printf("WALL part1 %.1f\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    return 0;
}
#else
// ---- device build: all four parts on the GPU ----------------------------------------------------------------------------------
namespace probe {

constexpr uint32_t kSafeBase = 0x21800000u;                 // bit pattern of 2^-60
constexpr uint64_t kSafeCount = 120ull << 23;               // biased exponents 67 .. 186

__device__ inline uint32_t pcg(uint32_t &s)
{
    s = s * 747796405u + 2891336453u;
    const uint32_t w = ((s >> ((s >> 28u) + 4u)) ^ s) * 277803737u;
    return (w >> 22u) ^ w;
}
__device__ inline float rand_safe(uint32_t &s) { return __uint_as_float((67u + pcg(s) % 120u) << 23 | (pcg(s) & 0x7fffffu)); }
__device__ inline uint64_t tid64() { return (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; }
__device__ inline uint64_t nthreads() { return (uint64_t)gridDim.x * blockDim.x; }
__device__ inline bool differ(float a, float b) { return __float_as_uint(a) != __float_as_uint(b); }
__device__ inline void flush(unsigned long long *dst, const unsigned long long *c, int n)
{
    for (int i = 0; i < n; i++)
        if (c[i]) atomicAdd(dst + i, c[i]);
}

__global__ void part1_kernel(unsigned long long *out)
{
    unsigned long long c[5] = {0, 0, 0, 0, 0};
    for (uint64_t u = tid64(); u < (1ull << 32); u += nthreads()) part1_one((uint32_t)u, c);
    flush(out, c, 5);
}

// c: rcp_fast, rcp2_fast_neg lane x, lane y, 1.0f / x
__global__ void part2_kernel(unsigned long long *out)
{
    unsigned long long c[4] = {0, 0, 0, 0};
    for (uint64_t i = tid64(); i < kSafeCount; i += nthreads()) {
        const float x = __uint_as_float(kSafeBase + (uint32_t)i), x2 = __uint_as_float(kSafeBase + (uint32_t)(kSafeCount - 1 - i));
        const float r = (float)(1.0 / (double)x), r2 = (float)(1.0 / (double)x2);
        const float2 p = rcp2_fast_neg(make_float2(-x, -x2));
        c[0] += differ(rcp_fast(x), r);
        c[1] += differ(p.x, r);
        c[2] += differ(p.y, r2);
        c[3] += differ(1.0f / x, r);
    }
    flush(out, c, 4);
}

// c[3k + 0..2] for a = 1, 3, 9: div_fast, div2_fast_neg lane x, lane y; c[9]: a / b
__global__ void part3_exhaustive_kernel(unsigned long long *out)
{
    unsigned long long c[10] = {};
    const float as[3] = {1.0f, 3.0f, 9.0f};
    for (uint64_t i = tid64(); i < kSafeCount; i += nthreads()) {
        const float b = __uint_as_float(kSafeBase + (uint32_t)i), b2 = __uint_as_float(kSafeBase + (uint32_t)(kSafeCount - 1 - i));
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float a = as[k];
            const float q = (float)((double)a / (double)b), q2 = (float)((double)a / (double)b2);
            const float2 p = div2_fast_neg(make_float2(a, a), make_float2(-b, -b2));
            c[3 * k] += differ(div_fast(a, b), q);
            c[3 * k + 1] += differ(p.x, q);
            c[3 * k + 2] += differ(p.y, q2);
            c[9] += differ(a / b, q);
        }
    }
    flush(out, c, 10);
}

// n draws of two pairs each; c: draws checked (both quotients in range), div_fast, div2_fast_neg lane x, lane y, a / b
__global__ void part3_random_kernel(uint64_t n, uint32_t seed, unsigned long long *out)
{
    unsigned long long c[5] = {0, 0, 0, 0, 0};
    uint32_t s = seed ^ (uint32_t)tid64() * 2654435761u;
    for (uint64_t i = tid64(); i < n; i += nthreads()) {
        const float a = rand_safe(s), b = rand_safe(s), a2 = rand_safe(s), b2 = rand_safe(s);
        const double qd = (double)a / (double)b, qd2 = (double)a2 / (double)b2;
        if (!(qd >= kLo && qd < kHi && qd2 >= kLo && qd2 < kHi)) continue;
        const float q = (float)qd, q2 = (float)qd2;
        const float2 p = div2_fast_neg(make_float2(a, a2), make_float2(-b, -b2));
        c[0] += 1;
        c[1] += differ(div_fast(a, b), q);
        c[2] += differ(p.x, q);
        c[3] += differ(p.y, q2);
        c[4] += differ(a / b, q);
    }
    flush(out, c, 5);
}

// ---- part 4: adversarial bilateral operands --------------------------------------------------------------------------------------
__device__ inline float half_bits(uint32_t h) { return __half2float(__ushort_as_half((unsigned short)h)); }
__device__ inline float rand_hi_depth(uint32_t &s)
{
    const uint32_t r = pcg(s) & 15u;
    if (r < 10) return half_bits(pcg(s) % 0x7c00u);                                   // any finite f16 >= 0 (subnormals included)
    if (r < 12) return half_bits(0x2000u + pcg(s) % 0x1c00u);                         // f16 in [2^-7, 1)
    if (r < 14) return __uint_as_float((107u + pcg(s) % 41u) << 23 | (pcg(s) & 0x7fffffu));   // any f32 in [2^-20, 2^21)
    if (r == 14) return __uint_as_float(0x7f800000u);                                  // sky: +inf
    return (pcg(s) & 1u) ? __uint_as_float(0x7fffffffu) : 0.0f;                       // NaN or 0
}
__device__ inline float rand_lo_depth(uint32_t &s, float hd)
{
    const uint32_t r = pcg(s) & 7u;
    if (r < 3) return hd;                                                              // exact tie: b_i = tol
    if (r < 5) {                                                                       // a few f16 ulps from hd
        const uint32_t h = __half_as_ushort(__float2half_rn(hd));
        const uint32_t d = 1u + (pcg(s) & 15u);
        return half_bits((pcg(s) & 1u) ? h + d : (h > d ? h - d : 0u));
    }
    if (r < 7) return rand_hi_depth(s);
    return half_bits(pcg(s) % 0x7c00u);
}
__device__ inline float rand_lo_ao(uint32_t &s)
{
    const uint32_t r = pcg(s) & 3u;
    return r == 0 ? 0.0f : (r == 1 ? 1.0f : unorm8_load(pcg(s) & 255u));
}
__device__ inline float rand_hi_ao(uint32_t &s)
{
    const uint32_t r = pcg(s) & 3u;
    return unorm8_load(r == 0 ? 0u : (r == 1 ? 1u : (r == 2 ? 255u : pcg(s) & 255u)));
}

struct Tols { float tol[3], nfs[2]; };

// n calls of two lanes each; c: lanes checked (guard passed), code mismatches, lanes whose pair failed the guard
template <bool BLEND>
__global__ void part4_kernel(uint64_t n, uint32_t seed, Tols t, unsigned long long *out)
{
    unsigned long long c[3] = {0, 0, 0};
    uint32_t s = seed ^ (uint32_t)tid64() * 2654435761u;
    for (uint64_t i = tid64(); i < n; i += nthreads()) {
        const float tol = t.tol[pcg(s) % 3u], nfs = t.nfs[pcg(s) & 1u];
        float hd[2], ha[2], ld[2][4], la[2][4];
        for (int l = 0; l < 2; l++) {
            hd[l] = rand_hi_depth(s);
            ha[l] = rand_hi_ao(s);
            for (int k = 0; k < 4; k++) { ld[l][k] = rand_lo_depth(s, hd[l]); la[l][k] = rand_lo_ao(s); }
        }
        int worst = (int)0x80000000u;
        const uint32_t codes = bilateral2<BLEND>(make_float2(hd[0], hd[1]), make_float2(ha[0], ha[1]),
                                                 make_float2(ld[0][0], ld[1][0]), make_float2(ld[0][1], ld[1][1]),
                                                 make_float2(ld[0][2], ld[1][2]), make_float2(ld[0][3], ld[1][3]),
                                                 make_float2(la[0][0], la[1][0]), make_float2(la[0][1], la[1][1]),
                                                 make_float2(la[0][2], la[1][2]), make_float2(la[0][3], la[1][3]), tol, nfs, worst);
        if (worst >= (int)0xdd800000u) { c[2] += 2; continue; }
        for (int l = 0; l < 2; l++) {
            const uint32_t want = unorm8_code(bilateral<BLEND>(hd[l], ha[l], ld[l][0], ld[l][1], ld[l][2], ld[l][3],
                                                               la[l][0], la[l][1], la[l][2], la[l][3], tol, nfs));
            c[0] += 1;
            c[1] += ((codes >> (16 * l)) & 0xffffu) != want;
        }
    }
    flush(out, c, 3);
}

#define CK(x)                                                                                           \
    do {                                                                                                \
        cudaError_t e_ = (x);                                                                           \
        if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(2); }   \
    } while (0)

struct Timer {
    cudaEvent_t a, b;
    Timer() { CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b)); CK(cudaEventRecord(a)); }
    float ms() { CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); float t; CK(cudaEventElapsedTime(&t, a, b)); return t; }
};

}  // namespace probe

int main(int argc, char **argv)
{
    const uint32_t seed = argc > 1 ? (uint32_t)strtoul(argv[1], nullptr, 0) : 20261016u;
    const auto t0 = std::chrono::steady_clock::now();
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int drv = 0, rtv = 0;
    CK(cudaDriverGetVersion(&drv));
    CK(cudaRuntimeGetVersion(&rtv));
    printf("DEVICE %s sm_%d%d driver_api=%d runtime=%d\n", prop.name, prop.major, prop.minor, drv, rtv);
    const int blocks = prop.multiProcessorCount * 8, threads = 256;
    unsigned long long *dc;
    CK(cudaMalloc(&dc, 64 * sizeof(unsigned long long)));
    CK(cudaMemset(dc, 0, 64 * sizeof(unsigned long long)));
    unsigned long long *c1 = dc, *c2 = dc + 8, *c3 = dc + 16, *c3r = dc + 32, *c4 = dc + 40, *c4b = dc + 48;

    { Timer t; part1_kernel<<<blocks, threads>>>(c1); CK(cudaGetLastError()); printf("WALL part1 %.1f\n", t.ms()); }
    { Timer t; part2_kernel<<<blocks, threads>>>(c2); CK(cudaGetLastError()); printf("WALL part2 %.1f\n", t.ms()); }
    { Timer t; part3_exhaustive_kernel<<<blocks, threads>>>(c3); CK(cudaGetLastError()); printf("WALL part3_exhaustive %.1f\n", t.ms()); }
    // 2^31 draws of two pairs
    { Timer t; part3_random_kernel<<<blocks, threads>>>(1ull << 31, seed, c3r); CK(cudaGetLastError()); printf("WALL part3_random %.1f\n", t.ms()); }

    const Tols tols{{0x1p-55f, 1e-12f, 0.1f}, {0x1p-52f, 0x1.fffffep57f}};
    for (float tol : tols.tol)
        for (float nfs : tols.nfs)
            if (!upsample_fast_div_ok(tol, nfs)) { printf("ERROR tol %g nfs %g outside upsample_fast_div_ok\n", tol, nfs); return 3; }
    const uint64_t calls = 1ull << 31;                                   // two lanes each: 2^32 operand sets per BLEND
    { Timer t; part4_kernel<false><<<blocks, threads>>>(calls, seed + 1, tols, c4); CK(cudaGetLastError()); printf("WALL part4_blend0 %.1f\n", t.ms()); }
    { Timer t; part4_kernel<true><<<blocks, threads>>>(calls, seed + 2, tols, c4b); CK(cudaGetLastError()); printf("WALL part4_blend1 %.1f\n", t.ms()); }
    CK(cudaDeviceSynchronize());

    unsigned long long h[64];
    CK(cudaMemcpy(h, dc, sizeof h, cudaMemcpyDeviceToHost));
    report("in_safe_range", 1ull << 32, h[0]);
    report("in_safe_range_neg", 1ull << 32, h[1]);
    report("pair_guard", h[4], h[2]);
    printf("COUNT in_range %llu\n", h[3]);
    report("rcp_fast", kSafeCount, h[8]);
    report("rcp2_fast_neg.x", kSafeCount, h[9]);
    report("rcp2_fast_neg.y", kSafeCount, h[10]);
    report("ieee_rcp", kSafeCount, h[11]);
    const char *an[3] = {"1", "3", "9"};
    for (int k = 0; k < 3; k++) {
        char n[64];
        snprintf(n, sizeof n, "div_fast.a%s", an[k]); report(n, kSafeCount, h[16 + 3 * k]);
        snprintf(n, sizeof n, "div2_fast_neg.x.a%s", an[k]); report(n, kSafeCount, h[17 + 3 * k]);
        snprintf(n, sizeof n, "div2_fast_neg.y.a%s", an[k]); report(n, kSafeCount, h[18 + 3 * k]);
    }
    report("ieee_div.a1_3_9", 3 * kSafeCount, h[25]);
    report("div_fast.random", h[32], h[33]);
    report("div2_fast_neg.x.random", h[32], h[34]);
    report("div2_fast_neg.y.random", h[32], h[35]);
    report("ieee_div.random", h[32], h[36]);
    report("bilateral2.blend0", h[40], h[41]);
    printf("COUNT bilateral2.blend0.fallback %llu\n", h[42]);
    report("bilateral2.blend1", h[48], h[49]);
    printf("COUNT bilateral2.blend1.fallback %llu\n", h[50]);
    CK(cudaFree(dc));
    printf("WALL total %.1f\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    return 0;
}
#endif
