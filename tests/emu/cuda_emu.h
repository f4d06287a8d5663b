// cuda_emu.h -- a minimal HOST stand-in for the CUDA constructs used by miniengineao_b200/csrc/*.cu.
//
// TEST INFRASTRUCTURE ONLY.  With -DMEAO_EMULATE the kernel sources are compiled by g++ into tests/emu/libmeao_emu.so,
// where every CTA runs as 256 cooperative fibers (ucontext) that switch at __syncthreads().  The CPU test-suite uses it
// to check the LOGIC of the kernels -- indexing, tiling, border handling, operation order, the variants' plumbing --
// against the oracle without a GPU.  It is never built into, linked with or loaded by libmeao.so: the product has no CPU
// path (include/meao.h), and nothing outside tests/ may use this directory.
//
// What is and is not emulated: fp32 arithmetic is IEEE on both sides, so results are bit-comparable; MUFU.RCP keeps the
// flush-to-zero behaviour of rcp.approx.ftz.f32 but returns the correctly rounded reciprocal in between (the refinement steps
// that follow make the quotient exact from any start within an ulp or two -- on the GPU tests/test_fast_div_exhaustive_gpu.py
// checks that for the real MUFU on every in-range operand); TMA box loads are emulated as synchronous copies with
// zero fill (mbarriers become no-ops), so both the TMA path and the gather path of every kernel can be run; timing, occupancy and memory behaviour mean nothing here.
#pragma once

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <functional>

// ---- qualifiers --------------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __grid_constant__
#define __restrict__
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static

// ---- vector types ---------------------------------------------------------------------------------------------------
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
struct uint3 { uint32_t x, y, z; };
struct dim3 { uint32_t x, y, z; dim3(uint32_t x_ = 1, uint32_t y_ = 1, uint32_t z_ = 1) : x(x_), y(y_), z(z_) {} };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

// ---- runtime bits the launchers touch -------------------------------------------------------------------------------------
typedef int cudaError_t;
typedef void *cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1 };
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
// a 2-D tiled tensor map, reduced to what cp.async.bulk.tensor.2d needs (cuTensorMapEncodeTiled's arguments)
struct alignas(64) CUtensorMap { const void *base; int elem, w, h; size_t pitch_bytes; int bw, bh; uint64_t pad_[3]; };

// ---- built-in variables + the fiber scheduler (tests/emu/emu_runtime.cpp) -------------------------------------------------------
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
namespace meao_emu {
void launch(dim3 grid, dim3 block, size_t dynamic_smem_bytes, const std::function<void()> &thread_body);
void syncthreads();
void *dynamic_smem();
[[noreturn]] void unsupported(const char *what);
extern long long tma_box_loads;      // number of emulated cp.async.bulk.tensor loads so far (tests assert the TMA branch really ran)
// The launch ledger: per kernel launched since the last reset, its address relative to the library's load base, its launch count,
// the TMA box loads issued during its launches and the CTAs of their grids (a persistent upsample grid is one wave of CTAs whatever
// its tile count; any other grid has one CTA per tile).  The emulated MEAO_LAUNCH (kernels.h) reports each kernel through note_launch
// just before its launch.  ledger_read fills up to cap entries and returns the number of kernels.
void ledger_reset();
int ledger_read(unsigned long long *offset, long long *launches, long long *tma_loads, long long *ctas, int cap);
}
inline void __syncthreads() { meao_emu::syncthreads(); }

// ---- fp16 (x86-64 GCC >= 12: _Float16 conversions are IEEE round-to-nearest-even) -------------------------------------------------
struct __half { _Float16 v; };
struct __half2 { __half x, y; };
inline __half __float2half_rn(float f) { return __half{(_Float16)f}; }
inline float __half2float(__half h) { return (float)h.v; }
inline __half2 __floats2half2_rn(float a, float b) { return __half2{__float2half_rn(a), __float2half_rn(b)}; }
inline float2 __half22float2(__half2 h) { return float2{__half2float(h.x), __half2float(h.y)}; }

// ---- scalar intrinsics (compile with -ffp-contract=off: nothing fuses unless the source says fmaf) -----------------------------------
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __saturatef(float x) { return x > 0.0f ? (x < 1.0f ? x : 1.0f) : 0.0f; }      // NaN -> +0, like .sat
inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
template <class T> inline T __ldg(const T *p) { return *p; }
using std::max;
using std::min;

namespace meao_emu {
// rcp.approx.ftz.f32 (PTX ISA): a subnormal operand counts as a zero of its sign (so its reciprocal is +-inf), a subnormal
// result flushes to a zero of its sign, +-inf -> +-0 and NaN -> NaN.  Between those edges the result here is correctly rounded;
// the hardware's approximation error is not modelled -- the exhaustive fast-division test checks it on the GPU.  So a range
// guard that lets a subnormal, zero or infinite operand into a fast path gives wrong results here as it does on the H100.
inline float rcp_approx(float x)
{
    if (std::fpclassify(x) == FP_SUBNORMAL) x = std::copysign(0.0f, x);
    const float r = (float)(1.0 / (double)x);
    return std::fpclassify(r) == FP_SUBNORMAL ? std::copysign(0.0f, r) : r;
}
// cp.async.bulk.tensor.2d (tiled, no swizzle): box whose first element is (x, y); out-of-bounds elements are zero-filled.
// Synchronous here: the issuing fiber (thread 0) runs before the others in every barrier phase, so the data is in place
// when they pass the (no-op) mbarrier wait.  Like the hardware, refuse a start coordinate that is not 16-byte aligned
// (DESIGN.md 2.4: the measured "illegal instruction").
inline void tma_load_2d(void *dst, const CUtensorMap *m, int x, int y)
{
    if (((long long)x * m->elem) % 16 != 0) unsupported("TMA start coordinate not 16-byte aligned (faults on the GPU)");
    if (((uintptr_t)dst) % 128 != 0) unsupported("TMA shared-memory destination not 128-byte aligned (misaligned-address fault on the GPU)");
    tma_box_loads++;
    for (int by = 0; by < m->bh; by++)
        for (int bx = 0; bx < m->bw; bx++) {
            char *d = (char *)dst + ((size_t)by * m->bw + bx) * m->elem;
            const int sx = x + bx, sy = y + by;
            if (sx >= 0 && sy >= 0 && sx < m->w && sy < m->h) memcpy(d, (const char *)m->base + (size_t)sy * m->pitch_bytes + (size_t)sx * m->elem, m->elem);
            else memset(d, 0, m->elem);
        }
}
}
