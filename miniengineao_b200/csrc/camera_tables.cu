// camera_tables.cu -- the per-layer camera tables (kernels.h LayerZ / LayerRender) derived on the device from a camera buffer in device
// memory (meao_bind_device_cameras), so that a frame recorded into a graph reads whatever cameras the buffer holds when it is replayed.
//
// Every entry is computed with the host planner's operations in the host planner's order (meao_api.cu camera_consts, frame_record.h
// layer_render): f32 IEEE products, quotients and differences, the one fmaf of the atlas padding and its f16 rounding.  With the build's
// -fmad=false, IEEE division and no flush-to-zero, each entry is the bytes camera_tables() writes for the same camera.  The
// SampleThickness values come from a double sqrt on the host and are kernel arguments, in the render stage's call order.
//
// Eight threads per layer, one per LayerRender row (k = 1..4, narrow then wide: row r = 2 (k - 1) + wide); row 0 also writes LayerZ.
// A camera that fails meao_set_camera's tests leaves its layer's entries as they were; the grid's last CTA folds the frame's lowest
// invalid (layer, field) into the status words (kernels.h CameraTableArgs).
// A translation unit of its own (build.py CAMERA_SOURCES): no other kernel changes.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

constexpr int kCamThreads = 256;

__device__ __forceinline__ void camera_tables_body(const CameraTableArgs &a, const LayerProjections *proj)
{
    const int t = blockIdx.x * kCamThreads + threadIdx.x;
    const int l = t >> 3, r = t & 7;
    if (l < a.layers) {
        const float n = __ldg(&a.cams[3 * l]), f = __ldg(&a.cams[3 * l + 1]), tan = __ldg(&a.cams[3 * l + 2]);
        const int bad = !(n > 0) ? 1 : !(f > n) ? 2 : !(tan > 0) ? 3 : 0;
        if (bad) {
            if (r == 0) atomic_max_u32(&a.status[4], ~(uint32_t)(l * 4 + bad));    // the largest complement: the lowest (layer, field)
        } else {
            const bool ortho = proj ? layer_is_ortho(*proj, l) : a.ortho != 0;
            float zb0, zb1;
            if (!ortho) {
                const float fpn = f / n;
                if (a.reversed_z) { zb0 = fpn - 1; zb1 = 1; } else { zb0 = 1 - fpn; zb1 = fpn; }
            } else {
                const float q = n / f;
                if (a.reversed_z) { zb0 = q - 1; zb1 = 1; } else { zb0 = 1 - q; zb1 = q; }
            }
            if (r == 0) a.zb[l] = LayerZ{zb0, zb1};
            const int k = 1 + (r >> 1);
            const bool wide = r & 1;
            const int wl = wide ? k : k + 2;
            int src_w = a.lw[1];
#pragma unroll
            for (int j = 2; j <= 6; j++) if (wl == j) src_w = a.lw[j];          // constant indices: the argument block stays in the parameter bank
            float tm = 2 * tan * 10.0f / (float)src_w;                          // AO.cs:678
            if (wide) tm *= 2;                                                  // AO.cs:679 (!source.isTiled)
            if (a.stereo) tm *= 2;                                              // AO.cs:680
            const float irf = ortho ? f / tm : 1 / tm;                          // AO.cs:683
            float pad = 0.0f;
            if (k <= 2) {
                if (ortho) pad = a.reversed_z ? 1e5f : fmaf(zb0, 0.0f, zb1);
                else pad = a.reversed_z ? 1e5f : 1.0f / fmaf(zb0, 0.0f, zb1);
            }
            float x[12], y[12];
#pragma unroll
            for (int i = 0; i < 12; i++) {
                x[i] = i < a.n ? irf / a.thick[i] : 0.0f;                      // AO.cs:687-688, in call order
                y[i] = i < a.n ? -(x[i] - 0.5f) : 0.0f;                         // Render.compute:85
            }
            // the 128-byte LayerRender row: it_nf[12] as {x, y} pairs, pad, pad_[7] zero
            float4 *dst = reinterpret_cast<float4 *>(a.ren + (size_t)r * a.layers + l);
#pragma unroll
            for (int j = 0; j < 6; j++) dst[j] = make_float4(x[2 * j], y[2 * j], x[2 * j + 1], y[2 * j + 1]);
            dst[6] = make_float4(f16_round(pad), 0.0f, 0.0f, 0.0f);
            dst[7] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
    }
    // the last CTA to finish reports the frame's lowest invalid (layer, field) and resets the per-launch words: every other CTA has
    // fenced its atomics before counting itself finished
    __shared__ bool last;
    threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) last = atomic_add_u32(&a.status[5], 1u) == gridDim.x - 1;
    __syncthreads();
    if (last && threadIdx.x == 0) {
        const uint32_t m = atomic_add_u32(&a.status[4], 0u);
        if (m) { a.status[0] += 1; a.status[1] = ~m >> 2; a.status[2] = ~m & 3; }
        a.status[4] = 0;
        a.status[5] = 0;
    }
}

__global__ void __launch_bounds__(kCamThreads) camera_tables_kernel(const CameraTableArgs a)
{
#ifdef MEAO_DEVICE_OK
    camera_tables_body(a, nullptr);
#endif
}

__global__ void __launch_bounds__(kCamThreads) camera_tables_mixed_kernel(const CameraTableArgs a, const __grid_constant__ LayerProjections proj)
{
#ifdef MEAO_DEVICE_OK
    camera_tables_body(a, &proj);
#endif
}

const struct {
    Kernel<CameraTableArgs> uniform;
    Kernel<CameraTableArgs, LayerProjections> mixed;
} kKernels = {camera_tables_kernel, camera_tables_mixed_kernel};

}  // namespace

cudaError_t launch_camera_tables(const CameraTableArgs &a, const LayerProjections *proj, cudaStream_t s)
{
    if (a.layers < 1 || a.layers > kMaxLayers || !a.cams || !a.zb || !a.ren || !a.status || a.n < 1 || a.n > 12) return cudaErrorInvalidValue;
    const dim3 grid(ceil_div(8 * a.layers, kCamThreads));
    if (proj) MEAO_LAUNCH((kKernels.mixed), grid, kCamThreads, 0, s, a, *proj);
    else MEAO_LAUNCH((kKernels.uniform), grid, kCamThreads, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kCameraTablesUnit = {"camera_tables.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels.uniform, kKernels.mixed); }};

}  // namespace meao
