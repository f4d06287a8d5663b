// halo.cu -- pack / unpack of the LowDepth border rows exchanged between neighbouring row bands
// (SURVEY.md 8e): up to 8 row blocks (4 levels x 2 sides) move in ONE launch, so a band step is
// two graph launches plus one neighbour send/recv.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

__global__ void __launch_bounds__(256) halo_copy_kernel(const HaloArgs a)
{
#ifdef MEAO_DEVICE_OK
    const HaloSeg s = a.seg[blockIdx.y];
    const int n = s.rows * s.width;
    pdl_wait();                     // the pack reads rows prepare_depth (the preceding grid) has just written
    pdl_launch_dependents();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = i / s.width, c = i - r * s.width;
        s.dst[(size_t)r * s.dst_pitch + c] = s.src[(size_t)r * s.src_pitch + c];
    }
#endif
}

const Kernel<HaloArgs> kKernels[] = {halo_copy_kernel};

}  // namespace

cudaError_t launch_halo_copy(const HaloArgs &a, cudaStream_t s)
{
    if (a.nseg <= 0) return cudaSuccess;
    int maxn = 0;
    for (int i = 0; i < a.nseg; i++) maxn = max(maxn, a.seg[i].rows * a.seg[i].width);
    dim3 grid(min(ceil_div(maxn, 256), 64), a.nseg);
    MEAO_LAUNCH((halo_copy_kernel), grid, 256, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kHaloUnit = {"halo.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
