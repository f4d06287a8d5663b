// band_exchange.cu -- the neighbour exchange of the row-band partition (SURVEY.md 8e) as ONE kernel inside the frame's graph.
//
// The pass list being partitioned is AmbientOcclusion.cs:511-531; its vertical dependency radii (Render.compute:162-168,
// Upsample.compute:89-146,213-232) make every band need <= ~24 border rows of LowDepth1..4 from each neighbour
// (meao_api.cu::compute_needs).  All band contexts keep those buffers in full-frame global coordinates with identical arena
// layouts, so "send my border rows" is: copy the rows to the SAME offset in the neighbour's arena through a peer mapping
// (NVLink stores; cudaIpc across processes, peer access within one), no pack / staging / unpack.
//
// Protocol (epoch e = 1, 2, ... counted on the device, so the captured graph replays unchanged):
//   1. every CTA announces to both neighbours "I am at epoch e" (ack): all kernels of this context's epoch e-1 have
//      completed (stream order), so the halo rows it RECEIVED may be overwritten;
//   2. a copying CTA waits until the neighbour it writes to has announced epoch >= e, copies its slice with 128-bit
//      stores, and fences at system scope;
//   3. the last CTA to finish publishes ready = e to both neighbours (st.release.sys) and then waits until both
//      neighbours' rows of epoch e have landed here (ld.acquire.sys) -- so when this grid completes, the render and
//      upsample kernels that follow it in the graph see their halo rows.
// No dependency cycle: step 1 of a context depends on nothing; step 2 only on the neighbour's step 1; step 3 only on the
// neighbour's step 2.  Every wait is bounded by a time-out that sets a sticky error instead of hanging the GPU.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

constexpr int kXchgThreads = 256;
constexpr int kXchgCtasPerSeg = 12;        // <= 96 CTAs in total: the spinning grid can never fill the GPU (no scheduling deadlock
                                           // with the neighbour band's kernels when two bands share a device, as in the tests)

__device__ __forceinline__ bool spin_until_ge(const uint32_t *flag, uint32_t e, unsigned long long timeout_ns)
{
    if (ld_acquire_sys(flag) >= e) return true;
    const unsigned long long t0 = global_timer_ns();
    for (;;) {
#pragma unroll 1
        for (int i = 0; i < 64; i++)
            if (ld_acquire_sys(flag) >= e) return true;
        if (global_timer_ns() - t0 > timeout_ns) return false;
    }
}

__global__ void __launch_bounds__(kXchgThreads) band_exchange_kernel(const XchgArgs a)
{
#ifdef MEAO_DEVICE_OK
    __shared__ uint32_t s_epoch, s_ok;
    const int tid = threadIdx.x;
    const XchgSeg seg = a.seg[blockIdx.y];
    BandFlags *fl = a.local;
    pdl_wait();                     // the rows copied below are written by prepare_depth, the preceding grid
    if (tid == 0) {
        const uint32_t e = *(volatile uint32_t *)&fl->epoch;        // stable: only the last CTA of this grid advances it
        bool ok = *(volatile uint32_t *)&fl->error == 0;
        // 1. announce (idempotent, every CTA: no CTA of the neighbour depends on a particular CTA of this grid being scheduled)
        if (a.peer[0]) st_release_sys(&a.peer[0]->ack[1], e);
        if (a.peer[1]) st_release_sys(&a.peer[1]->ack[0], e);
        // 2. the neighbour this CTA writes to must have consumed epoch e-1
        if (ok && !spin_until_ge(&fl->ack[seg.side], e, a.timeout_ns)) {
            ok = false; atomic_max_u32(&fl->error, 1u);
            if (a.host_error) *(volatile uint32_t *)a.host_error = 1u;
        }
        s_epoch = e; s_ok = ok ? 1u : 0u;
    }
    __syncthreads();
    if (s_ok) {
        for (uint32_t i = blockIdx.x * kXchgThreads + tid; i < seg.n16; i += gridDim.x * kXchgThreads) seg.dst[i] = seg.src[i];
    }
    threadfence_system();
    __syncthreads();
    if (tid == 0) {
        const uint32_t total = gridDim.x * gridDim.y;
        if (atomic_add_u32(&fl->done, 1u) == total - 1) {           // last CTA: every other CTA's stores are fenced
            const uint32_t e = s_epoch;
            threadfence_system();
            *(volatile uint32_t *)&fl->done = 0;
            // 3. publish, then wait for the neighbours' rows
            if (a.peer[0]) st_release_sys(&a.peer[0]->ready[1], e);
            if (a.peer[1]) st_release_sys(&a.peer[1]->ready[0], e);
            bool ok = *(volatile uint32_t *)&fl->error == 0;
            for (int side = 0; side < 2; side++)
                if (a.peer[side] && ok && !spin_until_ge(&fl->ready[side], e, a.timeout_ns)) {
                    ok = false; atomic_max_u32(&fl->error, 2u);
                    if (a.host_error) *(volatile uint32_t *)a.host_error = 2u;
                }
            *(volatile uint32_t *)&fl->epoch = e + 1;
            threadfence_system();
        }
    }
#endif
}

const Kernel<XchgArgs> kKernels[] = {band_exchange_kernel};

}  // namespace

cudaError_t launch_band_exchange(const XchgArgs &a, cudaStream_t s)
{
    if (a.nseg <= 0) return cudaSuccess;
    dim3 grid(kXchgCtasPerSeg, a.nseg);
    MEAO_LAUNCH((band_exchange_kernel), grid, kXchgThreads, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kBandExchangeUnit = {"band_exchange.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
