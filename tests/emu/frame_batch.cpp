// frame_batch.cpp -- batches (meao_render_arrays_batch / meao_render_batch) through the HOST-compiled kernel sources (TEST
// INFRASTRUCTURE ONLY, see cuda_emu.h).  Built by batch.py into libmeao_emu_batch.so together with the batch kernels' translation units
// (build.py BATCH_SOURCES), linked against libmeao_emu.so: every other kernel, the surface-access counter and the launch ledger are that
// library's.  A frame is launched the way libmeao launches it: the frame schedule, argument blocks and launcher choice of
// csrc/frame_record.h (launch_entry_batch), with the list in FrameIO.batch.
#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

extern "C" {

// An array batch on the frame `h` of frame_driver.cpp's frame_create (its frame type derives from FrameState, first and only base, so
// the handle is the FrameState).  Layer l reads depth[l], an emulated array of shape depth_shape[l] (0 2-D, 1 layered of one layer) of
// dw[l] x dh[l] elements (4 bytes: f32, 2 bytes: D16 codes) with rows dpitch[l] bytes apart, and writes ao[l] (1 byte per texel) likewise.
// The caller keeps every array at least W x H, as meao_api.cu check_batch_array does.
void frame_run_arrays_batch(void *h, int kind, void *const *depth, const int *depth_shape, const int *dw, const int *dh, const long long *dpitch,
                            void *const *ao, const int *ao_shape, const int *aw, const int *ah, const long long *apitch)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;                                     // the whole frame, as every batch
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    const int L = f.layers;
    std::vector<meao_emu::Surface> ds(L), as(L);
    std::unique_ptr<BatchIO> io(new BatchIO);
    io->arrays = true;
    auto surf_kind = [](int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : kSurfLayered; };
    for (int l = 0; l < L; l++) {
        ds[l] = meao_emu::Surface{depth[l], (int)depth_esize(kind), dw[l], dh[l], 1, (size_t)dpitch[l], depth_shape[l]};
        as[l] = meao_emu::Surface{ao[l], 1, aw[l], ah[l], 1, (size_t)apitch[l], ao_shape[l]};
        io->depth.e[l] = BatchSurf{(cudaSurfaceObject_t)&ds[l], surf_kind(depth_shape[l])};
        io->ao.e[l] = BatchSurf{(cudaSurfaceObject_t)&as[l], surf_kind(ao_shape[l])};
    }
    FrameIO fio;
    fio.kind = kind; fio.depth = depth_in(f, nullptr, kind);
    fio.batch = io.get();
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) launch_entry_batch(f, l, fio, -1, nullptr);
}

// A pointer batch (the fused frame of meao_render_batch) on the frame `h`: layer l reads depth[l], rows depth_row[l] bytes apart, and
// writes ao[l], rows ao_row[l] bytes apart.  The caller keeps the views apart, as meao_api.cu prepare_batch_pointers does.
void frame_run_pointers_batch(void *h, int kind, const void *const *depth, const long long *depth_row, void *const *ao, const long long *ao_row)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    std::unique_ptr<BatchIO> io(new BatchIO);
    for (int l = 0; l < f.layers; l++)
        io->ptr.e[l] = BatchPtr{depth[l], (uint8_t *)ao[l], (int)(depth_row[l] / depth_esize(kind)), (int)ao_row[l]};
    FrameIO fio;
    fio.kind = kind; fio.depth = depth_in(f, nullptr, kind);
    fio.low_only = fio.fused = true;
    fio.batch = io.get();
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) launch_entry_batch(f, l, fio, -1, nullptr);
}

// The batch kernels' units as this library builds them (kernels.h kBatchKernelUnits, which only libmeao lists): file names 32 bytes
// apart in names, kernel counts in counts; returns the number of units.
int frame_batch_kernel_units(char *names, int *counts, int cap)
{
    static const KernelUnit *const units[] = {&kPrepareDepthArrayBatchUnit, &kBlurUpsampleArrayBatchUnit, &kPrepareDepthBatchUnit,
                                              &kBlurUpsampleLinBatchUnit};
    int n = 0;
    for (const KernelUnit *u : units) {
        if (n >= cap) break;
        std::snprintf(names + 32 * n, 32, "%s", u->file);
        counts[n++] = u->walk(nullptr);
    }
    return n;
}

}  // extern "C"
