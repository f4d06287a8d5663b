// frame_layer_views.cpp -- layered CUDA-array frames with a layer-viewport table (meao_set_layer_viewports) through the HOST-compiled
// kernel sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  Built by layer_views.py into libmeao_emu_layer_views.so together with the
// table kernels' translation units (build.py VIEW_SOURCES), linked against libmeao_emu.so: every other kernel, the surface-access
// counter and the launch ledger are that library's.  A frame is launched the way libmeao launches it: the frame schedule, argument
// blocks and launcher choice of csrc/frame_record.h (launch_entry_views), with the table in FrameIO.views.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

extern "C" {

// A layered array frame with a viewport table on the frame `h` of frame_driver.cpp's frame_create (its frame type derives from
// FrameState, first and only base, so the handle is the FrameState).  depth: an emulated array of shape depth_shape (0 2-D, 1 layered,
// 2 cube) of depth_layers images of depth_w x depth_h elements (4 bytes: f32, 2 bytes: D16 codes) with rows depth_pitch bytes apart;
// ao: the same for the AO (1 byte per texel).  views: the frame's L table entries (kernels.h LayerView), which the caller keeps inside
// the arrays as meao_api.cu check_view_fit / check_ao_disjoint do; a texel outside an array would be dropped, not wrapped.
void frame_run_arrays_views(void *h, void *depth, int kind, int depth_shape, int depth_w, int depth_h, int depth_layers, long long depth_pitch,
                            void *ao, int ao_shape, int ao_w, int ao_h, int ao_layers, long long ao_pitch, const int *views)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;                                     // the whole frame, as every array frame
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    const meao_emu::Surface ds{depth, (int)depth_esize(kind), depth_w, depth_h, depth_layers, (size_t)depth_pitch, depth_shape};
    const meao_emu::Surface as{ao, 1, ao_w, ao_h, ao_layers, (size_t)ao_pitch, ao_shape};
    auto surf_kind = [](int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : shape == meao_emu::SURF_LAYERED ? kSurfLayered : kSurfCube; };
    ArrayIO aio{(cudaSurfaceObject_t)&ds, (cudaSurfaceObject_t)&as, surf_kind(depth_shape), surf_kind(ao_shape), ao};
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, nullptr, kind);
    io.aio = &aio;
    io.views = reinterpret_cast<const LayerView *>(views);
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) launch_entry_views(f, l, io, -1, nullptr);
}

// A fused pointer frame with a viewport table (meao_render_pitched with a table set) on the frame `h`: depth rows depth_row bytes and
// slices depth_layer bytes apart from `depth`, the AO likewise from `ao`, layer l at the rectangles and slices of views[l].  The caller
// keeps the rectangles inside the buffers, as meao_api.cu check_view_pitches does.
void frame_run_pitched_views(void *h, const void *depth, int kind, long long depth_row, long long depth_layer, void *ao, long long ao_row,
                             long long ao_layer, const int *views)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    const ViewPitch vp{depth_row, depth_layer, ao_row, ao_layer};
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, depth, kind, &vp);
    io.low_only = io.fused = true; io.ao = ao; io.vp = &vp;
    io.views = reinterpret_cast<const LayerView *>(views);
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) launch_entry_views(f, l, io, -1, nullptr);
}

// The table kernels' units as this library builds them (kernels.h kViewKernelUnits, which only libmeao lists): file
// names 32 bytes apart in names, kernel counts in counts; returns the number of units.
int frame_view_kernel_units(char *names, int *counts, int cap)
{
    static const KernelUnit *const units[] = {&kPrepareDepthArrayViewsUnit, &kBlurUpsampleArrayViewsUnit, &kPrepareDepthViewsUnit,
                                              &kBlurUpsampleLinViewsUnit};
    int n = 0;
    for (const KernelUnit *u : units) {
        if (n >= cap) break;
        std::snprintf(names + 32 * n, 32, "%s", u->file);
        counts[n++] = u->walk(nullptr);
    }
    return n;
}

}  // extern "C"
