// frame_views.cpp -- CUDA-array viewport frames (meao_render_arrays_at) through the HOST-compiled kernel sources (TEST INFRASTRUCTURE
// ONLY, see cuda_emu.h).  Built by views.py into libmeao_emu_views.so, which links against libmeao_emu.so: the kernels, their launchers,
// the surface-access counter and the launch ledger are that library's, so a viewport frame is counted and recorded like every other.
// A frame is launched the way libmeao launches it: the frame schedule, argument blocks and launcher choice of csrc/frame_record.h, with
// the viewport origins in ArrayIO.
#include <cstdint>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

extern "C" {

// A CUDA-array frame of viewports on the frame `h` of frame_driver.cpp's frame_create (its frame type derives from FrameState, first
// and only base, so the handle is the FrameState).  depth: an emulated array of shape depth_shape (0 2-D, 1 layered, 2 cube) of
// `layers` images of depth_w x depth_h elements (4 bytes: f32, 2 bytes: D16 codes) with rows depth_pitch bytes apart, read at texels
// [depth_x, depth_x + W) x [depth_y, depth_y + H); ao: the same for the AO (1 byte per texel), written at (ao_x, ao_y).  The caller
// keeps the viewports inside the arrays, as meao_api.cu check_array does; a texel outside an array would be dropped, not wrapped.
// Render tiles follow the planner's rule.
void frame_run_arrays_at(void *h, void *depth, int kind, int depth_shape, int depth_w, int depth_h, long long depth_pitch, int depth_x,
                         int depth_y, void *ao, int ao_shape, int ao_w, int ao_h, long long ao_pitch, int ao_x, int ao_y)
{
    FrameState &f = *static_cast<FrameState *>(h);
    f.band0 = 0; f.band1 = f.H;                                     // the whole frame, as every array frame
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    const int L = f.layers;
    const meao_emu::Surface ds{depth, (int)depth_esize(kind), depth_w, depth_h, depth_shape == 2 ? 6 : L, (size_t)depth_pitch, depth_shape};
    const meao_emu::Surface as{ao, 1, ao_w, ao_h, ao_shape == 2 ? 6 : L, (size_t)ao_pitch, ao_shape};
    // what meao_api.cu check_array derives from an array: how the kernels address its layers
    auto surf_kind = [](int shape) { return shape == meao_emu::SURF_2D ? kSurf2D : shape == meao_emu::SURF_LAYERED ? kSurfLayered : kSurfCube; };
    ArrayIO aio{(cudaSurfaceObject_t)&ds, (cudaSurfaceObject_t)&as, surf_kind(depth_shape), surf_kind(ao_shape), ao};
    aio.depth_x = depth_x; aio.depth_y = depth_y; aio.ao_x = ao_x; aio.ao_y = ao_y;
    FrameIO io;
    io.kind = kind; io.depth = depth_in(f, nullptr, kind);
    io.aio = &aio;
    for (const FrameLaunch &l : frame_schedule(f.plan.variants)) launch_entry(f, l, io, -1, nullptr);
}

}  // extern "C"
