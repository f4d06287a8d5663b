// render_ao_ortho.cu -- render_ao.cu's kernels under an orthographic projection (meao_set_projection): render_ao_kernel.inc with
// MEAO_ORTHO 1, a sampling sphere of constant size.  RenderArgs.inv_thickness carries it_i = (far / ThicknessMultiplier) /
// SampleThickness[i] (meao_api.cu camera_consts); neg_front is not read.  A translation unit of its own (build.py ORTHO_SOURCES) so
// that render_ao.cu compiles to exactly the code it did before.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

#define MEAO_ORTHO 1
#define MEAO_LAYERED 0
#define render_ao_kernel render_ao_ortho_kernel
#include "render_ao_kernel.inc"
#undef render_ao_kernel
#undef MEAO_LAYERED
#undef MEAO_ORTHO

// [render_slot]
const Kernel<CUtensorMap, RenderArgs, int> kKernels[kRenderSlots] = MEAO_RENDER_SLOTS(render_ao_ortho_kernel);

}  // namespace

cudaError_t launch_render_ao_ortho(const CUtensorMap &low_map, bool use_tma, const RenderArgs &a, cudaStream_t s)
{
    if (a.row1 <= a.row0) return cudaSuccess;
    const int k = render_slot(a);
    if (k < 0) return cudaErrorInvalidValue;
    const int ybase = a.row0 & ~3;
    const dim3 grid(ceil_div(a.lw, kTW), ceil_div(a.row1 - ybase, a.tile_h));
    MEAO_LAUNCH((kKernels[k]), grid, kThreads, render_smem_bytes(a.tile_h, a.wide), s, low_map, a, use_tma ? 1 : 0);
    return cudaGetLastError();
}

const KernelUnit kRenderAoOrthoUnit = {"render_ao_ortho.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels); }};

}  // namespace meao
