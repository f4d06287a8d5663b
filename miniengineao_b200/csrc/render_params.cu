// render_params.cu -- the render stage's two frame parameters derived on the device from a parameter buffer in device memory
// (meao_bind_device_params), so that a frame recorded into a graph renders with whatever thickness and intensity the buffer holds when it
// is replayed.
//
// The block is {thickness_modifier, intensity}.  One thread tests it with meao_set_params's test (thickness_modifier > 0; NaN fails) and
// writes {reject_fadeoff, intensity} into the context's slot, which the *_params_layered render kernels read once per CTA.
// reject_fadeoff is the host planner's -1 / thickness_modifier (meao_api.cu build_plan): an IEEE division without flush-to-zero, so a
// subnormal or infinite thickness gives the host's bits.  An invalid block leaves the slot as it was and is counted in the status words
// (kernels.h RenderParamArgs).  A translation unit of its own (build.py PARAM_SOURCES): no other kernel changes.
#include "common.cuh"
#include "kernels.h"

namespace meao {

namespace {

__global__ void __launch_bounds__(32) render_params_kernel(const RenderParamArgs a)
{
#ifdef MEAO_DEVICE_OK
    if (threadIdx.x != 0) return;
    const float tm = a.params[0], intensity = a.params[1];
    if (!(tm > 0.0f)) {
        atomic_add_u32(&a.status[0], 1u);
        a.status[1] = 1;                        // the field: thickness_modifier
        return;
    }
    a.derived[0] = -1 / tm;                                                 // AO.cs:733
    a.derived[1] = intensity;                                               // AO.cs:734
#endif
}

const struct {
    Kernel<RenderParamArgs> derive;
} kKernels = {render_params_kernel};

}  // namespace

cudaError_t launch_render_params(const RenderParamArgs &a, cudaStream_t s)
{
    if (!a.params || !a.derived || !a.status) return cudaErrorInvalidValue;
    MEAO_LAUNCH((kKernels.derive), dim3(1), 32, 0, s, a);
    return cudaGetLastError();
}

const KernelUnit kRenderParamsUnit = {"render_params.cu", [](cudaError_t *load) { return walk_kernels(load, kKernels.derive); }};

}  // namespace meao
