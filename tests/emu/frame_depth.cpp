// frame_depth.cpp -- the hierarchy depth (meao_set_hierarchy_depth) in the emulator (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  Built
// by depth.py into libmeao_emu_depth.so, which links against libmeao_emu.so.  Every emulated frame form hands its plan's variants to
// csrc/frame_record.h frame_schedule and reads the depth through effective_depth, so setting PlanVariants.levels on a frame of any
// front end (frame_driver.cpp, frame_ortho.cpp, frame_mixed.cpp, frame_batch.cpp, frame_device_cameras.cpp, ...) is all that is needed.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

extern "C" {

// The hierarchy depth of the frame `h` (frame_driver.cpp frame_create, whose frame type derives from FrameState, first and only base),
// as meao_api.cu build_plan plans it; frame_set_plan resets it to 4, so call it after every (re)load of the plan.
void frame_set_levels(void *h, int levels) { static_cast<FrameState *>(h)->plan.variants.levels = levels; }

// frame_schedule of variants4 = MeaoVariants {single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale} at hierarchy
// depth `levels`, with the camera stage when device_cameras: launch i as out5[5 i .. 5 i + 4] = stage, level, branch, wait, PDL class,
// and its meao_profile_frame name at names + 32 i.  Returns the count.
int frame_schedule_levels(const int *variants4, int levels, int device_cameras, int *out5, char *names, int cap)
{
    const PlanVariants v(MeaoVariants{variants4[0], variants4[1], variants4[2], variants4[3]}, levels);
    const std::vector<FrameLaunch> s = frame_schedule(v, device_cameras != 0);
    for (size_t i = 0; i < s.size() && (int)i < cap; i++) {
        const FrameLaunch &l = s[i];
        const int row[5] = {l.stage, l.level, l.branch, l.wait, l.pdl};
        memcpy(out5 + 5 * i, row, sizeof row);
        snprintf(names + 32 * i, 32, "%s", launch_name(l).c_str());
    }
    return (int)s.size();
}

}  // extern "C"
