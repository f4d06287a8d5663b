// frame_layers.cpp -- dynamic view counts (meao_reserve_layers) in the emulator (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  Built by
// tests/test_dynamic_layers_emulated.py into a library of its own, linked against libmeao_emu.so, whose frame_create makes the arena
// and whose frame_set_plan / frame_run / frame_get_buffer run the frames.  What this file adds is meao_api.cu's place_size under a
// layer reservation: a frame of W x H x L placed in an arena laid out for Wmax x Hmax x Lmax, with its camera tables in slot `slot` of
// the table region laid out for Lmax (arena_layout's table_layers).
#include <cstring>

#include "../../miniengineao_b200/csrc/common.cuh"
#include "../../miniengineao_b200/csrc/frame_record.h"

using namespace meao;

namespace {
// what meao_api.cu hands to cuTensorMapEncodeTiled (frame_driver.cpp's emu_map)
bool emu_map(CUtensorMap &m, const MapSpec &s)
{
    m = CUtensorMap{};
    m.base = s.base; m.elem = s.elem; m.w = s.w; m.h = s.h; m.pitch_bytes = (size_t)s.pitch_elems * s.elem; m.bw = s.bw; m.bh = s.bh;
    return true;
}
}  // namespace

extern "C" {

// Places a W x H x L frame in the arena of the frame `h` of frame_driver.cpp's frame_create (its frame type derives from FrameState,
// first and only base, so the handle is the FrameState).  The arena's base is where the tile counters sit minus their offset, which
// no size or layer count moves.  -1 if the frame does not fit an arena of `arena_bytes`.
int frame_place_layers(void *h, int W, int H, int L, int Lmax, int slot, long long arena_bytes)
{
    FrameState &f = *static_cast<FrameState *>(h);
    if (W < 1 || H < 1 || L < 1 || L > Lmax || slot < 0 || slot >= kSizeSlots) return -1;
    const ArenaLayout a = arena_layout(W, H, L, Lmax);
    if ((long long)a.bytes > arena_bytes) return -1;
    char *base = (char *)f.tile_ctr - arena_layout(1, 1, 1).ctr;
    f.W = W; f.H = H; f.layers = L;
    place_frame(f, a, base, slot);
    encode_maps(f, emu_map);
    f.band0 = 0; f.band1 = H;
    for (int k = 0; k <= 4; k++) f.need_c[k] = Range{0, f.lh[k]};
    return 0;
}

// The offsets of arena_layout(W, H, L, Lmax) that must not depend on W, H or L: out = {ctr, table0, table_stride, views, bytes}
void frame_layers_layout(int W, int H, int L, int Lmax, long long *out)
{
    const ArenaLayout a = arena_layout(W, H, L, Lmax);
    out[0] = (long long)a.ctr; out[1] = (long long)a.table0; out[2] = (long long)a.table_stride; out[3] = (long long)a.views;
    out[4] = (long long)a.bytes;
}

}  // extern "C"
