// arena_layout.h -- where every buffer of a context lives inside its one device allocation (the arena), as a pure function of the
// frame size and the layer count.  meao_api.cu lays out an arena with it and frame_record.h's place_frame places a frame's buffers
// by it -- in libmeao and in the emulator (tests/emu/frame_driver.cpp) alike.
//
// Order: BandFlags (offset 0 in every arena: the neighbour bands address it through their peer mapping), the tile counters of the
// persistent upsample grids, kSizeSlots per-layer camera table slots, the layer-viewport table, LinearDepth, the AO result, LowDepth / Occlusion / Combined /
// HighQuality of levels 1..4, and the two host-staging slots.  Every entry starts on a 256-byte boundary; rows start on 128-byte
// boundaries (pitches below).  Every entry's size is monotone in W and H, so the entries of a W' x H' frame with W' <= W and H' <= H
// lie inside the arena of W x H, each at an offset no larger than the W x H one (dynamic resolution, meao_reserve).  Every entry is
// monotone in L as well, and the camera table slots and the layer-viewport table are laid out for table_layers >= L layers: a context
// with a layer reservation (meao_reserve_layers) passes its maximum, so every (W, H, L) inside it finds the tables at the same offsets
// and its images inside the arena of (Wmax, Hmax, Lmax).
#ifndef MEAO_ARENA_LAYOUT_H
#define MEAO_ARENA_LAYOUT_H

#include <stddef.h>

namespace meao {

// Per-layer camera table slots in every arena: one per frame size a reserved context keeps planned (meao_reserve); an unreserved
// context uses slot 0.  Their offsets do not depend on the frame size.
constexpr int kSizeSlots = 8;

struct ArenaLayout {
    int lw[7], lh[7];                   // level sizes: ceil(W / 2^l) x ceil(H / 2^l) (AO.cs:276-281)
    int lin_pitch, result_pitch;        // elements (f16 / bytes)
    int low_pitch[5], occ_pitch[5];     // elements (f32 / bytes) of levels 1..4; comb and hq share occ_pitch
    size_t ctr;                         // 8 words: cursor + finished-CTA count of each persistent blur_upsample grid
    size_t table0, table_stride;        // slot s: LayerZ[L] at table0 + s * table_stride, then LayerRender[8 L] at table_ren below
    size_t table_ren;                   // offset of the LayerRender table inside a slot
    size_t views;                       // LayerView[L] (meao_set_layer_viewports): one table for every frame size
    size_t lin, result, low[5], occ[5], comb[4], hq[5];
    size_t depth_stage[2], ao_stage[2]; // L x W x H f32 (the largest depth element) and L x W x H bytes each
    size_t bytes;                       // the arena's size
};

inline int layout_align_up(int x, int a) { return (x + a - 1) / a * a; }

inline ArenaLayout arena_layout(int W, int H, int L, int table_layers)
{
    ArenaLayout a{};
    for (int l = 0; l < 7; l++) {
        const int div = 1 << l;
        a.lw[l] = (W + div - 1) / div;
        a.lh[l] = (H + div - 1) / div;
    }
    a.lin_pitch = layout_align_up(a.lw[0], 64);
    a.result_pitch = layout_align_up(a.lw[0], 128);
    // every image: L views of the same pitch, back to back ([L][h][pitch], kernels.h "layered frames")
    const size_t n = (size_t)L, nt = (size_t)(table_layers > L ? table_layers : L);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    take(sizeof(BandFlags));
    a.ctr = take(8 * sizeof(unsigned int));
    const size_t zb_bytes = (nt * sizeof(LayerZ) + 255) / 256 * 256, ren_bytes = 8 * nt * sizeof(LayerRender);
    a.table_ren = zb_bytes;
    a.table_stride = zb_bytes + (ren_bytes + 255) / 256 * 256;
    a.table0 = take(kSizeSlots * a.table_stride);
    a.views = take(nt * sizeof(LayerView));
    a.lin = take(n * a.lin_pitch * a.lh[0] * 2);
    a.result = take(n * a.result_pitch * a.lh[0]);
    for (int k = 1; k <= 4; k++) {
        a.low_pitch[k] = layout_align_up(a.lw[k], 32);
        a.occ_pitch[k] = layout_align_up(a.lw[k], 128);
        a.low[k] = take(n * a.low_pitch[k] * a.lh[k] * sizeof(float));
        a.occ[k] = take(n * a.occ_pitch[k] * a.lh[k]);
        if (k <= 3) a.comb[k] = take(n * a.occ_pitch[k] * a.lh[k]);
        a.hq[k] = take(n * a.occ_pitch[k] * a.lh[k]);
    }
    for (int i = 0; i < 2; i++) { a.depth_stage[i] = take(n * W * H * sizeof(float)); a.ao_stage[i] = take(n * W * H); }
    a.bytes = off;
    return a;
}

inline ArenaLayout arena_layout(int W, int H, int L) { return arena_layout(W, H, L, L); }

}  // namespace meao

#endif  // MEAO_ARENA_LAYOUT_H
