// drs_driver.cpp -- runs frames of several sizes inside ONE arena laid out for the largest (meao_reserve), through the host-compiled
// kernel sources (TEST INFRASTRUCTURE ONLY, see cuda_emu.h).  The frames are lin_driver.cpp's (fused) and layered_driver.cpp's (the
// whole-frame prepare_depth); what this driver adds is where the buffers live: before a frame of W x H the buffers are placed at the
// offsets and pitches arena_layout(W, H, L) gives -- the function meao_api.cu lays out its arena with -- inside an arena of
// arena_layout(Wmax, Hmax, L).bytes that still holds what larger frames (or a poison fill) left there.
#include "lin_driver.cpp"
#include "../../miniengineao_b200/csrc/arena_layout.h"

namespace {

struct DEmu : LEmu {
    char *arena = nullptr;
    size_t bytes = 0;
    int Wmax = 0, Hmax = 0;
};

DEmu *demu(void *h) { return static_cast<DEmu *>((LEmu *)h); }

}  // namespace

extern "C" {

void *demu_create(int Wmax, int Hmax, int layers)
{
    DEmu *d = new DEmu();
    d->L = layers; d->Wmax = Wmax; d->Hmax = Hmax;
    d->bytes = arena_layout(Wmax, Hmax, layers).bytes;
    void *p = nullptr;
    if (posix_memalign(&p, 256, d->bytes)) abort();
    memset(p, 0, d->bytes);
    d->arena = (char *)p;
    return (LEmu *)d;
}

void demu_destroy(void *h)
{
    DEmu *d = demu(h);
    free(d->arena);
    delete d;
}

size_t demu_arena_bytes(void *h) { return demu(h)->bytes; }

// every byte of the arena := fill
void demu_fill(void *h, int fill) { DEmu *d = demu(h); memset(d->arena, fill, d->bytes); }

// the buffers of a W x H frame, where meao_api.cu's place_size puts them; returns -1 if the size lies outside the arena's
int demu_resize(void *h, int W, int H)
{
    DEmu *d = demu(h);
    if (W < 1 || H < 1 || W > d->Wmax || H > d->Hmax) return -1;
    const ArenaLayout a = arena_layout(W, H, d->L);
    if (a.bytes > d->bytes) return -1;
    d->W = W; d->H = H;
    memcpy(d->lw, a.lw, sizeof d->lw);
    memcpy(d->lh, a.lh, sizeof d->lh);
    d->lin = (__half *)(d->arena + a.lin); d->lin_pitch = a.lin_pitch;
    d->result = (uint8_t *)(d->arena + a.result); d->result_pitch = a.result_pitch;
    for (int k = 1; k <= 4; k++) {
        d->low[k] = (float *)(d->arena + a.low[k]); d->low_pitch[k] = a.low_pitch[k];
        d->occ[k] = (uint8_t *)(d->arena + a.occ[k]); d->occ_pitch[k] = a.occ_pitch[k];
        d->hq[k] = (uint8_t *)(d->arena + a.hq[k]);
        if (k <= 3) d->comb[k] = (uint8_t *)(d->arena + a.comb[k]);
    }
    return 0;
}

}  // extern "C"
