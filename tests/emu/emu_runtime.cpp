// emu_runtime.cpp -- fiber scheduler behind tests/emu/cuda_emu.h (TEST INFRASTRUCTURE ONLY, see that header).
// One CTA at a time; its threads are ucontext fibers resumed round-robin, each running until it reaches __syncthreads()
// or returns, so one sweep over the live fibers is one barrier phase.
#include "cuda_emu.h"

#include <dlfcn.h>
#include <ucontext.h>
#include <map>
#include <vector>

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;

namespace meao_emu {
long long tma_box_loads = 0;
namespace {
constexpr size_t kStack = 256 * 1024;
struct Fiber { ucontext_t ctx; bool done; char *stack; };
std::vector<Fiber> g_fibers;
ucontext_t g_sched;
int g_current = -1;
const std::function<void()> *g_body = nullptr;
alignas(128) unsigned char g_dynamic_smem[64 * 1024];
// the launch ledger: kernel address relative to its library's load base -> its launches, the TMA box loads issued during them and the
// CTAs of their grids.  The kernels live in anonymous namespaces and have no dynamic symbols, so the test suite names them from the
// library's symbol table (nm).
struct LedgerEntry { long long launches, tma, ctas; };
std::map<uintptr_t, LedgerEntry> g_ledger;
uintptr_t g_next_kernel = 0;         // note_launch's kernel, the next launch's (0: none reported)

void trampoline()
{
    (*g_body)();
    g_fibers[g_current].done = true;
    swapcontext(&g_fibers[g_current].ctx, &g_sched);
}
}  // namespace

void *dynamic_smem() { return g_dynamic_smem; }

void syncthreads()
{
    const int me = g_current;
    swapcontext(&g_fibers[me].ctx, &g_sched);      // back to the scheduler; resumed in the next phase
}

void unsupported(const char *what)
{
    fprintf(stderr, "meao_emu: %s is not emulated (the emulator must run the kernels' non-TMA path)\n", what);
    abort();
}

void note_launch(const void *kernel)
{
    Dl_info info{};
    if (!kernel || !dladdr(kernel, &info) || !info.dli_fbase) unsupported("a launch of a kernel outside any loaded library");
    g_next_kernel = (uintptr_t)kernel - (uintptr_t)info.dli_fbase;
}

void launch(dim3 grid, dim3 block, size_t dynamic_smem_bytes, const std::function<void()> &body)
{
    const uintptr_t kernel = g_next_kernel;
    g_next_kernel = 0;
    const long long tma0 = tma_box_loads;
    if (dynamic_smem_bytes > sizeof g_dynamic_smem) unsupported("more than 64 KB of dynamic shared memory");
    const int n = (int)(block.x * block.y * block.z);
    if ((int)g_fibers.size() < n) {
        const size_t old = g_fibers.size();
        g_fibers.resize(n);
        for (size_t i = old; i < g_fibers.size(); i++) g_fibers[i].stack = (char *)malloc(kStack);
    }
    gridDim = grid; blockDim = block;
    g_body = &body;
    for (uint32_t bz = 0; bz < grid.z; bz++)
    for (uint32_t by = 0; by < grid.y; by++)
    for (uint32_t bx = 0; bx < grid.x; bx++) {
        blockIdx = uint3{bx, by, bz};
        for (int t = 0; t < n; t++) {
            Fiber &f = g_fibers[t];
            f.done = false;
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = f.stack;
            f.ctx.uc_stack.ss_size = kStack;
            f.ctx.uc_link = nullptr;
            makecontext(&f.ctx, trampoline, 0);
        }
        bool live = true;
        while (live) {
            live = false;
            for (int t = 0; t < n; t++) {
                if (g_fibers[t].done) continue;
                threadIdx = uint3{(uint32_t)t % block.x, ((uint32_t)t / block.x) % block.y, (uint32_t)t / (block.x * block.y)};
                g_current = t;
                swapcontext(&g_sched, &g_fibers[t].ctx);
                if (!g_fibers[t].done) live = true;
            }
        }
    }
    g_body = nullptr;
    g_current = -1;
    if (kernel) {
        LedgerEntry &e = g_ledger[kernel];
        e.launches++;
        e.tma += tma_box_loads - tma0;
        e.ctas += (long long)grid.x * grid.y * grid.z;
    }
}

void ledger_reset() { g_ledger.clear(); }

int ledger_read(unsigned long long *offset, long long *launches, long long *tma_loads, long long *ctas, int cap)
{
    int n = 0;
    for (const auto &kv : g_ledger) {
        if (n < cap) { offset[n] = kv.first; launches[n] = kv.second.launches; tma_loads[n] = kv.second.tma; ctas[n] = kv.second.ctas; }
        n++;
    }
    return n;
}

}  // namespace meao_emu
