// emu_runtime.cpp -- TEST-ONLY fiber scheduler behind tests/emu/cuda_shim.h.
// Every CUDA thread of the running block is a fiber on its own stack; fibers run
// until they reach a collective, the scheduler resolves a warp's collective once
// all 32 lanes have arrived with the same operation (strict: anything else aborts).
// jss_emu_set_schedule() picks the order in which ready fibers and blocks run and what
// shared and device memory hold before anything writes them (see README.md).
#include <setjmp.h>
#include <stdio.h>
#include <sys/mman.h>
#include <ucontext.h>

#include <vector>

#include "cuda_shim.h"

namespace emu {

thread_local dim3 threadIdx_, blockIdx_, blockDim_, gridDim_;
void *smem_ptr = nullptr;
int poison = -1;

namespace {
enum { READY = 0, WAITING = 1, DONE = 2 };
struct Fiber {
    ucontext_t ctx;
    jmp_buf jb;
    char *stack = nullptr;
    bool started = false;
    int state = READY;
    int op = 0;
    unsigned mask = 0;
    uint64_t value = 0, result = 0;
    int arg = 0;
};
constexpr size_t kStack = 256 * 1024;
std::vector<Fiber> fibers;
int cur = -1;
jmp_buf sched_jb;
ucontext_t sched_ctx;
void (*g_entry)(void *) = nullptr;
void *g_args = nullptr;
std::vector<char> smem_buf;
enum { ASCENDING = 0, DESCENDING = 1, SHUFFLED = 2 };
int sched_order = ASCENDING;
uint64_t sched_rng = 0;

uint64_t next_random() {   // splitmix64
    uint64_t z = (sched_rng += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// 0..n-1 in the order of the current schedule; a shuffle is drawn afresh on every call
void schedule_order(std::vector<int> &seq, int n) {
    seq.resize(n);
    for (int i = 0; i < n; i++) seq[i] = sched_order == DESCENDING ? n - 1 - i : i;
    if (sched_order == SHUFFLED)
        for (int i = n - 1; i > 0; i--) std::swap(seq[i], seq[next_random() % (uint64_t)(i + 1)]);
}

[[noreturn]] void die(const char *msg, int warp = -1) {
    fprintf(stderr, "[jss emu] FATAL: %s (block %u warp %d)\n", msg, blockIdx_.x, warp);
    abort();
}

void trampoline() {
    g_entry(g_args);
    fibers[cur].state = DONE;
    _longjmp(sched_jb, 1);
}

void run_fiber(int i) {
    Fiber &f = fibers[i];
    cur = i;
    threadIdx_ = dim3((unsigned)i, 1, 1);
    if (_setjmp(sched_jb) == 0) {
        if (!f.started) {
            f.started = true;
            swapcontext(&sched_ctx, &f.ctx);
        } else {
            _longjmp(f.jb, 1);
        }
    }
}

void resolve_warp(int w) {
    Fiber *l = &fibers[(size_t)w * 32];
    const int op = l[0].op;
    for (int i = 0; i < 32; i++) {
        if (l[i].op != op) {
            fprintf(stderr, "[jss emu] ops per lane:");
            for (int k = 0; k < 32; k++) fprintf(stderr, " %d", l[k].op);
            fprintf(stderr, "\n");
            die("lanes of one warp wait at different collectives (divergent collective)", w);
        }
        if (l[i].mask != 0xffffffffu) die("collective without a full mask", w);
    }
    uint64_t agg = 0;
    switch (op) {
    case OP_BALLOT: for (int i = 0; i < 32; i++) agg |= (uint64_t)(l[i].value != 0) << i; break;
    case OP_RED_MIN: agg = 0xffffffffu; for (int i = 0; i < 32; i++) agg = std::min<uint64_t>(agg, (uint32_t)l[i].value); break;
    case OP_RED_MAX: for (int i = 0; i < 32; i++) agg = std::max<uint64_t>(agg, (uint32_t)l[i].value); break;
    case OP_RED_ADD: for (int i = 0; i < 32; i++) agg = (uint32_t)(agg + (uint32_t)l[i].value); break;
    case OP_RED_OR: for (int i = 0; i < 32; i++) agg |= (uint32_t)l[i].value; break;
    default: break;
    }
    for (int i = 0; i < 32; i++) {
        switch (op) {
        case OP_SHFL: l[i].result = l[l[i].arg & 31].value; break;
        case OP_SHFL_XOR: l[i].result = l[(i ^ l[i].arg) & 31].value; break;
        case OP_SHFL_UP: l[i].result = (i >= l[i].arg) ? l[i - l[i].arg].value : l[i].value; break;
        case OP_SYNCWARP: l[i].result = 0; break;
        default: l[i].result = agg; break;
        }
    }
    for (int i = 0; i < 32; i++) l[i].state = READY;
}
}  // namespace

uint64_t collective(int op, unsigned mask, uint64_t value, int arg) {
    Fiber &f = fibers[cur];
    static const bool trace = getenv("JSS_EMU_TRACE") != nullptr;
    if (trace && (cur == 32 || cur == 33)) fprintf(stderr, "T%d op%d v=%llu a=%d\n", cur, op, (unsigned long long)value, arg);
    f.op = op; f.mask = mask; f.value = value; f.arg = arg; f.state = WAITING;
    if (_setjmp(f.jb) == 0) _longjmp(sched_jb, 1);
    return f.result;
}

void launch_impl(void (*entry)(void *), void *args, dim3 grid, dim3 block, size_t smem) {
    const int nt = (int)block.x;
    if (nt % 32 != 0) die("block size must be a multiple of 32");
    const int nw = nt / 32;
    if ((int)fibers.size() < nt) {
        fibers.resize(nt);
        for (auto &f : fibers)
            if (!f.stack) {
                f.stack = (char *)mmap(nullptr, kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
                if (f.stack == MAP_FAILED) die("mmap of a fiber stack failed");
            }
    }
    smem_buf.assign(smem + 64, 0);
    smem_ptr = (void *)(((uintptr_t)smem_buf.data() + 15) & ~(uintptr_t)15);
    g_entry = entry; g_args = args;
    blockDim_ = block; gridDim_ = grid;
    std::vector<int> blocks, seq;
    schedule_order(blocks, (int)grid.x);
    for (int b : blocks) {
        blockIdx_ = dim3((unsigned)b, 1, 1);
        if (poison >= 0) memset(smem_buf.data(), poison, smem_buf.size());   // a CTA starts with garbage
        for (int i = 0; i < nt; i++) {
            Fiber &f = fibers[i];
            f.started = false; f.state = READY;
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = f.stack;
            f.ctx.uc_stack.ss_size = kStack;
            f.ctx.uc_link = nullptr;
            makecontext(&f.ctx, trampoline, 0);
        }
        for (;;) {
            bool progress = false;
            schedule_order(seq, nt);
            for (int i : seq)
                if (fibers[i].state == READY) { run_fiber(i); progress = true; }
            int done = 0, at_bar = 0;
            for (int i = 0; i < nt; i++) {
                done += fibers[i].state == DONE;
                at_bar += fibers[i].state == WAITING && fibers[i].op == OP_SYNCTHREADS;
            }
            if (done == nt) break;
            if (at_bar > 0 && at_bar + done == nt) {      // block barrier complete
                for (int i = 0; i < nt; i++) if (fibers[i].state == WAITING) fibers[i].state = READY;
                continue;
            }
            for (int w = 0; w < nw; w++) {
                int nwait = 0, ndone = 0, nbar = 0;
                for (int i = 0; i < 32; i++) {
                    const Fiber &f = fibers[(size_t)w * 32 + i];
                    nwait += f.state == WAITING; ndone += f.state == DONE;
                    nbar += f.state == WAITING && f.op == OP_SYNCTHREADS;
                }
                if (nwait == 0) continue;
                if (nbar == 32 || (nbar > 0 && nbar + ndone == 32)) continue;   // whole warp parked at __syncthreads
                if (nbar > 0) die("some lanes at __syncthreads while others wait at a warp collective", w);
                if (ndone > 0) die("lanes exited while the rest of the warp waits at a full-mask collective", w);
                if (nwait == 32) { resolve_warp(w); progress = true; }
            }
            if (!progress) die("deadlock: no runnable fiber and no complete collective");
        }
    }
}

}  // namespace emu

// order: 0 ascending threads and blocks (the default), 1 descending, 2 a shuffle seeded by `seed`, redrawn on every
// scheduling pass and every launch.  poison: -1 zero-fills dynamic shared memory once per launch (the default), a
// byte value fills it at the start of every block and fills every cudaMalloc allocation.  Returns 0, or -1 if an
// argument is out of range (nothing changes then).
extern "C" int jss_emu_set_schedule(int order, uint64_t seed, int poison) {
    if (order < emu::ASCENDING || order > emu::SHUFFLED || poison < -1 || poison > 255) return -1;
    emu::sched_order = order;
    emu::sched_rng = seed;
    emu::poison = poison;
    return 0;
}
