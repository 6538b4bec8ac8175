// cuda_simt.h — TEST-ONLY: a small SIMT emulator, one step up from cuda_shim.h.  Every CUDA thread of a block is a fiber
// (ucontext) scheduled cooperatively on the calling OS thread; warp-level intrinsics (__match_any_sync, __ballot_sync,
// __reduce_*_sync, __shfl_sync, __syncwarp) are rendezvous points of the lanes named in their mask, and __syncthreads is
// a block barrier.  With it the DEVICE branches of the maintenance kernels — the warp-aggregated fast paths that
// cuda_shim.h compiles out (`#ifndef RL_SHIM`) — run on the host, without a GPU, against the same
// expectations as their plain paths.  Not shipped, not a fallback.
//
// Strict where the hardware is lenient: a lane that names an exited lane in a mask, lanes of one rendezvous that
// disagree on the operation or the mask, and a block that stops making progress are all reported (abort with a message),
// because on a GPU they are hangs or undefined behaviour.
//
// Interleaving mode (simt_interleave, off by default): a fiber otherwise gives way only at a rendezvous or a barrier, so
// a kernel without either runs each thread from start to finish.  With the mode on, every global atomic below and the
// memory helpers of rl_devmem.cuh (rlm_ld, rlm_ld64, rlm_cas128, rlm_or) first hand control back to the scheduler with
// probability p, and every pass of the scheduler visits the block's fibers in a seeded random order; p = 1 switches at
// every one of them.  A kernel whose threads claim and then write shared words thus runs under many interleavings of
// those steps, deterministically for one seed.  Blocks still run one after the other: only the threads of one block
// interleave, so a test puts the work that must collide inside one block.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <ucontext.h>

#include <functional>
#include <memory>
#include <utility>
#include <vector>

#define RL_SIMT 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

struct simt_dim3 {
    unsigned x = 0, y = 0, z = 0;
};
static simt_dim3 blockIdx, threadIdx, blockDim, gridDim;

struct ulonglong2 {
    unsigned long long x, y;
};
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }

namespace simt {
static void interleave_point();
}
#define RLM_EMU_SWITCH() simt::interleave_point()  // rl_devmem.cuh's memory helpers are switch points too

template <class T>
static inline T atomicAdd(T* p, T v) {
    simt::interleave_point();
    const T o = *p;
    *p = o + v;
    return o;
}
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned v) { return atomicAdd(p, (unsigned long long)v); }
template <class T>
static inline T atomicMax(T* p, T v) {
    simt::interleave_point();
    const T o = *p;
    if (v > o) *p = v;
    return o;
}
template <class T>
static inline T atomicMin(T* p, T v) {
    simt::interleave_point();
    const T o = *p;
    if (v < o) *p = v;
    return o;
}
template <class T>
static inline T atomicCAS(T* p, T cmp, T val) {
    simt::interleave_point();
    const T o = *p;
    if (o == cmp) *p = val;
    return o;
}
template <class T>
static inline T atomicExch(T* p, T v) {
    simt::interleave_point();
    const T o = *p;
    *p = v;
    return o;
}
static inline int __ffs(unsigned v) { return v ? __builtin_ctz(v) + 1 : 0; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }

namespace simt {

enum Op { OP_MATCH_ANY = 1, OP_BALLOT, OP_REDUCE_ADD, OP_REDUCE_MIN, OP_REDUCE_MAX, OP_SHFL, OP_SYNCWARP };

struct Warp {
    unsigned pending = 0;
    int op[32];
    unsigned mask[32];
    unsigned long long val[32];
    unsigned aux[32];
    unsigned long long res[32];
};

struct Fiber {
    ucontext_t ctx;
    std::unique_ptr<char[]> stack;  // uninitialised: a block of 256 threads would otherwise zero 16 MB per launch
    bool done = false;
    unsigned tid = 0;
};

struct Block {
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    ucontext_t sched;
    unsigned current = 0;
    unsigned long long progress = 0;  // bumped by every arrival, completion and exit: a pass without a bump is a deadlock
    unsigned bar_arrived = 0, bar_gen = 0, live = 0;
    std::function<void()> body;
};

static Block* g_block = nullptr;

// the interleaving mode (see the header comment)
struct Interleave {
    bool on = false;
    double p = 1.0;
    uint64_t state = 0;
};
static Interleave g_interleave;

static uint64_t next_random() {  // splitmix64
    uint64_t z = (g_interleave.state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

[[noreturn]] static void die(const char* what) {
    fprintf(stderr, "cuda_simt: %s (block %u, thread %u)\n", what, blockIdx.x, threadIdx.x);
    abort();
}

static void yield() {
    Block* b = g_block;
    swapcontext(&b->fibers[b->current].ctx, &b->sched);
}

// A switch point: with the interleaving mode on, inside a launch, give way to the other fibers with probability p.  A
// switch is progress (the fiber can always resume), so the deadlock check counts it.
static void interleave_point() {
    Block* b = g_block;
    if (!g_interleave.on || !b) return;
    if (g_interleave.p < 1.0 && (double)(next_random() >> 11) * 0x1.0p-53 >= g_interleave.p) return;
    b->progress++;
    yield();
}

static void trampoline() {
    Block* b = g_block;
    b->body();
    Fiber& f = b->fibers[b->current];
    f.done = true;
    b->live--;
    b->progress++;
    const unsigned lane = f.tid & 31u;
    if (b->warps[f.tid >> 5].pending & (1u << lane)) die("a thread exited inside a warp rendezvous");
    swapcontext(&f.ctx, &b->sched);
}

static unsigned long long compute(const Warp& w, int op, unsigned lane, unsigned mask) {
    switch (op) {
        case OP_MATCH_ANY: {
            unsigned r = 0;
            for (unsigned j = 0; j < 32; j++)
                if ((mask >> j & 1u) && w.val[j] == w.val[lane]) r |= 1u << j;
            return r;
        }
        case OP_BALLOT: {
            unsigned r = 0;
            for (unsigned j = 0; j < 32; j++)
                if ((mask >> j & 1u) && w.val[j]) r |= 1u << j;
            return r;
        }
        case OP_REDUCE_ADD: {
            unsigned r = 0;  // 32-bit wrapping, like redux.sync.add.u32
            for (unsigned j = 0; j < 32; j++)
                if (mask >> j & 1u) r += (unsigned)w.val[j];
            return r;
        }
        case OP_REDUCE_MIN:
        case OP_REDUCE_MAX: {
            unsigned r = op == OP_REDUCE_MIN ? 0xFFFFFFFFu : 0u;
            for (unsigned j = 0; j < 32; j++)
                if (mask >> j & 1u) r = op == OP_REDUCE_MIN ? (w.val[j] < r ? (unsigned)w.val[j] : r) : (w.val[j] > r ? (unsigned)w.val[j] : r);
            return r;
        }
        case OP_SHFL: {
            const unsigned src = w.aux[lane] & 31u;
            return (mask >> src & 1u) ? w.val[src] : w.val[lane];
        }
        default: return 0;
    }
}

// The lanes named in `mask` meet; the last one to arrive computes everybody's result.
static unsigned long long rendezvous(int op, unsigned mask, unsigned long long val, unsigned aux = 0) {
    Block* b = g_block;
    const unsigned tid = b->fibers[b->current].tid, lane = tid & 31u;
    Warp& w = b->warps[tid >> 5];
    if (!(mask >> lane & 1u)) die("a thread called a *_sync intrinsic with a mask that does not name it");
    const unsigned first = (tid >> 5) * 32u;
    for (unsigned j = 0; j < 32; j++)
        if ((mask >> j & 1u) && (first + j >= b->fibers.size() || b->fibers[first + j].done)) die("a *_sync mask names a thread that has exited or does not exist");
    w.op[lane] = op;
    w.mask[lane] = mask;
    w.val[lane] = val;
    w.aux[lane] = aux;
    w.pending |= 1u << lane;
    b->progress++;
    if ((w.pending & mask) == mask) {
        for (unsigned j = 0; j < 32; j++)
            if ((mask >> j & 1u) && (w.op[j] != op || w.mask[j] != mask)) die("the lanes of one rendezvous disagree on the intrinsic or on the mask");
        for (unsigned j = 0; j < 32; j++)
            if (mask >> j & 1u) w.res[j] = compute(w, op, j, mask);
        w.pending &= ~mask;
        b->progress++;
    } else {
        while (w.pending >> lane & 1u) yield();
    }
    return w.res[lane];
}

static void syncthreads() {
    Block* b = g_block;
    const unsigned gen = b->bar_gen;
    b->progress++;
    if (++b->bar_arrived == b->live) {
        b->bar_arrived = 0;
        b->bar_gen++;
    } else {
        while (b->bar_gen == gen) yield();
    }
}

}  // namespace simt

static inline unsigned __match_any_sync(unsigned mask, unsigned long long v) { return (unsigned)simt::rendezvous(simt::OP_MATCH_ANY, mask, v); }
static inline unsigned __ballot_sync(unsigned mask, int pred) { return (unsigned)simt::rendezvous(simt::OP_BALLOT, mask, pred ? 1 : 0); }
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_ADD, mask, v); }
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_MIN, mask, v); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_MAX, mask, v); }
static inline unsigned __shfl_sync(unsigned mask, unsigned v, int src) { return (unsigned)simt::rendezvous(simt::OP_SHFL, mask, v, (unsigned)src); }
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { simt::rendezvous(simt::OP_SYNCWARP, mask, 0); }
static inline void __syncthreads() { simt::syncthreads(); }

// Turn the interleaving mode on (seed, switch probability p in (0, 1]) or off.
static inline void simt_interleave(bool on, uint64_t seed = 0, double p = 1.0) {
    simt::g_interleave.on = on;
    simt::g_interleave.p = p;
    simt::g_interleave.state = seed;
}

// run body() once per thread of a <<<grid, block>>> launch: blocks one after the other, the threads of a block as fibers
template <class F>
static void simt_launch(unsigned grid, unsigned block, F&& body) {
    gridDim.x = grid;
    blockDim.x = block;
    for (unsigned bx = 0; bx < grid; bx++) {
        simt::Block B;
        B.body = body;
        B.fibers.resize(block);
        B.warps.resize((block + 31) / 32);
        B.live = block;
        simt::g_block = &B;
        for (unsigned t = 0; t < block; t++) {
            simt::Fiber& f = B.fibers[t];
            f.tid = t;
            constexpr size_t kStack = 64 * 1024;
            f.stack.reset(new char[kStack]);
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = f.stack.get();
            f.ctx.uc_stack.ss_size = kStack;
            f.ctx.uc_link = nullptr;
            makecontext(&f.ctx, simt::trampoline, 0);
        }
        std::vector<unsigned> order(block);
        while (B.live) {
            const unsigned long long before = B.progress;
            // the threads take turns, starting from a thread that depends on the block: no lane is always first; in the
            // interleaving mode every pass takes them in a fresh random order
            for (unsigned k = 0; k < block; k++) order[k] = (k + bx) % block;
            if (simt::g_interleave.on)
                for (unsigned k = block; k > 1; k--) std::swap(order[k - 1], order[simt::next_random() % k]);
            for (unsigned k = 0; k < block; k++) {
                const unsigned t = order[k];
                simt::Fiber& f = B.fibers[t];
                if (f.done) continue;
                B.current = t;
                blockIdx.x = bx;
                threadIdx.x = t;
                swapcontext(&B.sched, &f.ctx);
            }
            if (B.live && B.progress == before) simt::die("no thread of the block can make progress (a barrier or a *_sync some threads never reach)");
        }
        simt::g_block = nullptr;
    }
}
