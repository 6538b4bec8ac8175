// cuda_simt.h — TEST-ONLY: a small SIMT emulator, one step up from cuda_shim.h.  Every CUDA thread of a block is a fiber
// (its own stack, switched by a few instructions of x86-64 assembly) scheduled cooperatively on the calling OS thread; warp-level intrinsics (__match_any_sync, __ballot_sync,
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
// those steps, deterministically for one seed.  Global loads and stores (__ldcg, __ldcs, __ldg, __stcg),
// __threadfence and __threadfence_system are switch points too.
//
// Resident blocks (simt_launch_ex): a launch keeps up to R blocks live at once, as an SM keeps several CTAs, and
// dispatches the next block when one exits.  Every pass of the scheduler visits the fibers of all resident blocks (in
// a seeded random order in the interleaving mode); barriers and warp rendezvous stay per block.  With R = 1 (and in
// simt_launch) the blocks run one after the other.  A block's dynamic shared memory (simt_dyn_smem) is its own,
// filled with a poison pattern at its start, as the GPU leaves it uninitialised; statically declared __shared__
// variables are `static`, one copy for all blocks, so a kernel that has any may only run with R = 1.
//
// Wait loops: __nanosleep gives way.  A pass in which every block that did anything also slept is a pass of waiting;
// after kSpinPasses of them in a row the launch is reported (block and thread of a sleeper) and aborts: a block that
// waits for a flag that no resident block will set hangs a GPU.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <functional>
#include <memory>
#include <type_traits>
#include <utility>
#include <vector>

#define RL_SIMT 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

struct simt_dim3 {
    unsigned x = 0, y = 0, z = 0;
};
static simt_dim3 blockIdx, threadIdx, blockDim, gridDim;

struct ulonglong2 {
    unsigned long long x, y;
};
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }
struct uint4 {
    unsigned x, y, z, w;
};
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
// the device's min / max take mixed integer types
template <class A, class B>
static inline typename std::common_type<A, B>::type min(A a, B b) {
    return a < b ? a : b;
}
template <class A, class B>
static inline typename std::common_type<A, B>::type max(A a, B b) {
    return a < b ? b : a;
}

namespace simt {
static void interleave_point();
}

#if !defined(__x86_64__)
#error "cuda_simt.h switches fibers with x86-64 assembly"
#endif
// simt_fiber_switch(&from_sp, to_sp): saves the callee-saved registers on the current stack, stores the stack pointer
// in *from_sp and resumes the fiber whose stack pointer is to_sp (the system's swapcontext would also save the signal
// mask, a system call per switch).  Hidden: every library built from this header has its own copy.
extern "C" void simt_fiber_switch(void** from_sp, void* to_sp);
asm(R"(
    .text
    .globl simt_fiber_switch
    .hidden simt_fiber_switch
    .type simt_fiber_switch, @function
simt_fiber_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
    .size simt_fiber_switch, .-simt_fiber_switch
)");
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
template <class T>
static inline T atomicOr(T* p, T v) {
    simt::interleave_point();
    const T o = *p;
    *p = o | v;
    return o;
}
// global memory through the caches (the emulator has one memory: only the switch point differs from a plain access)
template <class T>
static inline T __ldcg(const T* p) {
    simt::interleave_point();
    return *p;
}
template <class T>
static inline T __ldcs(const T* p) {
    simt::interleave_point();
    return *p;
}
template <class T>
static inline T __ldg(const T* p) {
    simt::interleave_point();
    return *p;
}
template <class T>
static inline void __stcg(T* p, T v) {
    simt::interleave_point();
    *p = v;
}
static inline void __threadfence() { simt::interleave_point(); }
static inline void __threadfence_system() { simt::interleave_point(); }
static inline int __ffs(unsigned v) { return v ? __builtin_ctz(v) + 1 : 0; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }

namespace simt {

enum Op { OP_MATCH_ANY = 1, OP_BALLOT, OP_REDUCE_ADD, OP_REDUCE_MIN, OP_REDUCE_MAX, OP_SHFL, OP_SYNCWARP, OP_SHFL_UP };

struct Warp {
    unsigned pending = 0;
    int op[32];
    unsigned mask[32];
    unsigned long long val[32];
    unsigned aux[32];
    unsigned long long res[32];
};

struct Fiber {
    void* sp = nullptr;  // saved stack pointer (simt_fiber_switch)
    char* stack = nullptr;  // from the stack pool, uninitialised: a block of 256 threads would otherwise zero 16 MB
    bool done = false;
    unsigned tid = 0;
};

struct Block {
    unsigned idx = 0;  // blockIdx.x
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    unsigned current = 0;
    unsigned long long progress = 0;  // bumped by every arrival, completion and exit: a pass without a bump is a deadlock
    unsigned long long naps = 0;      // __nanosleep calls: a block that only naps is waiting for another one
    unsigned bar_arrived = 0, bar_gen = 0, live = 0;
    int bar_or = 0, bar_and = 1, bar_result = 0;  // __syncthreads_or / _and of the barrier being filled, and of the last one
    std::vector<unsigned char> smem;              // dynamic shared memory
    std::function<void()> body;
};

static Block* g_block = nullptr;
static void* g_sched = nullptr;  // the scheduler's saved stack pointer
static unsigned long long g_clock = 0;  // clock64(): a counter, monotonic per process

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
    simt_fiber_switch(&b->fibers[b->current].sp, g_sched);
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

static void nap() {
    Block* b = g_block;
    if (!b) return;
    b->naps++;
    yield();
}

static void trampoline() {
    Block* b = g_block;
    b->body();
    b = g_block;
    Fiber& f = b->fibers[b->current];
    f.done = true;
    b->live--;
    b->progress++;
    const unsigned lane = f.tid & 31u;
    if (b->warps[f.tid >> 5].pending & (1u << lane)) die("a thread exited inside a warp rendezvous");
    simt_fiber_switch(&f.sp, g_sched);  // never resumed
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
        case OP_SHFL_UP: {  // lanes below delta keep their own value
            const unsigned d = w.aux[lane];
            return (lane >= d && (mask >> (lane - d) & 1u)) ? w.val[lane - d] : w.val[lane];
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

// a block barrier; op 1 / 2 also reduces pred over the block (__syncthreads_or / __syncthreads_and)
static int syncthreads(int op = 0, int pred = 0) {
    Block* b = g_block;
    const unsigned gen = b->bar_gen;
    b->progress++;
    if (pred) b->bar_or = 1;
    else b->bar_and = 0;
    if (++b->bar_arrived == b->live) {
        b->bar_result = op == 1 ? b->bar_or : b->bar_and;
        b->bar_arrived = 0;
        b->bar_or = 0;
        b->bar_and = 1;
        b->bar_gen++;
    } else {
        while (b->bar_gen == gen) yield();
    }
    return op ? g_block->bar_result : 0;
}

}  // namespace simt

static inline unsigned __match_any_sync(unsigned mask, unsigned long long v) { return (unsigned)simt::rendezvous(simt::OP_MATCH_ANY, mask, v); }
static inline unsigned __ballot_sync(unsigned mask, int pred) { return (unsigned)simt::rendezvous(simt::OP_BALLOT, mask, pred ? 1 : 0); }
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_ADD, mask, v); }
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_MIN, mask, v); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) { return (unsigned)simt::rendezvous(simt::OP_REDUCE_MAX, mask, v); }
static inline unsigned __shfl_sync(unsigned mask, unsigned v, int src) { return (unsigned)simt::rendezvous(simt::OP_SHFL, mask, v, (unsigned)src); }
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu) { simt::rendezvous(simt::OP_SYNCWARP, mask, 0); }
static inline unsigned __shfl_up_sync(unsigned mask, unsigned v, unsigned delta) {
    return (unsigned)simt::rendezvous(simt::OP_SHFL_UP, mask, v, delta);
}
static inline void __syncthreads() { simt::syncthreads(); }
static inline int __syncthreads_or(int pred) { return simt::syncthreads(1, pred); }
static inline int __syncthreads_and(int pred) { return simt::syncthreads(2, pred); }
static inline void __nanosleep(unsigned) { simt::nap(); }
static inline long long clock64() { return (long long)++simt::g_clock; }
// the running block's dynamic shared memory
static inline void* simt_dyn_smem() { return simt::g_block->smem.data(); }

// Turn the interleaving mode on (seed, switch probability p in (0, 1]) or off.
static inline void simt_interleave(bool on, uint64_t seed = 0, double p = 1.0) {
    simt::g_interleave.on = on;
    simt::g_interleave.p = p;
    simt::g_interleave.state = seed;
}

namespace simt {
constexpr size_t kStack = 128 * 1024;
constexpr unsigned kSpinPasses = 256;  // passes of nothing but waiting before a launch is reported as hung
static std::vector<char*> g_stacks;    // free stacks, reused across blocks and launches

static std::unique_ptr<Block> start_block(unsigned bx, unsigned block, size_t smem, const std::function<void()>& body) {
    std::unique_ptr<Block> B(new Block());
    B->idx = bx;
    B->body = body;
    B->fibers.resize(block);
    B->warps.resize((block + 31) / 32);
    B->live = block;
    B->smem.assign(smem, 0xA5);  // poison: the GPU does not zero shared memory
    for (unsigned t = 0; t < block; t++) {
        Fiber& f = B->fibers[t];
        f.tid = t;
        if (g_stacks.empty()) {
            f.stack = new char[kStack];
        } else {
            f.stack = g_stacks.back();
            g_stacks.pop_back();
        }
        // the first switch to the fiber pops six zero registers and "returns" into trampoline with the stack
        // aligned as after a call
        uintptr_t top = ((uintptr_t)(f.stack + kStack)) & ~(uintptr_t)15;
        void** sp = reinterpret_cast<void**>(top - 16);
        sp[0] = reinterpret_cast<void*>(&trampoline);
        sp[1] = nullptr;
        sp -= 6;
        for (int k = 0; k < 6; k++) sp[k] = nullptr;
        f.sp = sp;
    }
    return B;
}
static void end_block(Block& B) {
    for (Fiber& f : B.fibers) g_stacks.push_back(f.stack);
    B.fibers.clear();
}
}  // namespace simt

// run body() once per thread of a <<<grid, block, smem>>> launch with up to `resident` blocks live at a time (see the
// header comment); each block gets `smem` bytes of dynamic shared memory
template <class F>
static void simt_launch_ex(unsigned grid, unsigned block, size_t smem, unsigned resident, F&& body) {
    gridDim.x = grid;
    blockDim.x = block;
    if (resident < 1) resident = 1;
    const std::function<void()> fn = body;
    std::vector<std::unique_ptr<simt::Block>> slots;
    unsigned next = 0, spin = 0;
    std::vector<std::pair<unsigned, unsigned>> order;
    std::vector<unsigned long long> before, naps_before;
    for (;;) {
        // dispatch: an exited block's place goes to the next block of the grid
        for (auto it = slots.begin(); it != slots.end();) {
            if ((*it)->live == 0) {
                simt::end_block(**it);
                it = slots.erase(it);
            } else {
                ++it;
            }
        }
        while (slots.size() < resident && next < grid) slots.push_back(simt::start_block(next++, block, smem, fn));
        if (slots.empty()) break;
        // one pass: every live fiber of every resident block gets a turn; the threads of a block start from a thread
        // that depends on the block (no lane is always first); in the interleaving mode the pass takes all the
        // fibers in a fresh random order
        order.clear();
        for (unsigned s = 0; s < slots.size(); s++)
            for (unsigned k = 0; k < block; k++) order.emplace_back(s, (k + slots[s]->idx) % block);
        if (simt::g_interleave.on)
            for (size_t k = order.size(); k > 1; k--) std::swap(order[k - 1], order[simt::next_random() % k]);
        before.resize(slots.size());
        naps_before.resize(slots.size());
        for (unsigned s = 0; s < slots.size(); s++) {
            before[s] = slots[s]->progress;
            naps_before[s] = slots[s]->naps;
        }
        for (const auto& o : order) {
            simt::Block& B = *slots[o.first];
            simt::Fiber& f = B.fibers[o.second];
            if (f.done) continue;
            B.current = o.second;
            simt::g_block = &B;
            blockIdx.x = B.idx;
            threadIdx.x = o.second;
            simt_fiber_switch(&simt::g_sched, f.sp);
        }
        simt::g_block = nullptr;
        bool worked = false, napped = false;
        for (unsigned s = 0; s < slots.size(); s++) {
            simt::Block& B = *slots[s];
            const bool moved = B.progress != before[s], slept = B.naps != naps_before[s];
            blockIdx.x = B.idx;
            threadIdx.x = B.current;
            if (B.live && !moved && !slept) simt::die("no thread of the block can make progress (a barrier or a *_sync some threads never reach)");
            if (slept) napped = true;
            else if (moved) worked = true;
        }
        spin = (napped && !worked) ? spin + 1 : 0;
        if (spin > simt::kSpinPasses) {
            for (auto& b : slots)
                if (b->naps) {
                    blockIdx.x = b->idx;
                    threadIdx.x = b->current;
                    break;
                }
            simt::die("a block waits in a __nanosleep loop that no resident block makes progress towards (a hang on a GPU)");
        }
    }
}

// run body() once per thread of a <<<grid, block>>> launch: blocks one after the other, the threads of a block as fibers
template <class F>
static void simt_launch(unsigned grid, unsigned block, F&& body) {
    simt_launch_ex(grid, block, 0, 1, body);
}
