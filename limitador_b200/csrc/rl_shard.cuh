// rl_shard.cuh — kernels of the namespace-sharded peer exchange (SURVEY.md §8e, DESIGN.md §8).
//
// One process per GPU.  Every rank owns an "exchange slab" in its HBM that all other ranks map
// (CUDA IPC over NVLink / NVSwitch peer access).  Per step a rank buckets its slice of the global
// batch by owner = rl_owner_of(ns_id, world) and STORES each 32-B record straight into the owner's
// inbox over NVLink — block (source rank) of the step's buffer, stable order — then publishes the
// block's fill and a step flag.  The owner waits for the flags of all sources, decides the inbox in
// (source rank, source index) order — the canonical stream order of the sharded store — and stores
// the verdict bytes straight back into the sources' verdict inboxes.  No NCCL call, no padding, no
// host round trip on the data path; the only cross-GPU synchronisation is a flag word per
// (source, owner, step) written with release and polled with acquire semantics at system scope.
#pragma once
#include "rl_kernels.cuh"
#ifdef RL_SIMT
#include <chrono>
#endif

#define RL_XCHG_MAX_WORLD 32
#ifndef RL_XCHG_TIMEOUT_NS
#define RL_XCHG_TIMEOUT_NS 30000000000ull  // a peer that does not show up in 30 s is an error, not a hang
#endif

struct RlXCtl {  // one per (buffer, peer rank) in every slab
    uint32_t cnt;    // records the peer put into its block of my inbox
    uint32_t rflag;  // step+1 once that block is complete
    uint32_t vflag;  // step+1 once the peer (as owner) has returned the verdicts of my records
    uint32_t _pad;
};

struct RlXchg {
    uint4* trace;                      // RL_FLAG_TRACE (see rl_kernels.cuh), else nullptr
    uint32_t* trace_pos;
    uint8_t* base[RL_XCHG_MAX_WORLD];  // slab of every rank, as mapped in this process
    unsigned long long off_recs, off_vin, off_ctl;
    uint32_t world, rank, cap, depth;
    __device__ __forceinline__ rl_record* inbox(uint32_t owner, uint32_t buf, uint32_t src) const {
        return reinterpret_cast<rl_record*>(base[owner] + off_recs) + ((size_t)buf * world + src) * cap;
    }
    __device__ __forceinline__ uint8_t* vin(uint32_t at_rank, uint32_t buf, uint32_t owner) const {
        return base[at_rank] + off_vin + ((size_t)buf * world + owner) * cap;
    }
    __device__ __forceinline__ RlXCtl* ctl(uint32_t at_rank, uint32_t buf, uint32_t peer) const {
        return reinterpret_cast<RlXCtl*>(base[at_rank] + off_ctl) + (size_t)buf * world + peer;
    }
};

// Under tests/emu/cuda_simt.h (RL_SIMT) the flag accesses are switch points of the emulator's interleaving mode around a
// plain access (it has one memory and runs one fiber at a time), and the timer is the host's steady clock.
__device__ __forceinline__ uint32_t rl_ld_acquire_sys(const uint32_t* p) {
#ifdef RL_SIMT
    RLM_EMU_SWITCH();
    return *(volatile const uint32_t*)p;
#else
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#endif
}
__device__ __forceinline__ void rl_st_release_sys(uint32_t* p, uint32_t v) {
#ifdef RL_SIMT
    RLM_EMU_SWITCH();
    *(volatile uint32_t*)p = v;
#else
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}
__device__ __forceinline__ unsigned long long rl_globaltimer() {
#ifdef RL_SIMT
    return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(
               std::chrono::steady_clock::now().time_since_epoch()).count();
#else
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
#endif
}
// spin until *p has reached `want` (step flags only grow); false on time-out
__device__ __forceinline__ bool rl_wait_flag(const uint32_t* p, uint32_t want) {
    if ((int32_t)(rl_ld_acquire_sys(p) - want) >= 0) return true;
    const unsigned long long t0 = rl_globaltimer();
    for (;;) {
        if ((int32_t)(rl_ld_acquire_sys(p) - want) >= 0) return true;
        __nanosleep(200);
        if (rl_globaltimer() - t0 > RL_XCHG_TIMEOUT_NS) return false;
    }
}

// Per-tile histogram of the owners; the last block turns it into exclusive prefixes over tiles and
// per-owner totals.  tile_cnt: [tiles][32], totals: [32].
__global__ void __launch_bounds__(RL_PART_THREADS) k_xcount(const rl_record* __restrict__ recs, uint32_t n,
                                                           uint32_t world, uint32_t tile, uint32_t* tile_cnt,
                                                           uint32_t* totals, uint32_t* ctr, uint4* trace,
                                                           uint32_t* trace_pos, uint32_t step) {
    __shared__ uint32_t wcnt[RL_PART_WARPS][32];
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t t0 = min(blockIdx.x * tile, n), t1 = min(t0 + tile, n);
    const uint32_t slice = tile / RL_PART_WARPS;
    const uint32_t s0 = min(t0 + warp * slice, t1), s1 = min(s0 + slice, t1);
    wcnt[warp][lane] = 0;
    if (blockIdx.x == 0 && tid == 0) rl_trace(trace, trace_pos, RL_EV_XCOUNT, 0, step);
    __syncthreads();
    for (uint32_t b = s0; b < s1; b += 32) {
        const uint32_t a = b + lane;
        const bool valid = a < s1;
        const uint32_t o = valid ? rl_owner_dev(recs[a].ns_id, world) : 0;
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const unsigned m = __match_any_sync(vmask, o);
            if (lane == (uint32_t)(__ffs(m) - 1)) wcnt[warp][o] += __popc(m);
        }
        __syncwarp();
    }
    __syncthreads();
    if (tid < 32) {
        uint32_t tot = 0;
        for (int w = 0; w < RL_PART_WARPS; w++) tot += wcnt[w][tid];
        tile_cnt[blockIdx.x * 32 + tid] = tot;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ctr, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // exclusive prefix over tiles, per owner (lane = owner): warp w takes the w-th slice of the tiles, its
    // loads are independent (16 in flight), the slices are stitched through shared memory
    {
        const uint32_t nt = gridDim.x;
        const uint32_t per = (nt + RL_PART_WARPS - 1) / RL_PART_WARPS;
        const uint32_t a0 = min(warp * per, nt), a1 = min(a0 + per, nt);
        uint32_t sum = 0;
        for (uint32_t tb = a0; tb < a1; tb += 16) {
            uint32_t c[16];
#pragma unroll
            for (int i = 0; i < 16; i++) c[i] = (tb + i < a1) ? __ldcg(&tile_cnt[(tb + i) * 32 + lane]) : 0;
#pragma unroll
            for (int i = 0; i < 16; i++) sum += c[i];
        }
        wcnt[warp][lane] = sum;
        __syncthreads();
        uint32_t run = 0;
        for (uint32_t w = 0; w < warp; w++) run += wcnt[w][lane];
        for (uint32_t tb = a0; tb < a1; tb += 16) {
            uint32_t c[16];
#pragma unroll
            for (int i = 0; i < 16; i++) c[i] = (tb + i < a1) ? __ldcg(&tile_cnt[(tb + i) * 32 + lane]) : 0;
#pragma unroll
            for (int i = 0; i < 16; i++) {
                if (tb + i < a1) tile_cnt[(tb + i) * 32 + lane] = run;
                run += c[i];
            }
        }
        if (warp == RL_PART_WARPS - 1) totals[lane] = run;
    }
    if (tid == 0) {
        *ctr = 0;
        rl_trace(trace, trace_pos, RL_EV_XCOUNT, 1, step);
    }
}

// Stable scatter of my records into the owners' inboxes (peer stores over NVLink); the last block
// publishes fills and step flags.  dest[a] = owner << 27 | position in the block.
__global__ void __launch_bounds__(RL_PART_THREADS) k_xscatter(RlXchg X, const rl_record* __restrict__ recs, uint32_t n,
                                                             uint32_t tile, const uint32_t* __restrict__ tile_cnt,
                                                             const uint32_t* __restrict__ totals, uint32_t buf,
                                                             uint32_t step, uint32_t* dest, uint32_t* ctr) {
    __shared__ uint32_t wcnt[RL_PART_WARPS][32];
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t world = X.world;
    const uint32_t t0 = min(blockIdx.x * tile, n), t1 = min(t0 + tile, n);
    const uint32_t slice = tile / RL_PART_WARPS;
    const uint32_t s0 = min(t0 + warp * slice, t1), s1 = min(s0 + slice, t1);
    wcnt[warp][lane] = 0;
    __syncthreads();
    for (uint32_t b = s0; b < s1; b += 32) {
        const uint32_t a = b + lane;
        const bool valid = a < s1;
        const uint32_t o = valid ? rl_owner_dev(recs[a].ns_id, world) : 0;
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const unsigned m = __match_any_sync(vmask, o);
            if (lane == (uint32_t)(__ffs(m) - 1)) wcnt[warp][o] += __popc(m);
        }
        __syncwarp();
    }
    __syncthreads();
    if (tid < 32) {
        uint32_t run = tile_cnt[blockIdx.x * 32 + tid];
        for (int w = 0; w < RL_PART_WARPS; w++) {
            const uint32_t c = wcnt[w][tid];
            wcnt[w][tid] = run;
            run += c;
        }
    }
    __syncthreads();
    for (uint32_t b = s0; b < s1; b += 32) {
        const uint32_t a = b + lane;
        const bool valid = a < s1;
        ulonglong2 w0 = make_ulonglong2(0ull, 0ull), w1 = w0;
        uint32_t o = 0;
        if (valid) {
            w0 = rl_ld_stream(&recs[a]);
            w1 = rl_ld_stream(reinterpret_cast<const ulonglong2*>(&recs[a]) + 1);
            o = rl_owner_dev((uint32_t)w0.x, world);
        }
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const unsigned m = __match_any_sync(vmask, o);
            const int leader = __ffs(m) - 1;
            uint32_t basepos = 0;
            if ((int)lane == leader) {
                basepos = wcnt[warp][o];
                wcnt[warp][o] = basepos + __popc(m);
            }
            basepos = __shfl_sync(m, basepos, leader);
            const uint32_t pos = basepos + __popc(m & ((1u << lane) - 1));
            ulonglong2* dst = reinterpret_cast<ulonglong2*>(X.inbox(o, buf, X.rank) + pos);
            dst[0] = w0;  // over NVLink when o != my rank
            dst[1] = w1;
            dest[a] = (o << 27) | pos;
        }
        __syncwarp();
    }
    // every CTA's peer stores are ordered before its arrival on the counter; the last block's flag
    // stores follow all of them (release at system scope)
    __threadfence_system();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ctr, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    if (tid < world) {
        RlXCtl* c = X.ctl(tid, buf, X.rank);
        c->cnt = totals[tid];
        rl_st_release_sys(&c->rflag, step + 1);
    }
    if (tid == 0) {
        *ctr = 0;
        rl_trace(X.trace, X.trace_pos, RL_EV_XSCATTER, 1, step);
    }
}

// Owner side: wait for the step's blocks of every source, publish the fills as an exclusive prefix
// (seg_prefix[0..world]) and the inbox size (n_dev) for the decision kernels.
__global__ void __launch_bounds__(32) k_xwait(RlXchg X, uint32_t buf, uint32_t step, uint32_t* seg_prefix,
                                             uint32_t* n_dev, uint32_t n_max, uint32_t* err) {
    const uint32_t lane = threadIdx.x;
    uint32_t cnt = 0;
    bool ok = true;
    if (lane == 0) rl_trace(X.trace, X.trace_pos, RL_EV_XWAIT, 0, step);
    if (lane < X.world) {
        const RlXCtl* c = X.ctl(X.rank, buf, lane);
        ok = rl_wait_flag(&c->rflag, step + 1);
        cnt = ok ? *(volatile const uint32_t*)&c->cnt : 0;
        if (cnt > X.cap) {
            cnt = 0;
            ok = false;
        }
    }
    if (!ok) {
        atomicMax(err, (uint32_t)RL_DEV_EXCHANGE);
        atomicCAS(err + 7, 0u, (1u << 28) | (lane << 20) | (step & 0xFFFFFu));  // detail: k_xwait, source rank, step
    }
    uint32_t x = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane >= o) x += y;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, x, X.world - 1);
    if (total > n_max) {  // more records than the engine was sized for (rl_config.max_batch): refuse the step
        if (lane == 0) {
            atomicMax(err, (uint32_t)RL_DEV_EXCHANGE);
            atomicCAS(err + 7, 0u, (3u << 28) | (step & 0xFFFFFu));  // detail: inbox larger than max_batch
        }
        x = 0;
        cnt = 0;
    }
    if (lane < X.world) seg_prefix[lane] = x - cnt;
    if (lane == X.world - 1) {
        seg_prefix[X.world] = x;
        *n_dev = x;
        rl_trace(X.trace, X.trace_pos, RL_EV_XWAIT, 1, step);
    }
}

// Owner side, verdict return.  The decision kernels write every verdict into a LOCAL mirror of the sources' verdict
// blocks (rl_store_verdict: request index -> (source, position) through the inbox prefix; a byte store to peer memory
// is a transaction of its own over NVLink — tens of thousands of them per step slow k_main down).  This kernel ships block s to
// source s with 16-byte stores — CTA (s, j) the j-th slice of block s — and the last block publishes the step flags.
#define RL_XRET_SLICES 8
__global__ void __launch_bounds__(256) k_xreturn(RlXchg X, const uint8_t* __restrict__ vmirror, const uint32_t* __restrict__ seg_prefix,
                                                uint32_t buf, uint32_t step, uint32_t* ctr) {
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x;
    const uint32_t s = blockIdx.x / RL_XRET_SLICES, j = blockIdx.x % RL_XRET_SLICES;
    const uint32_t n = seg_prefix[s + 1] - seg_prefix[s];
    const uint32_t nvec = (n + 15) / 16;  // whole 16-byte words of the block (blocks are 16-byte aligned, cap % 16 == 0)
    const uint4* src = reinterpret_cast<const uint4*>(vmirror + (size_t)s * X.cap);
    uint4* dst = reinterpret_cast<uint4*>(X.vin(s, buf, X.rank));
    for (uint32_t i = j * blockDim.x + tid; i < nvec; i += RL_XRET_SLICES * blockDim.x) dst[i] = __ldcg(src + i);
    __threadfence_system();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ctr, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    if (tid < X.world) rl_st_release_sys(&X.ctl(tid, buf, X.rank)->vflag, step + 1);
    if (tid == 0) {
        *ctr = 0;
        rl_trace(X.trace, X.trace_pos, RL_EV_XRETURN, 1, step);
    }
}

// Source side: wait for every owner's verdicts of the step ...
// Only single-warp kernels ever spin.  A spinning CTA pins its SM: the SM cannot change its shared-memory
// carveout while a CTA is resident, so a grid of spinners spread over all SMs keeps k_front / k_main (which
// need a larger carveout) from being scheduled at all — the very kernels whose results the spinners wait for.
__global__ void __launch_bounds__(32) k_xwaitv(RlXchg X, uint32_t buf, uint32_t step, uint32_t* err) {
    const uint32_t lane = threadIdx.x;
    if (lane == 0) rl_trace(X.trace, X.trace_pos, RL_EV_XWAITV, 0, step);
    if (lane < X.world && !rl_wait_flag(&X.ctl(X.rank, buf, lane)->vflag, step + 1)) {
        atomicMax(err, (uint32_t)RL_DEV_EXCHANGE);
        atomicCAS(err + 7, 0u, (2u << 28) | (lane << 20) | (step & 0xFFFFFu));  // detail: verdicts, owner rank, step
    }
    __syncwarp();
    if (lane == 0) rl_trace(X.trace, X.trace_pos, RL_EV_XWAITV, 1, step);
}
// ... then put them back in request order.
__global__ void __launch_bounds__(256) k_xgather(RlXchg X, uint32_t n, const uint32_t* __restrict__ dest, uint32_t buf,
                                                uint8_t* out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t d = dest[i];
        out[i] = __ldcg(X.vin(X.rank, buf, d >> 27) + (d & 0x07FFFFFFu));
    }
}
