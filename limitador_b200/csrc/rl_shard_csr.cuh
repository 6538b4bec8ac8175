// rl_shard_csr.cuh — the general (CSR) form of the namespace-sharded peer exchange (DESIGN.md §8c).
//
// The record exchange (rl_shard.cuh) moves 32-byte records: every limit of a namespace, one key.  A served request is a
// CSR row of rl_counter instead: the limits whose conditions held, each with the key of its own variable set, plus an
// operation (check_and_update, is_within_limits or update) and a load_counters flag.  Every counter of a request belongs
// to the request's namespace, so the request has exactly one owner: rl_owner_dev(ns of its first counter, world).
//
// A step (one buffer, no lag: a source sends step s+1 only after it has collected step s, and an owner reads its inbox
// only before it returns step s, so one buffer is never written while it is read):
//   source  k_ccount   stable bucketing by owner (one CTA): dest / counter position of every request, per-owner fills
//           k_cscatter request headers and counters STORED into the owners' inbox blocks; the last CTA publishes, per
//                      owner, the block's digest / counter fill / load bit, the request fill and the step flag
//   owner   k_xwait    (rl_shard.cuh) waits for every block; exclusive prefix of the request fills
//           k_cprep    exclusive prefix of the counter fills, registry digests compared (one warp, does not wait)
//           k_cunpack  the inbox laid out as ONE canonical CSR, (source rank, source index) order
//           k_cruns    the runs of equal op byte (one CTA); k_crebase: each run's offsets counted from 0
//           [host]     one read of the sizes and the runs, then one engine call per run (RL_MEM_DEVICE)
//           k_creturn  verdicts, first_limited and (for blocks that asked) remaining / ttl shipped to every source in
//                      16-byte stores; the last CTA publishes the verdict flags
//   source  k_xwaitv   (rl_shard.cuh) waits for every owner; k_cgather: back into request and counter order
// Only k_xwait and k_xwaitv spin (single warps: see the comment above k_xwaitv).
#pragma once
#include "rl_shard.cuh"

#define RL_COP_CHECK_AND_UPDATE 0u
#define RL_COP_IS_WITHIN 1u
#define RL_COP_UPDATE 2u
#define RL_COP_LOAD 0x10u     // with RL_COP_CHECK_AND_UPDATE: remaining / ttl wanted
#define RL_COP_REFUSED 0xFFu  // owner side: the source's registry digest differs, the request is not decided
#define RL_CRET_SLICES 8

struct RlCHdr {       // one request in an owner's inbox block
    uint32_t cpos;    // first counter, in the block's counter area
    uint32_t m_op;    // counters (bits 0..15) | op byte << 16
    uint64_t delta;
    uint64_t now_us;
};
struct RlCBlk {       // one per (owner, source), in the owner's slab, written by the source before its step flag
    unsigned long long digest;  // the source's limit registry
    uint32_t nctr;              // counters in the block
    uint32_t any_load;          // some request of the block wants remaining / ttl
};

// The CSR exchange's view of the slabs.  x carries the control words (RlXCtl at x.off_ctl, buffer 0) that k_xwait and
// k_xwaitv poll; the other areas are this exchange's own.
struct RlCXchg {
    RlXchg x;
    unsigned long long off_hdr, off_ctr, off_blk, off_ret, ret_stride;
    uint32_t cap_ctr;
    __device__ __forceinline__ RlCHdr* hdr(uint32_t owner, uint32_t src) const {
        return reinterpret_cast<RlCHdr*>(x.base[owner] + off_hdr) + (size_t)src * x.cap;
    }
    __device__ __forceinline__ rl_counter* ctr(uint32_t owner, uint32_t src) const {
        return reinterpret_cast<rl_counter*>(x.base[owner] + off_ctr) + (size_t)src * cap_ctr;
    }
    __device__ __forceinline__ RlCBlk* blk(uint32_t owner, uint32_t src) const {
        return reinterpret_cast<RlCBlk*>(x.base[owner] + off_blk) + src;
    }
    // the block owner `owner` returns to source `at`: verdicts [cap] | first [cap] u32 | remaining [cap_ctr] | ttl [cap_ctr]
    __device__ __forceinline__ uint8_t* ret(uint32_t at, uint32_t owner) const {
        return x.base[at] + off_ret + (size_t)owner * ret_stride;
    }
};

// The request's op byte at the source: one op for the batch; the load bit per request (load, nullable) or for all
__device__ __forceinline__ uint32_t rl_cop(uint32_t op, const uint8_t* load, uint32_t load_all, uint32_t i) {
    const bool lc = op == RL_COP_CHECK_AND_UPDATE && (load ? load[i] != 0 : load_all != 0);
    return op | (lc ? RL_COP_LOAD : 0u);
}

// Owner of a request: from its first counter's limit (an unknown limit, or no counter at all, stays with the source,
// whose engine refuses / answers it as the unsharded call would)
__device__ __forceinline__ uint32_t rl_csr_owner(const RlLimitDev* lims, uint32_t lims_cap, uint32_t m, const rl_counter* c,
                                                 uint32_t world, uint32_t rank) {
    if (m == 0) return rank;
    const uint32_t l = c->limit_id;
    if (l >= lims_cap || lims[l].group == 0) return rank;
    return rl_owner_dev(lims[l].ns_id, world);
}

// Source: stable bucketing of n requests by owner in one CTA of 1024 threads.  dest[i] = owner << 27 | position in the
// owner's block, cpos[i] = position of its first counter in the block's counter area; totals[0..31] requests,
// totals[32..63] counters, totals[64..95] any load, per owner.
__global__ void __launch_bounds__(1024) k_ccount(const RlLimitDev* __restrict__ lims, uint32_t lims_cap, uint32_t n,
                                                 const uint32_t* __restrict__ off, const rl_counter* __restrict__ ctrs,
                                                 uint32_t op, const uint8_t* __restrict__ load, uint32_t load_all,
                                                 uint32_t world, uint32_t rank, uint32_t* dest, uint32_t* cpos,
                                                 uint32_t* totals) {
    __shared__ uint32_t wreq[32][32], wctr[32][32];
    __shared__ uint32_t run_req[32], run_ctr[32], anyl[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 32) run_req[tid] = run_ctr[tid] = anyl[tid] = 0;
    for (uint32_t base = 0; base < n; base += 1024) {
        wreq[warp][lane] = 0;
        wctr[warp][lane] = 0;
        __syncthreads();
        const uint32_t i = base + tid;
        const bool valid = i < n;
        uint32_t o = 0, m = 0;
        if (valid) {
            const uint32_t c0 = off[i];
            m = off[i + 1] - c0;
            o = rl_csr_owner(lims, lims_cap, m, ctrs + c0, world, rank);
            if (rl_cop(op, load, load_all, i) & RL_COP_LOAD) atomicOr(&anyl[o], 1u);
        }
        // lanes of one owner, their rank among themselves and the counters of the lanes before them
        const unsigned vmask = __ballot_sync(0xffffffffu, valid);
        unsigned grp = 0;
        uint32_t cbefore = 0, csum = 0;
        if (valid) grp = __match_any_sync(vmask, o);
        for (uint32_t j = 0; j < 32; j++) {
            const uint32_t mj = __shfl_sync(0xffffffffu, m, j);
            if ((grp >> j) & 1u) {
                csum += mj;
                if (j < lane) cbefore += mj;
            }
        }
        if (valid && lane == (uint32_t)(__ffs(grp) - 1)) {
            wreq[warp][o] = __popc(grp);
            wctr[warp][o] = csum;
        }
        __syncthreads();
        if (tid < 32) {  // thread t: owner t, prefix over the warps in order (stable)
            uint32_t r = run_req[tid], c = run_ctr[tid];
            for (uint32_t w = 0; w < 32; w++) {
                const uint32_t a = wreq[w][tid], b = wctr[w][tid];
                wreq[w][tid] = r;
                wctr[w][tid] = c;
                r += a;
                c += b;
            }
            run_req[tid] = r;
            run_ctr[tid] = c;
        }
        __syncthreads();
        if (valid) {
            dest[i] = (o << 27) | (wreq[warp][o] + __popc(grp & ((1u << lane) - 1u)));
            cpos[i] = wctr[warp][o] + cbefore;
        }
        __syncthreads();
    }
    __syncthreads();
    if (tid < 32) {
        totals[tid] = tid < world ? run_req[tid] : 0;
        totals[32 + tid] = tid < world ? run_ctr[tid] : 0;
        totals[64 + tid] = tid < world ? anyl[tid] : 0;
    }
}

// Source: every request's header and counters stored into its owner's block (peer stores when the owner is another
// GPU); the last CTA publishes each owner's block: digest, counter fill, load bit, request fill, then the step flag.
__global__ void __launch_bounds__(256) k_cscatter(RlCXchg X, uint32_t n, const uint32_t* __restrict__ off,
                                                  const rl_counter* __restrict__ ctrs, const uint64_t* __restrict__ delta,
                                                  const uint64_t* __restrict__ now, uint32_t op, const uint8_t* __restrict__ load,
                                                  uint32_t load_all, const uint32_t* __restrict__ dest,
                                                  const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ totals,
                                                  unsigned long long digest, uint32_t step, uint32_t* ctr) {
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x, rank = X.x.rank;
    for (uint32_t i = blockIdx.x * blockDim.x + tid; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t d = dest[i], o = d >> 27, p = d & 0x07FFFFFFu, cp = cpos[i];
        const uint32_t c0 = off[i], m = off[i + 1] - c0;
        RlCHdr h;
        h.cpos = cp;
        h.m_op = m | (rl_cop(op, load, load_all, i) << 16);
        h.delta = delta[i];
        h.now_us = now[i];
        X.hdr(o, rank)[p] = h;
        rl_counter* dst = X.ctr(o, rank) + cp;
        for (uint32_t k = 0; k < m; k++) dst[k] = ctrs[c0 + k];
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ctr, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    if (tid < X.x.world) {
        RlCBlk* b = X.blk(tid, rank);
        b->digest = digest;
        b->nctr = totals[32 + tid];
        b->any_load = totals[64 + tid];
        RlXCtl* c = X.x.ctl(tid, 0, rank);
        c->cnt = totals[tid];
        __threadfence_system();
        rl_st_release_sys(&c->rflag, step + 1);
    }
    if (tid == 0) *ctr = 0;
}

// Owner, after k_xwait (seg[0..world] = request prefix, seg[36] = requests): cseg[0..world] = counter prefix, and
// head = {requests, counters, runs (k_cruns), sources whose registry digest differs (bit mask)}.  One warp, lane =
// source.  (world x cap_ctr <= the engine's max_counters: rl_shard_batch_create refuses more.)
__global__ void __launch_bounds__(32) k_cprep(RlCXchg X, const uint32_t* __restrict__ seg, unsigned long long digest,
                                              uint32_t* cseg, uint32_t* head) {
    const uint32_t lane = threadIdx.x, world = X.x.world;
    uint32_t c = 0;
    bool bad = false;
    if (lane < world) {
        const RlCBlk* b = X.blk(X.x.rank, lane);
        const uint32_t nreq = seg[lane + 1] - seg[lane];
        c = nreq ? min(*(volatile const uint32_t*)&b->nctr, X.cap_ctr) : 0;
        bad = *(volatile const unsigned long long*)&b->digest != digest;
    }
    uint32_t x = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane >= o) x += y;
    }
    const unsigned badmask = __ballot_sync(0xffffffffu, bad);
    const uint32_t total = __shfl_sync(0xffffffffu, x, world - 1);
    if (lane < world) cseg[lane] = x - c;
    if (lane == 0) {
        cseg[world] = total;
        head[0] = seg[36];
        head[1] = total;
        head[2] = 0;
        head[3] = badmask;
    }
}

// Owner: the inbox as one CSR in canonical order.  off[n] = counters; op[i] = the request's op byte, RL_COP_REFUSED for
// the requests of a source whose digest differs.
__global__ void __launch_bounds__(256) k_cunpack(RlCXchg X, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ cseg,
                                                 const uint32_t* __restrict__ head, uint32_t* off, rl_counter* ctrs,
                                                 uint64_t* delta, uint64_t* now, uint8_t* op) {
    const uint32_t n = head[0], world = X.x.world, bad = head[3];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) {
        if (i == n) {
            off[n] = cseg[world];
            continue;
        }
        uint32_t s = 0;
        while (s + 1 < world && seg[s + 1] <= i) s++;
        const RlCHdr h = X.hdr(X.x.rank, s)[i - seg[s]];
        const uint32_t m = h.m_op & 0xFFFFu, c0 = cseg[s] + h.cpos;
        off[i] = c0;
        delta[i] = h.delta;
        now[i] = h.now_us;
        op[i] = ((bad >> s) & 1u) ? (uint8_t)RL_COP_REFUSED : (uint8_t)(h.m_op >> 16);
        const rl_counter* src = X.ctr(X.x.rank, s) + h.cpos;
        for (uint32_t k = 0; k < m; k++) ctrs[c0 + k] = src[k];
    }
}

// Owner: the runs of equal op byte, in canonical order, one CTA.  runs[3k] = first request, runs[3k+1] = its first
// counter, runs[3k+2] = the op byte; head[2] = runs.
__global__ void __launch_bounds__(1024) k_cruns(const uint32_t* __restrict__ off, const uint8_t* __restrict__ op,
                                                uint32_t* head, uint32_t* runs) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t s_base;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n = head[0];
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + tid;
        const bool start = i < n && (i == 0 || op[i] != op[i - 1]);
        const unsigned b = __ballot_sync(0xffffffffu, start);
        if (lane == 0) wsum[warp] = __popc(b);
        __syncthreads();
        uint32_t before = s_base;
        for (uint32_t w = 0; w < warp; w++) before += wsum[w];
        if (start) {
            const uint32_t k = before + __popc(b & ((1u << lane) - 1u));
            runs[3 * k] = i;
            runs[3 * k + 1] = off[i];
            runs[3 * k + 2] = op[i];
        }
        __syncthreads();
        if (tid == 0)
            for (uint32_t w = 0; w < 32; w++) s_base += wsum[w];
        __syncthreads();
    }
    if (tid == 0) head[2] = s_base;
}

// Owner: roff[i + k] = off[i] - (run k's first counter) for request i of run k, and the run's end after its last request:
// run k's CSR offsets start at roff + runs[3k] + k and count from 0, as the engine's general form takes them.
__global__ void __launch_bounds__(256) k_crebase(const uint32_t* __restrict__ off, const uint32_t* __restrict__ head,
                                                 const uint32_t* __restrict__ runs, uint32_t* roff) {
    const uint32_t n = head[0], nr = head[2];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = nr;  // the last run starting at or before i
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) / 2;
            if (runs[3 * mid] <= i) lo = mid;
            else hi = mid;
        }
        const uint32_t c0 = runs[3 * lo + 1];
        roff[i + lo] = off[i] - c0;
        const uint32_t end = lo + 1 < nr ? runs[3 * (lo + 1)] : n;
        if (i + 1 == end) roff[i + lo + 1] = off[i + 1] - c0;
    }
}

// Owner: the local mirror (verdicts [n], first [n], remaining / ttl [counters], canonical positions) shipped to the
// sources, CTA (s, j) the j-th slice of source s's block, 16-byte stores.  remaining / ttl travel only for blocks whose
// source asked for them.  The last CTA publishes the verdict flags.
__global__ void __launch_bounds__(256) k_creturn(RlCXchg X, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ cseg,
                                                 const uint8_t* __restrict__ lim, const uint32_t* __restrict__ first,
                                                 const uint64_t* __restrict__ rem, const uint64_t* __restrict__ ttl,
                                                 uint32_t step, uint32_t* ctr) {
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x, rank = X.x.rank;
    const uint32_t s = blockIdx.x / RL_CRET_SLICES, j = blockIdx.x % RL_CRET_SLICES;
    const uint32_t r0 = seg[s], n = seg[s + 1] - r0, c0 = cseg[s], nc = cseg[s + 1] - c0;
    const bool lc = nc && n && X.blk(rank, s)->any_load;
    const uint32_t wl = (n + 15) / 16, wf = (n + 3) / 4, wr = lc ? (nc + 1) / 2 : 0;
    uint8_t* R = X.ret(s, rank);
    uint4* d_lim = reinterpret_cast<uint4*>(R);
    uint4* d_first = reinterpret_cast<uint4*>(R + X.x.cap);
    uint4* d_rem = reinterpret_cast<uint4*>(R + 5ull * X.x.cap);
    uint4* d_ttl = reinterpret_cast<uint4*>(R + 5ull * X.x.cap + 8ull * X.cap_ctr);
    for (uint32_t w = j * blockDim.x + tid; w < wl + wf + 2 * wr; w += RL_CRET_SLICES * blockDim.x) {
        uint32_t v[4] = {0, 0, 0, 0};
        if (w < wl) {
            for (uint32_t b = 0; b < 16 && 16 * w + b < n; b++) v[b / 4] |= (uint32_t)lim[r0 + 16 * w + b] << (8 * (b % 4));
            d_lim[w] = make_uint4(v[0], v[1], v[2], v[3]);
        } else if (w < wl + wf) {
            const uint32_t q = w - wl;
            for (uint32_t b = 0; b < 4 && 4 * q + b < n; b++) v[b] = first[r0 + 4 * q + b];
            d_first[q] = make_uint4(v[0], v[1], v[2], v[3]);
        } else {
            const uint32_t q = (w - wl - wf) % wr;
            const uint64_t* src = (w - wl - wf) < wr ? rem : ttl;
            uint64_t a = src[c0 + 2 * q], b = 2 * q + 1 < nc ? src[c0 + 2 * q + 1] : 0;
            const uint4 u = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
            ((w - wl - wf) < wr ? d_rem : d_ttl)[q] = u;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ctr, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence_system();
    if (tid < X.x.world) rl_st_release_sys(&X.x.ctl(tid, 0, rank)->vflag, step + 1);
    if (tid == 0) *ctr = 0;
}

// Source, after k_xwaitv: every request's outputs back in request order; remaining / ttl (when given) in counter order,
// for the requests that asked for them.
__global__ void __launch_bounds__(256) k_cgather(RlCXchg X, uint32_t n, const uint32_t* __restrict__ off, uint32_t op,
                                                 const uint8_t* __restrict__ load, uint32_t load_all,
                                                 const uint32_t* __restrict__ dest, const uint32_t* __restrict__ cpos,
                                                 uint8_t* out_lim, uint32_t* out_first, uint64_t* out_rem, uint64_t* out_ttl) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t d = dest[i], o = d >> 27, p = d & 0x07FFFFFFu;
        const uint8_t* R = X.ret(X.x.rank, o);
        if (out_lim) out_lim[i] = __ldcg(R + p);
        if (out_first) out_first[i] = __ldcg(reinterpret_cast<const uint32_t*>(R + X.x.cap) + p);
        if (out_rem && (rl_cop(op, load, load_all, i) & RL_COP_LOAD)) {
            const uint64_t* rem = reinterpret_cast<const uint64_t*>(R + 5ull * X.x.cap) + cpos[i];
            const uint64_t* ttl = reinterpret_cast<const uint64_t*>(R + 5ull * X.x.cap + 8ull * X.cap_ctr) + cpos[i];
            const uint32_t c0 = off[i], m = off[i + 1] - c0;
            for (uint32_t k = 0; k < m; k++) {
                out_rem[c0 + k] = __ldcg(rem + k);
                out_ttl[c0 + k] = __ldcg(ttl + k);
            }
        }
    }
}
