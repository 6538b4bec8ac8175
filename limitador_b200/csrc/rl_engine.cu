// rl_engine.cu — host side of librl_engine.so: the device tables of the limit registry (rl_registry.h), workspace,
// kernel launches and the C-ABI declared in include/rl_engine.h.
//
// There is NO CPU fallback: every entry point either runs the sm_90a kernels or returns
// an error.  The reference path this replaces: limitador/src/storage/in_memory.rs
// (InMemoryStorage) behind trait CounterStorage (limitador/src/storage/mod.rs:279-292).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <utility>
#include <vector>

#include "rl_cuda_host.h"
#include "rl_kernels.cuh"
#include "rl_shard.cuh"
#include "rl_internal.h"
#include "rl_registry.h"

#ifndef RL_SETS
#define RL_SETS 3  // RL_FLAG_PIPELINE: calls in flight on the device (>= 3: one per pipeline stage)
#endif
#ifndef RL_RING
#define RL_RING 4  // RL_MEM_HOST_ASYNC: staging slots (H2D of call i+RL_RING waits for the D2H of call i)
#endif

namespace {

constexpr uint32_t kMaxTiles = RL_MAX_TILES;
constexpr uint32_t kMaxRegions = 4096;

}  // namespace

// The per-batch workspace.  With RL_FLAG_PIPELINE there is one per call in flight: the partition kernels of
// batch s+1 run (on their own stream) while k_main of batch s is still replaying.
struct WorkSet {
    DevBuf<uint32_t> tile_loc, region_total, part_idx, part_row, row_of, chain_status,
        chain_wcnt, chain_w, small;  // small: [0] blocks-done counter of the probe, [1] item count, [2] ticket, [3] exit counter
    DevBuf<uint4> items;
};

struct rl_engine {
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    uint32_t cells = 1, log2P = 0, log2R = 0, row_bytes = 32;
    uint64_t capacity = 0;
    uint32_t max_batch = 0, max_counters = 0;
    uint32_t max_ctrs_req = RL_MAX_CTRS_PER_REQ;  // rl_config.max_counters_per_request (16: narrow encoding only)
    DevBuf<uint8_t> d_rows;

    RlRegistry reg;
    uint64_t structure_epoch = 0;  // calls that can move rows or re-map cells (rl_counters_drain: the next drain is full)
    RlTableShape shape;            // of the uploaded tables

    // device tables
    DevBuf<RlCellDesc> d_desc;
    DevBuf<RlLimitDev> d_limits;
    DevBuf<RlNsDev> d_ns;
    DevBuf<uint32_t> d_ns_limit_ids;
    DevBuf<uint32_t> d_group_ns;
    uint32_t limits_cap = 0, ns_cap = 0;

    // workspace
    DevBuf<uint32_t> d_misc;  // misc: err, flags, changed, exchange error detail (MISC_*)
    DevBuf<RlAccess> d_acc;
    // wide batches (max_ctrs_req > 16): perm[slot] = original index of the counter at that position (resolve);
    // remaining / ttl in processing order (k_main with load_counters), before k_wide_scatter
    DevBuf<uint8_t> d_perm;
    DevBuf<uint64_t> d_wide_rem, d_wide_ttl;
    DevBuf<uint64_t> d_delta, d_now;
    DevBuf<uint32_t> d_fl_prev, d_fl_next;
    DevBuf<unsigned long long> d_kstats;
    DevBuf<uint4> d_trace;     // RL_FLAG_TRACE: event ring
    DevBuf<uint32_t> d_hot;    // [RL_HOT_SLOTS] hot rows + [RL_HOT_CAND] candidates + [1] candidate count
    bool hot_rows = false;     // RL_HOT=1 enables the hot-row partitions (k_hot); see DESIGN.md §3.4 for why it is opt-in
    DevBuf<uint32_t> d_misc2;  // [0] trace write position
    uint32_t trace_seq = 0;
    DevBuf<uint8_t*> d_log_row;
    DevBuf<ulonglong2> d_log_state;
    // staging for RL_MEM_HOST calls
    DevBuf<rl_record> d_in_recs;
    DevBuf<uint32_t> d_in_off;
    DevBuf<rl_counter> d_in_ctrs;
    DevBuf<uint64_t> d_in_delta, d_in_now;
    DevBuf<uint8_t> d_out_limited;
    DevBuf<uint32_t> d_out_first;
    DevBuf<uint64_t> d_out_rem, d_out_ttl;
    // bucket helper
    DevBuf<uint32_t> d_bucket;
    DevBuf<unsigned long long> d_bucket_counts;
    PinnedBuf<uint32_t> h_misc;  // pinned mirror of d_misc

    rl_stats stats{};
    std::string last_error = "";
    bool pipeline = false;                 // RL_FLAG_PIPELINE
    bool kernel_stats = false;  // RL_FLAG_KERNEL_STATS
    static constexpr int kSets = RL_SETS;  // workspace sets = calls in flight (probe | scan+scatter | replay)
    WorkSet ws[kSets];                     // sets 1.. are allocated with RL_FLAG_PIPELINE only
    cudaStream_t sq = nullptr;       // scan + scatter stream
    cudaStream_t sp = nullptr, sm = nullptr;  // partition / replay streams
    cudaEvent_t ev_in = nullptr, ev_probe[kSets] = {}, ev_part[kSets] = {}, ev_main[kSets] = {};  // ev_probe: replay done, before a post_main hook
    uint64_t pipe_seq = 0;
    bool pipe_pending = false;
    // RL_MEM_HOST_ASYNC: ring of device staging slots; copies overlap the kernels of other calls
    static constexpr int kRing = RL_RING;
    DevBuf<rl_record> ring_recs[kRing];
    DevBuf<uint8_t> ring_lim[kRing];
    DevBuf<uint32_t> ring_first[kRing];
    cudaEvent_t ev_slot[kRing] = {};  // slot's D2H done
    uint64_t ring_seq = 0;
    bool d2h_pending = false;
    int d2h_last = 0;
    uint32_t weak_slots = 0;           // RL_FLAG_DEBUG_WEAK_TAGS
    uint32_t chunk = 128;              // accesses per k_main chunk (128 or 256; RL_CHUNK overrides)
    uint32_t part_target = 128;        // accesses per partition aimed at (RL_PART_TARGET)
    uint32_t main_grid_cap = 132 * 16;  // k_main CTAs launched at most (SMs x 16)
    uint32_t heavy_mult = 2;           // regions > heavy_mult x average are chained (0 = never; RL_HEAVY_MULT)
    bool profiling = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
    // rl_maint.cu: its per-engine state, and the per-namespace metrics hook (nullptr = off) called behind the replay
    // of a record call, on the stream that carries it
    void* ext = nullptr;
    void (*ext_free)(void*) = nullptr;
    rl_ns_hook_fn ns_hook = nullptr;
};

namespace {

enum { MISC_ERR = 0, MISC_FLAGS = 1, MISC_CHANGED = 3, MISC_XCHG = 7, MISC_N = 8 };

template <class... A>
int fail(rl_engine* e, int status, const char* fmt, A... a) {
    if (e) e->last_error = rl_format(fmt, a...);
    return status;
}

int pipe_fence(rl_engine* e);

#define RL_LAUNCH_CHECK(e)                    \
    do {                                      \
        (e)->stats.kernel_launches++;         \
        RL_CUDA((e), cudaGetLastError());     \
    } while (0)

uint32_t ceil_div(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }

uint32_t log2_ceil(uint64_t x) {
    uint32_t l = 0;
    while ((1ull << l) < x) l++;
    return l;
}

RlDev make_dev(rl_engine* e) {
    RlDev D;
    D.rows = e->d_rows.p;
    D.log2P = e->log2P;
    D.log2R = e->log2R;
    D.desc = e->d_desc.p;
    D.limits = e->d_limits.p;
    D.limits_cap = e->limits_cap;
    D.ns = e->d_ns.p;
    D.ns_cap = e->ns_cap;
    D.ns_limit_ids = e->d_ns_limit_ids.p;
    D.err = e->d_misc.p + MISC_ERR;
    D.flags = e->d_misc.p + MISC_FLAGS;
    D.kstats = e->kernel_stats ? e->d_kstats.p : nullptr;
    D.hot_rows = e->d_hot.p;
    D.hot_cand = e->d_hot.p + RL_HOT_SLOTS;
    D.hot_cand_n = e->d_hot.p + RL_HOT_SLOTS + RL_HOT_CAND;
    D.trace = e->d_trace.p;
    D.trace_pos = e->d_trace.p ? e->d_misc2.p : nullptr;
    D.seq = e->trace_seq;
    return D;
}

// Rebuild and upload the limit / group / namespace tables.
int upload_tables(rl_engine* e) {
    if (!e->reg.dirty) return RL_OK;
    const RlTableImage t = e->reg.image();
    e->shape = t.shape;
    RL_CUDA(e, e->d_desc.reserve(t.desc.size()));
    RL_CUDA(e, e->d_limits.reserve(t.lim.size()));
    RL_CUDA(e, e->d_ns.reserve(t.ns.size()));
    RL_CUDA(e, e->d_ns_limit_ids.reserve(t.ns_ids.size()));
    RL_CUDA(e, e->d_group_ns.reserve(t.group_ns.size()));
    // synchronous copies: the host vectors die at scope exit
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    RL_CUDA(e, cudaMemcpy(e->d_desc.p, t.desc.data(), t.desc.size() * sizeof(RlCellDesc), cudaMemcpyHostToDevice));
    RL_CUDA(e, cudaMemcpy(e->d_limits.p, t.lim.data(), t.lim.size() * sizeof(RlLimitDev), cudaMemcpyHostToDevice));
    RL_CUDA(e, cudaMemcpy(e->d_ns.p, t.ns.data(), t.ns.size() * sizeof(RlNsDev), cudaMemcpyHostToDevice));
    RL_CUDA(e, cudaMemcpy(e->d_ns_limit_ids.p, t.ns_ids.data(), t.ns_ids.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    RL_CUDA(e, cudaMemcpy(e->d_group_ns.p, t.group_ns.data(), t.group_ns.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    e->limits_cap = (uint32_t)t.lim.size();
    e->ns_cap = (uint32_t)t.ns.size();
    e->reg.dirty = false;
    return RL_OK;
}

// Translate the sticky device error (if any) into a status; clears it.
int check_device_error(rl_engine* e) {
    {
        int rf = pipe_fence(e);
        if (rf) return rf;
    }
    RL_CUDA(e, cudaMemcpyAsync(e->h_misc.p, e->d_misc.p, MISC_N * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    const uint32_t code = e->h_misc.p[MISC_ERR];
    if (code == RL_DEV_OK) return RL_OK;
    RL_CUDA(e, cudaMemsetAsync(e->d_misc.p + MISC_ERR, 0, sizeof(uint32_t), e->stream));
    switch (code) {
        case RL_DEV_TABLE_FULL:
            return fail(e, RL_TRANSIENT, "counter table region full (capacity_rows=%llu): batch partially applied",
                        (unsigned long long)e->capacity);
        case RL_DEV_UNKNOWN_LIMIT:
            return fail(e, RL_FATAL, "request names a limit_id that was never registered with rl_limits_set");
        case RL_DEV_KEY_RANGE:
            return fail(e, RL_FATAL, "key_hi bits 32..55 must be zero (counter identity is a 96-bit digest)");
        case RL_DEV_TOO_MANY_COUNTERS:
            return fail(e, RL_FATAL, "a request has more than %u counters", e->max_ctrs_req);
        case RL_DEV_EXCHANGE: {
            const uint32_t d = e->h_misc.p[MISC_XCHG];
            RL_CUDA(e, cudaMemsetAsync(e->d_misc.p + MISC_XCHG, 0, sizeof(uint32_t), e->stream));
            const char* what = (d >> 28) == 1 ? "records of source rank" : (d >> 28) == 2 ? "verdicts of owner rank" : "inbox larger than max_batch, rank";
            return fail(e, RL_FATAL, "peer exchange failed at step %u: %s %u did not arrive within %.0f s (or a block fill was out of range)",
                        d & 0xFFFFFu, what, (d >> 20) & 0xFFu, (double)RL_XCHG_TIMEOUT_NS * 1e-9);
        }
        default:
            return fail(e, RL_FATAL, "device error code %u", code);
    }
}

// A resolve kernel (request -> accesses) found a request the engine cannot take (unknown limit, more than
// max_counters_per_request counters, key out of range): refuse the WHOLE call before anything touches the
// table, so that the caller can fix the batch and retry without double counting (ADVICE r1).
int check_resolve_error(rl_engine* e) {
    RL_CUDA(e, cudaMemcpyAsync(e->h_misc.p, e->d_misc.p, MISC_N * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    if (e->h_misc.p[MISC_ERR] == RL_DEV_OK) return RL_OK;
    int r = check_device_error(e);
    if (r == RL_OK) r = RL_FATAL;
    e->last_error += " — the call was refused before the table was touched";
    return r;
}

struct Outs {
    uint8_t* limited = nullptr;
    uint32_t* first = nullptr;
    uint64_t* rem = nullptr;
    uint64_t* ttl = nullptr;
    const uint32_t* off = nullptr;
    uint32_t stride = 0;
};

RlBatch make_batch(rl_engine* e, uint32_t n_acc, uint32_t n_req, const Outs& o, int lc, int set = 0, uint32_t n_hint = 0,
                   bool hot_ok = true) {
    const WorkSet& w = e->ws[set];
    RlBatch B;
    B.nhot = (hot_ok && e->hot_rows) ? RL_HOT_SLOTS : 0;
    B.n_acc = n_acc;
    B.n_req = n_req;
    B.n_dev = nullptr;
    B.omap_prefix = nullptr;
    B.omap_n = 0;
    B.omap_stride = 0;
    B.tile_loc = w.tile_loc.p;
    B.region_total = w.region_total.p;
    B.part_idx = w.part_idx.p;
    B.row_of = w.row_of.p;
    B.part_row = w.part_row.p;
    B.scan_ctr = w.small.p + 0;
    B.ticket = w.small.p + 2;
    B.exit_ctr = w.small.p + 3;
    // n_hint (sharded steps): n_acc is only the upper bound of a device-side count (rl_batch_geom)
    const RlBatchGeom g = rl_batch_geom(n_acc, n_hint, e->log2P, e->part_target, e->chunk, e->heavy_mult);
    B.tile = g.tile;
    B.num_tiles = g.num_tiles;
    B.out_limited = o.limited;
    B.out_first_limited = o.first;
    B.out_remaining = o.rem;
    B.out_ttl = o.ttl;
    B.out_off = o.off;
    B.out_stride = o.stride;
    B.fl_prev = e->d_fl_prev.p;
    B.fl_next = e->d_fl_next.p;
    B.phase = RL_PHASE_COMMIT;
    B.load_counters = lc;
    B.items = w.items.p;
    B.n_items = w.small.p + 1;
    B.chain_status = w.chain_status.p;
    B.chain_wcnt = w.chain_wcnt.p;
    B.chain_w = w.chain_w.p;
    B.chunk = e->chunk;
    // a region is split into chained chunks only when it is far heavier than the average one; partition
    // granularity: about one k_main chunk per partition, never finer than the table's regions
    B.part_shift = g.part_shift;
    B.nparts = g.nparts;
    B.heavy_len = g.heavy_len;
    B.log_row = nullptr;
    B.log_state = nullptr;
    return B;
}

// probe + stable partition by table region (one launch)
template <class Src>
int launch_front(rl_engine* e, const RlDev& D, const RlBatch& B, const Src& src, cudaStream_t st = nullptr) {
    if (!st) st = e->stream;
    const size_t smem = rl_front_smem_bytes(B.nparts, B.nhot);
    return rl_with_cells(e->cells, [&](auto c) -> int {
        auto kern = k_front<decltype(c)::value, Src>;
        static int smem_limit[64] = {};  // per instantiation and device: raised as engines with more regions appear
        const int dv = e->device & 63;
        // (k_front also has ~8 KB of static shared memory: opt in well before the 48 KB default is reached)
        if (smem > 32 * 1024 && (int)smem > smem_limit[dv]) {
            const int max_smem = (int)rl_front_smem_bytes(1u << e->log2P, RL_HOT_SLOTS);
            RL_CUDA(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
            smem_limit[dv] = max_smem;
        }
        kern<<<B.num_tiles, RL_PART_THREADS, smem, st>>>(D, B, src);
        RL_LAUNCH_CHECK(e);
        return RL_OK;
    });
}

template <int GEO, int CELLS, class Src, int MODE, bool LC, int CH>
int launch_main_ch(rl_engine* e, const RlDev& D, const RlBatch& B, const Src& src, cudaStream_t st) {
    auto kern = k_main<GEO, CELLS, Src, MODE, CH, LC>;
    static bool attr_set[64] = {};  // per instantiation and device (function attributes are per device)
    const int dv = e->device & 63;
    if (!attr_set[dv]) {
        RL_CUDA(e, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)rl_main_smem_bytes<CELLS, CH>(RL_MAX_TILES)));
        attr_set[dv] = true;
    }
    // upper bound of the work-item count: one per partition + one per chunk of a heavy partition; CTAs take
    // items from a ticket, so a smaller grid only means that some CTAs take several
    // (capping the grid at one resident wave was tried: the CTAs that then take a second item make the kernel last
    // two chunk latencies instead of one)
    const uint32_t grid = rl_main_grid(B.nparts, B.n_acc, CH, e->main_grid_cap);
    kern<<<grid, CH, rl_main_smem_bytes<CELLS, CH>(B.num_tiles), st>>>(D, B, src, e->weak_slots);
    return RL_OK;
}

template <int GEO, int CELLS, class Src, int MODE, bool LC>
int launch_main_cells(rl_engine* e, const RlDev& D, const RlBatch& B, const Src& src, cudaStream_t st) {
    if constexpr (Src::kWide) {
        // wide batches get no hot rows (run_acc_pipeline) and run 128-access chunks only
        return launch_main_ch<GEO, CELLS, Src, MODE, LC, 128>(e, D, B, src, st);
    } else {
        if (B.nhot && B.phase == RL_PHASE_COMMIT) {
            // the hot rows' partitions: one CTA per hot slot (most exit at once), ahead of the cold partitions
            k_hot<GEO, CELLS, Src, MODE, LC><<<B.nhot, RL_HOT_THREADS, 0, st>>>(D, B, src);
            RL_LAUNCH_CHECK(e);
        }
        return e->chunk == 128 ? launch_main_ch<GEO, CELLS, Src, MODE, LC, 128>(e, D, B, src, st)
                               : launch_main_ch<GEO, CELLS, Src, MODE, LC, 256>(e, D, B, src, st);
    }
}

template <class Src, int MODE>
int launch_main(rl_engine* e, const RlDev& D, const RlBatch& B, const Src& src, cudaStream_t st = nullptr) {
    if (!st) st = e->stream;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (e->profiling) {
        RL_CUDA(e, cudaEventCreate(&ev0));
        RL_CUDA(e, cudaEventCreate(&ev1));
        RL_CUDA(e, cudaEventRecord(ev0, st));
    }
    const bool lc = (MODE == 0) && B.load_counters;
    const int r = rl_with_main_cells(e->cells, e->shape.max_cells_used, [&](auto g, auto c) {
        constexpr int G = decltype(g)::value, A = decltype(c)::value;
        return lc ? launch_main_cells<G, A, Src, MODE, MODE == 0>(e, D, B, src, st)
                  : launch_main_cells<G, A, Src, MODE, false>(e, D, B, src, st);
    });
    if (r) return r;
    RL_LAUNCH_CHECK(e);
    if (e->profiling) {
        RL_CUDA(e, cudaEventRecord(ev1, st));
        e->prof_events.emplace_back(ev0, ev1);
    }
    return RL_OK;
}

// Make the caller's stream wait for everything the pipeline still has in flight.
int pipe_fence(rl_engine* e) {
    if (!e->pipe_pending) return RL_OK;
    const int last = (int)((e->pipe_seq - 1) % rl_engine::kSets);
    RL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_main[last], 0));
    if (e->d2h_pending) RL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_slot[e->d2h_last], 0));
    e->d2h_pending = false;
    e->pipe_pending = false;
    return RL_OK;
}

// Runs partition + main for accesses that may contain multi-row requests (AccSrc).
// mode: 0 check_and_update, 2 update.  wide: the accesses were resolved with the wide position encoding
// (k_resolve_*_wide); check_and_update then runs the wide k_main, whose remaining / ttl go to scratch in processing
// order (slot = off[req] + position, or req * acc_stride + position for records) and are scattered into `o` at the
// end.  update_counters never reads positions: its k_main is the same for both encodings.
int run_acc_pipeline(rl_engine* e, uint32_t n_acc, uint32_t n_req, const uint64_t* d_delta, const uint64_t* d_now,
                     int mode, int lc, const Outs& o, bool wide = false, uint32_t acc_stride = 0) {
    RlDev D = make_dev(e);
    const bool scatter = wide && mode == 0 && lc && (o.rem || o.ttl);
    Outs ob = o;  // where k_main writes
    if (scatter) {
        RL_CUDA(e, e->d_wide_rem.reserve(e->max_counters));
        RL_CUDA(e, e->d_wide_ttl.reserve(e->max_counters));
        if (o.rem) ob.rem = e->d_wide_rem.p;
        if (o.ttl) ob.ttl = e->d_wide_ttl.p;
        if (!o.off) ob.stride = acc_stride;
    }
    // check_and_update in the general form may hold coupled (multi-row) requests, replayed in phases: partitions
    // stay sequential and no row gets a partition of its own
    RlBatch B = make_batch(e, n_acc, n_req, ob, lc, 0, 0, mode != 0);
    if (mode == 0) B.heavy_len = 0xFFFFFFFFu;
    AccSrc src{e->d_acc.p, d_delta, d_now};
    int r = launch_front(e, D, B, src);
    if (r) return r;
    if (mode == 2) return launch_main<AccSrc, 2>(e, D, B, src);
    auto main0 = [&]() { return wide ? launch_main<AccSrcWide, 0>(e, D, B, AccSrcWide{src}) : launch_main<AccSrc, 0>(e, D, B, src); };
    // does the batch contain coupled (multi-row) requests?
    RL_CUDA(e, cudaMemcpyAsync(e->h_misc.p, e->d_misc.p, MISC_N * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stats.fixed_point_rounds = 0;
    if (e->h_misc.p[MISC_FLAGS] & 1u) {
        RL_CUDA(e, cudaMemsetAsync(e->d_misc.p + MISC_FLAGS, 0, sizeof(uint32_t), e->stream));
        RL_CUDA(e, e->d_fl_prev.reserve(e->max_batch));
        RL_CUDA(e, e->d_fl_next.reserve(e->max_batch));
        B.fl_prev = e->d_fl_prev.p;
        B.fl_next = e->d_fl_next.p;
        RL_CUDA(e, cudaMemsetAsync(B.fl_prev, 0xFF, n_req * sizeof(uint32_t), e->stream));
        RL_CUDA(e, cudaMemsetAsync(B.fl_next, 0xFF, n_req * sizeof(uint32_t), e->stream));
        // undo log: original state of every row the batch touches
        const uint32_t buf_len = B.num_tiles * B.tile;  // positions of part_idx/part_row in use
        RL_CUDA(e, e->d_log_row.reserve(buf_len));
        RL_CUDA(e, e->d_log_state.reserve((size_t)buf_len * e->cells));
        B.log_row = e->d_log_row.p;
        B.log_state = e->d_log_state.p;
        RL_CUDA(e, cudaMemsetAsync(B.log_row, 0, (size_t)buf_len * sizeof(uint8_t*), e->stream));
        B.phase = RL_PHASE_SNAPSHOT;
        r = main0();
        if (r) return r;
        // Fixed-point iteration over the requests' first-limited positions (DESIGN.md §3.4):
        // each speculative round replays the batch from the committed table state.
        for (uint32_t round = 0;; round++) {
            if (round > n_req + 2) return fail(e, RL_FATAL, "fixed-point iteration did not converge");
            RL_CUDA(e, cudaMemsetAsync(e->d_misc.p + MISC_CHANGED, 0, sizeof(uint32_t), e->stream));
            B.phase = RL_PHASE_SPEC;
            r = main0();
            if (r) return r;
            rl_with_main_cells(e->cells, e->shape.max_cells_used, [&](auto g, auto c) {
                k_restore<decltype(g)::value><<<ceil_div(buf_len, 256), 256, 0, e->stream>>>(buf_len, decltype(c)::value,
                                                                                            B.log_row, B.log_state);
            });
            RL_LAUNCH_CHECK(e);
            k_fl_step<<<ceil_div(n_req, 256), 256, 0, e->stream>>>(n_req, B.fl_prev, B.fl_next,
                                                                    e->d_misc.p + MISC_CHANGED);
            RL_LAUNCH_CHECK(e);
            RL_CUDA(e, cudaMemcpyAsync(e->h_misc.p, e->d_misc.p, MISC_N * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                                       e->stream));
            RL_CUDA(e, cudaStreamSynchronize(e->stream));
            e->stats.fixed_point_rounds = round + 1;
            if (!(e->h_misc.p[MISC_CHANGED] & 1u)) break;
        }
    }
    B.phase = RL_PHASE_COMMIT;
    if ((r = main0()) || !scatter) return r;
    k_wide_scatter<<<ceil_div(n_req, 128), 128, 0, e->stream>>>(n_req, o.off, acc_stride, o.stride, e->d_perm.p, ob.rem,
                                                                 ob.ttl, o.rem, o.ttl);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

// Hooks of the sharded step (rl_shard_*): the owner's inbox is a segmented record source whose size is
// only known on the device; `pre_probe` runs on the probe stream right before the probe (it waits for
// the peers' blocks), `post_main` on the replay stream right behind k_main (it returns the verdicts).
struct PipeHooks {
    RecordSrc src;
    const uint32_t* n_dev = nullptr;
    std::function<void(RlBatch&)> patch_batch;  // verdict routing of a sharded step
    std::function<int(cudaStream_t, int)> pre_probe, post_main;  // (stream, workspace set)
};

// compact_now != 0: d_recs points at n 16-byte rl_record16 stamped with that one clock reading
int run_record_pipeline(rl_engine* e, uint32_t n, const rl_record* d_recs, int mode, int lc, const Outs& o,
                        bool may_pipeline = false, const PipeHooks* hooks = nullptr, uint32_t n_hint = 0,
                        uint64_t compact_now = 0) {
    RlDev D = make_dev(e);
    const bool pipelined = may_pipeline && e->pipeline && !e->shape.any_multi_ns;
    if (hooks && !pipelined) return fail(e, RL_FATAL, "sharded steps need RL_FLAG_PIPELINE and single-row namespaces");
    int r = pipelined ? RL_OK : pipe_fence(e);
    if (r) return r;
    if (e->shape.any_multi_ns) {
        if (compact_now) return fail(e, RL_FATAL, "16-byte records need single-row namespaces (use the 32-byte form)");
        // some namespace spans several rows: materialise accesses (stride = max limits per ns)
        const uint32_t stride = e->shape.record_stride(e->cells);
        if (stride > e->max_ctrs_req)
            return fail(e, RL_FATAL, "a namespace has more than %u limits", e->max_ctrs_req);
        const uint64_t n_acc = (uint64_t)n * stride;
        if (n_acc > e->d_acc.n)
            return fail(e, RL_FATAL, "batch of %u records x %u limits exceeds max_counters=%u", n, stride, e->max_counters);
        RlResolveOut O{e->d_acc.p, e->d_delta.p, e->d_now.p, o.limited, o.first};
        // the namespace with the most limits sets the stride, and with it the encoding of the whole batch
        const bool wide = stride > RL_MAX_CTRS_PER_REQ;
        if (wide)
            k_resolve_records_wide<<<ceil_div(n, 128), 128, 0, e->stream>>>(D, n, d_recs, stride, O, mode == 0, e->d_perm.p,
                                                                             e->max_ctrs_req);
        else
            k_resolve_records<<<ceil_div(n, 128), 128, 0, e->stream>>>(D, n, d_recs, stride, O, mode == 0);
        RL_LAUNCH_CHECK(e);
        if ((r = check_resolve_error(e))) return r;
        r = run_acc_pipeline(e, (uint32_t)n_acc, n, e->d_delta.p, e->d_now.p, mode, lc, o, wide, stride);
        if (r == RL_OK && e->ns_hook && mode == 0 && o.limited) r = e->ns_hook(e, e->stream, n, d_recs, 32, o.limited, o.first);
        return r;
    }
    // Pipelined, this is a two-stage software pipeline over successive calls: the front (probe + partition,
    // `sp`) of batch s+1 (and s+2) overlaps the replay of batch s (`sm`).  The front only reads row headers
    // and claims empty rows; the replay only touches the cells of rows found by ITS front, and replays stay
    // in call order on `sm`, so the table sees the batches in order.  Otherwise both run on the caller's stream.
    const int k = pipelined ? (int)(e->pipe_seq % rl_engine::kSets) : 0;
    const cudaStream_t sf = pipelined ? e->sp : e->stream, sr = pipelined ? e->sm : e->stream;  // front, replay
    RlBatch B = make_batch(e, n, n, o, lc, k, n_hint);
    RecordSrc src{d_recs, nullptr, 0, 0, compact_now ? 1u : 0u, compact_now};
    if (hooks) {
        // the inbox is filled by the peers' kernels and handed over through step flags, not through
        // anything on the caller's stream
        src = hooks->src;
        B.n_dev = hooks->n_dev;
        if (hooks->patch_batch) hooks->patch_batch(B);
    } else if (pipelined) {
        RL_CUDA(e, cudaEventRecord(e->ev_in, e->stream));  // inputs: whatever the caller enqueued so far
        RL_CUDA(e, cudaStreamWaitEvent(e->sp, e->ev_in, 0));
    }
    if (pipelined && e->pipe_seq >= (uint64_t)rl_engine::kSets)
        RL_CUDA(e, cudaStreamWaitEvent(e->sp, e->ev_main[k], 0));  // workspace set k is free again
    if (hooks && hooks->pre_probe && (r = hooks->pre_probe(e->sp, k))) return r;
    if ((r = launch_front(e, D, B, src, sf))) return r;
    if (pipelined) {
        RL_CUDA(e, cudaEventRecord(e->ev_part[k], e->sp));
        RL_CUDA(e, cudaStreamWaitEvent(e->sm, e->ev_part[k], 0));
    }
    r = mode == 2 ? launch_main<RecordSrc, 2>(e, D, B, src, sr) : launch_main<RecordSrc, 0>(e, D, B, src, sr);
    if (r) return r;
    // per-namespace metrics (rl_ns_metrics_enable): one reduction kernel right behind the replay, same stream
    if (e->ns_hook && !hooks && mode == 0 && o.limited &&
        (r = e->ns_hook(e, sr, n, d_recs, compact_now ? 16 : 32, o.limited, o.first)))
        return r;
    if (!pipelined) return RL_OK;
    if (hooks && hooks->post_main) {
        // the hook (a sharded step's verdict return) runs on its own stream: the replay of the next call does
        // not wait for it, only the reuse of this workspace set does
        RL_CUDA(e, cudaEventRecord(e->ev_probe[k], e->sm));
        RL_CUDA(e, cudaStreamWaitEvent(e->sq, e->ev_probe[k], 0));
        if ((r = hooks->post_main(e->sq, k))) return r;
        RL_CUDA(e, cudaEventRecord(e->ev_main[k], e->sq));
    } else {
        RL_CUDA(e, cudaEventRecord(e->ev_main[k], e->sm));
    }
    e->pipe_seq++;
    e->pipe_pending = true;
    return RL_OK;
}

int ensure_ready(rl_engine* e, uint64_t n, bool fence = true) {
    if (!e) return RL_FATAL;
    if (fence) {
        int rf = pipe_fence(e);
        if (rf) return rf;
    }
    if (n > e->max_batch) return fail(e, RL_FATAL, "batch of %llu exceeds max_batch=%u", (unsigned long long)n, e->max_batch);
    RL_CUDA(e, cudaSetDevice(e->device));
    if (e->reg.dirty && e->pipeline) {
        int r = pipe_fence(e);
        if (r) return r;
        RL_CUDA(e, cudaStreamSynchronize(e->sp));
        RL_CUDA(e, cudaStreamSynchronize(e->sq));
        RL_CUDA(e, cudaStreamSynchronize(e->sm));
    }
    return upload_tables(e);
}

// Force the (lazy) loading of the kernels a record-form check_and_update launches for this engine's geometry.
template <int GEO, int CELLS>
int preload_main(rl_engine* e) {
    cudaFuncAttributes fa;
    RL_CUDA(e, cudaFuncGetAttributes(&fa, k_hot<GEO, CELLS, RecordSrc, 0, false>));
    if (e->chunk == 128) {
        RL_CUDA(e, cudaFuncGetAttributes(&fa, k_main<GEO, CELLS, RecordSrc, 0, 128, false>));
        RL_CUDA(e, cudaFuncSetAttribute(k_main<GEO, CELLS, RecordSrc, 0, 128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)rl_main_smem_bytes<CELLS, 128>(RL_MAX_TILES)));
    } else {
        RL_CUDA(e, cudaFuncGetAttributes(&fa, k_main<GEO, CELLS, RecordSrc, 0, 256, false>));
        RL_CUDA(e, cudaFuncSetAttribute(k_main<GEO, CELLS, RecordSrc, 0, 256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)rl_main_smem_bytes<CELLS, 256>(RL_MAX_TILES)));
    }
    return RL_OK;
}
int preload_record_kernels(rl_engine* e) {
    int r = upload_tables(e);  // max_cells_used selects the k_main instantiation
    if (r) return r;
    cudaFuncAttributes fa;
    RL_CUDA(e, rl_with_cells(e->cells, [&](auto c) {
                return cudaFuncGetAttributes(&fa, k_front<decltype(c)::value, RecordSrc>);
            }));
    // k_main for the fewest and the most cells in use: every instantiation the limits set later can select
    for (const uint32_t used : {1u, (uint32_t)RL_MAX_CELLS})
        if ((r = rl_with_main_cells(e->cells, used,
                                    [&](auto g, auto c) { return preload_main<decltype(g)::value, decltype(c)::value>(e); })))
            return r;
    return RL_OK;
}

// Allocates one workspace set for batches of up to max_counters accesses.
int alloc_workset(rl_engine* e, WorkSet& w) {
    const uint32_t P1 = (1u << e->log2P) + RL_HOT_SLOTS + 1;  // cold partitions + hot slots + the no-row bucket
    const size_t maxA = e->max_counters;
    const size_t bufA = maxA + maxA / 128 + 256 * 1024 + 1024;  // part_idx/part_row: every tile's slice is a whole tile
    const size_t max_items = (size_t)(1u << e->log2P) + maxA / 128 + 2;
    RL_CUDA(e, w.tile_loc.reserve((size_t)(kMaxTiles + 1) * (P1 + 1)));
    RL_CUDA(e, w.region_total.reserve(P1 + 1));
    RL_CUDA(e, cudaMemsetAsync(w.region_total.p, 0, (P1 + 1) * sizeof(uint32_t), e->stream));
    RL_CUDA(e, w.part_idx.reserve(bufA));
    RL_CUDA(e, w.part_row.reserve(bufA));
    RL_CUDA(e, w.row_of.reserve(maxA));
    RL_CUDA(e, w.items.reserve(max_items));
    RL_CUDA(e, w.chain_status.reserve(max_items));
    RL_CUDA(e, w.chain_wcnt.reserve(max_items));
    RL_CUDA(e, w.chain_w.reserve(max_items * 256));
    RL_CUDA(e, w.small.reserve(8));
    RL_CUDA(e, cudaMemsetAsync(w.small.p, 0, 8 * sizeof(uint32_t), e->stream));
    return RL_OK;
}

}  // namespace

// =======================================================================================
extern "C" {

uint32_t rl_owner_of(uint32_t ns_id, uint32_t world) {
    return world ? (uint32_t)(rl_mix64((uint64_t)ns_id + 0x51ed270b0a1fULL) % world) : 0;
}

const char* rl_last_error(rl_engine* e) { return e ? e->last_error.c_str() : "null engine"; }

uint32_t rl_engine_max_counters_per_request(rl_engine* e) { return e ? e->max_ctrs_req : RL_MAX_COUNTERS_PER_REQUEST; }

int rl_engine_create(const rl_config* cfg, rl_engine** out) {
    if (!cfg || !out) return RL_FATAL;
    *out = nullptr;
    if (cfg->struct_size != sizeof(rl_config)) return RL_FATAL;
    if (cfg->cells_per_row != 1 && cfg->cells_per_row != 3 && cfg->cells_per_row != 7) return RL_FATAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device >= ndev || cfg->device < 0) {
        // No CPU fallback exists: without a CUDA device the engine cannot be created.
        return RL_FATAL;
    }
    rl_engine* e = new rl_engine();
    *out = e;  // returned even on failure so the caller can read rl_last_error, then destroy
    e->device = cfg->device;
    {
        const uint32_t w = cfg->max_counters_per_request;
        if (w != 0 && (w < RL_MAX_COUNTERS_PER_REQUEST || w > RL_MAX_COUNTERS_PER_REQUEST_WIDE))
            return fail(e, RL_FATAL, "max_counters_per_request=%u: must be 0 (= %d) or %d..%d", w, RL_MAX_COUNTERS_PER_REQUEST,
                        RL_MAX_COUNTERS_PER_REQUEST, RL_MAX_COUNTERS_PER_REQUEST_WIDE);
        if (w) e->max_ctrs_req = w;
    }
    RL_CUDA(e, cudaSetDevice(e->device));
    cudaDeviceProp prop;
    RL_CUDA(e, cudaGetDeviceProperties(&prop, e->device));
    // the library holds sm_90a code only, which no other architecture can load
    if (prop.major != 9 || prop.minor != 0) return fail(e, RL_FATAL, "device sm_%d%d is not sm_90a", prop.major, prop.minor);
    e->main_grid_cap = (uint32_t)prop.multiProcessorCount * 16u;
    // The table is read one random 32-B sector (a row header, a cell) at a time: ask the L2 not to fetch the
    // neighbouring sector from HBM along with it (the default granularity is 64 B).  A hint; per device.
    if (const char* v = getenv("RL_L2_FETCH")) {
        if (atoi(v) > 0) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(v));
    }
    RL_CUDA(e, cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    e->stream = e->own_stream;
    e->cells = cfg->cells_per_row;
    e->row_bytes = 16 * (1 + e->cells);
    uint32_t lg = std::max<uint32_t>(log2_ceil(std::max<uint64_t>(cfg->capacity_rows, 64)), 6);
    e->capacity = 1ull << lg;
    uint32_t regions = cfg->regions;
    if (regions == 0) {
        // auto: >= 1024 rows per region, at most 1024 regions
        regions = (uint32_t)std::min<uint64_t>(1024, std::max<uint64_t>(1, e->capacity / 1024));
    }
    if (regions & (regions - 1)) return fail(e, RL_FATAL, "regions must be a power of two");
    if (regions > kMaxRegions || (uint64_t)regions * 16 > e->capacity)
        return fail(e, RL_FATAL, "regions=%u out of range for capacity %llu", regions, (unsigned long long)e->capacity);
    e->log2P = log2_ceil(regions);
    e->log2R = lg - e->log2P;
    if (e->log2R > 31) return fail(e, RL_FATAL, "rows per region exceeds 2^31; raise regions");
    if (lg > 31) return fail(e, RL_FATAL, "capacity_rows must not exceed 2^31");
    e->max_batch = std::max<uint32_t>(cfg->max_batch, 1);
    e->max_counters = cfg->max_counters ? cfg->max_counters : 4 * e->max_batch;
    e->max_counters = std::max(e->max_counters, e->max_batch);
    e->reg.cells = e->cells;
    if (const char* v = getenv("RL_CHUNK")) e->chunk = (atoi(v) == 128) ? 128 : 256;
    if (const char* v = getenv("RL_HEAVY_MULT")) e->heavy_mult = (uint32_t)atoi(v);
    if (const char* v = getenv("RL_PART_TARGET")) e->part_target = std::max(16, atoi(v));
    if (cfg->flags & 1u) e->weak_slots = 1;  // RL_FLAG_DEBUG_WEAK_TAGS: four home slots in the grouping table

    const size_t bytes = (size_t)e->capacity * e->row_bytes;
    RL_CUDA(e, e->d_rows.reserve(bytes));
    RL_CUDA(e, cudaMemsetAsync(e->d_rows.p, 0, bytes, e->stream));

    int r = alloc_workset(e, e->ws[0]);
    if (r) return r;
    RL_CUDA(e, e->d_misc.reserve(MISC_N));
    RL_CUDA(e, cudaMemsetAsync(e->d_misc.p, 0, MISC_N * sizeof(uint32_t), e->stream));
    RL_CUDA(e, e->h_misc.exact(MISC_N));
    RL_CUDA(e, e->d_acc.reserve(e->max_counters));
    if (e->max_ctrs_req > RL_MAX_CTRS_PER_REQ) RL_CUDA(e, e->d_perm.reserve(e->max_counters));
    RL_CUDA(e, e->d_kstats.reserve(32));
    RL_CUDA(e, cudaMemsetAsync(e->d_kstats.p, 0, 32 * sizeof(unsigned long long), e->stream));
    RL_CUDA(e, e->d_delta.reserve(e->max_batch));
    RL_CUDA(e, e->d_now.reserve(e->max_batch));
    e->kernel_stats = (cfg->flags & RL_FLAG_KERNEL_STATS) != 0;
    e->hot_rows = (cfg->flags & RL_FLAG_HOT_ROWS) != 0;
    if (const char* v = getenv("RL_HOT")) e->hot_rows = atoi(v) != 0;
    RL_CUDA(e, e->d_hot.reserve(RL_HOT_SLOTS + RL_HOT_CAND + 4));
    if ((r = rl_internal_reset_hot_rows(e))) return r;
    RL_CUDA(e, e->d_misc2.reserve(4));
    RL_CUDA(e, cudaMemsetAsync(e->d_misc2.p, 0, 4 * sizeof(uint32_t), e->stream));
    if (cfg->flags & RL_FLAG_TRACE) {
        RL_CUDA(e, e->d_trace.reserve(RL_TRACE_CAP));
        RL_CUDA(e, cudaMemsetAsync(e->d_trace.p, 0, RL_TRACE_CAP * sizeof(uint4), e->stream));
    }
    if (cfg->flags & 2u) {  // RL_FLAG_PIPELINE
        e->pipeline = true;
        RL_CUDA(e, cudaStreamCreateWithFlags(&e->sp, cudaStreamNonBlocking));
        RL_CUDA(e, cudaStreamCreateWithFlags(&e->sm, cudaStreamNonBlocking));
        for (int k = 0; k < rl_engine::kRing; k++) RL_CUDA(e, cudaEventCreateWithFlags(&e->ev_slot[k], cudaEventDisableTiming));
        RL_CUDA(e, cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming));
        RL_CUDA(e, cudaStreamCreateWithFlags(&e->sq, cudaStreamNonBlocking));
        for (int k = 0; k < rl_engine::kSets; k++) {
            RL_CUDA(e, cudaEventCreateWithFlags(&e->ev_probe[k], cudaEventDisableTiming));
            RL_CUDA(e, cudaEventCreateWithFlags(&e->ev_part[k], cudaEventDisableTiming));
            RL_CUDA(e, cudaEventCreateWithFlags(&e->ev_main[k], cudaEventDisableTiming));
            if (k > 0 && (r = alloc_workset(e, e->ws[k]))) return r;  // set 0 is allocated above
        }
    }
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stats.capacity_rows = e->capacity;
    e->stats.regions = 1u << e->log2P;
    e->stats.row_bytes = e->row_bytes;
    return RL_OK;
}

void rl_engine_destroy(rl_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    for (cudaStream_t st : {e->sp, e->sm, e->sq, e->stream})
        if (st) cudaStreamSynchronize(st);
    // the maintenance state goes first, once its kernels (on e->stream and the replay stream) are done
    if (e->ext && e->ext_free) {
        e->ext_free(e->ext);
        e->ext = nullptr;
    }
    for (cudaEvent_t ev : e->ev_slot)
        if (ev) cudaEventDestroy(ev);
    if (e->ev_in) cudaEventDestroy(e->ev_in);
    for (int k = 0; k < rl_engine::kSets; k++) {
        if (e->ev_probe[k]) cudaEventDestroy(e->ev_probe[k]);
        if (e->ev_part[k]) cudaEventDestroy(e->ev_part[k]);
        if (e->ev_main[k]) cudaEventDestroy(e->ev_main[k]);
    }
    for (cudaStream_t st : {e->sq, e->sp, e->sm, e->own_stream})
        if (st) cudaStreamDestroy(st);
    delete e;  // frees the device and pinned buffers, on the device made current above
}

int rl_engine_set_stream(rl_engine* e, void* cuda_stream) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    {
        int rf = pipe_fence(e);
        if (rf) return rf;
    }
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stream = cuda_stream ? (cudaStream_t)cuda_stream : e->own_stream;
    return RL_OK;
}

void* rl_engine_stream(rl_engine* e) { return e ? (void*)e->stream : nullptr; }

int rl_sync(rl_engine* e) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    return check_device_error(e);
}

int rl_fence(rl_engine* e) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    return pipe_fence(e);
}

int rl_fence_call(rl_engine* e, uint32_t age) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (!e->pipeline || e->pipe_seq == 0) return RL_OK;
    if (age == 0) return pipe_fence(e);
    if (age >= (uint32_t)rl_engine::kSets) return fail(e, RL_FATAL, "rl_fence_call: age must be < %d", rl_engine::kSets);
    if (e->pipe_seq <= age) return RL_OK;
    // an earlier call: its replay event is still the one recorded for it
    RL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_main[(e->pipe_seq - 1 - age) % rl_engine::kSets], 0));
    return RL_OK;
}

int rl_profile_begin(rl_engine* e) {
    if (!e) return RL_FATAL;
    e->profiling = true;
    return RL_OK;
}

int rl_profile_end(rl_engine* e, double* out_main_ms, uint64_t* out_main_launches) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    e->profiling = false;
    {
        int rf = pipe_fence(e);
        if (rf) return rf;
    }
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    double ms = 0;
    for (auto& pr : e->prof_events) {
        float t = 0;
        RL_CUDA(e, cudaEventElapsedTime(&t, pr.first, pr.second));
        ms += t;
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    if (out_main_ms) *out_main_ms = ms;
    if (out_main_launches) *out_main_launches = e->prof_events.size();
    e->prof_events.clear();
    return RL_OK;
}

int rl_trace_dump(rl_engine* e, uint32_t cap, uint32_t* out_ev, uint32_t* out_seq, uint64_t* out_ns, uint32_t* out_count) {
    if (!e || !out_count) return RL_FATAL;
    *out_count = 0;
    if (!e->d_trace.p) return RL_OK;
    RL_CUDA(e, cudaSetDevice(e->device));
    RL_CUDA(e, cudaDeviceSynchronize());
    uint32_t pos = 0;
    RL_CUDA(e, cudaMemcpy(&pos, e->d_misc2.p, sizeof pos, cudaMemcpyDeviceToHost));
    const uint32_t n = std::min<uint32_t>(pos, RL_TRACE_CAP);
    std::vector<uint4> ev(n);
    if (n) RL_CUDA(e, cudaMemcpy(ev.data(), e->d_trace.p, (size_t)n * sizeof(uint4), cudaMemcpyDeviceToHost));
    const uint32_t m = std::min(n, cap);
    for (uint32_t i = 0; i < m; i++) {
        out_ev[i] = ev[i].x;
        out_seq[i] = ev[i].y;
        out_ns[i] = ((uint64_t)ev[i].w << 32) | ev[i].z;
    }
    *out_count = m;
    RL_CUDA(e, cudaMemset(e->d_misc2.p, 0, sizeof(uint32_t)));
    return RL_OK;
}

int rl_get_stats(rl_engine* e, rl_stats* out) {
    if (!e || !out) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    {
        int rf = pipe_fence(e);
        if (rf) return rf;
    }
    unsigned long long ks[32];
    RL_CUDA(e, cudaMemcpyAsync(ks, e->d_kstats.p, sizeof ks, cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stats.chunks = ks[0];
    e->stats.replay_rounds = ks[1];
    e->stats.chained_chunks = ks[2];
    e->stats.ordered_chunks = ks[3];
    for (int i = 0; i < 6; i++) e->stats.phase_cycles[i] = ks[8 + i];
    e->stats.phase_cycles[1] = ks[16];  // slot 1 (unused by k_main): ns spent in the front's last-block tail
    {
        uint32_t hot[RL_HOT_SLOTS];
        RL_CUDA(e, cudaMemcpyAsync(hot, e->d_hot.p, sizeof hot, cudaMemcpyDeviceToHost, e->stream));
        RL_CUDA(e, cudaStreamSynchronize(e->stream));
        e->stats.hot_rows = 0;
        for (uint32_t h : hot) e->stats.hot_rows += (h != 0xFFFFFFFFu);
    }
    *out = e->stats;
    return RL_OK;
}

int rl_limits_set(rl_engine* e, const rl_limit_desc* limits, uint32_t n) {
    if (!e || (!limits && n)) return RL_FATAL;
    e->structure_epoch++;
    std::string err;
    return e->reg.set(limits, n, &err) == RL_OK ? RL_OK : fail(e, RL_FATAL, "%s", err.c_str());
}

// One k_reset pass over the table, behind every pipelined call.  mode 0 resets the cells of the limits in `limit_sel`
// (indexed by limit id), mode 1 sweeps the qualified cells expired at now_us.  *out_dropped (nullable) = cells reset.
static int reset_table(rl_engine* e, int mode, uint64_t now_us, const std::vector<uint8_t>& limit_sel,
                       uint64_t* out_dropped) {
    int r = pipe_fence(e);
    if (r) return r;
    r = upload_tables(e);
    if (r) return r;
    DevBuf<uint8_t> d_sel;
    DevBuf<unsigned long long> d_cnt;
    if (!limit_sel.empty()) {
        RL_CUDA(e, d_sel.reserve(limit_sel.size()));
        RL_CUDA(e, cudaMemcpyAsync(d_sel.p, limit_sel.data(), limit_sel.size(), cudaMemcpyHostToDevice, e->stream));
    }
    if (out_dropped) {
        RL_CUDA(e, d_cnt.reserve(1));
        RL_CUDA(e, cudaMemsetAsync(d_cnt.p, 0, sizeof(unsigned long long), e->stream));
    }
    RlDev D = make_dev(e);
    const uint32_t blocks = ceil_div(e->capacity, 256);
    rl_with_cells(e->cells, [&](auto c) {
        k_reset<decltype(c)::value><<<blocks, 256, 0, e->stream>>>(D, e->capacity, mode, now_us, d_sel.p, d_cnt.p);
    });
    RL_LAUNCH_CHECK(e);
    unsigned long long cnt = 0;
    if (out_dropped) RL_CUDA(e, cudaMemcpyAsync(&cnt, d_cnt.p, sizeof cnt, cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    if (out_dropped) *out_dropped = cnt;
    return RL_OK;
}

int rl_delete_counters(rl_engine* e, const uint32_t* limit_ids, uint32_t n) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    e->structure_epoch++;
    std::vector<uint8_t> sel(std::max<size_t>(e->reg.limits.size(), 1), 0);
    bool any = false;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t id = limit_ids[i];
        if (!e->reg.find(id)) continue;
        sel[id] = 1;
        any = true;
        e->reg.set_simple_present(id, false);  // in_memory.rs:242-243
    }
    return any ? reset_table(e, 0, 0, sel, nullptr) : RL_OK;
}

int rl_limits_delete(rl_engine* e, const uint32_t* limit_ids, uint32_t n) {
    if (!e) return RL_FATAL;
    e->structure_epoch++;
    int r = rl_delete_counters(e, limit_ids, n);  // storage/mod.rs:104 — counters first
    if (r) return r;
    e->reg.remove(limit_ids, n);
    return RL_OK;
}

int rl_clear(rl_engine* e) {
    if (!e) return RL_FATAL;
    // in_memory.rs:197-201 — only simple_limits is cleared
    std::vector<uint32_t> ids;
    e->reg.each([&](uint32_t id, const HostLimit& l) {
        if (!l.qualified) ids.push_back(id);
    });
    return rl_delete_counters(e, ids.data(), (uint32_t)ids.size());
}

int rl_sweep(rl_engine* e, uint64_t now_us, uint64_t* out_invalidated) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    return reset_table(e, 1, now_us, {}, out_invalidated);
}

// The table reads behind rl_get_counters (live) and rl_counters_export: one k_scan pass over the rows of the
// namespaces in ns_sel (empty: every namespace), restricted to the limits whose counters exist.  live: (remaining,
// ttl) of the counters with ttl(now_us) > 0.  Otherwise (value, expiry), followed by the present unqualified limits
// whose row was never touched, as (l, 0, 0, 0, 0).  mem = RL_MEM_HOST stages at most capacity x cells entries on the
// device, RL_MEM_DEVICE writes the caller's arrays.  At most cap written; *out_count = number found.
static int read_table(rl_engine* e, bool live, uint64_t now_us, const std::vector<uint8_t>& ns_sel, uint64_t cap,
                      int mem, uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_a,
                      uint64_t* out_b, uint64_t* out_count) {
    if (mem != RL_MEM_HOST && mem != RL_MEM_DEVICE)
        return fail(e, RL_FATAL, "mem must be RL_MEM_HOST or RL_MEM_DEVICE (got %d)", mem);
    if (cap && (!out_limit_id || !out_key_lo || !out_key_hi || !out_a || !out_b))
        return fail(e, RL_FATAL, "cap > 0 needs all five output arrays");
    int r = pipe_fence(e);
    if (r) return r;
    r = upload_tables(e);
    if (r) return r;
    // present [L]: the limit's counters exist (RlRegistry::present) | seen [L]
    const uint32_t L = e->limits_cap;
    std::vector<uint8_t> flags(2 * (size_t)L, 0);
    for (uint32_t l = 0; l < L; l++) flags[l] = e->reg.present(l);
    DevBuf<uint8_t> d_sel, d_flags;
    DevBuf<unsigned long long> d_cnt;
    RL_CUDA(e, d_flags.reserve(flags.size()));
    RL_CUDA(e, d_cnt.reserve(1));
    RL_CUDA(e, cudaMemsetAsync(d_cnt.p, 0, sizeof(unsigned long long), e->stream));
    RL_CUDA(e, cudaMemcpyAsync(d_flags.p, flags.data(), flags.size(), cudaMemcpyHostToDevice, e->stream));
    if (!ns_sel.empty()) {
        RL_CUDA(e, d_sel.reserve(ns_sel.size()));
        RL_CUDA(e, cudaMemcpyAsync(d_sel.p, ns_sel.data(), ns_sel.size(), cudaMemcpyHostToDevice, e->stream));
    }
    // outputs: the caller's device arrays, or staging no larger than the table's cells
    uint64_t* out64[4] = {out_key_lo, out_key_hi, out_a, out_b};
    DevBuf<uint32_t> s_lid;
    DevBuf<uint64_t> s64[4];
    RlScanOut O{out_limit_id, out_key_lo, out_key_hi, out_a, out_b, d_cnt.p, cap, d_flags.p, d_flags.p + L};
    if (mem == RL_MEM_HOST) {
        const uint64_t n = std::min<uint64_t>(cap, e->capacity * e->cells);
        RL_CUDA(e, s_lid.reserve(n));
        for (auto& s : s64) RL_CUDA(e, s.reserve(n));
        O = RlScanOut{s_lid.p, s64[0].p, s64[1].p, s64[2].p, s64[3].p, d_cnt.p, n, d_flags.p, d_flags.p + L};
    }
    RlDev D = make_dev(e);
    const uint32_t blocks = ceil_div(e->capacity, 256);
    rl_with_cells(e->cells, [&](auto c) {
        k_scan<decltype(c)::value><<<blocks, 256, 0, e->stream>>>(D, e->capacity, live, now_us, d_sel.p, e->d_group_ns.p, O);
    });
    RL_LAUNCH_CHECK(e);
    unsigned long long cnt = 0;
    RL_CUDA(e, cudaMemcpyAsync(&cnt, d_cnt.p, sizeof cnt, cudaMemcpyDeviceToHost, e->stream));
    if (!live) RL_CUDA(e, cudaMemcpyAsync(flags.data() + L, d_flags.p + L, L, cudaMemcpyDeviceToHost, e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    const uint64_t got = std::min<uint64_t>(cnt, O.cap);
    if (mem == RL_MEM_HOST && got) {
        RL_CUDA(e, cudaMemcpy(out_limit_id, s_lid.p, got * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        for (int k = 0; k < 4; k++)
            RL_CUDA(e, cudaMemcpy(out64[k], s64[k].p, got * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    }
    // the export's present unqualified limits of the selected namespaces that no row showed, appended
    std::vector<uint32_t> extra;
    if (!live)
        e->reg.each([&](uint32_t l, const HostLimit& h) {
            if (flags[l] && !h.qualified && !flags[L + l] && (ns_sel.empty() || ns_sel[h.ns])) extra.push_back(l);
        });
    const uint64_t fit = cnt < cap ? std::min<uint64_t>(extra.size(), cap - cnt) : 0;
    if (fit && mem == RL_MEM_HOST) {
        std::copy(extra.begin(), extra.begin() + fit, out_limit_id + cnt);
        for (uint64_t* o : out64) std::fill(o + cnt, o + cnt + fit, 0);
    } else if (fit) {
        const std::vector<uint64_t> zero(fit, 0);
        RL_CUDA(e, cudaMemcpy(out_limit_id + cnt, extra.data(), fit * sizeof(uint32_t), cudaMemcpyHostToDevice));
        for (uint64_t* o : out64)
            RL_CUDA(e, cudaMemcpy(o + cnt, zero.data(), fit * sizeof(uint64_t), cudaMemcpyHostToDevice));
    }
    if (out_count) *out_count = cnt + extra.size();
    return RL_OK;
}

int rl_get_counters(rl_engine* e, const uint32_t* limit_ids, uint32_t n, uint64_t now_us, uint64_t cap,
                    uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_remaining,
                    uint64_t* out_ttl_us, uint64_t* out_count) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    // in_memory.rs:161-171: counters_in_namespace(limit.namespace()) for every given limit
    std::vector<uint8_t> ns_sel(std::max<size_t>(e->reg.ns_limits.size(), 1), 0);
    for (uint32_t i = 0; i < n; i++)
        if (const HostLimit* l = e->reg.find(limit_ids[i])) ns_sel[l->ns] = 1;
    return read_table(e, true, now_us, ns_sel, cap, RL_MEM_HOST, out_limit_id, out_key_lo, out_key_hi, out_remaining,
                      out_ttl_us, out_count);
}

int rl_counters_export(rl_engine* e, const uint32_t* ns_ids, uint32_t n_ns, uint64_t now_us, uint64_t cap, int mem,
                       uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_value,
                       uint64_t* out_expiry_us, uint64_t* out_count) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n_ns && !ns_ids) return fail(e, RL_FATAL, "rl_counters_export: n_ns > 0 with ns_ids == NULL");
    std::vector<uint8_t> ns_sel;  // empty: every namespace
    if (ns_ids) {
        ns_sel.assign(std::max<size_t>(e->reg.ns_limits.size(), 1), 0);
        for (uint32_t i = 0; i < n_ns; i++)
            if (ns_ids[i] < ns_sel.size()) ns_sel[ns_ids[i]] = 1;
    }
    return read_table(e, false, now_us, ns_sel, cap, mem, out_limit_id, out_key_lo, out_key_hi, out_value,
                      out_expiry_us, out_count);
}

int rl_limits_get(rl_engine* e, uint32_t cap, rl_limit_desc* out, uint32_t* out_n) {
    if (!e) return RL_FATAL;
    if (cap && !out) return fail(e, RL_FATAL, "rl_limits_get: cap > 0 with out == NULL");
    uint32_t n = 0;
    e->reg.each([&](uint32_t id, const HostLimit& l) {
        if (n < cap) out[n] = rl_limit_desc{id, l.ns, l.varset, l.qualified, l.max_value, l.window_us};
        n++;
    });
    if (out_n) *out_n = n;
    return RL_OK;
}

// ---------------------------------------------------------------------------------------
// Staging of the decision calls.  A call first normalises `mem`: RL_MEM_HOST_ASYNC stays only where the call can
// take it (async_ok) and is RL_MEM_HOST everywhere else, as rl_engine.h promises.
static int normalise_mem(rl_engine* e, int& mem, bool async_ok) {
    if (mem == RL_MEM_HOST_ASYNC && !async_ok) mem = RL_MEM_HOST;
    if (mem != RL_MEM_HOST && mem != RL_MEM_DEVICE && mem != RL_MEM_HOST_ASYNC)
        return fail(e, RL_FATAL, "mem must be RL_MEM_HOST, RL_MEM_DEVICE or RL_MEM_HOST_ASYNC (got %d)", mem);
    return RL_OK;
}

// A record call's input on the device: the caller's buffer (RL_MEM_DEVICE), the next ring slot (RL_MEM_HOST_ASYNC)
// or the staging buffer (RL_MEM_HOST).  rec_bytes: 32 (rl_record) or 16 (rl_record16).
static int stage_records(rl_engine* e, int mem, uint64_t n, const void* recs, size_t rec_bytes, const rl_record*& d_recs) {
    d_recs = static_cast<const rl_record*>(recs);
    if (mem == RL_MEM_DEVICE) return RL_OK;
    DevBuf<rl_record>* buf = &e->d_in_recs;
    if (mem == RL_MEM_HOST_ASYNC) {
        // H2D on the caller's stream (which carries nothing else of ours), kernels on the pipeline
        // streams, D2H behind the replay: the copies of one call overlap the kernels of its neighbours.
        const int slot = (int)(e->ring_seq % rl_engine::kRing);
        buf = &e->ring_recs[slot];
        if (e->ring_seq >= (uint64_t)rl_engine::kRing)
            RL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_slot[slot], 0));  // slot drained (its D2H done)
    }
    RL_CUDA(e, buf->reserve(e->max_batch));
    RL_CUDA(e, cudaMemcpyAsync(buf->p, recs, n * rec_bytes, cudaMemcpyHostToDevice, e->stream));
    d_recs = buf->p;
    return RL_OK;
}

// Where the kernels write a call's outputs: the caller's buffers (RL_MEM_DEVICE), the current ring slot
// (RL_MEM_HOST_ASYNC) or the staging buffers (RL_MEM_HOST; n_ctr remaining/ttl slots).  `user` holds the
// caller's pointers, null where an output is not wanted.
static int bind_outs(rl_engine* e, int mem, const Outs& user, uint64_t n_ctr, Outs& dev) {
    dev = user;
    if (mem == RL_MEM_DEVICE) return RL_OK;
    const int slot = (int)(e->ring_seq % rl_engine::kRing);
    DevBuf<uint8_t>& lim = mem == RL_MEM_HOST_ASYNC ? e->ring_lim[slot] : e->d_out_limited;
    DevBuf<uint32_t>& first = mem == RL_MEM_HOST_ASYNC ? e->ring_first[slot] : e->d_out_first;
    RL_CUDA(e, lim.reserve(e->max_batch));
    dev.limited = lim.p;
    if (user.first) {
        RL_CUDA(e, first.reserve(e->max_batch));
        dev.first = first.p;
    }
    if (user.rem || user.ttl) {  // RL_MEM_HOST only
        RL_CUDA(e, e->d_out_rem.reserve(std::max<uint64_t>(n_ctr, e->max_counters)));
        RL_CUDA(e, e->d_out_ttl.reserve(std::max<uint64_t>(n_ctr, e->max_counters)));
        dev.rem = e->d_out_rem.p;
        dev.ttl = e->d_out_ttl.p;
    }
    return RL_OK;
}

// Copies a host-memory call's outputs back to the caller.  RL_MEM_HOST: on the engine's stream, then the device
// error is checked.  RL_MEM_HOST_ASYNC: enqueued only, and the ring slot moves on.
static int copy_back(rl_engine* e, int mem, uint64_t n, uint64_t n_ctr, const Outs& dev, const Outs& user) {
    if (mem == RL_MEM_DEVICE) return RL_OK;
    // The verdicts of an RL_MEM_HOST_ASYNC call leave on the replay stream itself, right behind their k_main.
    // A dedicated copy stream parked on "replay done" looked cleaner, but streams share hardware queues:
    // whenever it landed on the queue of the stream carrying the next H2D, that copy waited for the replay
    // too and the whole pipeline serialised (the end-to-end rate fell to a fraction, one run in three).
    const cudaStream_t sd = mem == RL_MEM_HOST_ASYNC ? e->sm : e->stream;
    if (user.limited) RL_CUDA(e, cudaMemcpyAsync(user.limited, dev.limited, n, cudaMemcpyDeviceToHost, sd));
    if (user.first) RL_CUDA(e, cudaMemcpyAsync(user.first, dev.first, n * 4, cudaMemcpyDeviceToHost, sd));
    if (user.rem && n_ctr) RL_CUDA(e, cudaMemcpyAsync(user.rem, dev.rem, n_ctr * 8, cudaMemcpyDeviceToHost, sd));
    if (user.ttl && n_ctr) RL_CUDA(e, cudaMemcpyAsync(user.ttl, dev.ttl, n_ctr * 8, cudaMemcpyDeviceToHost, sd));
    if (mem == RL_MEM_HOST) return check_device_error(e);
    const int slot = (int)(e->ring_seq % rl_engine::kRing);
    RL_CUDA(e, cudaEventRecord(e->ev_slot[slot], sd));
    e->d2h_pending = true;
    e->d2h_last = slot;
    e->ring_seq++;
    return RL_OK;
}

int rl_check_and_update_records(rl_engine* e, uint64_t n, const rl_record* recs, int load_counters, int mem,
                                uint8_t* out_limited, uint32_t* out_first_limited, uint64_t* out_remaining,
                                uint64_t* out_ttl_us, uint32_t out_stride) {
    const bool lc = load_counters && (out_remaining || out_ttl_us);
    int r = normalise_mem(e, mem, e && e->pipeline && !e->shape.any_multi_ns && !lc);
    if (r) return r;
    if ((r = ensure_ready(e, n, mem == RL_MEM_HOST))) return r;
    if (n == 0) return RL_OK;
    if (!recs || !out_limited) return fail(e, RL_FATAL, "null recs/out_limited");
    if (lc && out_stride < e->shape.max_ns_limits)
        return fail(e, RL_FATAL, "out_stride %u < limits per namespace %u", out_stride, e->shape.max_ns_limits);
    e->stats.batches++;
    e->stats.requests += n;
    e->trace_seq = (uint32_t)e->stats.batches;
    const Outs user{out_limited, out_first_limited, lc ? out_remaining : nullptr, lc ? out_ttl_us : nullptr, nullptr,
                    out_stride};
    const uint64_t nout = lc ? n * out_stride : 0;
    const rl_record* d_recs;
    Outs o;
    if ((r = stage_records(e, mem, n, recs, sizeof(rl_record), d_recs)) || (r = bind_outs(e, mem, user, nout, o))) return r;
    if (lc && mem == RL_MEM_HOST) {
        // slots of limits a namespace does not have stay 0
        RL_CUDA(e, cudaMemsetAsync(o.rem, 0, nout * 8, e->stream));
        RL_CUDA(e, cudaMemsetAsync(o.ttl, 0, nout * 8, e->stream));
    }
    if ((r = run_record_pipeline(e, (uint32_t)n, d_recs, 0, load_counters ? 1 : 0, o, mem != RL_MEM_HOST))) return r;
    return copy_back(e, mem, n, nout, o, user);
}

int rl_check_and_update_compact(rl_engine* e, uint64_t n, const rl_record16* recs, uint64_t now_us, int mem,
                                uint8_t* out_limited, uint32_t* out_first_limited) {
    int r = normalise_mem(e, mem, e && e->pipeline && !e->shape.any_multi_ns);
    if (r) return r;
    if ((r = ensure_ready(e, n, mem == RL_MEM_HOST))) return r;
    if (n == 0) return RL_OK;
    if (!recs || !out_limited) return fail(e, RL_FATAL, "null recs/out_limited");
    if (now_us == 0) return fail(e, RL_FATAL, "now_us must be >= 1");
    e->stats.batches++;
    e->stats.requests += n;
    e->trace_seq = (uint32_t)e->stats.batches;
    const Outs user{out_limited, out_first_limited};
    const rl_record* d_recs;  // RecordSrc::compact reads 16-byte strides
    Outs o;
    if ((r = stage_records(e, mem, n, recs, sizeof(rl_record16), d_recs)) || (r = bind_outs(e, mem, user, 0, o))) return r;
    if ((r = run_record_pipeline(e, (uint32_t)n, d_recs, 0, 0, o, mem != RL_MEM_HOST, nullptr, 0, now_us))) return r;
    return copy_back(e, mem, n, 0, o, user);
}

// Brings a CSR batch onto the device (or aliases it) and returns the total counter count.
struct CsrDev {
    const uint32_t* off = nullptr;
    const rl_counter* ctrs = nullptr;
    const uint64_t* delta = nullptr;
    const uint64_t* now = nullptr;
    uint64_t total = 0;
};

static int stage_csr(rl_engine* e, uint64_t n, const uint32_t* off, const rl_counter* ctrs, const uint64_t* delta,
                     const uint64_t* now, int mem, CsrDev& d) {
    if (!off || !delta || !now) return fail(e, RL_FATAL, "null CSR arrays");
    d = CsrDev{off, ctrs, delta, now, 0};
    if (mem == RL_MEM_DEVICE) {
        uint32_t last = 0;
        RL_CUDA(e, cudaMemcpyAsync(&last, off + n, 4, cudaMemcpyDeviceToHost, e->stream));
        RL_CUDA(e, cudaStreamSynchronize(e->stream));
        d.total = last;
    } else {
        d.total = off[n];
    }
    if (d.total > e->max_counters)
        return fail(e, RL_FATAL, "batch has %llu counters > max_counters=%u", (unsigned long long)d.total, e->max_counters);
    if (mem == RL_MEM_DEVICE) return RL_OK;
    RL_CUDA(e, e->d_in_off.reserve(e->max_batch + 1));
    RL_CUDA(e, e->d_in_ctrs.reserve(e->max_counters));
    RL_CUDA(e, e->d_in_delta.reserve(e->max_batch));
    RL_CUDA(e, e->d_in_now.reserve(e->max_batch));
    RL_CUDA(e, cudaMemcpyAsync(e->d_in_off.p, off, (n + 1) * 4, cudaMemcpyHostToDevice, e->stream));
    if (d.total)
        RL_CUDA(e, cudaMemcpyAsync(e->d_in_ctrs.p, ctrs, d.total * sizeof(rl_counter), cudaMemcpyHostToDevice, e->stream));
    RL_CUDA(e, cudaMemcpyAsync(e->d_in_delta.p, delta, n * 8, cudaMemcpyHostToDevice, e->stream));
    RL_CUDA(e, cudaMemcpyAsync(e->d_in_now.p, now, n * 8, cudaMemcpyHostToDevice, e->stream));
    d = CsrDev{e->d_in_off.p, e->d_in_ctrs.p, e->d_in_delta.p, e->d_in_now.p, d.total};
    return RL_OK;
}

// The general form's resolve.  k_resolve_csr takes requests of up to 16 counters and reports a longer one as
// RL_DEV_TOO_MANY_COUNTERS.  On an engine created for more (max_counters_per_request > 16) that report is what
// selects the wide path: the batch is resolved again with the wide encoding and `wide` is set.  A batch without such
// a request runs exactly the kernels of a default engine.
static int resolve_csr(rl_engine* e, uint64_t n, const CsrDev& c, const RlResolveOut& O, int write_defaults, bool& wide) {
    RlDev D = make_dev(e);
    wide = false;
    k_resolve_csr<<<ceil_div(n, 128), 128, 0, e->stream>>>(D, (uint32_t)n, c.off, c.ctrs, O, write_defaults);
    RL_LAUNCH_CHECK(e);
    if (e->max_ctrs_req > RL_MAX_CTRS_PER_REQ) {
        RL_CUDA(e, cudaMemcpyAsync(e->h_misc.p, e->d_misc.p, MISC_N * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
        RL_CUDA(e, cudaStreamSynchronize(e->stream));
        if (e->h_misc.p[MISC_ERR] == RL_DEV_TOO_MANY_COUNTERS) {
            // every other refusal has a lower code (the error word is a sticky max): the wide pass finds it again
            RL_CUDA(e, cudaMemsetAsync(e->d_misc.p + MISC_ERR, 0, 2 * sizeof(uint32_t), e->stream));  // error + flags
            k_resolve_csr_wide<<<ceil_div(n, 128), 128, 0, e->stream>>>(D, (uint32_t)n, c.off, c.ctrs, O, write_defaults,
                                                                        e->d_perm.p, e->max_ctrs_req);
            RL_LAUNCH_CHECK(e);
            wide = true;
        }
    }
    return check_resolve_error(e);
}

int rl_check_and_update_batch(rl_engine* e, uint64_t n, const uint32_t* ctr_off, const rl_counter* ctrs,
                              const uint64_t* delta, const uint64_t* now_us, int load_counters, int mem,
                              uint8_t* out_limited, uint32_t* out_first_limited, uint64_t* out_remaining,
                              uint64_t* out_ttl_us) {
    int r = normalise_mem(e, mem, false);
    if (r) return r;
    if ((r = ensure_ready(e, n))) return r;
    if (n == 0) return RL_OK;
    if (!out_limited) return fail(e, RL_FATAL, "null out_limited");
    CsrDev c;
    if ((r = stage_csr(e, n, ctr_off, ctrs, delta, now_us, mem, c))) return r;
    const bool lc = load_counters && (out_remaining || out_ttl_us);
    e->stats.batches++;
    e->stats.requests += n;
    const Outs user{out_limited, out_first_limited, lc ? out_remaining : nullptr, lc ? out_ttl_us : nullptr};
    Outs o;
    if ((r = bind_outs(e, mem, user, c.total, o))) return r;
    o.off = c.off;
    RlResolveOut O{e->d_acc.p, nullptr, nullptr, o.limited, o.first};
    bool wide;
    if ((r = resolve_csr(e, n, c, O, 1, wide))) return r;
    if (c.total) {
        if ((r = run_acc_pipeline(e, (uint32_t)c.total, (uint32_t)n, c.delta, c.now, 0, load_counters ? 1 : 0, o, wide)))
            return r;
    }
    return copy_back(e, mem, n, c.total, o, user);
}

int rl_update_batch(rl_engine* e, uint64_t n, const uint32_t* ctr_off, const rl_counter* ctrs, const uint64_t* delta,
                    const uint64_t* now_us, int mem) {
    int r = normalise_mem(e, mem, false);
    if (r) return r;
    if ((r = ensure_ready(e, n))) return r;
    if (n == 0) return RL_OK;
    CsrDev c;
    if ((r = stage_csr(e, n, ctr_off, ctrs, delta, now_us, mem, c))) return r;
    e->stats.batches++;
    e->stats.requests += n;
    if (c.total == 0) return RL_OK;
    Outs o;
    RlResolveOut O{e->d_acc.p, nullptr, nullptr, nullptr, nullptr};
    bool wide;
    if ((r = resolve_csr(e, n, c, O, 0, wide))) return r;
    if ((r = run_acc_pipeline(e, (uint32_t)c.total, (uint32_t)n, c.delta, c.now, 2, 0, o, wide))) return r;
    return copy_back(e, mem, n, 0, o, o);
}

int rl_update_records(rl_engine* e, uint64_t n, const rl_record* recs, int mem) {
    int r = normalise_mem(e, mem, false);
    if (r) return r;
    if ((r = ensure_ready(e, n, mem != RL_MEM_DEVICE))) return r;
    if (n == 0) return RL_OK;
    if (!recs) return fail(e, RL_FATAL, "null recs");
    e->stats.batches++;
    e->stats.requests += n;
    const rl_record* d_recs;
    if ((r = stage_records(e, mem, n, recs, sizeof(rl_record), d_recs))) return r;
    Outs o;
    if ((r = run_record_pipeline(e, (uint32_t)n, d_recs, 2, 0, o, mem == RL_MEM_DEVICE))) return r;
    return copy_back(e, mem, n, 0, o, o);
}

int rl_is_within_limits_batch(rl_engine* e, uint64_t n, const uint32_t* ctr_off, const rl_counter* ctrs,
                              const uint64_t* delta, const uint64_t* now_us, int mem, uint8_t* out_limited,
                              uint32_t* out_first_limited) {
    int r = normalise_mem(e, mem, false);
    if (r) return r;
    if ((r = ensure_ready(e, n))) return r;
    if (n == 0) return RL_OK;
    if (!out_limited) return fail(e, RL_FATAL, "null out_limited");
    CsrDev c;
    if ((r = stage_csr(e, n, ctr_off, ctrs, delta, now_us, mem, c))) return r;
    const Outs user{out_limited, out_first_limited};
    Outs o;
    if ((r = bind_outs(e, mem, user, 0, o))) return r;
    RlDev D = make_dev(e);
    rl_with_cells(e->cells, [&](auto cl) {
        k_query_csr<decltype(cl)::value><<<ceil_div(n, 128), 128, 0, e->stream>>>(D, (uint32_t)n, c.off, c.ctrs, c.delta,
                                                                                   c.now, o.limited, o.first);
    });
    RL_LAUNCH_CHECK(e);
    return copy_back(e, mem, n, 0, o, user);
}

int rl_is_within_limits_records(rl_engine* e, uint64_t n, const rl_record* recs, int mem, uint8_t* out_limited,
                                uint32_t* out_first_limited) {
    int r = normalise_mem(e, mem, false);
    if (r) return r;
    if ((r = ensure_ready(e, n))) return r;
    if (n == 0) return RL_OK;
    if (!recs || !out_limited) return fail(e, RL_FATAL, "null recs/out_limited");
    const Outs user{out_limited, out_first_limited};
    const rl_record* d_recs;
    Outs o;
    if ((r = stage_records(e, mem, n, recs, sizeof(rl_record), d_recs)) || (r = bind_outs(e, mem, user, 0, o))) return r;
    RlDev D = make_dev(e);
    rl_with_cells(e->cells, [&](auto c) {
        k_query_records<decltype(c)::value><<<ceil_div(n, 128), 128, 0, e->stream>>>(D, (uint32_t)n, d_recs, o.limited,
                                                                                     o.first);
    });
    RL_LAUNCH_CHECK(e);
    return copy_back(e, mem, n, 0, o, user);
}

// ---------------------------------------------------------------------------------------
int rl_bucket_by_owner(rl_engine* e, uint64_t n, const rl_record* d_recs, uint32_t world, rl_record* d_out_recs,
                       uint32_t* d_out_src, uint64_t* h_counts) {
    if (!e) return RL_FATAL;
    if (world == 0 || world > 32) return fail(e, RL_FATAL, "world must be 1..32");
    RL_CUDA(e, cudaSetDevice(e->device));
    for (uint32_t w = 0; w < world; w++) h_counts[w] = 0;
    if (n == 0) return RL_OK;
    uint32_t tile = ceil_div(n, kMaxTiles);
    tile = std::max<uint32_t>(512, ((tile + 255) / 256) * 256);
    const uint32_t num_tiles = ceil_div(n, tile);
    RL_CUDA(e, e->d_bucket.reserve((size_t)(kMaxTiles + 1) * 32 + 32));
    RL_CUDA(e, e->d_bucket_counts.reserve(32));
    uint32_t* tile_cnt = e->d_bucket.p;
    uint32_t* owner_base = e->d_bucket.p + (size_t)(kMaxTiles + 1) * 32;
    k_bucket<false><<<num_tiles, RL_PART_THREADS, 0, e->stream>>>(d_recs, (uint32_t)n, world, tile, tile_cnt, owner_base,
                                                                  d_out_recs, d_out_src, 0, nullptr);
    RL_LAUNCH_CHECK(e);
    k_bucket_scan<<<1, 32, 0, e->stream>>>(num_tiles, world, tile_cnt, owner_base, e->d_bucket_counts.p, 0, nullptr);
    RL_LAUNCH_CHECK(e);
    k_bucket<true><<<num_tiles, RL_PART_THREADS, 0, e->stream>>>(d_recs, (uint32_t)n, world, tile, tile_cnt, owner_base,
                                                                 d_out_recs, d_out_src, 0, nullptr);
    RL_LAUNCH_CHECK(e);
    unsigned long long counts[32];
    RL_CUDA(e, cudaMemcpyAsync(counts, e->d_bucket_counts.p, world * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                               e->stream));
    RL_CUDA(e, cudaStreamSynchronize(e->stream));
    for (uint32_t w = 0; w < world; w++) h_counts[w] = counts[w];
    return RL_OK;
}

int rl_bucket_by_owner_padded(rl_engine* e, uint64_t n, const rl_record* d_recs, uint32_t world, uint32_t slot_cap,
                              rl_record* d_out_recs, uint32_t* d_out_pos, uint32_t* d_overflow) {
    if (!e) return RL_FATAL;
    if (world == 0 || world > 32 || slot_cap == 0) return fail(e, RL_FATAL, "world must be 1..32 and slot_cap > 0");
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n == 0) return RL_OK;
    uint32_t tile = ceil_div(n, kMaxTiles);
    tile = std::max<uint32_t>(512, ((tile + 255) / 256) * 256);
    const uint32_t num_tiles = ceil_div(n, tile);
    RL_CUDA(e, e->d_bucket.reserve((size_t)(kMaxTiles + 1) * 32 + 32));
    RL_CUDA(e, e->d_bucket_counts.reserve(32));
    uint32_t* tile_cnt = e->d_bucket.p;
    uint32_t* owner_base = e->d_bucket.p + (size_t)(kMaxTiles + 1) * 32;
    // unused slots = no-op records (ns_id 0xFFFFFFFF: a namespace without limits)
    RL_CUDA(e, cudaMemsetAsync(d_out_recs, 0xFF, (size_t)world * slot_cap * sizeof(rl_record), e->stream));
    k_bucket<false><<<num_tiles, RL_PART_THREADS, 0, e->stream>>>(d_recs, (uint32_t)n, world, tile, tile_cnt, owner_base,
                                                                  d_out_recs, nullptr, slot_cap, d_out_pos);
    RL_LAUNCH_CHECK(e);
    k_bucket_scan<<<1, 32, 0, e->stream>>>(num_tiles, world, tile_cnt, owner_base, e->d_bucket_counts.p, slot_cap,
                                           d_overflow);
    RL_LAUNCH_CHECK(e);
    k_bucket<true><<<num_tiles, RL_PART_THREADS, 0, e->stream>>>(d_recs, (uint32_t)n, world, tile, tile_cnt, owner_base,
                                                                 d_out_recs, nullptr, slot_cap, d_out_pos);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

int rl_gather_u8(rl_engine* e, uint64_t n, const uint8_t* d_in, const uint32_t* d_pos, uint8_t* d_out) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n == 0) return RL_OK;
    k_gather_u8<<<ceil_div(n, 256), 256, 0, e->stream>>>((uint32_t)n, d_in, d_pos, d_out);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

int rl_record_lane_put(rl_engine* e, uint64_t n_slots, rl_record* d_recs, const uint8_t* d_lane) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n_slots == 0) return RL_OK;
    k_lane_put<<<ceil_div(n_slots, 256), 256, 0, e->stream>>>((uint32_t)n_slots, d_recs, d_lane);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

int rl_record_lane_gather(rl_engine* e, uint64_t n, const rl_record* d_recs, const uint32_t* d_pos, uint8_t* d_out) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n == 0) return RL_OK;
    k_lane_gather<<<ceil_div(n, 256), 256, 0, e->stream>>>((uint32_t)n, d_recs, d_pos, d_out);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

int rl_unpermute_u8(rl_engine* e, uint64_t n, const uint8_t* d_in, const uint32_t* d_src, uint8_t* d_out) {
    if (!e) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    if (n == 0) return RL_OK;
    k_unpermute_u8<<<ceil_div(n, 256), 256, 0, e->stream>>>((uint32_t)n, d_in, d_src, d_out);
    RL_LAUNCH_CHECK(e);
    return RL_OK;
}

#include "rl_shard_host.inc"

}  // extern "C"

// ---- what rl_maint.cu may do with an engine (rl_internal.h) -------------------------------------------------------------
int rl_internal_view(rl_engine* e, RlTableView* out) {
    if (!e || !out) return RL_FATAL;
    RL_CUDA(e, cudaSetDevice(e->device));
    int r = pipe_fence(e);
    if (r) return r;
    r = upload_tables(e);
    if (r) return r;
    out->rows = e->d_rows.p;
    out->cells = e->cells;
    out->log2P = e->log2P;
    out->log2R = e->log2R;
    out->row_bytes = e->row_bytes;
    out->capacity = e->capacity;
    out->ns_cap = e->ns_cap;
    out->limits_cap = e->limits_cap;
    out->limits = e->d_limits.p;
    out->desc = e->d_desc.p;
    out->structure_epoch = e->structure_epoch;
    out->stream = e->stream;
    out->device = e->device;
    return RL_OK;
}
int rl_internal_fail(rl_engine* e, int status, const char* msg) { return fail(e, status, "%s", msg); }
void rl_internal_launched(rl_engine* e, uint32_t kernels) {
    if (e) e->stats.kernel_launches += kernels;
}
uint32_t rl_internal_sm_count(rl_engine* e) { return e->main_grid_cap / 16; }
void** rl_internal_ext(rl_engine* e, void (*ext_free)(void*)) {
    e->ext_free = ext_free;
    return &e->ext;
}
void rl_internal_set_ns_hook(rl_engine* e, rl_ns_hook_fn fn) { e->ns_hook = fn; }
int rl_internal_reset_hot_rows(rl_engine* e) {
    RL_CUDA(e, cudaMemsetAsync(e->d_hot.p, 0xFF, (RL_HOT_SLOTS + RL_HOT_CAND) * sizeof(uint32_t), e->stream));
    RL_CUDA(e, cudaMemsetAsync(e->d_hot.p + RL_HOT_SLOTS + RL_HOT_CAND, 0, 4 * sizeof(uint32_t), e->stream));
    return RL_OK;
}
void rl_internal_structure_changed(rl_engine* e) { e->structure_epoch++; }
void rl_internal_present(rl_engine* e, uint8_t* present, uint32_t n) {
    for (uint32_t l = 0; l < n; l++) present[l] = e->reg.present(l);
}
void rl_internal_mark_present(rl_engine* e, const uint8_t* flags, uint32_t n) {
    for (uint32_t l = 0; l < n; l++)
        if (flags[l]) e->reg.set_simple_present(l, true);
}
