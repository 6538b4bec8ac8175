// emu_engine.cpp — TEST-ONLY host driver of the decision kernels (limitador_b200/csrc/rl_kernels.cuh: k_front, k_hot,
// k_main, the resolve kernels, k_restore, k_fl_step, k_wide_scatter, k_scan) and of the peer exchange
// (limitador_b200/csrc/rl_shard.cuh: k_xcount .. k_xgather) under tests/emu/cuda_simt.h: the SAME kernel source the GPU
// runs, every CUDA thread a fiber, warp intrinsics as rendezvous, up to R k_main blocks resident at once.  Not shipped,
// not a fallback.  The call sequences follow rl_engine.cu (run_record_pipeline without the pipeline, run_acc_pipeline)
// and rl_shard_host.inc (rl_shard_send / _decide / _collect over `world` emulated engines and their slabs), the batch
// geometry is rl_batch_geom itself, and every call reports the geometry it reached.
#include "cuda_simt.h"
// (the emulator must come first: it defines __global__ & co. away)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../limitador_b200/csrc/rl_registry.h"
#include "../../limitador_b200/csrc/rl_shard.cuh"

namespace {

// what the report says about a call (indices of emu_engine's report array)
enum {
    G_TILES, G_TILE, G_MERGE_MAIN, G_MERGE_HOT, G_NPARTS, G_ITEMS, G_HEAVY_ITEMS, G_MAX_W, G_HOT_IN_USE, G_HOT_CAND,
    G_HOT_MAX_LIST, G_HOT_SWEEPS, G_FP_ROUNDS, G_CHUNKS, G_ROUNDS, G_CHAINED, G_ORDERED, G_HOT_AFTER, G_MAX_PART,
    G_CH, G_REARMED, G_N
};

}  // namespace

struct emu_engine {
    uint32_t cells = 1, log2P = 0, log2R = 0, row_bytes = 32;
    std::vector<uint8_t> rows;
    RlRegistry reg;
    RlTableImage t;  // the device tables of reg
    // knobs
    uint32_t chunk = 128, part_target = 128, heavy_mult = 2, main_grid_cap = 132 * 16, weak = 0, hot_on = 0, resident = 1;
    uint32_t n_dev = 0;  // sharded geometry on a plain call: the access count lives on the device, the tile is derived there
    bool interleave = false;
    uint64_t seed = 0;
    double p = 1.0;
    // device state that lives across calls
    std::vector<uint32_t> hot;  // hot_rows [RL_HOT_SLOTS] | hot_cand [RL_HOT_CAND] | hot_cand_n | pad
    std::vector<uint32_t> region_total, small;
    uint32_t err[8] = {}, flags = 0, changed = 0;  // err: sticky RL_DEV_* code; err[7]: the exchange's detail word
    unsigned long long kstats[32] = {};
    unsigned long long report[G_N] = {};
};

namespace {

RlDev make_dev(emu_engine* e) {
    RlDev D;
    D.rows = e->rows.data();
    D.log2P = e->log2P;
    D.log2R = e->log2R;
    D.desc = e->t.desc.data();
    D.limits = e->t.lim.data();
    D.limits_cap = (uint32_t)e->t.lim.size();
    D.ns = e->t.ns.data();
    D.ns_cap = (uint32_t)e->t.ns.size();
    D.ns_limit_ids = e->t.ns_ids.data();
    D.err = e->err;
    D.flags = &e->flags;
    D.kstats = e->kstats;
    D.hot_rows = e->hot.data();
    D.hot_cand = e->hot.data() + RL_HOT_SLOTS;
    D.hot_cand_n = e->hot.data() + RL_HOT_SLOTS + RL_HOT_CAND;
    D.trace = nullptr;
    D.trace_pos = nullptr;
    D.seq = 0;
    return D;
}

// the per-batch workspace: poisoned where the GPU's would hold the previous batch's data; region totals and the
// counters of `small` persist, as the kernels re-arm them
struct Work {
    std::vector<uint32_t> tile_loc, part_idx, part_row, row_of, chain_status, chain_wcnt, chain_w, fl_prev, fl_next;
    std::vector<uint4> items;
    std::vector<uint8_t*> log_row;
    std::vector<ulonglong2> log_state;
    uint32_t n_dev = 0;
};

// n_hint / n_dev (sharded steps, rl_shard_decide): n_acc is only the upper bound of the device-side count *n_dev, the
// partitions are sized for n_hint and the kernels derive the tile from *n_dev
RlBatch make_batch(emu_engine* e, Work& w, uint32_t n_acc, uint32_t n_req, uint8_t* lim, uint32_t* first, uint64_t* rem,
                   uint64_t* ttl, const uint32_t* off, uint32_t stride, int lc, bool hot_ok, uint32_t n_hint = 0,
                   const uint32_t* n_dev = nullptr) {
    RlBatch B;
    memset(&B, 0, sizeof B);
    B.nhot = (hot_ok && e->hot_on) ? RL_HOT_SLOTS : 0;
    B.n_acc = n_acc;
    B.n_req = n_req;
    const RlBatchGeom g = rl_batch_geom(n_acc, n_hint, e->log2P, e->part_target, e->chunk, e->heavy_mult);
    B.tile = g.tile;
    B.num_tiles = g.num_tiles;
    B.nparts = g.nparts;
    B.part_shift = g.part_shift;
    B.heavy_len = g.heavy_len;
    B.n_dev = n_dev;
    const uint32_t P1 = (1u << e->log2P) + RL_HOT_SLOTS + 1;
    const uint32_t tsz = n_dev ? std::max<uint32_t>(256, ((rl_ceil_div(n_acc, g.num_tiles) + 255) / 256) * 256) : g.tile;
    const size_t buf = (size_t)g.num_tiles * tsz;
    const size_t max_items = (size_t)(1u << e->log2P) + n_acc / 128 + 2 + g.nparts;
    w.tile_loc.assign((size_t)(g.num_tiles + 1) * (P1 + 1), 0xA5A5A5A5u);
    w.part_idx.assign(buf, 0xA5A5A5A5u);
    w.part_row.assign(buf, 0xA5A5A5A5u);
    w.row_of.assign(std::max<uint32_t>(n_acc, 1), 0xA5A5A5A5u);
    w.items.assign(max_items, uint4{0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u});
    w.chain_status.assign(max_items, 0xA5A5A5A5u);
    w.chain_wcnt.assign(max_items, 0xA5A5A5A5u);
    w.chain_w.assign(max_items * 256, 0xA5A5A5A5u);
    w.fl_prev.assign(std::max<uint32_t>(n_req, 1), RL_NONE_U32);
    w.fl_next.assign(std::max<uint32_t>(n_req, 1), RL_NONE_U32);
    B.tile_loc = w.tile_loc.data();
    B.region_total = e->region_total.data();
    B.row_of = w.row_of.data();
    B.part_idx = w.part_idx.data();
    B.part_row = w.part_row.data();
    B.scan_ctr = e->small.data() + 0;
    B.n_items = e->small.data() + 1;
    B.ticket = e->small.data() + 2;
    B.exit_ctr = e->small.data() + 3;
    B.out_limited = lim;
    B.out_first_limited = first;
    B.out_remaining = rem;
    B.out_ttl = ttl;
    B.out_off = off;
    B.out_stride = stride;
    B.fl_prev = w.fl_prev.data();
    B.fl_next = w.fl_next.data();
    B.phase = RL_PHASE_COMMIT;
    B.load_counters = lc;
    B.items = w.items.data();
    B.chain_status = w.chain_status.data();
    B.chain_wcnt = w.chain_wcnt.data();
    B.chain_w = w.chain_w.data();
    B.chunk = e->chunk;
    return B;
}

void interleave_on(emu_engine* e, uint64_t salt) {
    if (e->interleave) simt_interleave(true, e->seed * 0x9E3779B97F4A7C15ull + salt, e->p);
}
void interleave_off() { simt_interleave(false); }

template <class Src>
void launch_front(emu_engine* e, const RlDev& D, const RlBatch& B, const Src& src) {
    interleave_on(e, 1);
    rl_with_cells(e->cells, [&](auto c) {
        simt_launch_ex(B.num_tiles, RL_PART_THREADS, rl_front_smem_bytes(B.nparts, B.nhot), 1,
                       [&] { k_front<decltype(c)::value, Src>(D, B, src); });
    });
    interleave_off();
}

// what k_front's last block built: the work items, and the hot lists (partitions nparts ..)
void report_front(emu_engine* e, const RlBatch& B, const Work& w) {
    unsigned long long* g = e->report;
    g[G_TILES] = B.num_tiles;
    g[G_TILE] = B.n_dev ? std::max<uint32_t>(256, ((rl_ceil_div(*B.n_dev, B.num_tiles) + 255) / 256) * 256) : B.tile;
    g[G_NPARTS] = B.nparts;
    const uint32_t n_items = *B.n_items;
    g[G_ITEMS] = n_items;
    uint64_t heavy = 0, maxw = 0, maxpart = 0;
    for (uint32_t i = 0; i < n_items; i++) {
        const uint4 it = w.items[i];
        if (it.w != RL_NONE_U32) {
            heavy++;
            maxw = std::max<uint64_t>(maxw, it.w);
        }
    }
    const uint32_t TL = B.nparts + B.nhot + 2;
    std::vector<uint64_t> len(B.nparts + B.nhot, 0);
    for (uint32_t t = 0; t < B.num_tiles; t++)
        for (uint32_t q = 0; q < B.nparts + B.nhot; q++) len[q] += w.tile_loc[(size_t)t * TL + q + 1] - w.tile_loc[(size_t)t * TL + q];
    uint64_t hmax = 0, sweeps = 0;
    for (uint32_t q = 0; q < B.nparts; q++) maxpart = std::max(maxpart, len[q]);
    for (uint32_t h = 0; h < B.nhot; h++) {
        hmax = std::max(hmax, len[B.nparts + h]);
        sweeps = std::max<uint64_t>(sweeps, rl_ceil_div(len[B.nparts + h], RL_HOT_SWEEP));
    }
    g[G_HEAVY_ITEMS] = heavy;
    g[G_MAX_W] = maxw;
    g[G_HOT_MAX_LIST] = hmax;
    g[G_HOT_SWEEPS] = sweeps;  // at least: the longest list's whole-list sweeps
    g[G_MAX_PART] = maxpart;
    g[G_MERGE_HOT] = B.nhot ? rl_ceil_div(B.num_tiles, RL_HOT_THREADS) : 0;
}

template <int GEO, int CELLS, class Src, int MODE, bool LC, int CH>
void main_ch(emu_engine* e, const RlDev& D, const RlBatch& B, const Src& src) {
    const uint32_t grid = rl_main_grid(B.nparts, B.n_acc, CH, e->main_grid_cap);
    e->report[G_CH] = CH;
    e->report[G_MERGE_MAIN] = rl_ceil_div(B.num_tiles, CH);
    interleave_on(e, 3 + (uint64_t)B.phase);
    simt_launch_ex(grid, CH, rl_main_smem_bytes<CELLS, CH>(B.num_tiles), e->resident,
                   [&] { k_main<GEO, CELLS, Src, MODE, CH, LC>(D, B, src, e->weak); });
    interleave_off();
}

template <int GEO, int CELLS, class Src, int MODE, bool LC>
void main_lc(emu_engine* e, const RlDev& D, const RlBatch& B, const Src& src) {
    if constexpr (Src::kWide) {
        main_ch<GEO, CELLS, Src, MODE, LC, 128>(e, D, B, src);  // wide batches: no hot rows, 128-access chunks
    } else {
        if (B.nhot && B.phase == RL_PHASE_COMMIT) {
            // k_hot has static shared memory: one block at a time
            interleave_on(e, 2);
            simt_launch_ex(B.nhot, RL_HOT_THREADS, 0, 1, [&] { k_hot<GEO, CELLS, Src, MODE, LC>(D, B, src); });
            interleave_off();
        }
        if (e->chunk == 128) main_ch<GEO, CELLS, Src, MODE, LC, 128>(e, D, B, src);
        else main_ch<GEO, CELLS, Src, MODE, LC, 256>(e, D, B, src);
    }
}

// launch_main: the instantiation rl_with_main_cells selects
template <class Src, int MODE>
void launch_main(emu_engine* e, const RlDev& D, const RlBatch& B, const Src& src) {
    const bool lc = MODE == 0 && B.load_counters;
    rl_with_main_cells(e->cells, e->t.shape.max_cells_used, [&](auto g, auto c) {
        constexpr int G = decltype(g)::value, A = decltype(c)::value;
        lc ? main_lc<G, A, Src, MODE, MODE == 0>(e, D, B, src) : main_lc<G, A, Src, MODE, false>(e, D, B, src);
    });
}

void begin_call(emu_engine* e) {
    memset(e->report, 0, sizeof e->report);
    memset(e->kstats, 0, sizeof e->kstats);
    memset(e->err, 0, sizeof e->err);
    e->flags = 0;
    for (uint32_t h = 0; h < RL_HOT_SLOTS; h++) e->report[G_HOT_IN_USE] += e->hot[h] != 0xFFFFFFFFu;
}
int end_call(emu_engine* e) {
    unsigned long long* g = e->report;
    g[G_CHUNKS] = e->kstats[0];
    g[G_ROUNDS] = e->kstats[1];
    g[G_CHAINED] = e->kstats[2];
    g[G_ORDERED] = e->kstats[3];
    g[G_HOT_CAND] = e->hot[RL_HOT_SLOTS + RL_HOT_CAND];  // reported by this call's k_main, read by the next front
    for (uint32_t h = 0; h < RL_HOT_SLOTS; h++) g[G_HOT_AFTER] += e->hot[h] != 0xFFFFFFFFu;
    // the counters the kernels re-arm for the next batch
    bool rearmed = e->small[0] == 0 && e->small[2] == 0 && e->small[3] == 0;
    for (uint32_t v : e->region_total) rearmed = rearmed && v == 0;
    g[G_REARMED] = rearmed;
    return (int)e->err[0];
}

// run_acc_pipeline (rl_engine.cu): accesses that may hold coupled (multi-row) requests.  check_and_update with
// coupled requests: SNAPSHOT, SPEC rounds (k_restore, k_fl_step) until the first-limited positions settle, COMMIT.
int acc_pipeline(emu_engine* e, RlDev& D, std::vector<RlAccess>& acc, uint32_t n_req, const uint64_t* delta,
                 const uint64_t* now, int mode, int lc, uint8_t* lim, uint32_t* first, uint64_t* rem, uint64_t* ttl,
                 const uint32_t* off, uint32_t stride, bool wide, const std::vector<uint8_t>& perm, uint32_t acc_stride) {
    const uint32_t n_acc = (uint32_t)acc.size();
    const bool scatter = wide && mode == 0 && lc && (rem || ttl);
    std::vector<uint64_t> wrem(scatter ? n_acc + 1 : 0), wttl(scatter ? n_acc + 1 : 0);
    Work w;
    RlBatch B = make_batch(e, w, n_acc, n_req, lim, first, scatter && rem ? wrem.data() : rem, scatter && ttl ? wttl.data() : ttl,
                           off, scatter && !off ? acc_stride : stride, lc, mode != 0);
    if (mode == 0) B.heavy_len = 0xFFFFFFFFu;
    AccSrc src{acc.data(), delta, now};
    launch_front(e, D, B, src);
    report_front(e, B, w);
    if (mode == 2) {
        launch_main<AccSrc, 2>(e, D, B, src);
        return 0;
    }
    auto main0 = [&]() {
        if (wide) launch_main<AccSrcWide, 0>(e, D, B, AccSrcWide{src});
        else launch_main<AccSrc, 0>(e, D, B, src);
    };
    if (e->flags & 1u) {
        e->flags = 0;
        const uint32_t buf_len = B.num_tiles * B.tile;
        w.log_row.assign(buf_len, nullptr);
        w.log_state.assign((size_t)buf_len * e->cells, ulonglong2{0xA5A5A5A5A5A5A5A5ull, 0xA5A5A5A5A5A5A5A5ull});
        B.log_row = w.log_row.data();
        B.log_state = w.log_state.data();
        B.phase = RL_PHASE_SNAPSHOT;
        main0();
        for (uint32_t round = 0;; round++) {
            if (round > n_req + 2) return -1;  // did not converge
            e->changed = 0;
            B.phase = RL_PHASE_SPEC;
            main0();
            rl_with_main_cells(e->cells, e->t.shape.max_cells_used, [&](auto g, auto c) {
                simt_launch(rl_ceil_div(buf_len, 256), 256,
                            [&] { k_restore<decltype(g)::value>(buf_len, decltype(c)::value, B.log_row, B.log_state); });
            });
            simt_launch(rl_ceil_div(n_req, 256), 256, [&] { k_fl_step(n_req, B.fl_prev, B.fl_next, &e->changed); });
            e->report[G_FP_ROUNDS] = round + 1;
            if (!(e->changed & 1u)) break;
        }
    }
    B.phase = RL_PHASE_COMMIT;
    main0();
    if (scatter)
        simt_launch(rl_ceil_div(n_req, 128), 128, [&] {
            k_wide_scatter(n_req, off, acc_stride, stride, perm.data(), rem ? wrem.data() : nullptr, ttl ? wttl.data() : nullptr, rem, ttl);
        });
    return 0;
}

}  // namespace

extern "C" {

// capacity = 2^(log2P + log2R) rows of cells (1, 3 or 7) cells
emu_engine* emu_engine_create(uint32_t cells, uint32_t log2P, uint32_t log2R) {
    emu_engine* e = new emu_engine();
    e->cells = cells;
    e->log2P = log2P;
    e->log2R = log2R;
    e->row_bytes = 16 * (1 + cells);
    e->reg.cells = cells;
    e->rows.assign(((size_t)1 << (log2P + log2R)) * e->row_bytes, 0);
    e->hot.assign(RL_HOT_SLOTS + RL_HOT_CAND + 4, 0xFFFFFFFFu);  // rl_internal_reset_hot_rows
    for (uint32_t i = RL_HOT_SLOTS + RL_HOT_CAND; i < e->hot.size(); i++) e->hot[i] = 0;
    e->region_total.assign((1u << log2P) + RL_HOT_SLOTS + 2, 0);
    e->small.assign(8, 0);
    return e;
}
void emu_engine_destroy(emu_engine* e) { delete e; }

// rl_limits_set and the upload of the tables
int emu_engine_limits_set(emu_engine* e, const rl_limit_desc* d, uint32_t n) {
    std::string err;
    const int r = e->reg.set(d, n, &err);
    e->t = e->reg.image();
    return r;
}

// knobs: chunk (128/256), heavy_mult, part_target, hot rows, weak tags, sharded geometry, resident k_main blocks, grid cap
void emu_engine_knobs(emu_engine* e, uint32_t chunk, uint32_t heavy_mult, uint32_t part_target, uint32_t hot, uint32_t weak,
                      uint32_t n_dev, uint32_t resident, uint32_t main_grid_cap) {
    e->chunk = chunk;
    e->heavy_mult = heavy_mult;
    e->part_target = part_target;
    e->hot_on = hot;
    e->weak = weak;
    e->n_dev = n_dev;
    e->resident = resident;
    e->main_grid_cap = main_grid_cap;
}
// cuda_simt.h's interleaving mode for every launch of the calls that follow (the n-th launch of a call salts the seed)
void emu_engine_interleave(emu_engine* e, int on, uint64_t seed, double p) {
    e->interleave = on != 0;
    e->seed = seed;
    e->p = p;
}
const unsigned long long* emu_engine_report(emu_engine* e) { return e->report; }
uint32_t emu_engine_max_cells_used(emu_engine* e) { return e->t.shape.max_cells_used; }
// the table region of record r's row (single-row namespaces), or -1 when the record has no row
int64_t emu_engine_record_region(emu_engine* e, const rl_record* r) {
    if (r->ns_id >= e->t.ns.size() || e->t.ns[r->ns_id].mode != 1) return -1;
    const RlNsDev& ns = e->t.ns[r->ns_id];
    const uint64_t klo = ns.qualified_row ? r->key_lo : 0;
    const uint64_t hhi = ((uint64_t)ns.group << 32) | (ns.qualified_row ? (r->key_hi & 0xFFFFFFFFull) : 0);
    const uint64_t h = rl_row_hash(klo, hhi);
    return e->log2P ? (int64_t)(h >> (64 - e->log2P)) : 0;
}
// remaining / ttl slots per record (RlTableShape::record_stride)
uint32_t emu_engine_record_stride(emu_engine* e) { return e->t.shape.record_stride(e->cells); }

// check_and_update (mode 0) / update_counters (mode 2) over 32-byte records: run_record_pipeline (rl_engine.cu)
// without the pipeline — k_front, k_hot when hot rows are on, k_main — or, when some namespace spans several rows, the
// records resolved into accesses (k_resolve_records, narrow or wide) and run_acc_pipeline.  rem / ttl: [n * stride]
// with stride = emu_engine_record_stride.  compact_now != 0: recs points at n 16-byte rl_record16 stamped with that one
// clock reading (rl_check_and_update_compact; single-row namespaces only).  Returns the device error code.
int emu_engine_records(emu_engine* e, int mode, uint32_t n, const rl_record* recs, int lc, uint8_t* lim, uint32_t* first,
                       uint64_t* rem, uint64_t* ttl, uint64_t compact_now) {
    begin_call(e);
    RlDev D = make_dev(e);
    if (e->t.shape.any_multi_ns) {
        if (compact_now) return -1;  // run_record_pipeline refuses it
        const uint32_t stride = e->t.shape.record_stride(e->cells);
        const bool wide = stride > RL_MAX_CTRS_PER_REQ;
        std::vector<RlAccess> acc((size_t)n * stride);
        std::vector<uint64_t> delta(std::max<uint32_t>(n, 1)), now(std::max<uint32_t>(n, 1));
        std::vector<uint8_t> perm(wide ? acc.size() + 1 : 0);
        RlResolveOut O{acc.data(), delta.data(), now.data(), lim, first};
        const uint32_t blocks = rl_ceil_div(n, 128);
        if (wide) simt_launch(blocks, 128, [&] { k_resolve_records_wide(D, n, recs, stride, O, mode == 0, perm.data(), RL_MAX_CTRS_PER_REQ_WIDE); });
        else simt_launch(blocks, 128, [&] { k_resolve_records(D, n, recs, stride, O, mode == 0); });
        if (e->err[0]) return (int)e->err[0];
        if (acc_pipeline(e, D, acc, n, delta.data(), now.data(), mode, lc, lim, first, rem, ttl, nullptr, stride, wide, perm, stride))
            return -1;
        return end_call(e);
    }
    Work w;
    // the sharded knob: the count handed over on the device (n_hint = n_dev = n), the tile derived from it there
    w.n_dev = n;
    RlBatch B = make_batch(e, w, n, n, lim, first, rem, ttl, nullptr, e->cells, lc, true, e->n_dev ? n : 0,
                           e->n_dev ? &w.n_dev : nullptr);
    RecordSrc src{recs, nullptr, 0, 0, compact_now ? 1u : 0u, compact_now};
    launch_front(e, D, B, src);
    report_front(e, B, w);
    if (mode == 2) launch_main<RecordSrc, 2>(e, D, B, src);
    else launch_main<RecordSrc, 0>(e, D, B, src);
    return end_call(e);
}

// check_and_update / update_counters in the general (CSR) form: k_resolve_csr (or _wide when a request has more than 16
// counters) and run_acc_pipeline.  rem / ttl: [off[n]].
int emu_engine_csr(emu_engine* e, int mode, uint32_t n, const uint32_t* off, const rl_counter* ctrs, const uint64_t* delta,
                   const uint64_t* now, int lc, uint8_t* lim, uint32_t* first, uint64_t* rem, uint64_t* ttl) {
    begin_call(e);
    RlDev D = make_dev(e);
    uint32_t maxm = 0;
    for (uint32_t i = 0; i < n; i++) maxm = std::max(maxm, off[i + 1] - off[i]);
    const bool wide = maxm > RL_MAX_CTRS_PER_REQ;
    std::vector<RlAccess> acc(off[n]);
    std::vector<uint8_t> perm(wide ? off[n] + 1 : 0);
    RlResolveOut O{acc.data(), nullptr, nullptr, lim, first};
    const uint32_t blocks = rl_ceil_div(n, 128);
    if (wide) simt_launch(blocks, 128, [&] { k_resolve_csr_wide(D, n, off, ctrs, O, mode == 0, perm.data(), RL_MAX_CTRS_PER_REQ_WIDE); });
    else simt_launch(blocks, 128, [&] { k_resolve_csr(D, n, off, ctrs, O, mode == 0); });
    if (e->err[0]) return (int)e->err[0];
    if (acc.empty()) return end_call(e);
    if (acc_pipeline(e, D, acc, n, delta, now, mode, lc, lim, first, rem, ttl, off, 0, wide, perm, 0)) return -1;
    return end_call(e);
}

// is_within_limits over records (k_query_records): read-only
int emu_engine_query_records(emu_engine* e, uint32_t n, const rl_record* recs, uint8_t* lim, uint32_t* first) {
    begin_call(e);
    RlDev D = make_dev(e);
    rl_with_cells(e->cells, [&](auto c) {
        simt_launch(rl_ceil_div(n, 128), 128, [&] { k_query_records<decltype(c)::value>(D, n, recs, lim, first); });
    });
    return (int)e->err[0];
}

// the table through k_scan in export mode (read_table in rl_engine.cu, now = 0: every present cell as
// (value, expiry)); the present unqualified limits no row showed are left out, as a never-touched counter.
uint64_t emu_engine_export(emu_engine* e, uint64_t cap, uint32_t* lid, uint64_t* lo, uint64_t* hi, uint64_t* val, uint64_t* exp) {
    RlDev D = make_dev(e);
    const uint32_t L = (uint32_t)e->t.lim.size();
    std::vector<uint8_t> flags(2 * (size_t)L, 0);
    for (uint32_t l = 0; l < L; l++) flags[l] = e->reg.present(l);
    unsigned long long cnt = 0;
    RlScanOut O{lid, lo, hi, val, exp, &cnt, cap, flags.data(), flags.data() + L};
    const uint64_t nrows = e->rows.size() / e->row_bytes;
    rl_with_cells(e->cells, [&](auto c) {
        simt_launch(rl_ceil_div(nrows, 256), 256,
                    [&] { k_scan<decltype(c)::value>(D, nrows, false, 0, nullptr, e->t.group_ns.data(), O); });
    });
    return cnt;
}

}  // extern "C"

// ---- the namespace-sharded peer exchange (rl_shard_host.inc) over `world` emulated engines -------------------------
// Every rank has a host "slab" laid out as rl_shard_create lays out the device one (records | verdict inboxes | control
// words, depth = lag + 2 buffers) and its own exchange workspace; X.base[] of every rank names all the slabs, as
// rl_shard_connect_ptrs does.  The launches run in the caller's issue order, one at a time: a wait kernel issued before
// the kernels it waits for is reported by cuda_simt.h as a hang.
struct emu_shard_rank {
    emu_engine* e = nullptr;
    std::vector<uint8_t> slab;
    RlXchg X{};
    std::vector<uint32_t> tile_cnt, totals, ctrs, dest, seg;
    std::vector<uint8_t> verdict;  // the decide call's local mirror of the sources' verdict blocks [world][cap]
    uint64_t sent = 0, decided = 0, collected = 0;
    static constexpr int kRingN = 8;
    uint32_t n_of[kRingN] = {};
    uint8_t* out_of[kRingN] = {};
};
struct emu_shard {
    uint32_t world = 1, cap = 0, lag = 0, depth = 2, max_batch = 0;
    size_t recs_bytes = 0, vin_bytes = 0, ctl_bytes = 0;
    std::vector<emu_shard_rank> r;
};

namespace {
constexpr uint8_t kPoison = 0xA5;
size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
}  // namespace

extern "C" {

// world engines (one per rank, each with its limits set), cap records per source batch (a multiple of 16), lag 0..4,
// max_batch of every engine (an owner's inbox larger than min(world x cap, max_batch) fails the step).  NULL on bad input.
emu_shard* emu_shard_create(emu_engine** engines, uint32_t world, uint32_t cap, uint32_t lag, uint32_t max_batch) {
    if (world == 0 || world > RL_XCHG_MAX_WORLD || cap == 0 || (cap & 15u) || lag > 4) return nullptr;
    emu_shard* S = new emu_shard();
    S->world = world;
    S->cap = cap;
    S->lag = lag;
    S->depth = lag + 2;
    S->max_batch = max_batch;
    S->recs_bytes = align256((size_t)S->depth * world * cap * sizeof(rl_record));
    S->vin_bytes = align256((size_t)S->depth * world * cap);
    S->ctl_bytes = align256((size_t)S->depth * world * sizeof(RlXCtl));
    S->r.resize(world);
    for (uint32_t k = 0; k < world; k++) {
        emu_shard_rank& R = S->r[k];
        R.e = engines[k];
        R.slab.assign(S->recs_bytes + S->vin_bytes + S->ctl_bytes, 0);  // rl_shard_create zeroes the slab
        R.tile_cnt.assign((size_t)(RL_MAX_TILES + 1) * 32, 0);
        R.totals.assign(32, 0);
        R.ctrs.assign(4, 0);
        R.dest.assign((size_t)S->depth * cap, 0);
        R.seg.assign(40, 0);
        R.verdict.assign((size_t)world * cap, 0);
    }
    for (uint32_t k = 0; k < world; k++) {
        RlXchg& X = S->r[k].X;
        X.trace = nullptr;
        X.trace_pos = nullptr;
        for (auto& b : X.base) b = nullptr;
        for (uint32_t j = 0; j < world; j++) X.base[j] = S->r[j].slab.data();
        X.off_recs = 0;
        X.off_vin = S->recs_bytes;
        X.off_ctl = S->recs_bytes + S->vin_bytes;
        X.world = world;
        X.rank = k;
        X.cap = cap;
        X.depth = S->depth;
    }
    return S;
}
void emu_shard_destroy(emu_shard* S) { delete S; }

// rl_shard_send: bucket rank's n records by owner (k_xcount) and store them into the owners' inboxes (k_xscatter).  The
// blocks this step writes, the verdict blocks it will read and dest are poisoned first, so that a read past a fill or a
// missing verdict shows as a wrong result, not as a stale correct one.  out: n verdict bytes, filled by the collection.
int emu_shard_send(emu_shard* S, uint32_t rank, uint32_t n, const rl_record* recs, uint8_t* out) {
    emu_shard_rank& R = S->r[rank];
    if (n > S->cap || R.sent - R.collected > S->lag || (n && (!recs || !out))) return -1;
    const uint32_t step = (uint32_t)R.sent, buf = (uint32_t)(R.sent % S->depth), world = S->world;
    for (uint32_t o = 0; o < world; o++) {
        memset(R.X.inbox(o, buf, rank), kPoison, (size_t)S->cap * sizeof(rl_record));
        memset(R.X.vin(rank, buf, o), kPoison, S->cap);
    }
    std::fill(R.dest.begin() + (size_t)buf * S->cap, R.dest.begin() + (size_t)(buf + 1) * S->cap, 0xA5A5A5A5u);
    std::fill(R.tile_cnt.begin(), R.tile_cnt.end(), 0xA5A5A5A5u);
    std::fill(R.totals.begin(), R.totals.end(), 0xA5A5A5A5u);
    uint32_t tile = rl_ceil_div(std::max<uint64_t>(n, 1), RL_MAX_TILES);
    tile = std::max<uint32_t>(256, ((tile + 255) / 256) * 256);
    const uint32_t num_tiles = std::max<uint32_t>(1, rl_ceil_div(n, tile));
    // static __shared__ arrays: one copy for all blocks, so one block at a time
    simt_launch(num_tiles, RL_PART_THREADS, [&] {
        k_xcount(recs, n, world, tile, R.tile_cnt.data(), R.totals.data(), R.ctrs.data() + 0, nullptr, nullptr, step);
    });
    simt_launch(num_tiles, RL_PART_THREADS, [&] {
        k_xscatter(R.X, recs, n, tile, R.tile_cnt.data(), R.totals.data(), buf, step, R.dest.data() + (size_t)buf * S->cap,
                   R.ctrs.data() + 1);
    });
    R.n_of[R.sent % emu_shard_rank::kRingN] = n;
    R.out_of[R.sent % emu_shard_rank::kRingN] = out;
    R.sent++;
    return 0;
}

// rl_shard_decide: k_xwait, then the record path over the segmented inbox (n_acc = min(world x cap, max_batch), partitions
// sized for one source batch, the tile derived from the inbox fill on the device), the verdicts into the local mirror
// (poisoned first), then k_xreturn.  The engine's report holds the call's geometry; returns the device error code.
int emu_shard_decide(emu_shard* S, uint32_t rank) {
    emu_shard_rank& R = S->r[rank];
    emu_engine* e = R.e;
    if (R.decided >= R.sent || e->t.shape.any_multi_ns) return -1;
    const uint32_t step = (uint32_t)R.decided, buf = (uint32_t)(R.decided % S->depth), world = S->world, cap = S->cap;
    const uint32_t n_max = (uint32_t)std::min<uint64_t>((uint64_t)world * cap, S->max_batch);
    begin_call(e);
    RlDev D = make_dev(e);
    std::fill(R.seg.begin(), R.seg.end(), 0xA5A5A5A5u);
    std::fill(R.verdict.begin(), R.verdict.end(), kPoison);
    uint32_t* segp = R.seg.data();
    simt_launch(1, 32, [&] { k_xwait(R.X, buf, step, segp, segp + 36, n_max, e->err); });
    const RecordSrc src{R.X.inbox(rank, buf, 0), segp, world, cap, 0, 0};
    Work w;
    RlBatch B = make_batch(e, w, n_max, n_max, R.verdict.data(), nullptr, nullptr, nullptr, nullptr, 0, 0, true, cap, segp + 36);
    B.omap_prefix = segp;
    B.omap_n = world;
    B.omap_stride = cap;
    launch_front(e, D, B, src);
    report_front(e, B, w);
    launch_main<RecordSrc, 0>(e, D, B, src);
    simt_launch(world * RL_XRET_SLICES, 256, [&] { k_xreturn(R.X, R.verdict.data(), segp, buf, step, R.ctrs.data() + 2); });
    R.decided++;
    return end_call(e);
}

// rl_shard_collect (all = 0: only once more than `lag` decided steps are outstanding) / rl_shard_flush (all = 1): k_xwaitv,
// then k_xgather into the step's output.  Returns the steps collected.
int emu_shard_collect(emu_shard* S, uint32_t rank, int all) {
    emu_shard_rank& R = S->r[rank];
    emu_engine* e = R.e;
    int done = 0;
    while (R.collected < R.decided && (all || R.decided - R.collected > S->lag)) {
        const uint32_t step = (uint32_t)R.collected, buf = (uint32_t)(R.collected % S->depth);
        const uint32_t n = R.n_of[R.collected % emu_shard_rank::kRingN];
        uint8_t* out = R.out_of[R.collected % emu_shard_rank::kRingN];
        simt_launch(1, 32, [&] { k_xwaitv(R.X, buf, step, e->err); });
        if (n) {
            const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(rl_ceil_div(n, 256), e->main_grid_cap / 8));
            simt_launch(grid, 256, [&] { k_xgather(R.X, n, R.dest.data() + (size_t)buf * S->cap, buf, out); });
        }
        R.collected++;
        done++;
    }
    return done;
}

// k_xwait alone on rank's control words of (buf, step) (set them first with emu_shard_set_ctl, so that nothing waits):
// seg_out [40] = the exclusive prefix seg_prefix[0..world] and, at [36], n_dev; err_out [8] = the error words
void emu_shard_xwait(emu_shard* S, uint32_t rank, uint32_t buf, uint32_t step, uint32_t n_max, uint32_t* seg_out,
                     uint32_t* err_out) {
    emu_shard_rank& R = S->r[rank];
    std::fill(seg_out, seg_out + 40, 0xA5A5A5A5u);
    memset(err_out, 0, 8 * sizeof(uint32_t));
    simt_launch(1, 32, [&] { k_xwait(R.X, buf, step, seg_out, seg_out + 36, n_max, err_out); });
}

// rank's control words: [(buf * world + peer) * 4 + {0 cnt, 1 rflag, 2 vflag, 3 pad}], depth * world * 4 of them
void emu_shard_ctl(emu_shard* S, uint32_t rank, uint32_t* out) {
    memcpy(out, S->r[rank].slab.data() + S->recs_bytes + S->vin_bytes, (size_t)S->depth * S->world * sizeof(RlXCtl));
}
void emu_shard_set_ctl(emu_shard* S, uint32_t rank, const uint32_t* in) {
    memcpy(S->r[rank].slab.data() + S->recs_bytes + S->vin_bytes, in, (size_t)S->depth * S->world * sizeof(RlXCtl));
}
// block `src` of owner's inbox `buf` (cap records), rank's dest of `buf` (cap words), its blocks-done counters (4 words:
// k_xcount, k_xscatter, k_xreturn, unused) and its error words of the last decide / collect (8 words)
void emu_shard_inbox(emu_shard* S, uint32_t owner, uint32_t buf, uint32_t src, rl_record* out) {
    memcpy(out, S->r[owner].X.inbox(owner, buf, src), (size_t)S->cap * sizeof(rl_record));
}
void emu_shard_dest(emu_shard* S, uint32_t rank, uint32_t buf, uint32_t* out) {
    memcpy(out, S->r[rank].dest.data() + (size_t)buf * S->cap, (size_t)S->cap * sizeof(uint32_t));
}
void emu_shard_ctrs(emu_shard* S, uint32_t rank, uint32_t* out) { memcpy(out, S->r[rank].ctrs.data(), 4 * sizeof(uint32_t)); }
void emu_shard_err(emu_shard* S, uint32_t rank, uint32_t* out) { memcpy(out, S->r[rank].e->err, 8 * sizeof(uint32_t)); }

}  // extern "C"
