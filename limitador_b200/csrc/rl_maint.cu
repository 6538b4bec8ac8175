// rl_maint.cu — host side of the maintenance kernels (rl_maint.cuh): tombstone reclamation (rl_compact), the
// per-namespace metrics reduction (rl_ns_metrics_*), counter import and change tracking (rl_counters_track / _drain).  A translation unit of its own: it sees an engine only through
// rl_internal.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "rl_cuda_host.h"
#include "rl_internal.h"
#include "rl_maint.cuh"

namespace {

struct MaintState {
    int device = 0;
    // metrics accumulators (device): authorized_calls | authorized_hits | limited_calls [ns_cap], limited_by_limit
    // [limits_cap], dropped [1]
    DevBuf<unsigned long long> d_metrics;
    uint32_t ns_cap = 0, limits_cap = 0;
    bool metrics_on = false;
    // change tracking: the table as the last drain saw it; the next drain is full until one ran at epoch_seen
    DevBuf<uint8_t> d_shadow;
    bool full_next = true;
    uint64_t epoch_seen = 0;
};

void maint_free(void* p) {
    MaintState* s = static_cast<MaintState*>(p);
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;  // frees the accumulators, on the device made current above
}

MaintState* state_of(rl_engine* e, int device) {
    void** slot = rl_internal_ext(e, maint_free);
    if (!*slot) {
        MaintState* s = new MaintState();
        s->device = device;
        *slot = s;
    }
    return static_cast<MaintState*>(*slot);
}

template <class... A>
int fail(rl_engine* e, int status, const char* fmt, A... a) {
    return rl_internal_fail(e, status, rl_format(fmt, a...).c_str());
}

size_t metrics_words(uint32_t ns_cap, uint32_t limits_cap) { return (size_t)3 * ns_cap + limits_cap + 1; }

RlNsMetricsDev metrics_dev(const MaintState* s) {
    RlNsMetricsDev M;
    M.authorized_calls = s->d_metrics.p;
    M.authorized_hits = s->d_metrics.p + s->ns_cap;
    M.limited_calls = s->d_metrics.p + 2 * (size_t)s->ns_cap;
    M.limited_by_limit = s->d_metrics.p + 3 * (size_t)s->ns_cap;
    M.dropped = s->d_metrics.p + 3 * (size_t)s->ns_cap + s->limits_cap;
    M.ns_cap = s->ns_cap;
    M.limits_cap = s->limits_cap;
    return M;
}

// Make the accumulators cover ns_cap namespaces and limits_cap limits; growing keeps the counts (rare: a full
// device synchronisation, then a copy).
int metrics_reserve(rl_engine* e, MaintState* s, uint32_t ns_cap, uint32_t limits_cap) {
    if (s->d_metrics.p && ns_cap <= s->ns_cap && limits_cap <= s->limits_cap) return RL_OK;
    const uint32_t new_ns = std::max<uint32_t>({ns_cap, s->ns_cap, 1024u}), new_lim = std::max<uint32_t>({limits_cap, s->limits_cap, 1024u});
    const uint32_t grow_ns = s->d_metrics.p && new_ns > s->ns_cap ? std::max(new_ns, 2 * s->ns_cap) : new_ns;
    const uint32_t grow_lim = s->d_metrics.p && new_lim > s->limits_cap ? std::max(new_lim, 2 * s->limits_cap) : new_lim;
    if (grow_ns >= (1u << 31)) return rl_internal_fail(e, RL_FATAL, "namespace ids must stay below 2^31 for the metrics reduction");
    DevBuf<unsigned long long> d_new;
    RL_CUDA(e, cudaDeviceSynchronize());
    RL_CUDA(e, d_new.exact(metrics_words(grow_ns, grow_lim)));
    RL_CUDA(e, cudaMemset(d_new.p, 0, metrics_words(grow_ns, grow_lim) * sizeof(unsigned long long)));
    if (s->d_metrics.p) {
        const size_t w = sizeof(unsigned long long);
        for (int k = 0; k < 3; k++)
            RL_CUDA(e, cudaMemcpy(d_new.p + (size_t)k * grow_ns, s->d_metrics.p + (size_t)k * s->ns_cap, s->ns_cap * w, cudaMemcpyDeviceToDevice));
        RL_CUDA(e, cudaMemcpy(d_new.p + 3 * (size_t)grow_ns, s->d_metrics.p + 3 * (size_t)s->ns_cap, s->limits_cap * w, cudaMemcpyDeviceToDevice));
        RL_CUDA(e, cudaMemcpy(d_new.p + 3 * (size_t)grow_ns + grow_lim, s->d_metrics.p + 3 * (size_t)s->ns_cap + s->limits_cap, w, cudaMemcpyDeviceToDevice));
    }
    s->d_metrics.swap(d_new);  // the old accumulators are freed on return
    s->ns_cap = grow_ns;
    s->limits_cap = grow_lim;
    return RL_OK;
}

int launch_metrics(rl_engine* e, MaintState* s, cudaStream_t st, uint32_t n, const void* d_recs, int record_bytes,
                   const uint8_t* d_limited, const uint32_t* d_first) {
    if (n == 0) return RL_OK;
    const uint32_t threads = 256;
    const uint32_t blocks = std::min<uint32_t>((n + threads - 1) / threads, rl_internal_sm_count(e) * 8u);  // grid-stride beyond 8 CTAs per SM
    k_ns_metrics<<<blocks, threads, 0, st>>>(static_cast<const unsigned long long*>(d_recs), record_bytes == 16 ? 2u : 4u, n,
                                             d_limited, d_first, metrics_dev(s));
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    return RL_OK;
}

// the hook rl_engine.cu calls behind the replay of a record call (rl_ns_metrics_enable)
int ns_hook(rl_engine* e, cudaStream_t st, uint32_t n, const void* d_recs, int record_bytes, const uint8_t* d_limited,
            const uint32_t* d_first) {
    void** slot = rl_internal_ext(e, maint_free);
    MaintState* s = static_cast<MaintState*>(*slot);
    if (!s || !s->metrics_on) return RL_OK;
    return launch_metrics(e, s, st, n, d_recs, record_bytes, d_limited, d_first);
}

}  // namespace

extern "C" {

int rl_ns_metrics_enable(rl_engine* e, int on) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    MaintState* s = state_of(e, v.device);
    if (on) {
        r = metrics_reserve(e, s, std::max<uint32_t>(v.ns_cap, 1u << 16), std::max<uint32_t>(v.limits_cap, 1u << 16));
        if (r) return r;
    }
    s->metrics_on = on != 0;
    rl_internal_set_ns_hook(e, on ? ns_hook : nullptr);
    return RL_OK;
}

int rl_ns_metrics_accumulate(rl_engine* e, uint64_t n, const void* recs, uint32_t record_bytes, const uint8_t* limited,
                             const uint32_t* first_limited, int mem) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    if (record_bytes != 32 && record_bytes != 16) return rl_internal_fail(e, RL_FATAL, "record_bytes must be 32 (rl_record) or 16 (rl_record16)");
    if (n > 0xFFFFFFFFull || (n && (!recs || !limited))) return rl_internal_fail(e, RL_FATAL, "rl_ns_metrics_accumulate: bad arguments");
    MaintState* s = state_of(e, v.device);
    r = metrics_reserve(e, s, std::max<uint32_t>(v.ns_cap, 1u << 16), std::max<uint32_t>(v.limits_cap, 1u << 16));
    if (r || n == 0) return r;
    if (mem == RL_MEM_DEVICE) return launch_metrics(e, s, v.stream, (uint32_t)n, recs, (int)record_bytes, limited, first_limited);
    // host arrays: staged for the call
    In<uint8_t> d_recs, d_lim;
    In<uint32_t> d_first;
    RL_CUDA(e, d_recs.set(static_cast<const uint8_t*>(recs), n * record_bytes, mem, v.stream));
    RL_CUDA(e, d_lim.set(limited, n, mem, v.stream));
    RL_CUDA(e, d_first.set(first_limited, n, mem, v.stream));
    r = launch_metrics(e, s, v.stream, (uint32_t)n, d_recs.p, (int)record_bytes, d_lim.p, d_first.p);
    RL_CUDA(e, cudaStreamSynchronize(v.stream));  // before the staged copies are freed
    return r;
}

int rl_ns_metrics_read(rl_engine* e, uint32_t ns_cap, uint64_t* out_authorized_calls, uint64_t* out_authorized_hits,
                       uint64_t* out_limited_calls, uint32_t limits_cap, uint64_t* out_limited_by_limit,
                       uint64_t* out_dropped, int reset) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    MaintState* s = state_of(e, v.device);
    if (out_dropped) *out_dropped = 0;
    for (uint32_t i = 0; i < ns_cap; i++) {
        if (out_authorized_calls) out_authorized_calls[i] = 0;
        if (out_authorized_hits) out_authorized_hits[i] = 0;
        if (out_limited_calls) out_limited_calls[i] = 0;
    }
    if (out_limited_by_limit)
        for (uint32_t i = 0; i < limits_cap; i++) out_limited_by_limit[i] = 0;
    if (!s->d_metrics.p) return RL_OK;
    RL_CUDA(e, cudaStreamSynchronize(v.stream));  // the view fenced the pipeline onto this stream
    std::vector<unsigned long long> h(metrics_words(s->ns_cap, s->limits_cap));
    RL_CUDA(e, cudaMemcpy(h.data(), s->d_metrics.p, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    const uint32_t nn = std::min(ns_cap, s->ns_cap), nl = std::min(limits_cap, s->limits_cap);
    for (uint32_t i = 0; i < nn; i++) {
        if (out_authorized_calls) out_authorized_calls[i] = h[i];
        if (out_authorized_hits) out_authorized_hits[i] = h[(size_t)s->ns_cap + i];
        if (out_limited_calls) out_limited_calls[i] = h[2 * (size_t)s->ns_cap + i];
    }
    if (out_limited_by_limit)
        for (uint32_t i = 0; i < nl; i++) out_limited_by_limit[i] = h[3 * (size_t)s->ns_cap + i];
    if (out_dropped) *out_dropped = h[3 * (size_t)s->ns_cap + s->limits_cap];
    if (reset) RL_CUDA(e, cudaMemset(s->d_metrics.p, 0, h.size() * sizeof(unsigned long long)));
    return RL_OK;
}

int rl_compact(rl_engine* e, uint32_t min_tombstone_pct, rl_compact_stats* out) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    if (out) memset(out, 0, sizeof *out);
    const uint32_t P = 1u << v.log2P;
    const uint64_t R = 1ull << v.log2R;
    DevBuf<uint32_t> d_census;  // live[P] | tomb[P]
    RL_CUDA(e, d_census.alloc(2 * (size_t)P));
    RL_CUDA(e, cudaMemsetAsync(d_census.p, 0, 2 * (size_t)P * sizeof(uint32_t), v.stream));
    const uint32_t threads = 256;
    const uint32_t blocks = (uint32_t)((v.capacity + threads - 1) / threads);
    k_region_census<<<blocks, threads, 0, v.stream>>>(v.rows, v.row_bytes, v.log2R, v.capacity, d_census.p, d_census.p + P);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    std::vector<uint32_t> census(2 * (size_t)P);
    RL_CUDA(e, cudaMemcpyAsync(census.data(), d_census.p, census.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));
    std::vector<uint8_t> sel(P, 0);
    uint64_t live = 0, tomb = 0, chosen = 0, tomb_chosen = 0;
    for (uint32_t g = 0; g < P; g++) {
        live += census[g];
        tomb += census[P + g];
        // a region is rebuilt when its tombstones reach min_tombstone_pct % of its rows (0 = any tombstone at all)
        if (census[P + g] && (uint64_t)census[P + g] * 100 >= (uint64_t)min_tombstone_pct * R) {
            sel[g] = 1;
            chosen++;
            tomb_chosen += census[P + g];
        }
    }
    if (out) {
        out->regions = P;
        out->rows_live = live;
        out->rows_tombstoned = tomb;
        out->regions_rebuilt = chosen;
    }
    if (!chosen) return RL_OK;
    DevBuf<uint8_t> d_sel, d_scratch;
    DevBuf<unsigned long long> d_counts;
    RL_CUDA(e, d_sel.alloc(P));
    if (d_scratch.alloc((size_t)v.capacity * v.row_bytes) != cudaSuccess) {
        cudaGetLastError();
        return rl_internal_fail(e, RL_TRANSIENT, "rl_compact: no device memory for the scratch slab (one copy of the table)");
    }
    RL_CUDA(e, d_counts.alloc(3));
    RL_CUDA(e, cudaMemcpyAsync(d_sel.p, sel.data(), P, cudaMemcpyHostToDevice, v.stream));
    RL_CUDA(e, cudaMemsetAsync(d_counts.p, 0, 3 * sizeof(unsigned long long), v.stream));
    k_compact_move<<<blocks, threads, 0, v.stream>>>(v.rows, d_scratch.p, v.row_bytes, v.log2R, v.capacity, d_sel.p);
    RL_CUDA(e, cudaGetLastError());
    k_compact_reinsert<<<blocks, threads, 0, v.stream>>>(v.rows, d_scratch.p, v.row_bytes, v.log2P, v.log2R, v.capacity, d_sel.p, d_counts.p);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 2);
    rl_internal_structure_changed(e);
    r = rl_internal_reset_hot_rows(e);  // table row indices changed
    unsigned long long counts[3] = {0, 0, 0};
    RL_CUDA(e, cudaMemcpyAsync(counts, d_counts.p, sizeof counts, cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));  // before the scratch slab is freed
    if (r) return r;
    if (out) {
        out->rows_moved = counts[0];
        out->rows_reclaimed = tomb_chosen + counts[1];
    }
    if (counts[2]) return rl_internal_fail(e, RL_FATAL, "rl_compact: a row could not be placed again (table corrupt?)");
    return RL_OK;
}

int rl_counters_import(rl_engine* e, uint64_t n, const uint32_t* limit_id, const uint64_t* key_lo, const uint64_t* key_hi,
                       const uint64_t* value, const uint64_t* expiry_us, int mem) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    if (mem != RL_MEM_HOST && mem != RL_MEM_DEVICE)
        return rl_internal_fail(e, RL_FATAL, "rl_counters_import: mem must be RL_MEM_HOST or RL_MEM_DEVICE");
    if (n && (!limit_id || !key_lo || !key_hi || !value || !expiry_us))
        return rl_internal_fail(e, RL_FATAL, "rl_counters_import: n > 0 needs all five input arrays");
    if (n >= (1ull << 48)) return rl_internal_fail(e, RL_FATAL, "rl_counters_import: n must stay below 2^48");
    if (n == 0) return RL_OK;
    rl_internal_structure_changed(e);
    // inputs on the device: the caller's arrays, or staged for the call
    In<uint32_t> lid;
    In<uint64_t> lo, hi, val, exp;
    RL_CUDA(e, lid.set(limit_id, n, mem, v.stream));
    RL_CUDA(e, lo.set(key_lo, n, mem, v.stream));
    RL_CUDA(e, hi.set(key_hi, n, mem, v.stream));
    RL_CUDA(e, val.set(value, n, mem, v.stream));
    RL_CUDA(e, exp.set(expiry_us, n, mem, v.stream));
    const RlImportIn I{lid.p, lo.p, hi.p, val.p, exp.p, n};
    const RlImportTab T{v.rows, v.row_bytes, v.log2P, v.log2R, v.limits, v.limits_cap};
    DevBuf<unsigned long long> d_err, d_row_of;
    DevBuf<uint8_t> d_unq;
    DevBuf<unsigned> d_mask;  // per-row cell mask of this call
    RL_CUDA(e, d_err.alloc(1));
    RL_CUDA(e, d_unq.alloc(v.limits_cap));
    RL_CUDA(e, cudaMemsetAsync(d_err.p, 0xFF, sizeof(unsigned long long), v.stream));
    RL_CUDA(e, cudaMemsetAsync(d_unq.p, 0, v.limits_cap, v.stream));
    const uint32_t threads = 256;
    const uint32_t blocks = (uint32_t)((n + threads - 1) / threads);
    unsigned long long err = ~0ull;
    auto report = [&](const char* pass) {
        const uint64_t idx = err >> 8;
        const uint32_t why = (uint32_t)(err & 0xFF);
        static const char* const reason[] = {"", "limit id not registered in this engine", "qualified counter with key_hi >= 2^32",
                                             "qualified counter with expiry 0", "the same counter appears twice",
                                             "its table region is full"};
        return fail(e, why == RLM_IMP_TABLE_FULL ? RL_TRANSIENT : RL_FATAL,
                    "rl_counters_import: entry %llu refused (%s) in the %s pass; no counter changed", (unsigned long long)idx,
                    why <= RLM_IMP_TABLE_FULL ? reason[why] : "?", pass);
    };
    // pass 1: every entry names a registered limit and a valid key / expiry
    k_import_resolve<<<blocks, threads, 0, v.stream>>>(T, I, d_err.p, d_unq.p);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    RL_CUDA(e, cudaMemcpyAsync(&err, d_err.p, sizeof err, cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));
    if (err != ~0ull) return report("resolve");
    // pass 2: find or claim the rows; duplicates and full regions are found before any cell is written
    RL_CUDA(e, d_row_of.alloc(n));
    if (d_mask.alloc(v.capacity) != cudaSuccess) {
        cudaGetLastError();
        return rl_internal_fail(e, RL_TRANSIENT, "rl_counters_import: no device memory for the per-row cell mask");
    }
    RL_CUDA(e, cudaMemsetAsync(d_mask.p, 0, v.capacity * sizeof(unsigned), v.stream));
    RL_CUDA(e, cudaMemsetAsync(d_row_of.p, 0, n * sizeof(unsigned long long), v.stream));
    k_import_claim<<<blocks, threads, 0, v.stream>>>(T, I, d_row_of.p, d_mask.p, d_err.p);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    RL_CUDA(e, cudaMemcpyAsync(&err, d_err.p, sizeof err, cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));
    if (err != ~0ull) {  // give back the rows this call claimed: the table is byte-identical to before the call
        k_import_release<<<blocks, threads, 0, v.stream>>>(T, n, d_row_of.p);
        RL_CUDA(e, cudaGetLastError());
        rl_internal_launched(e, 1);
        RL_CUDA(e, cudaStreamSynchronize(v.stream));
        return report("claim");
    }
    // pass 3: the cells
    k_import_write<<<blocks, threads, 0, v.stream>>>(T, I, d_row_of.p);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    std::vector<uint8_t> unq(v.limits_cap);
    RL_CUDA(e, cudaMemcpyAsync(unq.data(), d_unq.p, unq.size(), cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));  // before the staged inputs are freed
    rl_internal_mark_present(e, unq.data(), v.limits_cap);
    return RL_OK;
}

int rl_counters_track(rl_engine* e, int on) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    MaintState* s = state_of(e, v.device);
    RL_CUDA(e, cudaStreamSynchronize(v.stream));
    if (!on) {
        RL_CUDA(e, s->d_shadow.exact(0));
        return RL_OK;
    }
    if (!s->d_shadow.p && s->d_shadow.exact((size_t)v.capacity * v.row_bytes) != cudaSuccess) {
        cudaGetLastError();
        return rl_internal_fail(e, RL_TRANSIENT, "rl_counters_track: no device memory for the shadow (one copy of the table)");
    }
    s->full_next = true;
    return RL_OK;
}

int rl_counters_drain(rl_engine* e, uint64_t cap, int mem, uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi,
                      uint64_t* out_value, uint64_t* out_expiry_us, uint64_t* out_count, int* out_full) {
    RlTableView v;
    int r = rl_internal_view(e, &v);
    if (r) return r;
    if (!out_count || !out_full) return rl_internal_fail(e, RL_FATAL, "rl_counters_drain: out_count and out_full are needed");
    *out_count = 0;
    *out_full = 0;
    MaintState* s = state_of(e, v.device);
    if (!s->d_shadow.p) return rl_internal_fail(e, RL_FATAL, "rl_counters_drain: change tracking is off (rl_counters_track)");
    if (mem != RL_MEM_HOST && mem != RL_MEM_DEVICE)
        return rl_internal_fail(e, RL_FATAL, "rl_counters_drain: mem must be RL_MEM_HOST or RL_MEM_DEVICE");
    if (cap && (!out_limit_id || !out_key_lo || !out_key_hi || !out_value || !out_expiry_us))
        return rl_internal_fail(e, RL_FATAL, "rl_counters_drain: cap > 0 needs all five output arrays");
    const size_t table_bytes = (size_t)v.capacity * v.row_bytes;
    if (s->full_next || s->epoch_seen != v.structure_epoch) {
        // full: the export itself, and the table into the shadow only when the caller got all of it
        *out_full = 1;
        if ((r = rl_counters_export(e, nullptr, 0, 0, cap, mem, out_limit_id, out_key_lo, out_key_hi, out_value, out_expiry_us,
                                    out_count)))
            return r;
        if (*out_count > cap) return RL_OK;
        RL_CUDA(e, cudaMemcpyAsync(s->d_shadow.p, v.rows, table_bytes, cudaMemcpyDeviceToDevice, v.stream));
        RL_CUDA(e, cudaStreamSynchronize(v.stream));
        s->full_next = false;
        s->epoch_seen = v.structure_epoch;
        return RL_OK;
    }
    std::vector<uint8_t> present(std::max<uint32_t>(v.limits_cap, 1));
    rl_internal_present(e, present.data(), (uint32_t)present.size());
    DevBuf<uint8_t> d_present;
    DevBuf<unsigned long long> d_cnt;
    RL_CUDA(e, d_present.alloc(present.size()));
    RL_CUDA(e, d_cnt.alloc(1));
    RL_CUDA(e, cudaMemcpyAsync(d_present.p, present.data(), present.size(), cudaMemcpyHostToDevice, v.stream));
    RL_CUDA(e, cudaMemsetAsync(d_cnt.p, 0, sizeof(unsigned long long), v.stream));
    const RlChangeTab T{v.rows, s->d_shadow.p, v.row_bytes, v.cells, v.capacity, v.desc, d_present.p};
    const uint32_t threads = 256;
    const uint32_t blocks = (uint32_t)((v.capacity + threads - 1) / threads);
    // count first: a drain that does not fit leaves the shadow as it was, so the call can be repeated with a larger cap
    RlChangeOut O{nullptr, nullptr, nullptr, nullptr, nullptr, d_cnt.p};
    k_changes<<<blocks, threads, 0, v.stream>>>(T, O, 0);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    unsigned long long cnt = 0;
    RL_CUDA(e, cudaMemcpyAsync(&cnt, d_cnt.p, sizeof cnt, cudaMemcpyDeviceToHost, v.stream));
    RL_CUDA(e, cudaStreamSynchronize(v.stream));
    *out_count = cnt;
    if (cnt > cap) return RL_OK;
    // then emit, into the caller's device arrays or staging of exactly the count
    DevBuf<uint32_t> s_lid;
    DevBuf<uint64_t> s64[4];
    O = RlChangeOut{out_limit_id, out_key_lo, out_key_hi, out_value, out_expiry_us, d_cnt.p};
    if (mem == RL_MEM_HOST) {
        RL_CUDA(e, s_lid.alloc(cnt));
        for (auto& b : s64) RL_CUDA(e, b.alloc(cnt));
        O = RlChangeOut{s_lid.p, s64[0].p, s64[1].p, s64[2].p, s64[3].p, d_cnt.p};
    }
    RL_CUDA(e, cudaMemsetAsync(d_cnt.p, 0, sizeof(unsigned long long), v.stream));
    k_changes<<<blocks, threads, 0, v.stream>>>(T, O, 1);
    RL_CUDA(e, cudaGetLastError());
    rl_internal_launched(e, 1);
    if (mem == RL_MEM_HOST && cnt) {
        RL_CUDA(e, cudaMemcpyAsync(out_limit_id, s_lid.p, cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, v.stream));
        uint64_t* out64[4] = {out_key_lo, out_key_hi, out_value, out_expiry_us};
        for (int k = 0; k < 4; k++) RL_CUDA(e, cudaMemcpyAsync(out64[k], s64[k].p, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, v.stream));
    }
    RL_CUDA(e, cudaStreamSynchronize(v.stream));  // before the staging is freed
    return RL_OK;
}

}  // extern "C"
