// emu_maint.cpp — TEST-ONLY host driver of the maintenance, counter-import and CRDT kernels
// (limitador_b200/csrc/rl_maint.cuh, rl_crdt.cuh) under tests/emu/cuda_shim.h: the SAME kernel source the GPU runs, one
// CUDA thread after the other in a shuffled order.  Not shipped, not a fallback.  The launch geometry and the call
// sequences follow rl_maint.cu / rl_crdt.cu; the table helpers restate rl_kernels.cuh's rl_probe so that a rebuilt region is checked by the rule the
// hot path looks rows up with.
// Built twice: plain (cuda_shim.h: one thread after the other, the kernels' `#ifndef RL_SHIM` fast paths compiled out) and
// with -DEMU_SIMT (cuda_simt.h: the threads of a block as fibers, warp intrinsics as rendezvous — the DEVICE branches run).
#ifdef EMU_SIMT
#include "cuda_simt.h"
#define shim_launch simt_launch
static uint64_t shim_seed = 0;
#else
#include "cuda_shim.h"
#endif
// (the shim must come first: it defines __global__ & co. away)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../limitador_b200/csrc/rl_crdt.cuh"
#include "../../limitador_b200/csrc/rl_maint.cuh"

extern "C" {

void emu_seed(uint64_t s) { shim_seed = s; }
#ifdef EMU_SIMT
// cuda_simt.h's interleaving mode for the launches that follow (on = 0: off, the default)
void emu_simt_interleave(int on, uint64_t seed, double p) { simt_interleave(on != 0, seed, p); }
#endif

// ---- per-namespace metrics ------------------------------------------------------------------------------------------
// out = authorized_calls[ns_cap] | authorized_hits[ns_cap] | limited_calls[ns_cap] | limited_by_limit[limits_cap] | dropped
void emu_ns_metrics(const unsigned long long* recs, uint32_t rec_words, uint32_t n, const uint8_t* limited,
                    const uint32_t* first_limited, uint32_t ns_cap, uint32_t limits_cap, unsigned long long* out) {
    RlNsMetricsDev M;
    M.authorized_calls = out;
    M.authorized_hits = out + ns_cap;
    M.limited_calls = out + 2 * (size_t)ns_cap;
    M.limited_by_limit = out + 3 * (size_t)ns_cap;
    M.dropped = out + 3 * (size_t)ns_cap + limits_cap;
    M.ns_cap = ns_cap;
    M.limits_cap = limits_cap;
    const uint32_t threads = 256;
    const uint32_t blocks = std::min<uint32_t>((n + threads - 1) / threads, 7u);  // few blocks: the grid-stride loop gets trips
    if (n) shim_launch(blocks, threads, [&] { k_ns_metrics(recs, rec_words, n, limited, first_limited, M); });
}

// ---- the counter table, as the hot path lays it out ------------------------------------------------------------------
struct emu_table {
    std::vector<uint8_t> rows;
    uint32_t cells, log2P, log2R, row_bytes;
    uint64_t capacity;
};

emu_table* emu_table_create(uint32_t cells, uint32_t log2P, uint32_t log2R) {
    emu_table* t = new emu_table();
    t->cells = cells;
    t->log2P = log2P;
    t->log2R = log2R;
    t->row_bytes = 16 * (1 + cells);
    t->capacity = 1ull << (log2P + log2R);
    t->rows.assign(t->capacity * t->row_bytes, 0);
    return t;
}
void emu_table_destroy(emu_table* t) { delete t; }
uint8_t* emu_table_raw(emu_table* t) { return t->rows.data(); }
uint64_t emu_table_bytes(emu_table* t) { return t->rows.size(); }

// rl_probe (rl_kernels.cuh): home = low hash bits inside the region the high bits pick, linear probing, the first
// tombstone passed is reused on insert, an empty row ends the search.  Returns the row index or -1.
static int64_t table_probe(emu_table* t, uint64_t key_lo, uint64_t hdr_hi, bool create) {
    const uint64_t h = rl_row_hash(key_lo, hdr_hi);
    const uint64_t R = 1ull << t->log2R;
    const uint64_t base = (t->log2P ? (h >> (64 - t->log2P)) : 0ull) << t->log2R;
    const uint64_t idx = (uint32_t)h & (R - 1);
    int64_t tomb = -1;
    for (uint64_t i = 0; i < R; i++) {
        const uint64_t r = base + ((idx + i) & (R - 1));
        unsigned long long* hdr = reinterpret_cast<unsigned long long*>(t->rows.data() + r * t->row_bytes);
        if (hdr[0] == key_lo && hdr[1] == hdr_hi) return (int64_t)r;
        if (hdr[0] == 0 && hdr[1] == 0) {
            if (!create) return -1;
            const uint64_t target = tomb >= 0 ? (uint64_t)tomb : r;
            unsigned long long* th = reinterpret_cast<unsigned long long*>(t->rows.data() + target * t->row_bytes);
            th[0] = key_lo;
            th[1] = hdr_hi;
            return (int64_t)target;
        }
        if (hdr[1] == RLM_TOMB_HI && tomb < 0) tomb = (int64_t)r;
    }
    if (create && tomb >= 0) {
        unsigned long long* th = reinterpret_cast<unsigned long long*>(t->rows.data() + (uint64_t)tomb * t->row_bytes);
        th[0] = key_lo;
        th[1] = hdr_hi;
        return tomb;
    }
    return -1;
}

// cells: 2 words (value, expiry) per cell
int64_t emu_table_put(emu_table* t, uint64_t key_lo, uint64_t hdr_hi, const unsigned long long* cells) {
    const int64_t r = table_probe(t, key_lo, hdr_hi, true);
    if (r >= 0) memcpy(t->rows.data() + (uint64_t)r * t->row_bytes + 16, cells, 16 * t->cells);
    return r;
}
int64_t emu_table_get(emu_table* t, uint64_t key_lo, uint64_t hdr_hi, unsigned long long* cells) {
    const int64_t r = table_probe(t, key_lo, hdr_hi, false);
    if (r >= 0 && cells) memcpy(cells, t->rows.data() + (uint64_t)r * t->row_bytes + 16, 16 * t->cells);
    return r;
}
// what rl_sweep's k_reset does to a row whose last counter expired: cells cleared, header = tombstone
int64_t emu_table_tombstone(emu_table* t, uint64_t key_lo, uint64_t hdr_hi) {
    const int64_t r = table_probe(t, key_lo, hdr_hi, false);
    if (r < 0) return r;
    uint8_t* row = t->rows.data() + (uint64_t)r * t->row_bytes;
    memset(row, 0, t->row_bytes);
    reinterpret_cast<unsigned long long*>(row)[1] = RLM_TOMB_HI;
    return r;
}

// rl_compact (rl_maint.cu), same sequence.  stats: regions, regions_rebuilt, rows_live, rows_tombstoned, rows_moved,
// rows_reclaimed, failures.
void emu_table_compact(emu_table* t, uint32_t min_tombstone_pct, unsigned long long* stats, uint8_t* sel_out) {
    const uint32_t P = 1u << t->log2P;
    const uint64_t R = 1ull << t->log2R;
    std::vector<uint32_t> census(2 * (size_t)P, 0);
    const uint32_t threads = 256, blocks = (uint32_t)((t->capacity + threads - 1) / threads);
    shim_launch(blocks, threads, [&] { k_region_census(t->rows.data(), t->row_bytes, t->log2R, t->capacity, census.data(), census.data() + P); });
    std::vector<uint8_t> sel(P, 0);
    unsigned long long live = 0, tomb = 0, chosen = 0, tomb_chosen = 0;
    for (uint32_t g = 0; g < P; g++) {
        live += census[g];
        tomb += census[P + g];
        if (census[P + g] && (uint64_t)census[P + g] * 100 >= (uint64_t)min_tombstone_pct * R) {
            sel[g] = 1;
            chosen++;
            tomb_chosen += census[P + g];
        }
    }
    if (sel_out) memcpy(sel_out, sel.data(), P);
    unsigned long long counts[3] = {0, 0, 0};
    if (chosen) {
        std::vector<uint8_t> scratch(t->rows.size(), 0xAB);  // uninitialised on the device: poison it here
        shim_launch(blocks, threads, [&] { k_compact_move(t->rows.data(), scratch.data(), t->row_bytes, t->log2R, t->capacity, sel.data()); });
        shim_launch(blocks, threads, [&] {
            k_compact_reinsert(t->rows.data(), scratch.data(), t->row_bytes, t->log2P, t->log2R, t->capacity, sel.data(), counts);
        });
    }
    stats[0] = P;
    stats[1] = chosen;
    stats[2] = live;
    stats[3] = tomb;
    stats[4] = counts[0];
    stats[5] = chosen ? tomb_chosen + counts[1] : 0;
    stats[6] = counts[2];
}

// rl_counters_import (rl_maint.cu), same launch geometry and pass sequence.  rows: the table (capacity =
// 2^(log2P + log2R) rows of 16 * (1 + cells) bytes), changed in place; limits: RlLimitDev[limits_cap].  Returns the
// error word ((index << 8) | reason, ~0 = imported); unq_out[limits_cap] = the unqualified limits the call makes present.
unsigned long long emu_import(uint8_t* rows, uint32_t cells, uint32_t log2P, uint32_t log2R, const RlLimitDev* limits,
                              uint32_t limits_cap, uint64_t n, const uint32_t* limit_id, const uint64_t* key_lo,
                              const uint64_t* key_hi, const uint64_t* value, const uint64_t* expiry_us,
                              uint8_t* unq_out) {
    const RlImportTab T{rows, 16u * (1 + cells), log2P, log2R, limits, limits_cap};
    const RlImportIn I{limit_id, key_lo, key_hi, value, expiry_us, n};
    const uint64_t capacity = 1ull << (log2P + log2R);
    unsigned long long err = ~0ull;
    std::vector<uint8_t> unq(limits_cap, 0);
    const uint32_t threads = 256, blocks = (uint32_t)((n + threads - 1) / threads);
    if (n == 0) return err;
    shim_launch(blocks, threads, [&] { k_import_resolve(T, I, &err, unq.data()); });
    if (err != ~0ull) return err;
    std::vector<unsigned long long> row_of(n, 0);
    std::vector<unsigned> mask(capacity, 0);
    shim_launch(blocks, threads, [&] { k_import_claim(T, I, row_of.data(), mask.data(), &err); });
    if (err != ~0ull) {
        shim_launch(blocks, threads, [&] { k_import_release(T, n, row_of.data()); });
        return err;
    }
    shim_launch(blocks, threads, [&] { k_import_write(T, I, row_of.data()); });
    for (uint32_t l = 0; l < limits_cap; l++) unq_out[l] = unq[l];
    return err;
}

// ---- the replicated counter value ------------------------------------------------------------------------------------
struct emu_crdt {
    std::vector<uint8_t> rows;
    uint32_t err = 0;
    RlCrdtTab T;
};

emu_crdt* emu_crdt_create(uint64_t capacity_rows, uint32_t actors, uint32_t self_actor) {
    emu_crdt* c = new emu_crdt();
    uint64_t cap = 1;
    while (cap < capacity_rows) cap <<= 1;
    c->T.actors = actors;
    c->T.actors_pad = (actors + 1u) & ~1u;
    c->T.self_actor = self_actor;
    c->T.row_bytes = 32 + 8 * c->T.actors_pad;
    c->T.mask = cap - 1;
    c->rows.assign(cap * c->T.row_bytes, 0);
    c->T.rows = c->rows.data();
    c->T.err = &c->err;
    return c;
}
void emu_crdt_destroy(emu_crdt* c) { delete c; }

static uint32_t take_err(emu_crdt* c) {
    const uint32_t e = c->err;
    c->err = 0;
    return e;
}
static uint32_t blocks_for(uint64_t n) { return (uint32_t)((n + 255) / 256); }

uint32_t emu_crdt_inc(emu_crdt* c, uint32_t n, const rl_crdt_key* keys, const uint32_t* actor, const uint64_t* inc,
                      const uint64_t* window_us, uint64_t now) {
    if (n) shim_launch(blocks_for(n), 256, [&] { k_crdt_inc(c->T, n, keys, actor, inc, window_us, now); });
    return take_err(c);
}
uint32_t emu_crdt_merge(emu_crdt* c, uint32_t n, const rl_crdt_update* ups, const uint32_t* actors, const uint64_t* values,
                        uint64_t n_values, uint64_t now) {
    if (!n) return 0;
    std::vector<unsigned long long> row_of(n, 0x5555555555555555ull);
    shim_launch(blocks_for(n), 256, [&] { k_crdt_merge_expiry(c->T, n, ups, now, row_of.data()); });
    shim_launch(blocks_for(n), 256, [&] { k_crdt_merge_values(c->T, n, ups, actors, values, n_values, row_of.data()); });
    return take_err(c);
}
uint32_t emu_crdt_read(emu_crdt* c, uint32_t n, const rl_crdt_key* keys, uint64_t now, uint64_t* out_value, uint64_t* out_expiry) {
    if (n) shim_launch(blocks_for(n), 256, [&] { k_crdt_read(c->T, n, keys, now, out_value, out_expiry); });
    return take_err(c);
}
// mode 0 export, 1 dump; returns the count
uint64_t emu_crdt_scan(emu_crdt* c, int mode, uint64_t now, uint64_t cap, rl_crdt_key* out_keys, uint64_t* out_a,
                       uint64_t* out_expiry, uint64_t* out_values) {
    unsigned long long count = 0;
    shim_launch(blocks_for(c->T.mask + 1), 256, [&] { k_crdt_scan(c->T, mode, now, cap, out_keys, out_a, out_expiry, out_values, &count); });
    return count;
}

}  // extern "C"
