// rl_maint.cuh — maintenance kernels beside the hot path (SURVEY.md §8 f3 and VERDICT r1 item 10):
//   k_ns_metrics        per-namespace authorized_calls / authorized_hits / limited_calls of a decided batch as ONE
//                       segmented reduction (limitador-server/src/prometheus_metrics.rs:93-125 increments them
//                       once per request on the host, after the decision: envoy_rls/server.rs:183-195)
//   k_region_census     live rows and tombstones per table region
//   k_compact_move /    tombstone reclamation: a region whose probe chains are lengthened by tombstones (rl_sweep
//   k_compact_reinsert  leaves them) is rebuilt in place — its rows go to a scratch slab, the region is cleared, the
//                       rows that still hold a counter are inserted again by the rule the hot path probes by
//                       (rl_kernels.cuh rl_probe: home = low hash bits, linear probing inside the region, 128-bit
//                       CAS on the header).  No reference analog (moka evicts, in_memory.rs:205-212); observable
//                       state is unchanged: what rl_counters_export(..., now_us = 0) lists before == after.
//   k_import_resolve /  counter import (rl_counters_import): set counters to exported (value, expiry) pairs in three
//   k_import_claim /    passes — check every entry, find or claim every row by rl_probe's rule, then write the cells —
//   k_import_write      so that a refused call has written no cell (DESIGN.md §9f).
//
// Written so that the SAME source runs under tests/emu/cuda_shim.h (one CUDA thread after the other on the host):
// grid-stride / one-item-per-thread kernels, global atomics only; warp-aggregated fast paths sit inside
// `#ifndef RL_SHIM` and produce the same sums.
#pragma once
#include <stdint.h>

#include "rl_core.h"
#include "rl_devmem.cuh"

// ---------------------------------------------------------------------------------------------------------------------
// Per-namespace metrics.
struct RlNsMetricsDev {
    unsigned long long* authorized_calls;  // [ns_cap]   requests allowed
    unsigned long long* authorized_hits;   // [ns_cap]   sum of their hits_addend
    unsigned long long* limited_calls;     // [ns_cap]   requests limited
    unsigned long long* limited_by_limit;  // [limits_cap] limited requests by the limit named (limit_name label), nullable
    unsigned long long* dropped;           // [1] requests not counted: error verdict, or a namespace id out of range
    uint32_t ns_cap, limits_cap;
};

// rec_words = 4: 32-byte rl_record (word 0 = ns_id | hits_addend << 32); 2: 16-byte rl_record16 (word 0 = ns_id:24 |
// hits:8 | key_hi:32).  One request per thread and loop trip; every lane of a warp makes the same number of trips.
__global__ void k_ns_metrics(const unsigned long long* __restrict__ recs, uint32_t rec_words, uint32_t n,
                             const uint8_t* __restrict__ limited, const uint32_t* __restrict__ first_limited,
                             RlNsMetricsDev M) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t n_up = ((uint64_t)n + 31u) & ~31ull;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += stride) {
        bool valid = i < n;
        uint32_t ns = 0, hits = 0, v = 0, fl = RL_NONE_U32;
        if (valid) {
            const unsigned long long w0 = recs[i * rec_words];
            if (rec_words == 4) {
                ns = (uint32_t)w0;
                hits = (uint32_t)(w0 >> 32);
            } else {
                ns = (uint32_t)w0 & 0x00FFFFFFu;
                hits = (uint32_t)(w0 >> 24) & 0xFFu;
            }
            v = limited[i];
            if (v == 0xFFu || ns >= M.ns_cap) {  // RL_VERDICT_ERROR: the request was not decided
                valid = false;
                atomicAdd(M.dropped, 1ull);
            } else if (v && first_limited) {
                fl = first_limited[i];
            }
        }
#ifndef RL_SHIM
        // warp-aggregated: the lanes that hold the same (namespace, verdict) add once
        const unsigned lane = threadIdx.x & 31u;
        const unsigned key = valid ? ((ns << 1) | (v ? 1u : 0u)) : 0xFFFFFFFFu;
        const unsigned grp = __match_any_sync(0xFFFFFFFFu, key);
        const unsigned lo = __reduce_add_sync(grp, hits & 0xFFFFu), hi = __reduce_add_sync(grp, hits >> 16);
        if (valid && (unsigned)(__ffs(grp) - 1) == lane) {
            const unsigned long long cnt = (unsigned long long)__popc(grp);
            if (v) {
                atomicAdd(&M.limited_calls[ns], cnt);
            } else {
                atomicAdd(&M.authorized_calls[ns], cnt);
                atomicAdd(&M.authorized_hits[ns], (unsigned long long)lo + ((unsigned long long)hi << 16));
            }
        }
        if (M.limited_by_limit) {
            const bool named = valid && v && fl < M.limits_cap;
            const unsigned g2 = __match_any_sync(0xFFFFFFFFu, named ? fl : 0xFFFFFFFFu);
            if (named && (unsigned)(__ffs(g2) - 1) == lane) atomicAdd(&M.limited_by_limit[fl], (unsigned long long)__popc(g2));
        }
#else
        if (valid) {
            if (v) {
                atomicAdd(&M.limited_calls[ns], 1ull);
                if (M.limited_by_limit && fl < M.limits_cap) atomicAdd(&M.limited_by_limit[fl], 1ull);
            } else {
                atomicAdd(&M.authorized_calls[ns], 1ull);
                atomicAdd(&M.authorized_hits[ns], (unsigned long long)hits);
            }
        }
#endif
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Tombstone reclamation.
#define RLM_TOMB_HI 0xFFFFFFFFFFFFFFFFull

// live[g] / tomb[g] += rows of region g that hold a key / a tombstone.  One row per thread; threads past the table
// keep going to the warp-wide step.
__global__ void k_region_census(const uint8_t* __restrict__ rows, uint32_t row_bytes, uint32_t log2R, uint64_t nrows,
                                uint32_t* live, uint32_t* tomb) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = r < nrows;
    bool is_tomb = false, is_live = false;
    uint32_t region = 0;
    if (in) {
        const ulonglong2 hdr = rlm_ld(rows + r * row_bytes);
        is_tomb = hdr.y == RLM_TOMB_HI;
        is_live = !is_tomb && hdr.y != 0;
        region = (uint32_t)(r >> log2R);
    }
#ifndef RL_SHIM
    const unsigned lane = threadIdx.x & 31u;
    const unsigned grp = __match_any_sync(0xFFFFFFFFu, in ? region : 0xFFFFFFFFu);
    const unsigned t = __popc(__ballot_sync(0xFFFFFFFFu, is_tomb) & grp), l = __popc(__ballot_sync(0xFFFFFFFFu, is_live) & grp);
    if (in && (unsigned)(__ffs(grp) - 1) == lane) {
        if (t) atomicAdd(&tomb[region], t);
        if (l) atomicAdd(&live[region], l);
    }
#else
    if (is_tomb) atomicAdd(&tomb[region], 1u);
    if (is_live) atomicAdd(&live[region], 1u);
#endif
}

// Rows of the selected regions -> scratch (same row index), region cleared.
__global__ void k_compact_move(uint8_t* rows, uint8_t* scratch, uint32_t row_bytes, uint32_t log2R, uint64_t nrows,
                               const uint8_t* __restrict__ sel) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows || !sel[r >> log2R]) return;
    uint8_t* src = rows + r * row_bytes;
    uint8_t* dst = scratch + r * row_bytes;
    for (uint32_t q = 0; q < row_bytes; q += 16) {
        const ulonglong2 v = rlm_ld(src + q);
        rlm_st(dst + q, v.x, v.y);
        rlm_st(src + q, 0ull, 0ull);
    }
}

// counts[0] rows inserted again, [1] rows dropped because every cell was (0, 0) (they hold no counter: a qualified
// cell with expiry 0 is absent, an unqualified (0, EPOCH) is the default the next access recreates), [2] failures.
__global__ void k_compact_reinsert(uint8_t* rows, const uint8_t* __restrict__ scratch, uint32_t row_bytes, uint32_t log2P,
                                   uint32_t log2R, uint64_t nrows, const uint8_t* __restrict__ sel,
                                   unsigned long long* counts) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows || !sel[r >> log2R]) return;
    const uint8_t* src = scratch + r * row_bytes;
    const ulonglong2 hdr = rlm_ld(src);
    if (hdr.y == 0 || hdr.y == RLM_TOMB_HI) return;
    bool any = false;
    for (uint32_t q = 16; q < row_bytes; q += 16) {
        const ulonglong2 c = rlm_ld(src + q);
        any = any || c.x != 0 || c.y != 0;
    }
    if (!any) {
        atomicAdd(&counts[1], 1ull);
        return;
    }
    const uint64_t h = rl_row_hash(hdr.x, hdr.y);
    const uint64_t region = log2P ? (h >> (64 - log2P)) : 0ull;
    const uint32_t R = 1u << log2R;
    const uint64_t base = region << log2R;
    const uint32_t idx = (uint32_t)h & (R - 1);
    if (region != (r >> log2R)) {  // the row was not where its hash puts it: never rebuilt wrongly, reported
        atomicAdd(&counts[2], 1ull);
        return;
    }
    for (uint32_t i = 0; i < R; i++) {
        uint8_t* dst = rows + (base + ((idx + i) & (R - 1))) * row_bytes;
        const ulonglong2 cur = rlm_ld(dst);
        if (cur.x != 0 || cur.y != 0) continue;  // taken by another row of the region (keys are distinct)
        const ulonglong2 old = rlm_cas128(dst, make_ulonglong2(0ull, 0ull), hdr);
        if (old.x != 0 || old.y != 0) continue;  // lost the race for this slot: the next one
        for (uint32_t q = 16; q < row_bytes; q += 16) {
            const ulonglong2 c = rlm_ld(src + q);
            rlm_st(dst + q, c.x, c.y);
        }
        atomicAdd(&counts[0], 1ull);
        return;
    }
    atomicAdd(&counts[2], 1ull);  // cannot happen: the region held this row before
}

// ---------------------------------------------------------------------------------------------------------------------
// Counter import.  The entries are the five arrays rl_counters_export returns; every error is one word,
// (index << 8) | reason, lowered with atomicMin so that the host learns the first bad index (~0 = no error).
enum : uint32_t {
    RLM_IMP_UNKNOWN_LIMIT = 1,  // limit id not registered in this engine
    RLM_IMP_KEY_RANGE = 2,      // qualified counter with key_hi >= 2^32
    RLM_IMP_NO_EXPIRY = 3,      // qualified counter with expiry 0 (that is an absent counter)
    RLM_IMP_DUPLICATE = 4,      // the same counter twice in one call
    RLM_IMP_TABLE_FULL = 5,     // the row's region has no free row
};

struct RlImportIn {
    const uint32_t* limit_id;
    const uint64_t* key_lo;
    const uint64_t* key_hi;
    const uint64_t* value;
    const uint64_t* expiry;
    uint64_t n;
};

struct RlImportTab {
    uint8_t* rows;
    uint32_t row_bytes, log2P, log2R;
    const RlLimitDev* limits;  // [limits_cap], group 0 = not registered
    uint32_t limits_cap;
};

// Entry i -> row header (key_lo, hdr_hi = group << 32 | key_hi; key 0 for unqualified limits) and cell, or a reason.
__device__ __forceinline__ uint32_t rlm_import_entry(const RlImportTab& T, const RlImportIn& I, uint64_t i, uint64_t& klo,
                                                     uint64_t& hhi, uint32_t& cell, bool& qualified) {
    const uint32_t lid = I.limit_id[i];
    if (lid >= T.limits_cap) return RLM_IMP_UNKNOWN_LIMIT;
    const RlLimitDev l = T.limits[lid];
    if (l.group == 0) return RLM_IMP_UNKNOWN_LIMIT;
    qualified = l.qualified != 0;
    cell = l.cell;
    klo = 0;
    hhi = (uint64_t)l.group << 32;
    if (qualified) {
        const uint64_t khi = I.key_hi[i];
        if (khi >> 32) return RLM_IMP_KEY_RANGE;
        if (I.expiry[i] == 0) return RLM_IMP_NO_EXPIRY;
        klo = I.key_lo[i];
        hhi |= khi;
    }
    return 0;
}

// Pass 1: check every entry; unq[limit] = 1 for the unqualified limits named (they become present on success).
__global__ void k_import_resolve(RlImportTab T, RlImportIn I, unsigned long long* err, uint8_t* unq) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= I.n) return;
    uint64_t klo, hhi;
    uint32_t cell;
    bool q = false;
    const uint32_t why = rlm_import_entry(T, I, i, klo, hhi, cell, q);
    if (why) {
        atomicMin(err, ((unsigned long long)i << 8) | why);
        return;
    }
    if (!q) unq[I.limit_id[i]] = 1;
}

// row_of[] words: the row index, plus whether this call claimed the row and what the row was before
#define RLM_ROW_CLAIMED (1ull << 63)
#define RLM_ROW_WAS_TOMB (1ull << 62)
#define RLM_ROW_INDEX(w) ((w) & ((1ull << 62) - 1))
#define RLM_ROW_NONE 0xFFFFFFFFFFFFFFFFull  // the region is full

// rl_probe (rl_kernels.cuh) with create: linear probing inside the key's region from its home row, the first tombstone
// passed is reused once the key is known to be absent, rows are claimed with a 128-bit CAS on the header.
__device__ __forceinline__ uint64_t rlm_claim_row(const RlImportTab& T, uint64_t h, uint64_t klo, uint64_t hhi) {
    const uint32_t R = 1u << T.log2R;
    const uint64_t base = (T.log2P ? (h >> (64 - T.log2P)) : 0ull) << T.log2R;
    const uint32_t idx = (uint32_t)h & (R - 1);
    int64_t tomb = -1;
    uint32_t restarts = 0;
    for (uint32_t i = 0; i < R;) {
        const uint64_t r = base + ((idx + i) & (R - 1));
        const ulonglong2 cur = rlm_ld(T.rows + r * T.row_bytes);
        if (cur.x == klo && cur.y == hhi) return r;
        if (cur.x == 0 && cur.y == 0) {
            const uint64_t target = tomb >= 0 ? (uint64_t)tomb : r;
            const ulonglong2 expect = make_ulonglong2(0ull, tomb >= 0 ? RLM_TOMB_HI : 0ull);
            const ulonglong2 old = rlm_cas128(T.rows + target * T.row_bytes, expect, make_ulonglong2(klo, hhi));
            if (old.x == expect.x && old.y == expect.y) return target | RLM_ROW_CLAIMED | (tomb >= 0 ? RLM_ROW_WAS_TOMB : 0ull);
            if (++restarts > 4 * R) break;  // another thread took the row first: rescan
            tomb = -1;
            i = 0;
            continue;
        }
        if (cur.y == RLM_TOMB_HI && tomb < 0) tomb = (int64_t)r;
        i++;
    }
    if (tomb >= 0) {
        const ulonglong2 old = rlm_cas128(T.rows + (uint64_t)tomb * T.row_bytes, make_ulonglong2(0ull, RLM_TOMB_HI),
                                          make_ulonglong2(klo, hhi));
        if (old.x == 0 && old.y == RLM_TOMB_HI) return (uint64_t)tomb | RLM_ROW_CLAIMED | RLM_ROW_WAS_TOMB;
        if (old.x == klo && old.y == hhi) return (uint64_t)tomb;
    }
    return RLM_ROW_NONE;
}

// Pass 2: find or claim every entry's row (row_of[i], zeroed for the call) and mark its cell in cellmask[row] (zeroed
// too); a cell marked twice is a duplicate.  Claimed rows keep the cells they had (all zero) until pass 3, which runs
// only if this pass reported nothing.  Device path: the lanes of a warp that name the same row probe once.
__global__ void k_import_claim(RlImportTab T, RlImportIn I, unsigned long long* row_of, unsigned* cellmask,
                               unsigned long long* err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t klo = 0, hhi = 0;
    uint32_t cell = 0;
    bool q = false;
    const bool valid = i < I.n && rlm_import_entry(T, I, i, klo, hhi, cell, q) == 0;
    uint64_t row = RLM_ROW_NONE;
#ifndef RL_SHIM
    // every lane of the warp reaches this point (blockDim is a multiple of 32, no thread returned)
    const unsigned lane = threadIdx.x & 31u;
    const unsigned vmask = __ballot_sync(0xFFFFFFFFu, valid);
    const unsigned grp = __match_any_sync(0xFFFFFFFFu, klo) & __match_any_sync(0xFFFFFFFFu, hhi) & (valid ? vmask : ~vmask);
    const unsigned leader = (unsigned)(__ffs(grp) - 1);
    if (valid && lane == leader) row = rlm_claim_row(T, rl_row_hash(klo, hhi), klo, hhi);
    const unsigned r_lo = __shfl_sync(0xFFFFFFFFu, (unsigned)(row & 0xFFFFFFFFull), (int)leader);
    const unsigned r_hi = __shfl_sync(0xFFFFFFFFu, (unsigned)(row >> 32), (int)leader);
    row = ((uint64_t)r_hi << 32) | r_lo;
    if (lane != leader && row != RLM_ROW_NONE) row &= ~(RLM_ROW_CLAIMED | RLM_ROW_WAS_TOMB);  // the leader claimed it
#else
    if (valid) row = rlm_claim_row(T, rl_row_hash(klo, hhi), klo, hhi);
#endif
    if (!valid) return;
    if (row == RLM_ROW_NONE) {
        atomicMin(err, ((unsigned long long)i << 8) | RLM_IMP_TABLE_FULL);
        return;
    }
    row_of[i] = row;
    const unsigned old = rlm_or(&cellmask[RLM_ROW_INDEX(row)], 1u << cell);
    if (old >> cell & 1u) atomicMin(err, ((unsigned long long)i << 8) | RLM_IMP_DUPLICATE);
}

// After a refused pass 2: every row the call claimed gets its old header back (empty or tombstone; its cells were never
// written).  A row that was empty before the call lies on no older key's probe chain, so the table is as it was.
__global__ void k_import_release(RlImportTab T, uint64_t n, const unsigned long long* __restrict__ row_of) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !(row_of[i] & RLM_ROW_CLAIMED)) return;
    rlm_st(T.rows + RLM_ROW_INDEX(row_of[i]) * T.row_bytes, 0ull, (row_of[i] & RLM_ROW_WAS_TOMB) ? RLM_TOMB_HI : 0ull);
}

// Pass 3: (value, expiry) into every entry's cell.
__global__ void k_import_write(RlImportTab T, RlImportIn I, const unsigned long long* __restrict__ row_of) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= I.n) return;
    const uint32_t cell = T.limits[I.limit_id[i]].cell;
    rlm_st(T.rows + RLM_ROW_INDEX(row_of[i]) * T.row_bytes + 16 + 16 * cell, I.value[i], I.expiry[i]);
}

// ---------------------------------------------------------------------------------------------------------------------
// Change tracking (rl_counters_drain): the table against its shadow, a copy taken at the previous drain.  Between two
// calls that move rows or re-map cells only the decision calls and rl_sweep change the table, and neither moves a row,
// so row r of the shadow and row r of the table are read with the same (row group, cell) -> limit mapping.
struct RlChangeTab {
    const uint8_t* rows;
    uint8_t* shadow;             // [nrows * row_bytes]
    uint32_t row_bytes, cells;
    uint64_t nrows;
    const RlCellDesc* desc;      // [row groups][8]
    const uint8_t* present;      // [limits] 1 = the limit's counters exist (rl_counters_export's rule)
};

struct RlChangeOut {
    uint32_t* limit_id;
    uint64_t* key_lo;
    uint64_t* key_hi;
    uint64_t* value;
    uint64_t* expiry;
    unsigned long long* count;
};

// The cells of a row that rl_counters_export(now_us = 0) lists, as a bit mask; cell[c] = (value, expiry) of cell c.
__device__ __forceinline__ uint32_t rlm_listed(const RlChangeTab& T, const uint8_t* row, ulonglong2& hdr, ulonglong2* cell) {
    hdr = rlm_ld(row);
    if (hdr.y == 0 || hdr.y == RLM_TOMB_HI) return 0;
    const RlCellDesc* d = T.desc + (size_t)(hdr.y >> 32) * 8;
    uint32_t m = 0;
    for (uint32_t c = 0; c < T.cells; c++) {
        cell[c] = rlm_ld(row + 16 + 16 * c);
        const uint32_t lid = d[c].limit_id;
        if (lid == RL_NONE_U32 || !T.present[lid]) continue;
        if (d[c].qualified && cell[c].y == 0) continue;  // logically absent
        m |= 1u << c;
    }
    return m;
}

// One thread per row.  A row whose bytes equal the shadow's is skipped.  Otherwise the counters it lists now and
// listed then are compared: the same key in both keeps the cells whose (value, expiry) moved, and a listed cell that
// is gone is absent, (limit, key, 0, 0).  A row that holds another key than its shadow (empty, tombstone, key A then
// key B) lists every old counter as absent and every new one as present: a journal applies a drain's absents before
// its presents.  emit = 0: *O.count += the entries.  emit = 1: the entries are written at reserved positions (the
// count pass found them to fit) and the row is copied into the shadow.
__global__ void k_changes(RlChangeTab T, RlChangeOut O, int emit) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.nrows) return;
    const uint8_t* row = T.rows + r * T.row_bytes;
    uint8_t* old = T.shadow + r * T.row_bytes;
    bool same = true;
    for (uint32_t q = 0; q < T.row_bytes && same; q += 16) {
        const ulonglong2 a = rlm_ld(row + q), b = rlm_ld(old + q);
        same = a.x == b.x && a.y == b.y;
    }
    if (same) return;
    ulonglong2 hn, ho, cn[RL_MAX_CELLS], co[RL_MAX_CELLS];
    const uint32_t mn = rlm_listed(T, row, hn, cn), mo = rlm_listed(T, old, ho, co);
    const bool same_key = mn && mo && hn.x == ho.x && hn.y == ho.y;
    const RlCellDesc* dn = mn ? T.desc + (size_t)(hn.y >> 32) * 8 : T.desc;
    const RlCellDesc* d_o = mo ? T.desc + (size_t)(ho.y >> 32) * 8 : T.desc;
    uint32_t gone = 0, now = 0;  // cells emitted as absent (old key) / as present (new key)
    if (same_key) {
        for (uint32_t c = 0; c < T.cells; c++) {
            if (mn >> c & 1u) {
                if (!(mo >> c & 1u) || cn[c].x != co[c].x || cn[c].y != co[c].y) now |= 1u << c;
            } else if (mo >> c & 1u) {
                gone |= 1u << c;
            }
        }
    } else {
        gone = mo;
        now = mn;
    }
    uint32_t n = 0;
    for (uint32_t c = 0; c < T.cells; c++) n += (gone >> c & 1u) + (now >> c & 1u);
    if (!emit) {
        if (n) atomicAdd(O.count, (unsigned long long)n);
        return;
    }
    if (n) {
        unsigned long long pos = atomicAdd(O.count, (unsigned long long)n);
        for (uint32_t c = 0; c < T.cells; c++) {
            if (!(gone >> c & 1u)) continue;
            O.limit_id[pos] = d_o[c].limit_id;
            O.key_lo[pos] = ho.x;
            O.key_hi[pos] = ho.y & 0xFFFFFFFFull;
            O.value[pos] = 0;
            O.expiry[pos] = 0;
            pos++;
        }
        for (uint32_t c = 0; c < T.cells; c++) {
            if (!(now >> c & 1u)) continue;
            O.limit_id[pos] = dn[c].limit_id;
            O.key_lo[pos] = hn.x;
            O.key_hi[pos] = hn.y & 0xFFFFFFFFull;
            O.value[pos] = cn[c].x;
            O.expiry[pos] = cn[c].y;
            pos++;
        }
    }
    for (uint32_t q = 0; q < T.row_bytes; q += 16) {
        const ulonglong2 a = rlm_ld(row + q);
        rlm_st(old + q, a.x, a.y);
    }
}
