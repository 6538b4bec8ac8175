// rl_crdt.cuh — kernels of the replicated counter value (include/rl_crdt.h; SURVEY.md §8 f4).
//
// Reference semantics restated (paths relative to limitador/src/storage/ of the reference repository):
//   distributed/cr_counter_value.rs:38-46   read_at
//   distributed/cr_counter_value.rs:54-75   inc_at / inc_actor_at
//   distributed/cr_counter_value.rs:81-115  merge_at (+ :142-147 reset)
//   atomic_expiring_value.rs:76-99          expired_at (inclusive), update_if_expired (CAS; only the winner stores)
//   atomic_expiring_value.rs:113-130        AtomicExpiryTime::merge_at (the earlier unexpired expiry wins)
//
// Row = | key_lo key_hi | expiry_us pad | value[actor 0] ... value[actors_pad-1] |, 32 + 8 * actors_pad bytes; the table is
// open-addressed with linear probing, rows are claimed with a 128-bit CAS on the key and never removed.  The same
// source runs under tests/emu/cuda_shim.h (see rl_maint.cuh): one item per thread, global atomics only.
#pragma once
#include <stdint.h>

#include "../../include/rl_crdt.h"
#include "rl_core.h"
#include "rl_devmem.cuh"

struct RlCrdtTab {
    uint8_t* rows;
    uint64_t mask;        // capacity - 1 (capacity = 2^k rows)
    uint32_t row_bytes;   // 32 + 8 * actors_pad
    uint32_t actors, actors_pad, self_actor;
    uint32_t* err;        // sticky max: 1 table full, 2 actor out of range, 3 bad key, 4 value index out of range
};

// Find the row of key (lo, hi); with create, claim an empty one for it.  nullptr = absent (or the table is full).
__device__ __forceinline__ uint8_t* rl_crdt_row(const RlCrdtTab& T, uint64_t lo, uint64_t hi, bool create) {
    const uint64_t h = rl_row_hash(lo, hi);
    for (uint64_t i = 0; i <= T.mask; i++) {
        uint8_t* row = T.rows + ((h + i) & T.mask) * T.row_bytes;
        const ulonglong2 hdr = rlm_ld(row);
        if (hdr.x == lo && hdr.y == hi) return row;
        if (hdr.x == 0 && hdr.y == 0) {
            if (!create) return nullptr;
            const ulonglong2 old = rlm_cas128(row, make_ulonglong2(0ull, 0ull), make_ulonglong2(lo, hi));
            if ((old.x == 0 && old.y == 0) || (old.x == lo && old.y == hi)) return row;
            // another key took the slot first: keep probing
        }
    }
    return nullptr;
}
__device__ __forceinline__ bool rl_crdt_key_ok(uint64_t lo, uint64_t hi) { return (lo != 0 || hi != 0) && hi != 0xFFFFFFFFFFFFFFFFull; }
__device__ __forceinline__ unsigned long long* rl_crdt_expiry(uint8_t* row) { return reinterpret_cast<unsigned long long*>(row + 16); }
__device__ __forceinline__ unsigned long long* rl_crdt_values(uint8_t* row) { return reinterpret_cast<unsigned long long*>(row + 32); }

// inc_actor_at (cr_counter_value.rs:66-75; :54-60 for ourselves — the same rule on our own slot)
__global__ void k_crdt_inc(RlCrdtTab T, uint32_t n, const rl_crdt_key* __restrict__ keys, const uint32_t* __restrict__ actor,
                           const uint64_t* __restrict__ increment, const uint64_t* __restrict__ window_us, uint64_t now) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t a = actor[i];
    if (a >= T.actors) {
        atomicMax(T.err, 2u);
        return;
    }
    if (!rl_crdt_key_ok(keys[i].lo, keys[i].hi)) {
        atomicMax(T.err, 3u);
        return;
    }
    uint8_t* row = rl_crdt_row(T, keys[i].lo, keys[i].hi, true);
    if (!row) {
        atomicMax(T.err, 1u);
        return;
    }
    unsigned long long* exp = rl_crdt_expiry(row);
    unsigned long long* val = rl_crdt_values(row) + a;
    const unsigned long long cur = rlm_ld64(exp);
    if (cur <= now) {  // expired_at is inclusive; a fresh row (expiry 0) starts its first window here
        // update_if_expired: only the thread whose CAS moves the expiry stores, the others add (:55-59, :70-74).  The
        // store is an add of (increment - the stale value read before the CAS): the other threads of this call that
        // target the slot add only after they have seen the CAS, and an exchange landing after their adds would erase
        // them.  The fence keeps the stale read before the CAS for every observer.
        const unsigned long long stale = rlm_ld64(val);
        rlm_fence();
        if (atomicCAS(exp, cur, (unsigned long long)(now + window_us[i])) == cur) {
            atomicAdd(val, (unsigned long long)increment[i] - stale);
            return;
        }
    }
    atomicAdd(val, (unsigned long long)increment[i]);
}

// merge_at, first half (:83-88): expiry.  row_of[i] = the update's row index, or ~0 for an update that is ignored
// because it has already expired (:83).  A locally expired (or new) row is reset to the remote window: expiry = theirs,
// every value 0 (:85-87, :142-147); otherwise the earlier of the two expiries is kept (atomic_expiring_value.rs:116).
__global__ void k_crdt_merge_expiry(RlCrdtTab T, uint32_t n, const rl_crdt_update* __restrict__ ups, uint64_t now,
                                    unsigned long long* row_of) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    row_of[i] = ~0ull;
    const rl_crdt_update u = ups[i];
    if (u.expires_at_us <= now) return;
    if (!rl_crdt_key_ok(u.key_lo, u.key_hi)) {
        atomicMax(T.err, 3u);
        return;
    }
    uint8_t* row = rl_crdt_row(T, u.key_lo, u.key_hi, true);
    if (!row) {
        atomicMax(T.err, 1u);
        return;
    }
    unsigned long long* exp = rl_crdt_expiry(row);
    const unsigned long long e = u.expires_at_us;
    unsigned long long cur = rlm_ld64(exp);
    for (;;) {
        if (cur <= now) {
            const unsigned long long old = atomicCAS(exp, cur, e);
            if (old == cur) {  // we reset the row: nobody merges values before the second kernel
                unsigned long long* val = rl_crdt_values(row);
                for (uint32_t a = 0; a < T.actors_pad; a++) atomicExch(val + a, 0ull);
                break;
            }
            cur = old;
        } else if (e < cur) {
            const unsigned long long old = atomicCAS(exp, cur, e);
            if (old == cur) break;
            cur = old;
        } else {
            break;
        }
    }
    row_of[i] = (unsigned long long)((row - T.rows) / T.row_bytes);
}

// merge_at, second half (:89-113): every actor keeps the larger value (ours: `if other > ours: fetch_add(other - ours)`;
// the others: insert if vacant and non-zero, else max — all of them a maximum over a slot that starts at 0)
__global__ void k_crdt_merge_values(RlCrdtTab T, uint32_t n, const rl_crdt_update* __restrict__ ups,
                                    const uint32_t* __restrict__ actors, const uint64_t* __restrict__ values, uint64_t n_values,
                                    const unsigned long long* __restrict__ row_of) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long r = row_of[i];
    if (r == ~0ull) return;
    const rl_crdt_update u = ups[i];
    unsigned long long* val = rl_crdt_values(T.rows + r * T.row_bytes);
    for (uint32_t j = 0; j < u.n_vals; j++) {
        const uint64_t idx = (uint64_t)u.val_off + j;
        if (idx >= n_values) {
            atomicMax(T.err, 4u);
            return;
        }
        const uint32_t a = actors[idx];
        if (a >= T.actors) {
            atomicMax(T.err, 2u);
            continue;
        }
        atomicMax(val + a, (unsigned long long)values[idx]);
    }
}

// read_at (:38-46)
__global__ void k_crdt_read(RlCrdtTab T, uint32_t n, const rl_crdt_key* __restrict__ keys, uint64_t now, uint64_t* out_value,
                            uint64_t* out_expiry) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t sum = 0, e = 0;
    uint8_t* row = rl_crdt_key_ok(keys[i].lo, keys[i].hi) ? rl_crdt_row(T, keys[i].lo, keys[i].hi, false) : nullptr;
    if (row) {
        e = rlm_ld64(rl_crdt_expiry(row));
        if (e > now) {
            const unsigned long long* val = rl_crdt_values(row);
            for (uint32_t a = 0; a < T.actors; a++) sum += rlm_ld64(val + a);
        }
    }
    out_value[i] = sum;
    if (out_expiry) out_expiry[i] = e;
}

// mode 0: the re-sync stream (distributed/mod.rs:302-318): our own value, if non-zero and unexpired.  mode 1: every row.
__global__ void k_crdt_scan(RlCrdtTab T, int mode, uint64_t now, uint64_t cap, rl_crdt_key* out_keys, uint64_t* out_a,
                            uint64_t* out_expiry, uint64_t* out_values, unsigned long long* count) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > T.mask) return;
    uint8_t* row = T.rows + r * T.row_bytes;
    const ulonglong2 hdr = rlm_ld(row);
    if (hdr.x == 0 && hdr.y == 0) return;
    const unsigned long long e = rlm_ld64(rl_crdt_expiry(row));
    const unsigned long long* val = rl_crdt_values(row);
    if (mode == 0) {
        const unsigned long long mine = rlm_ld64(val + T.self_actor);
        if (mine == 0 || e <= now) return;
        const unsigned long long pos = atomicAdd(count, 1ull);
        if (pos < cap) {
            out_keys[pos].lo = hdr.x;
            out_keys[pos].hi = hdr.y;
            out_a[pos] = mine;
            out_expiry[pos] = e;
        }
    } else {
        const unsigned long long pos = atomicAdd(count, 1ull);
        if (pos < cap) {
            out_keys[pos].lo = hdr.x;
            out_keys[pos].hi = hdr.y;
            out_expiry[pos] = e;
            for (uint32_t a = 0; a < T.actors; a++) out_values[pos * T.actors + a] = rlm_ld64(val + a);
        }
    }
}
