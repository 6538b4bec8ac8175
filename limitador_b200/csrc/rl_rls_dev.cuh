// rl_rls_dev.cuh — the RLS plan stage on the device (include/rl_rls.h: rl_rls_plan_device, rl_rls_serve).
//
// One thread per request restates the CPU plan (rl_rls.cpp plan_range + rl_match.cpp match_one) exactly:
//   k_rls_plan     decode (rl_wire.h, the CPU plan's decoder), the request's kind, then counters_that_apply against the
//                  matcher image (rl_match_image.h) with the counter keys digested by rl_blake2b.h; the counters go to a
//                  per-request scratch slice, and the request's (is_store << 32 | counters) word to `count`
//   (scan)         exclusive sum over `count` (CUB on the device; a host loop under the shim) -> every store request's
//                  position in the store call and its first counter
//   k_rls_scatter  the store call in batch order: store_index, ctr_off, ctrs, delta, now
// The match after the decode (rl_match_ctx) is also the HTTP plan's (rl_http_dev.cuh).
// Written so that the SAME source runs under tests/emu/cuda_shim.h (one CUDA thread after the other on the host): plain
// per-thread code, no shared memory, no warp intrinsics, nothing that recurses.
#pragma once
#include <stdint.h>

#include "../../include/rl_rls.h"
#include "rl_blake2b.h"
#include "rl_match_image.h"
#include "rl_rls_dev.h"
#include "rl_wire.h"

struct RlsPlanArgs {
    const uint8_t* buf;          // the batch's wire bytes: request i = buf[off[i] .. off[i+1])
    const uint64_t* off;         // [n + 1]
    uint64_t n;
    RlImage img;
    uint32_t per_req;            // counters one request may carry: min(matcher cap, engine maximum)
    rl_rls_entry* ent;           // entry scratch: request i's entries at ent[off[i] / 2] (an entry takes >= 2 wire bytes)
    rl_counter* scratch;         // [n * per_req]: request i's counters at i * per_req
    RlsDevReq* req;              // [n]
    unsigned long long* count;   // [n + 1]: (1 << 32) | counters for a store request, 0 otherwise; count[n] = 0
};

__device__ __forceinline__ bool rls_has_nul(const uint8_t* p, uint32_t n) {
    for (uint32_t i = 0; i < n; i++)
        if (p[i] == 0) return true;
    return false;
}

// The entry bound to `slot` (entries hold their slot in `descriptor` once bound): the last one wins, as a HashMap keeps
// the last value inserted (server.rs:121-127).  nullptr: unbound.
__device__ __forceinline__ const rl_rls_entry* rls_bound(const rl_rls_entry* E, uint32_t ne, uint32_t slot) {
    for (uint32_t k = ne; k-- > 0;)
        if (E[k].descriptor == slot) return &E[k];
    return nullptr;
}

// The match body of both device plans (RLS and HTTP): plan_range's checks after the decode, then match_one.  The context
// is E[0 .. ne) (byte ranges inside msg), the namespace msg[ns_off .. ns_off + ns_len); a.img is the matcher, a.per_req the
// counters a request may carry.  Returns the request's kind; its counters at out[0 .. n_out).
template <class Args>
__device__ __forceinline__ uint8_t rl_match_ctx(const Args& a, const uint8_t* msg, uint32_t ns_off, uint32_t ns_len,
                                                rl_rls_entry* E, uint32_t ne, rl_counter* out, uint32_t& n_out) {
    n_out = 0;
    // no namespace the matcher knows holds a NUL: nothing applies (lib.rs:434-440)
    if (rls_has_nul(msg + ns_off, ns_len)) return REQ_NO_LIMITS;
    // the matcher compares NUL-terminated strings: an embedded NUL anywhere in the context is refused
    for (uint32_t k = 0; k < ne; k++)
        if (rls_has_nul(msg + E[k].key_off, E[k].key_len) || rls_has_nul(msg + E[k].val_off, E[k].val_len)) return REQ_UNSUPPORTED;
    const RlImage& I = a.img;
    const uint32_t ns = rl_img_find_ns(I, msg + ns_off, ns_len);
    if (ns == RL_IMG_EMPTY) return REQ_NO_LIMITS;  // no limit was ever added for the namespace
    for (uint32_t k = 0; k < ne; k++)  // bind: from here on an entry's `descriptor` holds its slot
        E[k].descriptor = rl_img_find_slot(I, E[k].descriptor, msg + E[k].key_off, E[k].key_len);
    for (uint32_t x = I.ns_lim_off[ns]; x < I.ns_lim_off[ns + 1]; x++) {
        const uint32_t lid = I.ns_lims[x];
        const uint32_t* L = I.lims + 5ull * lid;
        bool ok = true;
        for (uint32_t p = L[0]; ok && p < L[0] + L[1]; p++) {
            const uint32_t* P = I.preds + 4ull * p;
            const rl_rls_entry* b = rls_bound(E, ne, P[0]);
            // an unbound name / missing key makes the predicate false (cel.rs:315-331)
            ok = b && (b->val_len == P[3] && rl_img_bytes_eq(msg + b->val_off, I.arena + P[2], P[3])) != (P[1] != 0);
        }
        for (uint32_t v = L[2]; ok && v < L[2] + L[3]; v++) ok = rls_bound(E, ne, I.vars[3ull * v]) != nullptr;  // limit.rs:133-148
        if (!ok) continue;
        if (n_out >= a.per_req) {  // more counters than one request may carry: the request gets none
            n_out = 0;
            return REQ_UNSUPPORTED;
        }
        rl_counter& c = out[n_out];
        c.limit_id = lid;
        c._pad = 0;
        c.key_lo = c.key_hi = 0;
        if (L[3]) {  // one key per variable set: an earlier counter of the request may have it already
            bool hit = false;
            for (uint32_t k = 0; k < n_out && !hit; k++)
                if (I.lims[5ull * out[k].limit_id + 4] == L[4]) {
                    c.key_lo = out[k].key_lo;
                    c.key_hi = out[k].key_hi;
                    hit = true;
                }
            if (!hit) {
                rl_b2::KeyDigest d;
                for (uint32_t v = L[2]; v < L[2] + L[3]; v++) {
                    const uint32_t* V = I.vars + 3ull * v;
                    const rl_rls_entry* b = rls_bound(E, ne, V[0]);
                    d.str((const char*)I.arena + V[1], V[2]);
                    d.str((const char*)msg + b->val_off, b->val_len);
                }
                d.finish(c.key_lo, c.key_hi);
            }
        }
        n_out++;
    }
    return n_out ? REQ_STORE : REQ_NO_LIMITS;
}

// the RLS plan after the decode: an empty domain is answered UNKNOWN before the match (server.rs:106-116)
__device__ __forceinline__ uint8_t rls_match(const RlsPlanArgs& a, const uint8_t* msg, const rl_rls_request& q,
                                             rl_rls_entry* E, uint32_t ne, rl_counter* out, uint32_t& n_out) {
    n_out = 0;
    if (q.domain_len == 0) return REQ_UNKNOWN_DOMAIN;
    return rl_match_ctx(a, msg, q.domain_off, q.domain_len, E, ne, out, n_out);
}

__global__ void k_rls_plan(RlsPlanArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    if (i == a.n) {
        a.count[i] = 0;
        return;
    }
    const uint8_t* msg = a.buf + a.off[i];
    const uint64_t len = a.off[i + 1] - a.off[i];
    rl_rls_entry* E = a.ent + a.off[i] / 2;
    rl_wire::EntrySink sink{E, (uint32_t)(len / 2 < 0xFFFFFFFFull ? len / 2 : 0xFFFFFFFFull), 0};
    rl_rls_request q;
    RlsDevReq R{REQ_BAD_WIRE, 1, RL_RLS_NO_STORE, 0, 0};
    unsigned long long cnt = 0;
    if (rl_wire::decode_request(msg, len, q, sink)) {
        R.hits = q.hits_addend ? q.hits_addend : 1;  // server.rs:131-135
        R.dom_off = q.domain_off;
        R.dom_len = q.domain_len;
        uint32_t n_ctr = 0;
        R.kind = rls_match(a, msg, q, E, sink.n, a.scratch + i * a.per_req, n_ctr);
        if (R.kind == REQ_STORE) cnt = (1ull << 32) | n_ctr;
    }
    a.req[i] = R;
    a.count[i] = cnt;
}

struct RlsScatterArgs {
    RlsDevReq* req;                  // [n]: the store index is filled in
    const rl_counter* scratch;       // k_rls_plan's per-request counters
    const unsigned long long* start; // [n + 1]: exclusive sum of k_rls_plan's count: (store index << 32) | first counter
    uint64_t n;
    uint32_t per_req;
    int method;
    uint64_t now_us;
    uint32_t* ctr_off;               // [n_store + 1]
    rl_counter* ctrs;                // [n_ctr]
    uint64_t* delta;                 // [n_store]
    uint64_t* now;                   // [n_store]
};

__global__ void k_rls_scatter(RlsScatterArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    const unsigned long long s = a.start[i];
    if (i == a.n) {
        a.ctr_off[s >> 32] = (uint32_t)s;
        return;
    }
    RlsDevReq& R = a.req[i];
    if (R.kind != REQ_STORE) return;
    const uint32_t j = (uint32_t)(s >> 32), c = (uint32_t)s, k = (uint32_t)(a.start[i + 1] - s);
    R.store = j;
    a.ctr_off[j] = c;
    for (uint32_t x = 0; x < k; x++) a.ctrs[(uint64_t)c + x] = a.scratch[i * a.per_req + x];
    // CheckRateLimit asks with delta 1 whatever hits_addend says (kuadrant_service.rs:62-65)
    a.delta[j] = a.method == RL_RLS_CHECK_RATE_LIMIT ? 1 : R.hits;
    a.now[j] = a.now_us;
}
