// rl_http_dev.cuh — the HTTP plan stage on the device (include/rl_http.h: rl_http_plan_device, rl_http_serve).
//
// One thread per body restates the CPU plan (rl_rls.cpp plan_range over rl_json.h):
//   k_http_plan     decode (rl_json.h), then the match body the RLS plan runs (rl_match_ctx); the counters go to a
//                   per-request scratch slice, the request's HttpScan element to `count`
//   (scan)          exclusive scan of HttpScanOp over `count` (CUB on the device; a host loop under the shim): every store
//                   request's position, first counter and store call (a run of equal load_counters flags)
//   k_http_runs     the store calls' table and the batch's totals, in one block the host reads once
//   k_http_scatter  the store requests in batch order: store_index, ctr_off, the per-call ctr_off, ctrs, delta, now, load
// Written, like rl_rls_dev.cuh, so that the same source runs under tests/emu/cuda_shim.h.
#pragma once
#include <stdint.h>

#include "../../include/rl_http.h"
#include "rl_json.h"
#include "rl_rls_dev.cuh"

// A prefix of the batch's requests: its store requests, their counters, the store calls they form (runs of equal
// load_counters flags) and the flags of its first and last store request.  Associative; {0} is the identity.
struct HttpScan {
    uint32_t n_store, n_ctr, n_runs;
    uint8_t first, last, _pad[2];
};

struct HttpScanOp {
    RL_HD HttpScan operator()(const HttpScan& a, const HttpScan& b) const {
        HttpScan o = a.n_store ? a : b;
        o.n_ctr = a.n_ctr + b.n_ctr;
        if (a.n_store && b.n_store) {
            o.n_store = a.n_store + b.n_store;
            o.n_runs = a.n_runs + b.n_runs - (a.last == b.first ? 1u : 0u);
            o.last = b.last;
        }
        return o;
    }
};

// the words before the store calls in the block k_http_runs writes (the batch's HttpScan)
#define RL_HTTP_RUNS_HEAD 4u

struct HttpPlanArgs {
    const uint8_t* buf;          // the batch's bodies: body i = buf[off[i] .. off[i+1])
    const uint64_t* off;         // [n + 1]
    uint64_t n;
    RlImage img;
    uint32_t per_req;            // counters one request may carry: min(matcher cap, engine maximum)
    int endpoint;
    uint8_t* txt;                // [bytes]: the unescaped strings at their source offsets
    uint8_t* bits;               // [bytes / 8 + n + 1]: body i's skip stack at off[i] / 8 + i
    rl_rls_entry* ent;           // entry scratch: body i's entries at ent[off[i] / 2]
    rl_counter* scratch;         // [n * per_req]
    HttpDevReq* req;             // [n]
    HttpScan* count;             // [n + 1]; count[n] = {0}
};

__global__ void k_http_plan(HttpPlanArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    HttpScan cnt{0, 0, 0, 0, 0, {0, 0}};
    if (i == a.n) {
        a.count[i] = cnt;
        return;
    }
    const uint8_t* body = a.buf + a.off[i];
    const uint64_t len = a.off[i + 1] - a.off[i];
    uint8_t* txt = a.txt + a.off[i];
    rl_rls_entry* E = a.ent + a.off[i] / 2;
    rl_wire::EntrySink sink{E, (uint32_t)(len / 2 < 0xFFFFFFFFull ? len / 2 : 0xFFFFFFFFull), 0};
    rl_json::Info q;
    HttpDevReq R{REQ_BAD_WIRE, RL_RLS_NO_STORE, 0, 0, 0, 0, 0};
    if (rl_json::decode_info(body, len, txt, a.bits + a.off[i] / 8 + i, q, sink)) {
        R.dom_off = q.ns_off;
        R.dom_len = q.ns_len;
        R.headers = q.headers;
        R.delta = q.delta;
        uint32_t n_ctr = 0;
        R.kind = rl_match_ctx(a, txt, q.ns_off, q.ns_len, E, sink.n, a.scratch + i * a.per_req, n_ctr);
        if (R.kind == REQ_STORE) {
            const uint8_t lc = rl_json::load_counters(a.endpoint, q.headers);
            cnt = HttpScan{1, n_ctr, 1, lc, lc, {0, 0}};
        }
    }
    a.req[i] = R;
    a.count[i] = cnt;
}

struct HttpRunsArgs {
    const HttpScan* count;       // k_http_plan's elements
    const HttpScan* start;       // [n + 1]: their exclusive scan
    uint64_t n;
    uint32_t* block;             // [RL_HTTP_RUNS_HEAD + 3 * runs]: the batch's HttpScan, then one HttpRun per store call
};

__device__ __forceinline__ bool http_starts_run(const HttpScan& prefix, uint8_t load) {
    return prefix.n_store == 0 || prefix.last != load;
}

__global__ void k_http_runs(HttpRunsArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    const HttpScan P = a.start[i];
    if (i == a.n) {
        const uint32_t w[RL_HTTP_RUNS_HEAD] = {P.n_store, P.n_ctr, P.n_runs, P.first};
        for (uint32_t k = 0; k < RL_HTTP_RUNS_HEAD; k++) a.block[k] = w[k];
        return;
    }
    const HttpScan c = a.count[i];
    if (!c.n_store || !http_starts_run(P, c.first)) return;
    uint32_t* run = a.block + RL_HTTP_RUNS_HEAD + 3ull * P.n_runs;
    run[0] = P.n_store;
    run[1] = P.n_ctr;
    run[2] = c.first;
}

struct HttpScatterArgs {
    HttpDevReq* req;             // [n]: the store index is filled in
    const rl_counter* scratch;   // k_http_plan's per-request counters
    const HttpScan* start;       // [n + 1]: the exclusive scan
    const uint32_t* runs;        // the store calls (k_http_runs' block past its head)
    uint64_t n;
    uint32_t per_req;
    int endpoint;
    uint64_t now_us;
    uint32_t* ctr_off;           // [n_store + 1]: the batch's CSR
    uint32_t* ctr_run;           // [n_store + n_runs]: store call r's CSR offsets at ctr_run[runs[r].store + r ..], from 0
    rl_counter* ctrs;            // [n_ctr]
    uint64_t* delta;             // [n_store]
    uint64_t* now;               // [n_store]
    uint8_t* load;               // [n_store]
};

__global__ void k_http_scatter(HttpScatterArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    const HttpScan P = a.start[i];
    if (i == a.n) {  // the ends of the batch and of its last store call
        a.ctr_off[P.n_store] = P.n_ctr;
        if (P.n_store) a.ctr_run[P.n_store + P.n_runs - 1] = P.n_ctr - a.runs[3ull * (P.n_runs - 1) + 1];
        return;
    }
    HttpDevReq& R = a.req[i];
    if (R.kind != REQ_STORE) return;
    const uint8_t lc = rl_json::load_counters(a.endpoint, R.headers);
    const bool first = http_starts_run(P, lc);
    const uint32_t j = P.n_store, c = P.n_ctr, k = a.start[i + 1].n_ctr - c, r = first ? P.n_runs : P.n_runs - 1;
    R.store = j;
    a.ctr_off[j] = c;
    a.ctr_run[j + r] = c - a.runs[3ull * r + 1];
    if (first && r) a.ctr_run[j + r - 1] = c - a.runs[3ull * (r - 1) + 1];  // the end of the call before
    for (uint32_t x = 0; x < k; x++) a.ctrs[(uint64_t)c + x] = a.scratch[i * a.per_req + x];
    a.delta[j] = R.delta;  // the request's own delta, also for /check (server.rs:144)
    a.now[j] = a.now_us;
    a.load[j] = lc;
}
