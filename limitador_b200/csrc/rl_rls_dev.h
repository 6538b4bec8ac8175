// rl_rls_dev.h — what the RLS service (rl_rls.cpp) and the device plan (rl_rls_dev.cu, kernels in rl_rls_dev.cuh) share.
// Library-internal.  rl_rls.cpp reaches the rl_rls_dev_* functions through weak references, so that the wire surface still
// links without the CUDA units (the sanitizer build of tests/san): there they are null and only the CPU plan exists.
#pragma once
#include <stdint.h>

#include "../../include/rl_rls.h"

// what the plan decided for one request
enum : uint8_t { REQ_BAD_WIRE = 1, REQ_UNKNOWN_DOMAIN = 2, REQ_NO_LIMITS = 3, REQ_STORE = 4, REQ_UNSUPPORTED = 5 };

// One request of a device plan, as the finish reads it: its kind, hits (hits_addend, 0 -> 1), position in the store
// call (RL_RLS_NO_STORE if none) and its domain's byte range inside the message.
struct RlsDevReq {
    uint32_t kind, hits, store, dom_off, dom_len;
};

// One body of an HTTP device plan (include/rl_http.h): kind, position in the store requests, the namespace's position in
// the body (dom_off: first byte after its opening quote; dom_len: its unescaped length), response_headers (RL_HTTP_HEADERS_*)
// and delta.
struct HttpDevReq {
    uint32_t kind, store, dom_off, dom_len, headers, _pad;
    uint64_t delta;
};
// One store call of an HTTP batch: its first store request, its first counter and its load_counters flag.
struct HttpRun {
    uint32_t store, ctr, load;
};

struct rl_rls_dev;  // per-service device state (shared by the RLS and HTTP surfaces): the matcher image, staging and scratch buffers

extern "C" {
// Stage 1 on the engine's device and stream: the wire bytes go up through a pinned staging buffer, the kernels decode,
// match and lay the store call out in device memory.  Returns after one synchronisation (the read of the batch's store
// request and counter counts) with the per-request array's address: pinned host memory owned by *st, filled once
// rl_rls_dev_copy_plan or rl_rls_dev_wait returned, valid until the next plan.  *st is created on first use.  RL_OK or
// an error status (rl_rls_dev_error).
int rl_rls_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int method, uint64_t n, const uint8_t* buf,
                    const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                    const RlsDevReq** out_req);
// Host copies of the planned store requests of either plan: ctr_off [n_store + 1], ctrs [n_ctr], delta [n_store], and
// unless load is NULL (an HTTP plan's) load_counters flags [n_store].
int rl_rls_dev_copy_plan(rl_rls_dev* st, uint32_t* ctr_off, rl_counter* ctrs, uint64_t* delta, uint8_t* load);
// The store call of the planned batch from its device arrays (RL_MEM_DEVICE), then its outputs copied back: limited and
// first_limited [n_store] (not for Report), and with load_counters remaining / ttl_us [n_ctr] together with ctr_off
// [n_store + 1] and ctrs [n_ctr], which the headers are formatted from.  Returns the store call's status;
// rl_last_error(e) tells why it failed.
int rl_rls_dev_decide(rl_rls_dev* st, rl_engine* e, int method, int load_counters, uint8_t* limited, uint32_t* first_limited,
                      uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs);
// Wait for everything the plan and the store call enqueued (the per-request array and the outputs are then on the host).
int rl_rls_dev_wait(rl_rls_dev* st);
/* The planned batch's store requests through the sharded exchange (rl_shard_batch_send): method / endpoint -> op, with the
 * HTTP plan's per-request load flags or load_counters for all.  empty != 0 (or no planned state): an empty batch, so that
 * a rank whose plan failed still takes part in the step; *out_failed = the status that made a planned batch go out empty.  _collect: rl_shard_batch_collect into the plan's output arrays,
 * then the verdicts (always: error verdicts mark the requests that were not decided) and, with load_counters, remaining /
 * ttl and the CSR to the host.  Returns the collect's status. */
int rl_rls_dev_shard_send(rl_rls_dev* st, rl_shard_batch* sb, int empty, int http, int method, int load_counters,
                          int* out_failed);
int rl_rls_dev_shard_collect(rl_rls_dev* st, rl_shard_batch* sb, int load_counters, uint8_t* limited, uint32_t* first_limited,
                             uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs);
// The HTTP plan on the same state (rl_http_dev.cuh): as rl_rls_dev_plan, and the one read before the store call also
// brings the store calls back: *out_runs[0 .. *out_n_runs) (pinned host memory owned by *st, valid until the next plan).
int rl_http_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int endpoint, uint64_t n, const uint8_t* buf,
                     const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                     const HttpDevReq** out_req, const HttpRun** out_runs, uint32_t* out_n_runs);
// One store call per run from the device arrays, then the outputs back as rl_rls_dev_decide copies them (remaining / ttl,
// ctr_off and ctrs when a run loads counters).  run_status[r] = the status of run r's call.
int rl_http_dev_decide(rl_rls_dev* st, rl_engine* e, int endpoint, int* run_status, uint8_t* limited, uint32_t* first_limited,
                       uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs);
// The counter variable dictionary (rl_cvars_dev.cuh) on the same state, on the engine's device.  Both plans record into it
// after their scatter while it is on.  configure: (0, 0) turns it off and frees it; otherwise max_keys (rounded up to a
// power of two: the slots) and the arena's bytes.
int rl_cv_dev_configure(rl_rls_dev** st, rl_engine* e, uint64_t max_keys, uint64_t arena_bytes);
int rl_cv_dev_stats(rl_rls_dev* st, uint64_t* out_slots, uint64_t* out_keys, uint64_t* out_arena_used, uint64_t* out_dropped);
// The blobs of n counters: counter i's at (*out_blobs)[(*out_blob_off)[i] .. [i + 1]); (*out_unnamed)[i] = 1 for a
// qualified counter without an entry (every qualified counter while keeping is off).  Host memory owned by *st, valid
// until the next call on it.
int rl_cv_dev_lookup(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* limit_id, const uint64_t* key_lo,
                     const uint64_t* key_hi, const uint8_t** out_blobs, const uint64_t** out_blob_off, const uint8_t** out_unnamed);
// Keep exactly the entries the engine's counters reference (rl_counters_export(NULL, now_us)), in a fresh table and a
// compacted arena.
int rl_cv_dev_gc(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t now_us, uint64_t* out_kept, uint64_t* out_freed);
// Snapshots (include/rl_rls.h: rl_rls_counter_vars_export / _import).  Export: the entries the counters
// rl_counters_export(ns_ids, now_us) lists reference, into host arrays.  Import: every entry checked against the image
// (variable set, blob, UTF-8, digest), then committed all or nothing into a fresh table.
int rl_cv_dev_export(rl_rls_dev** st, rl_engine* e, rl_matcher* m, const uint32_t* ns_ids, uint32_t n_ns, uint64_t now_us,
                     uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset, uint64_t* out_key_lo, uint64_t* out_key_hi,
                     uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count, uint64_t* out_bytes);
int rl_cv_dev_import(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* varset, const uint64_t* key_lo,
                     const uint64_t* key_hi, const uint64_t* blob_off, const uint8_t* blobs, uint64_t* out_added);
// Drains (include/rl_rls.h: rl_rls_counter_vars_drain): the entries recorded since the last drain, in the export's layout.
int rl_cv_dev_drain(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset,
                    uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count,
                    uint64_t* out_bytes, int* out_full);
const char* rl_rls_dev_error(rl_rls_dev* st);
void rl_rls_dev_destroy(rl_rls_dev* st);
}
