/* rl_rls.h — the Envoy RLS v3 wire surface in front of the engine (SURVEY.md §8 f2, with the f1 matcher inside).
 *
 * Replaces, batched and without a protobuf runtime,
 *   MyRateLimiter::should_rate_limit        limitador-server/src/envoy_rls/server.rs:91-208
 *   KuadrantService::check_rate_limit       limitador-server/src/envoy_rls/kuadrant_service.rs:27-107
 *   KuadrantService::report                 limitador-server/src/envoy_rls/kuadrant_service.rs:109-186
 *   PrometheusMetrics::incr_*               limitador-server/src/prometheus_metrics.rs:93-125 (namespace and
 *                                           limit-name labels; CEL custom labels are out of scope)
 * over the messages of
 *   envoy.service.ratelimit.v3.RateLimitRequest / RateLimitResponse
 *       limitador-server/vendor/protobufs/data-plane-api/envoy/service/ratelimit/v3/rls.proto
 *   envoy.extensions.common.ratelimit.v3.RateLimitDescriptor (entries key/value)
 *   envoy.config.core.v3.HeaderValue (key, value)
 *
 * A batch of n wire requests is served in three stages:
 *   plan    (GPU in rl_rls_serve, CPU in rl_rls_plan): decode every request, build its CEL context
 *           (`descriptors[i]` = the i-th descriptor's entries as a map, last duplicate key wins — server.rs:121-127),
 *           run counters_that_apply (include/rl_match.h) and lay the counters out as the CSR that
 *           rl_check_and_update_batch / rl_is_within_limits_batch / rl_update_batch take.  Requests that never reach
 *           the store are answered here: domain "" -> overall_code UNKNOWN (server.rs:106-116); no limit applies ->
 *           OK (lib.rs:434-440); hits_addend 0 -> 1 (server.rs:131-135).
 *   decide  (GPU): ONE engine call for the whole batch; array order is the stream order that defines the result.
 *   finish  (CPU): verdicts (+ remaining / ttl with draft-03 headers) -> RateLimitResponse bytes, the three
 *           X-RateLimit-* headers sorted by key (server.rs:45-57, lib.rs:235-275), per-namespace metrics.
 * rl_rls_serve runs the three stages through the engine given at creation: the plan runs on the engine's device
 * (rl_rls_plan_device: one thread per request, the same decoder and digest as the CPU plan, the matcher as a device
 * image uploaded when its limits change), the store call reads the counters where the plan left them, and only what
 * the finish reads comes back to the host.  rl_rls_plan (the CPU plan on `threads` workers) and rl_rls_finish are
 * exported on their own so that the CPU stages can be driven (and tested) without a GPU; the product never decides on
 * the CPU.
 *
 * gRPC status per request (what tonic would put in grpc-status): 0 OK with a response body; 13 INTERNAL for a
 * message that does not decode (prost DecodeError); 14 UNAVAILABLE "Service unavailable" when the store call fails
 * (server.rs:160-172) — those two have no body.
 */
#ifndef RL_RLS_H
#define RL_RLS_H

#include <stdint.h>

#include "rl_engine.h"
#include "rl_match.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rl_rls rl_rls;

enum { RL_RLS_CODE_UNKNOWN = 0, RL_RLS_CODE_OK = 1, RL_RLS_CODE_OVER_LIMIT = 2 }; /* RateLimitResponse.Code */
enum { RL_RLS_HEADERS_NONE = 0, RL_RLS_HEADERS_DRAFT_VERSION_03 = 1 };            /* server.rs:38-42 */
enum {
    RL_RLS_SHOULD_RATE_LIMIT = 0, /* check_rate_limited_and_update(ns, ctx, hits_addend, headers != NONE) */
    RL_RLS_CHECK_RATE_LIMIT = 1,  /* is_rate_limited(ns, ctx, 1): read-only, no headers */
    RL_RLS_REPORT = 2             /* update_counters(ns, ctx, hits_addend): always OK */
};
enum { RL_GRPC_OK = 0, RL_GRPC_INTERNAL = 13, RL_GRPC_UNAVAILABLE = 14 };
#define RL_RLS_NO_STORE 0xFFFFFFFFu

/* ---- wire codec (usable on its own) ------------------------------------------------------------------------ */
typedef struct rl_rls_entry {
    uint32_t descriptor;        /* index of the descriptor the entry belongs to */
    uint32_t key_off, key_len;  /* byte ranges inside the request buffer (not NUL-terminated) */
    uint32_t val_off, val_len;
} rl_rls_entry;
typedef struct rl_rls_request {
    uint32_t domain_off, domain_len;
    uint32_t hits_addend;   /* as on the wire: 0 when absent (the service turns it into 1) */
    uint32_t n_descriptors; /* descriptors without entries count too: they shift the indices of the later ones */
    uint32_t n_entries;     /* entries found (may exceed cap_entries: then only the first cap_entries are written) */
} rl_rls_request;
/* Decode one RateLimitRequest.  RL_OK, or RL_FATAL for a malformed message (truncated varint / length, wire type
 * that does not fit the field, field number 0, group nesting, invalid UTF-8 in a string field — what prost refuses). */
int rl_rls_decode_request(const uint8_t *buf, uint64_t len, rl_rls_request *out, rl_rls_entry *entries,
                          uint32_t cap_entries);
/* Encode a RateLimitResponse {overall_code, response_headers_to_add = n_headers x HeaderValue{key, value}} (proto3:
 * zero / empty fields are not written).  *out_len = bytes needed; RL_FATAL if cap is too small. */
int rl_rls_encode_response(uint32_t overall_code, const char *const *keys, const char *const *values,
                           uint32_t n_headers, uint8_t *out, uint64_t cap, uint64_t *out_len);

/* ---- the service ---------------------------------------------------------------------------------------------- */
/* engine may be NULL (plan / finish only).  threads = workers of the plan and finish stages (0 = one per online CPU,
 * at most 64).  use_limit_name_label: limited_calls carries limit_name too (prometheus_metrics.rs:109-117). */
int rl_rls_create(rl_matcher *m, rl_engine *engine, int header_mode, uint32_t threads, int use_limit_name_label,
                  rl_rls **out);
void rl_rls_destroy(rl_rls *s);
const char *rl_rls_last_error(rl_rls *s);

/* Stage 1 on the CPU workers.  Request i = buf[off[i] .. off[i+1]).  now_us = the batch's clock reading (0 = wall
 * clock now). */
int rl_rls_plan(rl_rls *s, int method, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
/* Stage 1 on the engine's device (needs a service created with an engine); afterwards rl_rls_plan_view and
 * rl_rls_finish behave exactly as after rl_rls_plan, and every array equals rl_rls_plan's.  One difference, in a
 * misconfiguration only: with the matcher's counter cap raised above the engine's max_counters_per_request, the CPU
 * plan refuses whole worker ranges (which ones depends on the thread count), the device plan refuses exactly the
 * requests with more counters than the engine takes (gRPC 14 UNAVAILABLE). */
int rl_rls_plan_device(rl_rls *s, int method, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
/* The store call of the planned batch: n_store requests (a subset of the batch, in batch order) as CSR arrays owned by
 * the service, valid until the next plan.  store_index[i] (nullable out, n entries) = position of request i in the
 * store call or RL_RLS_NO_STORE. */
int rl_rls_plan_view(rl_rls *s, uint64_t *out_n_store, const uint32_t **out_ctr_off, const rl_counter **out_ctrs,
                     const uint64_t **out_delta, const uint64_t **out_now_us, int *out_load_counters,
                     const uint32_t **out_store_index);
/* Stage 3 (once per planned batch).  store_status = status of the store call (non-OK: every store request is answered
 * UNAVAILABLE); limited / first_limited: n_store entries; remaining / ttl_us: one per counter (only read with headers). */
int rl_rls_finish(rl_rls *s, int store_status, const uint8_t *limited, const uint32_t *first_limited,
                  const uint64_t *remaining, const uint64_t *ttl_us);
/* Responses of the last finished batch: response i = (*out_buf)[(*out_off)[i] .. (*out_off)[i+1]) (empty for a
 * non-OK gRPC status and for overall_code UNKNOWN, which encodes to zero bytes), (*out_grpc)[i] its status,
 * (*out_code)[i] the overall_code.  Valid until the next plan. */
int rl_rls_responses(rl_rls *s, const uint8_t **out_buf, const uint64_t **out_off, const uint8_t **out_grpc,
                     const uint8_t **out_code);
/* rl_rls_plan_device -> the engine (RL_MEM_DEVICE: one device->host read of the store request count before it) ->
 * finish. */
int rl_rls_serve(rl_rls *s, int method, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);

/* ---- serving on a namespace-sharded store (rl_shard_batch, include/rl_engine.h) --------------------------------------
 * Every rank runs its own service (matcher and engine, configured with the same limits) and attaches its rank's
 * rl_shard_batch; all ranks issue the same sequence of serve calls (a rank without traffic serves an empty batch).  Each
 * rank plans its batch on its own GPU, ships every store request to the owner of its namespace and finishes its own
 * responses and metrics from the outputs that come back.  The responses, metrics and the union of the owners' tables are
 * those of serving the ranks' batches one after another, in rank order, through one service on one engine.  A store
 * request that was not decided (a batch over the exchange's caps, a source whose limits differ from the owner's, a failed
 * engine call on its owner) is answered UNAVAILABLE (gRPC 14), never allowed.
 *   rl_rls_attach_shard   from now on rl_rls_serve runs rl_rls_serve_sharded (NULL detaches).  A sharded service does
 *                         not keep counter variables: rl_rls_keep_counter_vars, the counter variable export, import and
 *                         drain and GET /counters are refused (RL_FATAL).
 *   rl_rls_serve_sharded  send, decide, collect.  RL_FATAL (after the responses are finished) when the owner found a
 *                         source with other limits: rl_rls_last_error names both ranks.
 *   rl_rls_send           plan on the device and send (buf / off are not read after it returns); rl_rls_decide: decide
 *                         the owner's inbox; rl_rls_collect: collect and finish.  A one-process driver of several ranks
 *                         calls every rank's send, then every decide, then every collect. */
int rl_rls_attach_shard(rl_rls *s, rl_shard_batch *shard);
int rl_rls_serve_sharded(rl_rls *s, int method, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
int rl_rls_send(rl_rls *s, int method, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
int rl_rls_decide(rl_rls *s);
int rl_rls_collect(rl_rls *s);

/* ---- counter variables (GET /counters, include/rl_http.h) ------------------------------------------------------
 * The store keeps a counter's 96-bit key digest only.  With keeping on, every device plan (rl_rls_serve,
 * rl_rls_plan_device and their HTTP counterparts on the same service) records the variable values behind the keys it
 * produced in a dictionary on the engine's device: (variable set, key) -> the values, in the order of the limit's sorted
 * variables.  A key is recorded once, on the batch that first produced it (one device probe per variable set per store
 * request after that).  The CPU plans (rl_rls_plan, rl_http_plan) do not record.
 *   rl_rls_keep_counter_vars   off by default; max_keys slots (rounded up to a power of two; size it about twice the
 *                              live qualified counters: a key probes at most 64 slots) and arena_bytes of values, both
 *                              fixed until the next call.  (0, 0) turns it off and frees the memory; any call starts empty.
 *   rl_rls_counter_vars_stats  entries, arena bytes in use, and keys dropped since it was turned on: a full table or
 *                              arena never fails or delays a serve call, the key is simply not recorded (and its
 *                              counters are "unnamed" in GET /counters until a later batch records it after a GC).
 *   rl_rls_counter_vars_gc     keep exactly the entries the engine's present counters reference
 *                              (rl_counters_export(NULL, now_us)) in a fresh table and a compacted arena (needs a second
 *                              arena of the same size for the length of the call).  Serialise with serve, as rl_compact.
 *   rl_rls_counter_vars_export / _import   carry the dictionary through a counter snapshot (rl_counters_export /
 *                              rl_counters_import), so that a restored counter is named in GET /counters at once.  Export
 *                              with the same ns_ids and now_us as the counters; import before the counters.  The import
 *                              checks every entry against the matcher's limits as they stand (the variable set, the blob's
 *                              layout, UTF-8 without NUL, and BLAKE2b-96 over (source, value) equal to the key), so a
 *                              file from another configuration, or a corrupted one, can never name a counter wrongly.
 *                              Serialise both with serve, as rl_compact.
 * Needs a service created with an engine. */
int rl_rls_keep_counter_vars(rl_rls *s, uint64_t max_keys, uint64_t arena_bytes);
int rl_rls_counter_vars_stats(rl_rls *s, uint64_t *out_keys, uint64_t *out_arena_used, uint64_t *out_dropped);
int rl_rls_counter_vars_gc(rl_rls *s, uint64_t now_us, uint64_t *out_kept, uint64_t *out_freed);
/* The dictionary entries that the counters rl_counters_export(e, ns_ids, n_ns, now_us, ...) would list refer to,
 * each entry once, in no particular order.  Host memory.  blob_off has cap + 1 entries; blob i is
 * blobs[blob_off[i] .. blob_off[i+1]), in the dictionary's own format: for each variable of the variable set,
 * in digest order, a u32 LE length and then the bytes.  With cap = 0, or with cap / bytes_cap too small, nothing is
 * written and only *out_count / *out_bytes are set.  With keeping off the count is 0.  Changes nothing. */
int rl_rls_counter_vars_export(rl_rls *s, const uint32_t *ns_ids, uint32_t n_ns, uint64_t now_us,
                               uint64_t cap, uint64_t bytes_cap,
                               uint32_t *out_varset, uint64_t *out_key_lo, uint64_t *out_key_hi,
                               uint64_t *out_blob_off, uint8_t *out_blobs,
                               uint64_t *out_count, uint64_t *out_bytes);
/* Add entries to the dictionary.  All or nothing.  Keeping must be on.  blob_off has n + 1 entries, non-decreasing.
 * RL_FATAL, with nothing changed and rl_rls_last_error naming the first refused entry and why: a variable set that is
 * not a qualified limit's, a blob that is not exactly one (length, value) per variable, a value that is not UTF-8 or
 * holds a NUL, values that do not digest to the key, a key named twice.  RL_TRANSIENT, with nothing changed (the
 * dropped count included): no room in the arena, or a key without a free slot within 64 probes.  A key the dictionary
 * holds already is skipped (by the digest its values are the same) and does not count in *out_added. */
int rl_rls_counter_vars_import(rl_rls *s, uint64_t n, const uint32_t *varset, const uint64_t *key_lo,
                               const uint64_t *key_hi, const uint64_t *blob_off, const uint8_t *blobs,
                               uint64_t *out_added);
/* The entries recorded since the last drain, in rl_rls_counter_vars_export's layout, beside rl_counters_drain (a
 * journal on disk keeps both).  The arena is append-only between a GC and an import, so those are the slots whose blob
 * starts at or past the arena cursor the previous drain read.  *out_full = 1 (and no entry) on the first drain after
 * rl_rls_keep_counter_vars, rl_rls_counter_vars_gc or rl_rls_counter_vars_import: take a full
 * rl_rls_counter_vars_export then; the next drain starts from this one.  When *out_count > cap or *out_bytes >
 * bytes_cap nothing is written and the drain is not consumed (repeat it with larger caps).  With keeping off the
 * count is 0.  Serialise with serve, as rl_compact. */
int rl_rls_counter_vars_drain(rl_rls *s, uint64_t cap, uint64_t bytes_cap,
                              uint32_t *out_varset, uint64_t *out_key_lo, uint64_t *out_key_hi,
                              uint64_t *out_blob_off, uint8_t *out_blobs,
                              uint64_t *out_count, uint64_t *out_bytes, int *out_full);

/* ---- configuration (RateLimiter::configure_with, limitador/src/lib.rs:475-505) -----------------------------------
 * rl_rls_configure makes the service's matcher and engine hold exactly the limits of `limits`, as limitador-server does
 * with its limits file at start and on every change of it:
 *   - a limit's identity is (namespace, seconds, set of conditions, set of variables); of two entries with one identity
 *     the first wins (HashSet::insert);
 *   - a live limit of the new set is kept: its limit_id, counters (value and expiry) and position in its namespace stay.
 *     If its max_value or name differs it takes the entry's max_value, name and id; if only the id differs nothing
 *     changes (Storage::update_limit, storage/mod.rs:67-83);
 *   - a live limit absent from the new set is deleted with its counters, qualified and unqualified (rl_limits_delete,
 *     ONE call for all of them); added again later, it starts from fresh counters under its old limit_id;
 *   - added limits follow the kept ones of their namespace, in the given order (the order of the counters of a request,
 *     of X-RateLimit-Limit and of GET /limits);
 *   - all or nothing: nothing changes (matcher, engine, device match image, counters, metrics) unless every entry is
 *     accepted.  Refused: an expression the matcher's dialect does not accept; a namespace that would hold more limits
 *     than one request may carry counters (the smaller of the matcher's counter cap and the engine's
 *     max_counters_per_request; 16 without an engine); anything rl_limits_set refuses (the limits set before it are
 *     dropped again and the old maxima restored).  RL_FATAL, report->first_refused = the entry's index, and
 *     rl_rls_last_error says "entry <index>: <reason>".  A failure of the engine's delete call itself returns its status
 *     with first_refused = RL_NONE.
 * dry_run != 0 (limitador-server --validate): the entries are parsed, checked against the matcher and counted, nothing
 * changes, and the engine is not asked.  engine == NULL: the matcher alone changes.  The matcher's generation is bumped
 * once, so the next device plan uploads the new match image.  Pipelined record calls issued before are fenced first
 * (RL_FLAG_PIPELINE).  The counter-variable dictionary is not collected: after a call with deleted > 0, run
 * rl_rls_counter_vars_gc to get the deleted counters' entries back.  Serialise with serve, as rl_compact. */
typedef struct rl_limit_spec {
    const char *ns;
    uint64_t max_value;
    uint64_t seconds;
    const char *const *conditions;
    uint32_t n_cond;
    uint32_t _pad0;
    const char *const *variables;
    uint32_t n_var;
    uint32_t _pad1;
    const char *name; /* nullable */
    const char *id;   /* nullable; GET /limits renders it */
} rl_limit_spec;
typedef struct rl_configure_report {
    uint32_t kept;          /* live limits of the new set with max_value and name unchanged */
    uint32_t added;         /* new limits, and deleted ones that came back */
    uint32_t updated;       /* kept limits that took a new max_value or name */
    uint32_t deleted;       /* live limits deleted, with their counters */
    uint32_t first_refused; /* index of the refused entry, or RL_NONE */
    uint32_t _pad;
} rl_configure_report;
int rl_rls_configure(rl_rls *s, const rl_limit_spec *limits, uint32_t n, int dry_run, rl_configure_report *out_report);
/* Status::config_version / config_err_since (limitador-server/src/main.rs:218-235): successful rl_rls_configure calls,
 * and failed ones since the last success.  Dry runs do not count. */
int rl_rls_config_status(rl_rls *s, uint64_t *out_version, uint64_t *out_err_since);

/* Prometheus text exposition of authorized_calls / authorized_hits / limited_calls (sorted by label values) plus
 * `limitador_up 1`: lines `name{limitador_namespace="ns"[,limit_name="x"]} value` as
 * metrics_exporter_prometheus renders them (prometheus_metrics.rs:415-447).  *out_len = bytes needed incl. NUL. */
int rl_rls_metrics_render(rl_rls *s, char *out, uint64_t cap, uint64_t *out_len);
/* Stage timings of the last serve call in microseconds: plan (the device plan, and taking its per-request outcomes in),
 * store call (with the copies of its outputs), finish. */
int rl_rls_last_timings(rl_rls *s, double *out_plan_us, double *out_store_us, double *out_finish_us);

#ifdef __cplusplus
}
#endif
#endif /* RL_RLS_H */
