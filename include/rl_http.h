/* rl_http.h — Limitador's HTTP API in front of the engine: POST /check, /report and /check_and_report.
 *
 * Replaces, batched,
 *   check / report / check_and_report      limitador-server/src/http_api/server.rs:129-260
 *   add_response_header                    limitador-server/src/http_api/server.rs:262-280
 *   get_limits / get_counters              limitador-server/src/http_api/server.rs:88-125 (types request_types.rs:18-96)
 * over the JSON body CheckAndReportInfo {namespace, values, delta, response_headers}
 * (limitador-server/src/http_api/request_types.rs:10-16).  The HTTP server itself (routing, content type, body size
 * limit, /status, /metrics) stays with the caller: a batch here is a list of request bodies of one endpoint.
 *
 * The service hangs off an rl_rls service and shares its matcher, engine, workers, device state and metrics registry
 * (the reference has one PrometheusMetrics for both servers, so rl_rls_metrics_render covers both).  Batches of the two
 * surfaces are issued from one thread, as the engine requires.
 *
 * A batch of n bodies is served in three stages, as for RLS (include/rl_rls.h):
 *   plan    decode every body (the JSON rules are stated in limitador_b200/csrc/rl_json.h), bind `values` as
 *           descriptors[0] (server.rs:140-141), run counters_that_apply, lay the counters out as a CSR.  The request's own
 *           delta goes to the store as it is (no 0 -> 1 rule, also for /check).  On the engine's device in rl_http_serve
 *           and rl_http_plan_device, on the CPU workers in rl_http_plan; every array of the two is equal.
 *   decide  /check: is_rate_limited (rl_is_within_limits_batch); /report: update_counters (rl_update_batch);
 *           /check_and_report: check_rate_limited_and_update (rl_check_and_update_batch) with load_counters =
 *           response_headers.is_some() request by request (server.rs:206,210).  Since that flag changes which counters a
 *           store call inserts, the store requests are split into maximal runs of consecutive requests with the same flag
 *           and every run is one store call, in batch order.  A batch whose requests agree is one call.
 *   finish  per request: the HTTP status, the body and the X-RateLimit-* headers; the metrics of /check_and_report.
 *
 * Outcomes (server.rs:51-74,129-260):
 *   /check             200 `null` | 429 `Too many requests` | 500 `Internal server error`
 *   /report            200 `null` | 500 `Internal server error`
 *   /check_and_report  200 `null` | 429 `null` | 500 `null`; with response_headers == "DraftVersion03" the three
 *                      X-RateLimit-* headers on 200 and 429 (none when no limit applies); another string loads the
 *                      counters but adds no headers.
 *   any                400 for a body the JSON extractor refuses (serde's message text is not reproduced: empty body).
 * 500 covers a failed store call, an RL_VERDICT_ERROR verdict and a request the plan cannot ship: one with a NUL (from
 * `\u0000`) in a key or value of `values`, or with more counters than the engine takes.
 */
#ifndef RL_HTTP_H
#define RL_HTTP_H

#include <stdint.h>

#include "rl_rls.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rl_http rl_http;

enum { RL_HTTP_CHECK = 0, RL_HTTP_REPORT = 1, RL_HTTP_CHECK_AND_REPORT = 2 };
/* response_headers: absent or null (None), "DraftVersion03", another string */
enum { RL_HTTP_HEADERS_NONE = 0, RL_HTTP_HEADERS_DRAFT_VERSION_03 = 1, RL_HTTP_HEADERS_OTHER = 2 };

/* ---- the JSON codec (usable on its own) ------------------------------------------------------------------------- */
typedef struct rl_http_info {
    uint32_t ns_off, ns_len;   /* the namespace, unescaped, inside txt */
    uint64_t delta;
    uint32_t n_entries;        /* entries of values (may exceed cap_entries: then only the first cap_entries are written) */
    uint32_t response_headers; /* RL_HTTP_HEADERS_* */
} rl_http_info;
/* Decode one CheckAndReportInfo body.  txt: len bytes of the caller's; every deserialized string is written there
 * unescaped at its own source offset, and the entries (descriptor 0) and the namespace are byte ranges inside txt.
 * RL_OK, or RL_FATAL for a body the extractor refuses (HTTP 400). */
int rl_http_decode_body(const uint8_t *body, uint64_t len, uint8_t *txt, rl_http_info *out, rl_rls_entry *entries,
                        uint32_t cap_entries);

/* ---- the service ---------------------------------------------------------------------------------------------- */
/* rls outlives the HTTP service. */
int rl_http_create(rl_rls *rls, rl_http **out);
void rl_http_destroy(rl_http *h);
const char *rl_http_last_error(rl_http *h);

/* Stage 1 on the CPU workers.  Body i = buf[off[i] .. off[i+1]).  now_us = the batch's clock reading (0 = wall clock). */
int rl_http_plan(rl_http *h, int endpoint, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
/* Stage 1 on the engine's device; afterwards rl_http_plan_view and rl_http_finish behave exactly as after rl_http_plan. */
int rl_http_plan_device(rl_http *h, int endpoint, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
/* The store requests of the planned batch (a subset, in batch order) as CSR arrays owned by the service, valid until the
 * next plan; load_counters[j] (n_store) is store request j's flag: consecutive equal flags form one store call.
 * store_index[i] (n entries) = position of body i in the store requests or RL_RLS_NO_STORE. */
int rl_http_plan_view(rl_http *h, uint64_t *out_n_store, const uint32_t **out_ctr_off, const rl_counter **out_ctrs,
                      const uint64_t **out_delta, const uint64_t **out_now_us, const uint8_t **out_load_counters,
                      const uint32_t **out_store_index);
/* Stage 3 (once per planned batch).  store_status: n_store statuses (the status of the store call that decided the
 * request; NULL = all RL_OK); limited / first_limited: n_store entries (not read for /report); remaining / ttl_us: one
 * per counter (read for /check_and_report requests with load_counters). */
int rl_http_finish(rl_http *h, const int32_t *store_status, const uint8_t *limited, const uint32_t *first_limited,
                   const uint64_t *remaining, const uint64_t *ttl_us);
/* Responses of the last finished batch: status[i]; body i = body[body_off[i] .. body_off[i+1]); header k of response i
 * (0 X-RateLimit-Limit, 1 X-RateLimit-Remaining, 2 X-RateLimit-Reset) = hdr[hdr_off[3i+k] .. hdr_off[3i+k+1]), empty
 * when absent.  Valid until the next plan. */
int rl_http_responses(rl_http *h, const uint16_t **out_status, const uint8_t **out_body, const uint64_t **out_body_off,
                      const uint8_t **out_hdr, const uint64_t **out_hdr_off);
/* rl_http_plan_device -> the engine (RL_MEM_DEVICE, one call per run of equal load_counters flags) -> finish. */
int rl_http_serve(rl_http *h, int endpoint, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
/* Over the RLS service's sharded store (rl_rls_attach_shard; rl_http_serve runs rl_http_serve_sharded then): one step
 * covers the whole batch, however many load_counters runs it has.  Phases as rl_rls_send / _decide / _collect. */
int rl_http_serve_sharded(rl_http *h, int endpoint, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
int rl_http_send(rl_http *h, int endpoint, uint64_t n, const uint8_t *buf, const uint64_t *off, uint64_t now_us);
int rl_http_decide(rl_http *h);
int rl_http_collect(rl_http *h);
/* Stage timings of the last serve call in microseconds, and the store calls it made. */
int rl_http_last_timings(rl_http *h, double *out_plan_us, double *out_store_us, double *out_finish_us,
                         uint32_t *out_store_calls);

/* ---- GET /limits/{namespace} and GET /counters/{namespace} --------------------------------------------------------
 * ns[0 .. ns_len) is the path segment as the caller's router decoded it.  Bodies as actix Json + serde_json write them:
 * compact, fields in declaration order, strings with the short escapes and lower-case \u00XX, everything else raw.
 *   Limit    {"id":null,"namespace":..,"max_value":..,"seconds":..,"name":null|"..","conditions":[..],"variables":[..]}
 *            (id: the matcher keeps no limit ids; conditions / variables: the sorted identity sources)
 *   Counter  {"limit":{..},"set_variables":{source:value, sorted by source},"remaining":..,"expires_in_seconds":..}
 * Arrays in a deterministic order: limits in counter order; counters by (the limit's position, key_lo, key_hi).
 * Outcomes: 200 with the array (an unknown namespace: 200 []); /counters answers 500 `Internal server error` when the
 * engine call fails or when a listed qualified counter has no recorded variables (keeping off, a dropped key, or a
 * counter that came from an import or a direct engine call: see rl_rls_keep_counter_vars), never a counter with empty
 * or guessed variables.  The response is read with rl_http_get_response. */
int rl_http_get_limits(rl_http *h, const char *ns, uint32_t ns_len);
/* The namespace's counters with ttl(now_us) > 0 (rl_get_counters; 0 = wall clock), the live limits' only, joined with the
 * recorded variables on the engine's device. */
int rl_http_get_counters(rl_http *h, const char *ns, uint32_t ns_len, uint64_t now_us);
/* The rendering of GET /counters on its own (no engine needed): n counters with their remaining / ttl_us (as
 * rl_get_counters reports them), counter i's recorded blob at blobs[blob_off[i] .. blob_off[i+1]) (the values in the
 * order of the limit's variables, each a u32 little-endian length then the bytes) and unnamed[i] != 0 for a qualified
 * counter without one.  Counters of other namespaces' or deleted limits are left out. */
int rl_http_render_counters(rl_http *h, const char *ns, uint32_t ns_len, uint64_t n, const rl_counter *ctrs,
                            const uint64_t *remaining, const uint64_t *ttl_us, const uint8_t *blobs, const uint64_t *blob_off,
                            const uint8_t *unnamed);
/* The last GET response: status, body (valid until the next GET call), and the qualified counters it found unnamed. */
int rl_http_get_response(rl_http *h, uint16_t *out_status, const uint8_t **out_body, uint64_t *out_len,
                         uint64_t *out_unnamed);

#ifdef __cplusplus
}
#endif
#endif /* RL_HTTP_H */
