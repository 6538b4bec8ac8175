/* rl_match.h — CPU front of the engine: limits -> counters (SURVEY.md §8 f1).
 *
 * Replaces, for a table-driven subset of the reference's CEL expressions,
 *   RateLimiter::counters_that_apply          limitador/src/lib.rs:507-522
 *     = Storage::get_limits                   limitador/src/storage/mod.rs:85-91
 *     + Limit::applies                        limitador/src/limit.rs:157-174
 *         (Predicate::test                    limitador/src/limit/cel.rs:314-334: a condition over an unbound
 *                                             name or a missing key is false, never an error)
 *     + Counter::new / resolve_variables      limitador/src/counter.rs:20-32, limit.rs:133-148 (a variable
 *                                             without a value drops the counter)
 *   and the interning a GPU-backed CounterStorage needs: Limit identity (limit.rs:177-214: namespace,
 *   seconds, conditions, variables — max_value, name and id excluded) -> dense limit_id, namespace -> ns_id,
 *   (namespace, variable set) -> varset_id, resolved variable values -> 96-bit counter key.
 *
 * Expressions accepted (anything else is refused at rl_matcher_add_limit with RL_FATAL "unsupported condition
 * expression", so that a deployment can keep such limits on the reference's interpreter).  Two dialects, chosen per
 * matcher with rl_matcher_set_dialect (rl_match_dialect.h); variables take the same grammar in both.
 *
 * RL_MATCH_DIALECT_TABLE (the default):
 *   operand   := IDENT                                      a root binding (ASCII identifier, NO dots: `req.method`
 *                                                           is CEL member access on the variable `req`, which the
 *                                                           reference never binds — limit/cel.rs:314-322)
 *              | 'descriptors[' N '].' IDENT                the Envoy descriptor list (cel.rs:102-114)
 *              | 'descriptors[' N '][' QUOTED ']'
 *   condition := operand ('==' | '!=') QUOTED               QUOTED = '...' or "..." closed by the quote that opened
 *                                                           it, without any backslash (CEL escape processing is not
 *                                                           done here: such literals and keys are refused, not
 *                                                           reinterpreted)
 *   variable  := operand
 *
 * RL_MATCH_DIALECT_BOOLEAN: the table dialect's conditions and boolean formulas whose result provably does not depend on
 * how a CEL implementation propagates errors through && / || (DESIGN.md §9b).  Tokens may be separated by whitespace;
 * operand and QUOTED are as above (a QUOTED also holds no line break; raw, byte and triple-quoted strings are refused);
 * IDENT is no CEL reserved word, nor `descriptors` or `has`.
 *   atom      := operand ('==' | '!=') QUOTED | QUOTED ('==' | '!=') operand
 *              | operand '.' ('startsWith' | 'endsWith' | 'contains') '(' QUOTED ')'
 *              | operand 'in' '[' [QUOTED (',' QUOTED)*] ']'
 *   group     := any formula of atoms with '&&', '||', '!' and parentheses in which every atom has the SAME operand and
 *                which holds at most RL_MATCH_MAX_ATOMS (6) atoms; a '!' directly before an ==, != or `in` needs
 *                parentheses (CEL reads `!x == 'a'` as `(!x) == 'a'`).  An unbound or missing operand (a descriptor
 *                index past the request's list included) makes the whole group false, whatever its formula: every
 *                atom errors, and the reference's Predicate::test turns that into false (cel.rs:321-339).
 *   presence  := 'has(descriptors[' N '].' IDENT ')' | QUOTED 'in descriptors[' N ']'
 *                true iff descriptor N exists and holds the key; only positively, and only as a top-level conjunct
 *   condition := (group | presence) ('&&' (group | presence))*
 * Refused: || or ! across two operands, a presence test under ! or ||, `matches`, `size`, any literal that is not a
 * string, `limit.name` / `limit.id`, dotted root operands, more than 6 atoms in one group, and all other CEL.
 *
 * Output = exactly the inputs of rl_check_and_update_batch (include/rl_engine.h): a CSR of rl_counter.
 * Counters come out in the limits' registration order (the reference iterates a HashSet: unspecified).
 * Pure host code; no CUDA call is made by anything in this header.
 */
#ifndef RL_MATCH_H
#define RL_MATCH_H

#include <stdint.h>

#include "rl_engine.h"
#include "rl_match_dialect.h" /* rl_matcher_set_dialect: which of the two grammars below later limits are parsed in */

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rl_matcher rl_matcher;

#define RL_BIND_ROOT 0xFFFFFFFFu
/* One (key, value) of a request's context: a root binding (Context::from(HashMap), cel.rs:156-160) or an
 * entry of descriptors[descriptor] (Context::list_binding, cel.rs:102-114).  Strings are NUL-terminated
 * UTF-8 owned by the caller. */
typedef struct rl_binding {
    uint32_t descriptor; /* index into the descriptor list, or RL_BIND_ROOT */
    uint32_t _pad;
    const char *key;
    const char *value;
} rl_binding;

int rl_matcher_create(rl_matcher **out);
void rl_matcher_destroy(rl_matcher *m);
/* The returned pointer is valid until the next failing call on this matcher (any thread): callers that share a
 * matcher between threads use the _copy form. */
const char *rl_matcher_last_error(rl_matcher *m);
int rl_matcher_last_error_copy(rl_matcher *m, char *out, uint32_t cap);

/* Limit::new + Storage::add_limit / update_limit (storage/mod.rs:60-83).  A limit with a known identity keeps
 * its limit_id and takes the new max_value / name.  *out_desc is what rl_limits_set needs. */
int rl_matcher_add_limit(rl_matcher *m, const char *ns, uint64_t max_value, uint64_t seconds,
                         const char *const *conditions, uint32_t n_cond, const char *const *variables,
                         uint32_t n_var, const char *name /* nullable */, rl_limit_desc *out_desc);
/* Storage::delete_limit (storage/mod.rs:93-117): the id is retired, never reused. */
/* The same with the reference's two entry points told apart: keep_existing != 0 is Storage::add_limit — a
 * HashSet::insert, i.e. a no-op that KEEPS the old max_value / name when an equal live limit exists
 * (storage/mod.rs:60-65) — keep_existing == 0 is update_limit (:67-83).  *out_existed (nullable) = 1 if an equal
 * live limit was already registered.  *out_desc always describes the limit as it now stands. */
int rl_matcher_add_limit_ex(rl_matcher *m, const char *ns, uint64_t max_value, uint64_t seconds,
                            const char *const *conditions, uint32_t n_cond, const char *const *variables,
                            uint32_t n_var, const char *name /* nullable */, int keep_existing,
                            rl_limit_desc *out_desc, int *out_existed /* nullable */);
int rl_matcher_delete_limit(rl_matcher *m, uint32_t limit_id);
/* Counters one request may produce before matching fails (default RL_MAX_COUNTERS_PER_REQUEST = what a default engine
 * takes per request, so that an oversized request is refused here, before anything is enqueued).  A caller whose engine
 * was created with a larger rl_config.max_counters_per_request (up to 64) raises it to match: the reference's "50
 * limits per namespace" scenarios (limitador/benches/bench.rs:65-90) then run end to end.  Raised past the engine's
 * maximum, requests over the latter match but cannot be shipped to the engine. */
int rl_matcher_set_counter_cap(rl_matcher *m, uint32_t cap);
/* RL_OK and *out_ns_id, or RL_FATAL if no limit was ever added for the namespace (no limits => allow,
 * lib.rs:434-440: the caller skips the engine). */
int rl_matcher_namespace_id(rl_matcher *m, const char *ns, uint32_t *out_ns_id);
/* Name of a limit (Authorization::Limited(name)), or NULL.  The pointer is valid only while no
 * rl_matcher_add_limit / _delete_limit runs; concurrent callers use the _copy form (*out_has_name nullable). */
const char *rl_matcher_limit_name(rl_matcher *m, uint32_t limit_id);
int rl_matcher_limit_name_copy(rl_matcher *m, uint32_t limit_id, char *out, uint32_t cap, int *out_has_name);

/* counters_that_apply for one request: *out_n counters written to out_ctrs (RL_FATAL if more than cap). */
int rl_matcher_counters(rl_matcher *m, uint32_t ns_id, const rl_binding *binds, uint32_t n_binds,
                        rl_counter *out_ctrs, uint32_t cap, uint32_t *out_n);
/* The same for n requests: request i owns binds[bind_off[i] .. bind_off[i+1]); fills out_ctr_off[0..n] and
 * out_ctrs (capacity cap counters) — pass both straight to rl_check_and_update_batch.  Thread-safe against
 * other matching calls; rl_matcher_add_limit / _delete_limit take the matcher exclusively. */
int rl_matcher_counters_batch(rl_matcher *m, uint64_t n, const uint32_t *ns_id, const uint32_t *bind_off,
                              const rl_binding *binds, uint32_t *out_ctr_off, rl_counter *out_ctrs, uint64_t cap);
/* counters_that_apply for n requests named by their namespace STRING, under ONE reader section (a batching stage matches
 * thousands of requests per call: no lock traffic per request — per-request calls from many threads bounce the matcher's
 * reader/writer lock between cores and stop scaling).  out_status[i]: 0 = matched (possibly no counter); 1 = no limit was
 * ever added for the namespace (nothing applies, lib.rs:434-440); 2 = more counters apply than one request may carry (the
 * request gets none).  out_ctr_off has n + 1 entries; out_ctrs needs room for the counter cap beyond the counters written. */
int rl_matcher_counters_batch_ns(rl_matcher *m, uint64_t n, const char *const *ns, const uint32_t *bind_off,
                                 const rl_binding *binds, uint32_t *out_ctr_off, rl_counter *out_ctrs, uint64_t cap,
                                 uint8_t *out_status);
/* CheckResult::response_header (lib.rs:235-275) for one request, from the load_counters outputs of
 * rl_check_and_update_batch: the request's counters are ordered by remaining (stable), then
 *   X-RateLimit-Limit     = "<max>, <max>;w=<seconds>[;name=\"<name>\"], ..."  (most restrictive first; a '"' in a
 *                            name becomes '\'')
 *   X-RateLimit-Remaining = remaining of the most restrictive counter
 *   X-RateLimit-Reset     = its ttl in whole seconds
 * max, seconds and name come from the matcher's limits.  Each buffer receives a NUL-terminated string (all
 * empty when n == 0); RL_FATAL if one is too small or a limit_id is unknown. */
int rl_matcher_response_headers(rl_matcher *m, const rl_counter *ctrs, const uint64_t *remaining,
                                const uint64_t *ttl_us, uint32_t n, char *out_limit, uint32_t cap_limit,
                                char *out_remaining, uint32_t cap_remaining, char *out_reset, uint32_t cap_reset);
/* The same for the n requests of a CSR (request i owns ctrs[ctr_off[i] .. ctr_off[i+1]), remaining / ttl_us indexed like
 * ctrs) under one reader section: request i's three values are written NUL-terminated, one after the other (Limit,
 * Remaining, Reset), at out + out_off[i]; out_off has n + 1 entries; a request without counters gets three empty strings.
 * *out_len = bytes needed; RL_FATAL if cap is too small (out_len still set). */
int rl_matcher_response_headers_batch(rl_matcher *m, uint64_t n, const uint32_t *ctr_off, const rl_counter *ctrs,
                                      const uint64_t *remaining, const uint64_t *ttl_us, char *out, uint64_t cap,
                                      uint64_t *out_off, uint64_t *out_len);
/* The matcher inside the batching front (SURVEY §8 f1 + §8b "Threading"): one request as the reference's callers have it
 * — a namespace and a context — through counters_that_apply on the CALLING thread (matching threads run in parallel:
 * the matcher is read-shared) and then through the front's queue (include/rl_engine.h: rl_front_check_and_update), i.e.
 * RateLimiter::check_rate_limited_and_update (lib.rs:425-464) end to end.  out_ctrs (nullable, capacity
 * RL_MAX_COUNTERS_PER_REQUEST) / *out_n_ctrs (nullable) receive the counters that applied; out_remaining / out_ttl_us
 * are indexed like them.  This helper matches at most RL_MAX_COUNTERS_PER_REQUEST counters whatever the engine's
 * max_counters_per_request: a wider request is matched by the caller (rl_matcher_counters) and shipped with
 * rl_front_check_and_update, which takes up to the engine's maximum.  A namespace without limits, or a context no limit applies to, is "not limited" without
 * touching the store (lib.rs:434-440). */
int rl_front_check_and_update_bindings(rl_front *f, rl_matcher *m, const char *ns, const rl_binding *binds, uint32_t n_binds,
                                       uint64_t delta, uint64_t now_us, int load_counters, uint8_t *out_limited,
                                       uint32_t *out_first_limited, rl_counter *out_ctrs, uint32_t *out_n_ctrs,
                                       uint64_t *out_remaining, uint64_t *out_ttl_us, uint64_t *out_seq);

/* The 96-bit counter key of n (variable source, value) pairs (any order): key_lo = digest bits 0..63,
 * key_hi = bits 64..95.  BLAKE2b-96 over the pairs sorted by source, each string length-prefixed (u32 LE).
 * (0, 0) for n == 0 (unqualified counter). */
void rl_counter_key(const char *const *sources, const char *const *values, uint32_t n, uint64_t *key_lo,
                    uint64_t *key_hi);

#ifdef __cplusplus
}
#endif
#endif /* RL_MATCH_H */
