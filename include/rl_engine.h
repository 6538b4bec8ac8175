/*
 * rl_engine.h — C-ABI of the H100-native batched rate-limit engine (librl_engine.so).
 *
 * This is the drop-in boundary for ONE path of Kuadrant/limitador:
 *   RateLimiter::check_rate_limited_and_update  (limitador/src/lib.rs:425-464)
 *   = is_rate_limited + update_counters over the in-memory CounterStorage
 *   (limitador/src/storage/in_memory.rs, atomic_expiring_value.rs).
 *
 * Each entry point replaces one method of `trait CounterStorage`
 * (limitador/src/storage/mod.rs:279-292), batched: the caller (the Rust crate's batching
 * front, see INTEGRATION.md) performs limit matching on the CPU (lib.rs:507-522) and
 * ships plain arrays; the engine owns an HBM-resident counter table and runs hand-written
 * sm_90a kernels.  A batch is applied EXACTLY as if its requests had been submitted one
 * at a time, in array order, to the reference's InMemoryStorage with the clock reading
 * now_us[i] at request i.
 *
 * Conventions
 *   - All functions return RL_OK / RL_TRANSIENT / RL_FATAL (storage/mod.rs:312-339:
 *     StorageErr{msg, transient}); rl_last_error() gives the message.  A full table is an
 *     error (RL_TRANSIENT), never a silent allow or eviction.
 *   - No pointer is retained after a call returns.  `mem` says where EVERY array argument
 *     of that call lives: RL_MEM_HOST (pageable or pinned) or RL_MEM_DEVICE (same device
 *     as the engine).  RL_MEM_DEVICE calls are enqueued on the engine's stream and return
 *     immediately; rl_sync() waits and reports deferred errors.
 *   - Time is µs since the UNIX epoch (atomic_expiring_value.rs:62-66); 1 <= now_us < 2^62.
 *   - Counter identity = (limit_id, key_lo, key_hi) with key_hi < 2^32: a 96-bit digest of
 *     the counter's resolved variable values (counter.rs:123-138); ignored for
 *     unqualified limits (no variables).
 *   - The engine handle may be used from one thread at a time (the batching front owns it).
 */
#ifndef RL_ENGINE_H
#define RL_ENGINE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rl_engine rl_engine;

enum { RL_OK = 0, RL_TRANSIENT = 1, RL_FATAL = 2 };
enum { RL_MEM_HOST = 0, RL_MEM_DEVICE = 1,
       /* pinned host buffers that stay valid until rl_sync(): rl_check_and_update_records returns after
        * ENQUEUEING the H2D copy, the kernels and the D2H copy of the verdicts (needs RL_FLAG_PIPELINE;
        * otherwise, or with load_counters outputs, it behaves like RL_MEM_HOST) */
       RL_MEM_HOST_ASYNC = 2 };
#define RL_NONE 0xFFFFFFFFu
/* out_limited[i] of a request that could NOT be evaluated (malformed key, full table region, exchange block
 * overflow): the call (or the next rl_sync) also reports the error; the byte is never a silent 0 = allowed */
#define RL_VERDICT_ERROR 0xFFu
#define RL_MAX_COUNTERS_PER_REQUEST 16 /* counters one request may name (general form) on a default engine; the matcher
                                          refuses more unless its cap is raised */
#define RL_MAX_COUNTERS_PER_REQUEST_WIDE 64 /* the most rl_config.max_counters_per_request may ask for */
/* test aid: the in-kernel row grouping table gives every row one of only four home slots, so that
 * distinct rows collide and its linear probing is exercised to full length */
#define RL_FLAG_DEBUG_WEAK_TAGS 1u
/* Record calls with RL_MEM_DEVICE / RL_MEM_HOST_ASYNC buffers are software-pipelined over three internal
 * streams: probe+count of call s+2 and scan+scatter of call s+1 overlap the replay of call s.  Results are
 * the same; outputs of such calls are ordered on the caller's stream only after rl_fence() (or rl_sync). */
#define RL_FLAG_PIPELINE 2u
/* rl_stats.chunks / replay_rounds / chained_chunks / ordered_chunks / phase_cycles are accounted by the
 * replay kernel (a few atomics per chunk, ~7 % of a 65536-request step); without the flag they stay 0. */
#define RL_FLAG_KERNEL_STATS 4u
/* Device-side event trace: the kernels of a step stamp the GPU's nanosecond timer at their start and end into a
 * ring of 65536 events (rl_trace_dump), so the timeline of a pipelined / sharded step can be read without a
 * profiler.  One atomic and one 16-B store per kernel and event. */
#define RL_FLAG_TRACE 8u
/* Hot rows (DESIGN.md §3.4): a table row that dominates its replay chunks gets a partition of its own and is replayed
 * by one CTA of k_hot over its whole request list — the hot-key regime of BASELINE.json configs[4].  Opt-in (also
 * RL_HOT=1 in the environment): for Zipf(1.1) traffic at batch 65536 the chained chunks of k_main are as fast. */
#define RL_FLAG_HOT_ROWS 16u

typedef struct rl_config {
    uint32_t struct_size;    /* sizeof(rl_config) */
    int32_t device;          /* CUDA device ordinal */
    uint64_t capacity_rows;  /* table rows (distinct counter keys per row group); rounded up to 2^k.
                                Replaces InMemoryStorage::new(cache_size), in_memory.rs:205-212 */
    uint32_t cells_per_row;  /* 1, 3 or 7: limits of one namespace sharing one variable set live
                                in one row (row bytes = 16 * (1 + cells)) */
    uint32_t max_batch;      /* max requests per call */
    uint32_t max_counters;   /* max total counters per CSR call (0 = 4 * max_batch) */
    uint32_t regions;        /* 0 = auto; power of two */
    uint32_t flags;          /* RL_FLAG_* */
    uint32_t max_counters_per_request; /* counters one request may name, and limits one namespace may have on the record
                                          path: 0 or 16 = RL_MAX_COUNTERS_PER_REQUEST (a 17-counter request is refused
                                          before the table is touched); 17..64 = a wide engine; anything else is refused
                                          by rl_engine_create.  Declares a maximum, it does not choose a code path: a
                                          batch runs the wide kernels only if it holds a request of more than 16
                                          counters (DESIGN.md §9g), so narrow traffic costs the same on a wide engine */
} rl_config;

/* A limit as the storage sees it (limit.rs:177-214: identity excludes max_value/name).
 * limit_id is a dense id interned by the caller; (ns_id, varset_id) tells the engine
 * which limits share a variable set (varset_id 0 = no variables = unqualified). */
typedef struct rl_limit_desc {
    uint32_t limit_id;
    uint32_t ns_id;
    uint32_t varset_id;
    uint32_t qualified; /* !variables.is_empty(), counter.rs:108-110 */
    uint64_t max_value;
    uint64_t window_us; /* seconds * 1e6, counter.rs:76-78 */
} rl_limit_desc;

/* 32-byte request record (SURVEY §8d): limit set implied by ns_id (every limit of the
 * namespace applies, registration order), one key for all qualified limits. */
typedef struct rl_record {
    uint32_t ns_id;
    uint32_t hits_addend; /* RLS uint32 hits_addend (envoy_rls/server.rs:131-135), used as delta */
    uint64_t key_lo;
    uint64_t key_hi;      /* bits 0..31: digest bits 64..95; bits 32..55: must be 0; bits 56..63: the lane
                             byte, opaque to every decision call (rl_record_lane_put/_gather use it) */
    uint64_t now_us;
} rl_record;
#define RL_RECORD_LANE_BYTE 23 /* byte offset of the lane byte inside rl_record */
#define RL_RECORD_KEY_HI_MASK 0x00FFFFFFFFFFFFFFull

/* 16-byte wire form of rl_record for batches stamped with ONE clock reading (what a batching front does: it reads
 * the clock once when it drains its queue): halves the bytes a host-fed step moves over PCIe.
 *   word0 = ns_id (bits 0..23) | hits_addend (bits 24..31, 1..255) | key_hi (bits 32..63: digest bits 64..95)
 *   word1 = key_lo
 * Namespaces with id >= 2^24 or hits_addend > 255 use the 32-byte form. */
typedef struct rl_record16 {
    uint64_t ns_hits_keyhi;
    uint64_t key_lo;
} rl_record16;

/* One counter of a request in the general (CSR) form: Counter = limit + set_variables. */
typedef struct rl_counter {
    uint32_t limit_id;
    uint32_t _pad;
    uint64_t key_lo;
    uint64_t key_hi;
} rl_counter;

typedef struct rl_stats {
    uint64_t kernel_launches; /* kernels launched by this engine since creation */
    uint64_t batches;
    uint64_t requests;
    uint64_t capacity_rows;
    uint32_t regions;
    uint32_t row_bytes;
    uint32_t fixed_point_rounds; /* speculative rounds run for multi-row requests (last batch) */
    uint32_t _pad;
    uint64_t chunks;         /* (RL_FLAG_KERNEL_STATS) k_main: chunks of <= 256 accesses replayed */
    uint64_t replay_rounds;  /* k_main: run-length rounds summed over chunks */
    uint64_t chained_chunks; /* chunks of heavy regions (optimistic concurrency control) */
    uint64_t ordered_chunks; /* ... of which had to commit in order */
    uint64_t phase_cycles[6]; /* k_main SM cycles summed over chunks: load, group, stage, replay, commit protocol, write-back */
    uint32_t hot_rows;        /* table rows that currently have a partition of their own (k_hot), of 256 slots */
    uint32_t _pad2;
} rl_stats;

int rl_engine_create(const rl_config *cfg, rl_engine **out);
void rl_engine_destroy(rl_engine *e);
/* The engine's max_counters_per_request (16 for a default engine, and for e == NULL). */
uint32_t rl_engine_max_counters_per_request(rl_engine *e);
/* Message of the last non-OK status on this engine (never NULL). */
const char *rl_last_error(rl_engine *e);
/* Use the caller's CUDA stream (a cudaStream_t) for all subsequent work; NULL = the
 * engine's own stream.  rl_engine_stream returns the stream in use. */
int rl_engine_set_stream(rl_engine *e, void *cuda_stream);
void *rl_engine_stream(rl_engine *e);
/* Make the engine's stream wait for every pipelined call issued so far (RL_FLAG_PIPELINE);
 * a no-op otherwise.  Does not block the host. */
int rl_fence(rl_engine *e);
/* Same for one call only: age 0 = the last pipelined call, 1 = the one before it (later calls keep
 * running).  Lets a caller overlap the post-processing of call s with the kernels of call s+1. */
int rl_fence_call(rl_engine *e, uint32_t age);
/* Wait for all enqueued work; returns and clears any deferred device-side error. */
int rl_sync(rl_engine *e);
int rl_get_stats(rl_engine *e, rl_stats *out);
/* RL_FLAG_TRACE: copy (and clear) the event ring.  out_ev[i] = event id | end << 8 (ids: 1 front, 2 replay,
 * 3 exchange count, 4 exchange scatter, 5 inbox wait, 6 verdict return, 7 verdict wait, 8 verdict gather),
 * out_seq[i] = call / exchange step number, out_ns[i] = GPU nanosecond timer.  Synchronises the device. */
int rl_trace_dump(rl_engine *e, uint32_t cap, uint32_t *out_ev, uint32_t *out_seq, uint64_t *out_ns, uint32_t *out_count);

/* CounterStorage::add_counter (storage/mod.rs:281, in_memory.rs:38-44) + Storage::update_limit
 * (storage/mod.rs:67-83): new ids are registered (unqualified ⇒ counter pre-created as
 * (0, EPOCH)); for a live id only max_value may change. */
int rl_limits_set(rl_engine *e, const rl_limit_desc *limits, uint32_t n);
/* Storage::delete_limit (storage/mod.rs:93-117): delete_counters + forget the limits. */
int rl_limits_delete(rl_engine *e, const uint32_t *limit_ids, uint32_t n);

/* CounterStorage::check_and_update (storage/mod.rs:283-288, in_memory.rs:72-156), batched.
 * Record form.  out_limited[i] = 1 iff Authorization::Limited; out_first_limited[i] =
 * limit id the reference would name (in_memory.rs:91-94,99-101) or RL_NONE;
 * with load_counters != 0, out_remaining/out_ttl_us[i*out_stride + k] describe the k-th
 * limit of the namespace (Counter::set_remaining / set_expires_in).  Nullable outputs:
 * out_first_limited, out_remaining, out_ttl_us. */
int rl_check_and_update_records(rl_engine *e, uint64_t n, const rl_record *recs, int load_counters,
                                int mem, uint8_t *out_limited, uint32_t *out_first_limited,
                                uint64_t *out_remaining, uint64_t *out_ttl_us, uint32_t out_stride);
/* The record form over 16-byte records, all stamped now_us (single-row namespaces only, no load_counters). */
int rl_check_and_update_compact(rl_engine *e, uint64_t n, const rl_record16 *recs, uint64_t now_us, int mem,
                                uint8_t *out_limited, uint32_t *out_first_limited);
/* General form: request i owns ctrs[ctr_off[i] .. ctr_off[i+1]) (at most max_counters_per_request), counters are
 * processed unqualified-first then in the given order (in_memory.rs:105,121);
 * out_remaining/out_ttl_us are indexed like ctrs.  An empty counter list is "not limited"
 * (lib.rs:434-440). */
int rl_check_and_update_batch(rl_engine *e, uint64_t n, const uint32_t *ctr_off, const rl_counter *ctrs,
                              const uint64_t *delta, const uint64_t *now_us, int load_counters, int mem,
                              uint8_t *out_limited, uint32_t *out_first_limited,
                              uint64_t *out_remaining, uint64_t *out_ttl_us);

/* CounterStorage::is_within_limits (in_memory.rs:20-35) folded over a request's counters
 * as RateLimiter::is_rate_limited does (lib.rs:362-409): read-only, given order, first
 * counter over its limit wins.  Any number of counters per request, on every engine. */
int rl_is_within_limits_batch(rl_engine *e, uint64_t n, const uint32_t *ctr_off, const rl_counter *ctrs,
                              const uint64_t *delta, const uint64_t *now_us, int mem,
                              uint8_t *out_limited, uint32_t *out_first_limited);
int rl_is_within_limits_records(rl_engine *e, uint64_t n, const rl_record *recs, int mem,
                                uint8_t *out_limited, uint32_t *out_first_limited);

/* CounterStorage::update_counter (in_memory.rs:47-69) for every counter of every request
 * (RateLimiter::update_counters, lib.rs:411-423): unconditional, may exceed max_value. */
int rl_update_batch(rl_engine *e, uint64_t n, const uint32_t *ctr_off, const rl_counter *ctrs,
                    const uint64_t *delta, const uint64_t *now_us, int mem);
int rl_update_records(rl_engine *e, uint64_t n, const rl_record *recs, int mem);

/* CounterStorage::get_counters (in_memory.rs:158-187): every counter of the namespaces of
 * the given limits with ttl(now_us) > 0.  Host output arrays of capacity cap; *out_count =
 * number found (may exceed cap). */
int rl_get_counters(rl_engine *e, const uint32_t *limit_ids, uint32_t n, uint64_t now_us, uint64_t cap,
                    uint32_t *out_limit_id, uint64_t *out_key_lo, uint64_t *out_key_hi,
                    uint64_t *out_remaining, uint64_t *out_ttl_us, uint64_t *out_count);
/* CounterStorage::delete_counters (in_memory.rs:189-195,241-257). */
int rl_delete_counters(rl_engine *e, const uint32_t *limit_ids, uint32_t n);
/* CounterStorage::clear (in_memory.rs:197-201): drops ONLY unqualified counters. */
int rl_clear(rl_engine *e);
/* TTL sweep (no reference function; north_star's companion kernel): invalidate every
 * qualified counter with expiry <= now_us and free rows left empty.  Mirrored in the
 * oracle as lo_invalidate_expired.  *out_invalidated (nullable) = counters dropped. */
int rl_sweep(rl_engine *e, uint64_t now_us, uint64_t *out_invalidated);
/* Tombstone reclamation (no reference function: moka evicts, in_memory.rs:205-212).  rl_sweep turns emptied rows into
 * tombstones, which keep lengthening the probe chains of their region.  rl_compact rebuilds, in place, every region whose
 * tombstones reach min_tombstone_pct percent of its rows (0 = any region with a tombstone): the region's rows go to a
 * scratch slab (one table-sized device allocation for the call), the region is cleared and the rows that still hold a
 * counter are inserted again by the hot path's own probing rule.  Rows whose cells are all (0, 0) hold nothing and are
 * dropped as well.  Observable state is unchanged: what rl_counters_export(..., now_us = 0) lists before == after.
 * Serialise with the request path. */
typedef struct rl_compact_stats {
    uint64_t regions;          /* table regions */
    uint64_t regions_rebuilt;
    uint64_t rows_live;        /* rows holding a key before the call, whole table */
    uint64_t rows_tombstoned;  /* tombstones before the call, whole table */
    uint64_t rows_moved;       /* rows inserted again in the rebuilt regions */
    uint64_t rows_reclaimed;   /* slots freed in the rebuilt regions: tombstones + rows without any counter */
} rl_compact_stats;
int rl_compact(rl_engine *e, uint32_t min_tombstone_pct, rl_compact_stats *out /* nullable */);

/* ---- Per-namespace metrics on the device (SURVEY §8 f3) ----------------------------------------------------------
 * The reference increments authorized_calls / authorized_hits / limited_calls once per request on the host, after the
 * decision (limitador-server/src/prometheus_metrics.rs:93-125, called at envoy_rls/server.rs:183-195).  Here they are ONE
 * segmented reduction per decided batch, keyed by the records' ns_id (and, for limited_calls by limit name, by the limit
 * named in out_first_limited), accumulated in device memory until read.
 *   rl_ns_metrics_enable    : from now on every rl_check_and_update_records / _compact call adds its batch, with one
 *                             kernel enqueued right behind the replay (same stream; nothing blocks).  Sharded steps
 *                             decide other ranks' requests: there the SOURCE rank accumulates what it collected with
 *                             rl_ns_metrics_accumulate.
 *   rl_ns_metrics_accumulate: add an already decided batch: n records of record_bytes (32 = rl_record, 16 = rl_record16),
 *                             their verdict bytes (RL_VERDICT_ERROR entries are not counted) and, nullable, the limit ids
 *                             named.  mem = RL_MEM_HOST or RL_MEM_DEVICE for all three arrays.
 *   rl_ns_metrics_read      : copy out (and optionally reset) the counts of namespaces [0, ns_cap) and limits
 *                             [0, limits_cap); *out_dropped = requests not counted (error verdicts).  Nullable outputs. */
int rl_ns_metrics_enable(rl_engine *e, int on);
int rl_ns_metrics_accumulate(rl_engine *e, uint64_t n, const void *recs, uint32_t record_bytes, const uint8_t *limited,
                             const uint32_t *first_limited, int mem);
int rl_ns_metrics_read(rl_engine *e, uint32_t ns_cap, uint64_t *out_authorized_calls, uint64_t *out_authorized_hits,
                       uint64_t *out_limited_calls, uint32_t limits_cap, uint64_t *out_limited_by_limit,
                       uint64_t *out_dropped, int reset);

/* ---- Counter snapshots: restart, resize or re-shard an engine without losing counters -----------------------------
 * A snapshot is the five arrays rl_counters_export returns.  Export it from one engine and import it into another (one
 * with another capacity, cells_per_row or region count, or another rank of a sharded store): the counters go on exactly
 * where they were.  Limit ids are the caller's: the target must register the same limits under the same ids
 * (rl_limits_get lists them) before the import.  No reference function: the reference keeps counters across restarts
 * only in its disk store (limitador/src/storage/disk/rocksdb_storage.rs). */
/* Every present counter of the selected namespaces (ns_ids == NULL: all) as (limit_id, key, value, expiry_us); an
 * unqualified counter whose row was never touched is (limit_id, 0, 0, 0, 0).  now_us == 0: the exact state.
 * now_us > 0: qualified counters with 0 < expiry <= now_us are left out, i.e. the state rl_sweep(now_us) would leave.
 * mem = RL_MEM_HOST or RL_MEM_DEVICE for the five outputs; unordered (the counters of one row are adjacent), at most
 * cap written, *out_count = number found (may exceed cap).  Does not change the table. */
int rl_counters_export(rl_engine *e, const uint32_t *ns_ids, uint32_t n_ns, uint64_t now_us, uint64_t cap, int mem,
                       uint32_t *out_limit_id, uint64_t *out_key_lo, uint64_t *out_key_hi,
                       uint64_t *out_value, uint64_t *out_expiry_us, uint64_t *out_count);
/* Set n counters to exactly (value, expiry_us).  A present counter is replaced; other counters are untouched (import
 * into a fresh engine for a clone).  limit_id is resolved against THIS engine's registry, so the target may have
 * another capacity, cells_per_row, region count or row-group assignment.  The key is ignored for unqualified limits,
 * whose counters become present (as after add_counter).  Refused with RL_FATAL before any counter changes: unknown
 * limit id, key_hi >= 2^32, a qualified counter with expiry 0, the same counter twice.  A full region: RL_TRANSIENT,
 * and again no counter changes (a refused call leaves the table as it was, rows included).  rl_last_error names the
 * first refused entry.  Serialise with the request path (as
 * rl_compact). */
int rl_counters_import(rl_engine *e, uint64_t n, const uint32_t *limit_id, const uint64_t *key_lo,
                       const uint64_t *key_hi, const uint64_t *value, const uint64_t *expiry_us, int mem);
/* Every registered limit, ascending id (what a snapshot must be restored against).  At most cap written,
 * *out_n = number registered. */
int rl_limits_get(rl_engine *e, uint32_t cap, rl_limit_desc *out, uint32_t *out_n);

/* ---- Change tracking: the counters changed since the last drain (DESIGN.md §9k) ------------------------------------
 * What a journal on disk needs to bring a service's counters back after a crash, without moving the whole table each
 * time.  The decision kernels do not take part: a drain compares the table with a shadow copy in one pass of its own,
 * so an engine that never drains pays nothing.  No reference function: the reference's disk store writes every update
 * through RocksDB's write-ahead log (limitador/src/storage/disk/rocksdb_storage.rs).
 *   rl_counters_track  on = 1: allocate the shadow, capacity_rows x row bytes of device memory (RL_TRANSIENT when there
 *                      is no room), and make the next drain full.  on = 0: free it.
 *   rl_counters_drain  full drain (*out_full = 1): exactly rl_counters_export(e, NULL, 0, 0, cap, mem, ...).  It is the
 *                      first drain after rl_counters_track, and the first after any call that can move rows or re-map
 *                      cells: rl_limits_set, rl_limits_delete, rl_delete_counters, rl_clear, rl_compact and
 *                      rl_counters_import (rl_rls_configure runs through them).
 *                      delta drain (*out_full = 0): every counter whose (value, expiry) differs from what the previous
 *                      drain saw, as (limit_id, key, value, expiry_us); a counter that is no longer listed is
 *                      (limit_id, key, 0, 0).  One row position can go from key A to a tombstone to key B between two
 *                      drains: then A's counters come out absent and B's present, so apply a delta's absents before its
 *                      presents.  Replaying the full drain and then every delta in order gives exactly what
 *                      rl_counters_export(e, NULL, 0, 0, ...) lists at the last drain.
 *                      Both: mem = RL_MEM_HOST or RL_MEM_DEVICE for the five outputs, unordered, *out_count = entries
 *                      found, at most cap written.  When *out_count > cap the drain is not consumed (the shadow stays
 *                      as it was): the same drain can be repeated with a larger cap.  Needs tracking on.  Serialise with the request path (as rl_compact);
 *                      pipelined record calls are fenced first. */
int rl_counters_track(rl_engine *e, int on);
int rl_counters_drain(rl_engine *e, uint64_t cap, int mem, uint32_t *out_limit_id, uint64_t *out_key_lo,
                      uint64_t *out_key_hi, uint64_t *out_value, uint64_t *out_expiry_us, uint64_t *out_count,
                      int *out_full);

/* Measurement aid (bench.py roofline leg): between begin and end the engine brackets every
 * launch of its dominant kernel (k_main) with CUDA events on the launching stream;
 * end() synchronises and returns the summed device time and the launch count. */
int rl_profile_begin(rl_engine *e);
int rl_profile_end(rl_engine *e, double *out_main_ms, uint64_t *out_main_launches);

/* Multi-GPU exchange helper (SURVEY §8e): stable bucketing of n device-resident records by
 * owner = rl_owner_of(ns_id, world).  Writes the permuted records to d_out_recs, the
 * source index of every permuted record to d_out_src (uint32), and the per-owner counts
 * to h_counts[world] (host).  All d_* pointers are device memory. */
int rl_bucket_by_owner(rl_engine *e, uint64_t n, const rl_record *d_recs, uint32_t world,
                       rl_record *d_out_recs, uint32_t *d_out_src, uint64_t *h_counts);
/* Sync-free variant for fixed-size exchanges: owner o's records go to d_out_recs[o*slot_cap ...]
 * (stable, at most slot_cap of them; the unused slots of d_out_recs[world*slot_cap] are filled with
 * 0xFF bytes = records of a namespace without limits, which the engine ignores).  d_out_pos[i] = slot
 * of record i (or ~0 when its block overflowed, in which case *d_overflow |= 1).  Enqueued on
 * the engine's stream; nothing is copied to the host. */
int rl_bucket_by_owner_padded(rl_engine *e, uint64_t n, const rl_record *d_recs, uint32_t world, uint32_t slot_cap,
                              rl_record *d_out_recs, uint32_t *d_out_pos, uint32_t *d_overflow);
/* out[i] = in[pos[i]] (0 where pos[i] == ~0), device pointers. */
int rl_gather_u8(rl_engine *e, uint64_t n, const uint8_t *d_in, const uint32_t *d_pos, uint8_t *d_out);
/* Pipelined exchange: the verdict bytes of an earlier step travel back in the lane byte of this
 * step's records, so a sharded step costs one all-to-all instead of two.
 *   rl_record_lane_put   : lane byte of d_recs[i] = d_lane[i], i < n_slots (after rl_bucket_by_owner_padded)
 *   rl_record_lane_gather: d_out[i] = lane byte of d_recs[d_pos[i]] (0 where d_pos[i] == ~0) */
int rl_record_lane_put(rl_engine *e, uint64_t n_slots, rl_record *d_recs, const uint8_t *d_lane);
int rl_record_lane_gather(rl_engine *e, uint64_t n, const rl_record *d_recs, const uint32_t *d_pos, uint8_t *d_out);
/* out[src[i]] = in[i] for i < n (device pointers): return verdict bytes to request order. */
int rl_unpermute_u8(rl_engine *e, uint64_t n, const uint8_t *d_in, const uint32_t *d_src, uint8_t *d_out);
uint32_t rl_owner_of(uint32_t ns_id, uint32_t world);

/* ---- Namespace-sharded peer exchange (SURVEY §8e) ----------------------------------------------
 * One process (and one engine) per GPU; the key space shards by rl_owner_of(ns_id, world) — every counter
 * of a request belongs to its namespace (lib.rs:512), the property the reference relies on for Redis
 * Cluster hash tags (storage/keys.rs:1-13).  Every rank owns an exchange slab in its HBM which the other
 * ranks map (CUDA IPC; NVLink / NVSwitch peer access).  A step:
 *   send    : bucket my slice of the global batch by owner (stable) and STORE the 32-B records straight
 *             into the owners' inboxes over NVLink, then publish fill + step flag;
 *   decide  : wait (on the device) for the blocks of all sources, run check_and_update over the inbox in
 *             (source rank, source index) order — the canonical stream order of the sharded store — and
 *             store the verdict bytes straight back into the sources' verdict inboxes;
 *   collect : wait (on the device) for every owner's verdicts of the step sent `lag` steps ago and put them
 *             back in request order into the out_limited buffer given with that step.
 * No NCCL call, no padding and no host synchronisation on the data path; `lag`+1 steps are in flight (`lag`+2
 * buffers, so that a send never waits for an earlier step's delivery).
 * Every rank must issue the same sequence of calls.  cap = max records per rank and step; an owner can
 * receive up to world*cap records in a step (rl_config.max_batch bounds it: more is an error, RL_FATAL at
 * the next rl_sync).  All d_* pointers are device memory; everything is enqueued, nothing blocks the host. */
typedef struct rl_shard rl_shard;
int rl_shard_create(rl_engine *e, uint32_t rank, uint32_t world, uint32_t cap, uint32_t lag, rl_shard **out);
void rl_shard_destroy(rl_shard *s);
/* 64-byte CUDA IPC handle (cudaIpcGetMemHandle) of this rank's slab, to be all-gathered by the caller */
int rl_shard_ipc_handle(rl_shard *s, void *out64);
/* handles64: world x 64 bytes, rank-major; opens every peer's slab (cudaIpcOpenMemHandle) */
int rl_shard_connect_ipc(rl_shard *s, const void *handles64);
/* same-process peers (several engines in one process): slabs[r] = rl_shard_slab of rank r */
int rl_shard_connect_ptrs(rl_shard *s, void *const *slabs);
void *rl_shard_slab(rl_shard *s);
uint64_t rl_shard_slab_bytes(rl_shard *s);
int rl_shard_send(rl_shard *s, uint64_t n, const rl_record *d_recs, uint8_t *d_out_limited);
int rl_shard_decide(rl_shard *s);
/* *out_done (nullable) = the out_limited buffer whose delivery was enqueued by this call, or NULL.  Deliveries run on
 * a stream of the shard's own (the caller's stream, which carries the sends, never parks on a verdict wait):
 * rl_shard_fence orders the caller's stream after every delivery enqueued so far (it does not block the host);
 * rl_shard_flush does it too. */
int rl_shard_collect(rl_shard *s, uint8_t **out_done);
int rl_shard_fence(rl_shard *s);
/* send + decide + collect: the one call of the one-process-per-GPU deployment */
int rl_shard_step(rl_shard *s, uint64_t n, const rl_record *d_recs, uint8_t *d_out_limited, uint8_t **out_done);
/* deliver every step still in flight (all ranks must have issued the same steps) */
int rl_shard_flush(rl_shard *s);
/* debugging aid: host copy of this rank's control words, out[(buf*world + peer)*4 + {0 fill, 1 record flag,
 * 2 verdict flag}] for buf < lag+2, then the steps sent, decided, collected; out holds (lag+2)*world*4 + 3 words */
int rl_shard_debug(rl_shard *s, uint32_t *out);

/* ---- The general (CSR) form of the sharded exchange: served requests on a namespace-sharded store ----------------
 * What rl_rls_serve and rl_http_serve hand their engine: request i owns counters ctrs[ctr_off[i] .. ctr_off[i+1]), with
 * its own delta and now_us.  Its owner is rl_owner_of(ns of its first counter's limit, world): every counter of a request
 * belongs to the request's namespace (lib.rs:512).  A step:
 *   send    : bucket the batch by owner (stable) and STORE each request (a header: counter count, delta, now_us, op and
 *             load flag; then its counters in their order) into its owner's inbox block, then publish the block (request
 *             and counter fill, the digest of this rank's limit registry) and the step flag;
 *   decide  : wait (on the device) for every source's block, lay the inbox out as one CSR in (source rank, index at the
 *             source) order -- the canonical order -- and run one general-form engine call per run of equal (op, load)
 *             (one read of the sizes and runs to the host); the outputs go back to every source;
 *   collect : wait (on the device) for every owner and put verdicts, first_limited and, for requests with load_counters,
 *             remaining / ttl back in request and counter order.  Synchronises the engine's stream.
 * Results are those of the ranks' batches applied one after another, in rank order, to one engine.  Every rank issues
 * the same calls (a rank without traffic sends n = 0), one step at a time (no lag).
 * Guards, each for whole steps so that no peer is ever left waiting:
 *   - cap_requests / cap_counters per source and step (multiples of 16); create refuses world x cap beyond the engine's
 *     max_batch / max_counters.  A batch over its caps sends empty blocks; its requests get RL_VERDICT_ERROR and collect
 *     returns RL_TRANSIENT.
 *   - a source whose registry digest (limit ids, ns, varset, qualified, window, max_value) differs from the owner's: its
 *     requests get RL_VERDICT_ERROR and the owner's decide returns RL_FATAL naming both ranks.
 *   - a failed engine call (a full region, ...): its run's requests get RL_VERDICT_ERROR at their sources, decide returns
 *     RL_TRANSIENT with the call's message; other runs and owners are unaffected.
 * Only a call refused for its own arguments sends nothing (no peers connected, the previous step not collected, an
 * unknown op, decide before send): that is a broken protocol and leaves the group out of step.  Any other failure on
 * a rank (null or over-cap arrays, an engine that cannot run, a failed engine call) still sends and returns its step,
 * with error verdicts, so that no peer is left waiting.
 * All d_* pointers are device memory of the engine's device and stay valid until collect returns; d_load (nullable) =
 * one load_counters flag per request, else load_all for every request; load_counters applies to
 * RL_SHARD_CHECK_AND_UPDATE only.  Nullable outputs: d_first_limited, d_remaining / d_ttl_us (indexed like ctrs). */
enum { RL_SHARD_CHECK_AND_UPDATE = 0, RL_SHARD_IS_WITHIN = 1, RL_SHARD_UPDATE = 2 };
typedef struct rl_shard_batch rl_shard_batch;
int rl_shard_batch_create(rl_engine *e, uint32_t rank, uint32_t world, uint32_t cap_requests, uint32_t cap_counters,
                          rl_shard_batch **out);
void rl_shard_batch_destroy(rl_shard_batch *s);
void *rl_shard_batch_slab(rl_shard_batch *s);
rl_engine *rl_shard_batch_engine(rl_shard_batch *s); /* the engine it was created on */
/* as rl_shard_ipc_handle / rl_shard_connect_ipc / rl_shard_connect_ptrs */
int rl_shard_batch_ipc_handle(rl_shard_batch *s, void *out64);
int rl_shard_batch_connect_ipc(rl_shard_batch *s, const void *handles64);
int rl_shard_batch_connect_ptrs(rl_shard_batch *s, void *const *slabs);
int rl_shard_batch_send(rl_shard_batch *s, uint64_t n, uint64_t n_ctr, const uint32_t *d_ctr_off, const rl_counter *d_ctrs,
                        const uint64_t *d_delta, const uint64_t *d_now_us, int op, const uint8_t *d_load, int load_all);
int rl_shard_batch_decide(rl_shard_batch *s);
int rl_shard_batch_collect(rl_shard_batch *s, uint8_t *d_limited, uint32_t *d_first_limited, uint64_t *d_remaining,
                           uint64_t *d_ttl_us);
/* send + decide + collect: the one call of the one-process-per-GPU deployment (returns the worse status) */
int rl_shard_batch_step(rl_shard_batch *s, uint64_t n, uint64_t n_ctr, const uint32_t *d_ctr_off, const rl_counter *d_ctrs,
                        const uint64_t *d_delta, const uint64_t *d_now_us, int op, const uint8_t *d_load, int load_all,
                        uint8_t *d_limited, uint32_t *d_first_limited, uint64_t *d_remaining, uint64_t *d_ttl_us);

/* ---- Batching front (SURVEY §8b threading row) ---------------------------------------------
 * Thread-safe, blocking, one request per call: concurrent callers are coalesced by a dispatcher
 * thread into batches of at most max_batch requests (waiting at most max_delay_us for company)
 * and shipped through rl_check_and_update_batch.  The drain order is the stream order that
 * defines the result; *out_seq returns the caller's position in it.  now_us == 0 = the front
 * stamps the batch with the wall clock when it drains it.  While a front exists, it owns the
 * engine's request path (maintenance calls must be serialised by the caller). */
typedef struct rl_front rl_front;
int rl_front_create(rl_engine *e, uint32_t max_batch, uint32_t max_delay_us, rl_front **out);
void rl_front_destroy(rl_front *f);
/* m: up to the engine's max_counters_per_request (the matched counters of one request) */
int rl_front_check_and_update(rl_front *f, const rl_counter *ctrs, uint32_t m, uint64_t delta, uint64_t now_us,
                              int load_counters, uint8_t *out_limited, uint32_t *out_first_limited,
                              uint64_t *out_remaining, uint64_t *out_ttl_us, uint64_t *out_seq);
int rl_front_stats(rl_front *f, uint64_t *out_batches, uint64_t *out_requests);

#ifdef __cplusplus
}
#endif
#endif
