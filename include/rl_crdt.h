/* rl_crdt.h — cross-box replication: per-actor counter values merged on the GPU (SURVEY.md §8 f4).
 *
 * Replaces, batched, the value type of the reference's replicated store and the two streams that feed it:
 *   CrCounterValue<A>                 limitador/src/storage/distributed/cr_counter_value.rs:10-150
 *       read_at      :38-46   expired ? 0 : own value + sum of the other actors' values
 *       inc_actor_at :66-75   (inc_at :54-60 for ourselves) window roll-over through AtomicExpiryTime::update_if_expired
 *       merge_at     :81-115  a remote (expiry, {actor: value}) set: ignored when already expired; the EARLIER
 *                             unexpired expiry wins (atomic_expiring_value.rs:113-130); a locally expired value is reset
 *                             to the remote window; then every actor keeps the LARGER of the two values
 *   the gossip stream                 CounterUpdate{key, values, expires_at}: limitador/proto/distributed.proto:54-58,
 *                                     applied at distributed/mod.rs:236-246
 *   the re-sync stream                process_re_sync, distributed/mod.rs:294-332: our own non-zero unexpired values
 *
 * One table row per counter key: 16-B key | expiry_us | per-actor values (actors fixed at creation, ours one of them).
 * The semantics are eventually consistent, not bit-exact against a single stream: the reference applies concurrent
 * increments and merges in whatever order its threads run.  What IS exact, and tested against the CPU restatement
 * (oracle/crdt_oracle.c, pinned by the reference's own eleven unit tests): a batch in which every key appears once
 * equals the reference applied to that batch in any order; an inc batch that repeats keys equals one such order (see
 * rl_crdt_inc); merge batches may repeat keys (merge_at commutes for one clock reading: the earliest unexpired expiry
 * and the per-actor maxima do not depend on the order).
 *
 * Differences a caller can observe: the reference PANICS when a gossiped key has no local counter
 * (`limits.get(&update.key).unwrap()`, distributed/mod.rs:242); here the row is created and treated as locally
 * expired (the remote window and values are taken).  A full table is RL_TRANSIENT, never a dropped update.
 *
 * Time is microseconds since the epoch, as everywhere in this library (the wire carries whole seconds in expires_at:
 * the caller multiplies, as mod.rs:245 does with Duration::from_secs).  `mem` = RL_MEM_HOST or RL_MEM_DEVICE for every
 * array of the call (include/rl_engine.h).  One thread at a time per handle.
 */
#ifndef RL_CRDT_H
#define RL_CRDT_H

#include <stdint.h>

#include "rl_engine.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rl_crdt rl_crdt;

#define RL_CRDT_MAX_ACTORS 16

typedef struct rl_crdt_config {
    uint32_t struct_size;   /* sizeof(rl_crdt_config) */
    int32_t device;         /* CUDA device ordinal */
    uint64_t capacity_rows; /* counters the table can hold; rounded up to 2^k */
    uint32_t actors;        /* replicas in the cluster, ourselves included: 1..RL_CRDT_MAX_ACTORS */
    uint32_t self_actor;    /* our index in [0, actors) — CrCounterValue::ourselves */
} rl_crdt_config;

/* counter identity: any non-zero 128-bit value with hi != ~0 (e.g. rl_counter's (key_lo, limit_id << 32 | key_hi)) */
typedef struct rl_crdt_key {
    uint64_t lo, hi;
} rl_crdt_key;

/* one CounterUpdate: the values are actors[val_off .. val_off + n_vals) / values[...] of the call's flat arrays */
typedef struct rl_crdt_update {
    uint64_t key_lo, key_hi;
    uint64_t expires_at_us;
    uint32_t val_off, n_vals;
} rl_crdt_update;

int rl_crdt_create(const rl_crdt_config *cfg, rl_crdt **out);
void rl_crdt_destroy(rl_crdt *c);
const char *rl_crdt_last_error(rl_crdt *c);

/* inc_actor_at for n counters, all at the clock reading now_us: counter keys[i] of actor[i] += increment[i] within a
 * window of window_us[i] (a counter that is absent or expired starts a new window at now_us and takes the increment as
 * its value).  Keys may repeat, and every increment counts:
 *   - one actor's repeats of a key are exact: the sum of its increments on an absent or expired counter, its old value
 *     plus that sum on a live one (wrapping mod 2^64), which is what every order of them gives;
 *   - repeats of a key by several actors equal the sequential order that starts with one of them, like concurrent
 *     callers of the reference: on an absent or expired counter that request's window starts and its actor's value
 *     becomes the sum of that actor's increments, while the other actors add theirs onto the values they held.
 * Except: a window that leaves the expiry at or before now_us (window_us 0, or now_us + window_us wrapping past 2^64)
 * starts over at every increment, and the result of repeating such a key within one call is unspecified. */
int rl_crdt_inc(rl_crdt *c, uint64_t n, const rl_crdt_key *keys, const uint32_t *actor, const uint64_t *increment,
                const uint64_t *window_us, uint64_t now_us, int mem);
/* merge_at for n updates at the clock reading now_us.  Keys may repeat. */
int rl_crdt_merge(rl_crdt *c, uint64_t n, const rl_crdt_update *updates, const uint32_t *actors, const uint64_t *values,
                  uint64_t n_values, uint64_t now_us, int mem);
/* read_at: out_value[i] = 0 for an absent or expired counter, else the sum over the actors (wrapping);
 * out_expiry_us[i] (nullable) = its expiry, 0 when absent. */
int rl_crdt_read(rl_crdt *c, uint64_t n, const rl_crdt_key *keys, uint64_t now_us, int mem, uint64_t *out_value,
                 uint64_t *out_expiry_us);
/* The re-sync stream: every counter whose OWN value is non-zero and whose expiry is later than now_us, as (key, our
 * value, expiry) — what a peer merges as CounterUpdate{key, {self_actor: value}, expiry}.  Host outputs of capacity cap;
 * *out_count = counters found (may exceed cap). */
int rl_crdt_export(rl_crdt *c, uint64_t now_us, uint64_t cap, rl_crdt_key *out_keys, uint64_t *out_value,
                   uint64_t *out_expiry_us, uint64_t *out_count);
/* Parity aid: every row as (key, expiry, values[actors]); out_values holds cap * actors words.  Host outputs. */
int rl_crdt_dump(rl_crdt *c, uint64_t cap, rl_crdt_key *out_keys, uint64_t *out_expiry_us, uint64_t *out_values,
                 uint64_t *out_count);
/* CounterStorage::clear of the replicated store (distributed/mod.rs:210-213): every counter is forgotten. */
int rl_crdt_clear(rl_crdt *c);
/* kernels launched by this handle since creation */
uint64_t rl_crdt_kernel_launches(rl_crdt *c);

#ifdef __cplusplus
}
#endif
#endif /* RL_CRDT_H */
