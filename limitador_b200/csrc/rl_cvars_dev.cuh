// rl_cvars_dev.cuh — the counter variable dictionary on the device (include/rl_rls.h: rl_rls_keep_counter_vars; read by
// include/rl_http.h: rl_http_get_counters).
//
// The store keeps a counter's 96-bit key digest only; the variable values behind it exist on the device, in a plan's
// scratch, for the length of one batch.  With keeping on, the service records them after every device plan:
//   dictionary          (varset_id, key_lo, key_hi) -> blob.  Open addressing over a power-of-two slot array; a slot is
//                       claimed by a CAS of its fingerprint word (0 = empty) within RL_CV_PROBE steps of its home.  The
//                       blob lives in a byte arena whose cursor is an atomic add: the variable set's values in the order
//                       of the image's `vars` for the limit (the digest order), each a u32 length then the bytes.
//   k_counter_vars_record   one thread per request of the batch, after k_rls_scatter / k_http_scatter: for every
//                       qualified variable set of a store request (its first counter), probe; on a miss decode the
//                       request again with the plan's own decoder, bind it by the plan's rule (rls_bound: last duplicate
//                       wins), reserve the blob, write it, and only then claim a slot.  A blob that does not fit, or a
//                       key that finds no slot, is counted in `dropped`: no slot is ever claimed without its blob.  Two
//                       threads with the same key in one batch: the CAS loser sees the winner's fingerprint and stops
//                       (its reserved bytes stay unused until the next GC).
//   k_counter_vars_lookup / _gather   GET /counters: per counter the blob's length or "unnamed", a scan, the packed blobs
//   k_counter_vars_mark / _rebuild    GC: mark the entries the engine's live counters reference, then copy them into a
//                       fresh table and a compacted arena
//   k_counter_vars_export / _check / _import   snapshots: the GC's mark, then the marked entries laid out for the host;
//                       an import checks every entry against the image (rl_cv_check_entry), then copies the dictionary
//                       into a fresh table (_occupied, _kept, _rebuild) and claims the new entries there
//   k_counter_vars_since   drains (rl_rls_counter_vars_drain): the entries recorded since the last drain, laid out by
//                       the export's kernels
// Written, like rl_rls_dev.cuh, so that the same source runs under tests/emu/cuda_shim.h: per-thread code and global
// atomics only.
#pragma once
#include <stdint.h>

#include "rl_http_dev.cuh"

#define RL_CV_PROBE 64u                  // probe steps before a key is dropped (the whole table when smaller)
#define RL_CV_NONE 0xFFFFFFFFFFFFFFFFull  // lookup: no entry

struct CvSlot {
    unsigned long long fp;  // fingerprint of the key; 0 = empty, claimed by CAS
    uint64_t key_lo;
    uint32_t key_hi, varset;
    uint64_t off;           // the blob: arena[off .. off + len)
    uint32_t len, _pad;
};

// the dictionary's control words
enum : uint32_t { RL_CV_CURSOR = 0, RL_CV_KEYS = 1, RL_CV_DROPPED = 2, RL_CV_CTL_WORDS = 4 };

struct CvDict {
    CvSlot* slots;
    uint64_t mask;               // slots - 1
    uint8_t* arena;
    uint64_t arena_bytes;
    unsigned long long* ctl;     // [RL_CV_CTL_WORDS]
};

RL_HD unsigned long long rl_cv_fp(uint32_t varset, uint64_t lo, uint64_t hi) {
    uint64_t f = lo ^ ((hi << 32 | varset) * 0x9E3779B97F4A7C15ull);
    f ^= f >> 29;
    return f ? f : 1;
}
RL_HD uint64_t rl_cv_probe_len(const CvDict& D) { return D.mask + 1 < RL_CV_PROBE ? D.mask + 1 : RL_CV_PROBE; }

// the slot holding exactly (varset, lo, hi), or RL_CV_NONE (for kernels after the recording one: slots are complete)
RL_HD uint64_t rl_cv_find(const CvDict& D, uint32_t varset, uint64_t lo, uint64_t hi) {
    const unsigned long long fp = rl_cv_fp(varset, lo, hi);
    for (uint64_t k = 0, P = rl_cv_probe_len(D); k < P; k++) {
        const uint64_t p = (fp + k) & D.mask;
        const CvSlot& s = D.slots[p];
        if (s.fp == 0) return RL_CV_NONE;
        if (s.fp == fp && s.key_lo == lo && s.key_hi == (uint32_t)hi && s.varset == varset) return p;
    }
    return RL_CV_NONE;
}

enum : int { RL_CV_NO_ROOM = 0, RL_CV_CLAIMED = 1, RL_CV_HELD = 2 };

// Claim a slot for a key whose blob is already written: RL_CV_CLAIMED, RL_CV_NO_ROOM (no free slot within the probe
// length) or RL_CV_HELD (a slot already holds the fingerprint).
__device__ __forceinline__ int rl_cv_claim_slot(const CvDict& D, uint32_t varset, uint64_t lo, uint64_t hi, uint64_t off,
                                                uint32_t len) {
    const unsigned long long fp = rl_cv_fp(varset, lo, hi);
    for (uint64_t k = 0, P = rl_cv_probe_len(D); k < P; k++) {
        const uint64_t p = (fp + k) & D.mask;
        const unsigned long long prev = atomicCAS(&D.slots[p].fp, 0ull, fp);
        if (prev == fp) return RL_CV_HELD;
        if (prev != 0) continue;
        CvSlot& s = D.slots[p];
        s.key_lo = lo;
        s.key_hi = (uint32_t)hi;
        s.varset = varset;
        s.off = off;
        s.len = len;
        atomicAdd(&D.ctl[RL_CV_KEYS], 1ull);
        return RL_CV_CLAIMED;
    }
    return RL_CV_NO_ROOM;
}
// The recording and the GC: a slot that already holds the fingerprint is the key's own (recorded by another thread of
// the batch): nothing to do.  false: no free slot within the probe length.
__device__ __forceinline__ bool rl_cv_claim(const CvDict& D, uint32_t varset, uint64_t lo, uint64_t hi, uint64_t off,
                                            uint32_t len) {
    return rl_cv_claim_slot(D, varset, lo, hi, off, len) != RL_CV_NO_ROOM;
}

struct CvRecordArgs {
    const uint8_t* buf;          // the batch as the plan staged it
    const uint64_t* off;         // [n + 1]
    uint64_t n;
    RlImage img;
    uint32_t per_req;
    rl_rls_entry* ent;           // the plan's entry scratch (request i's at ent[off[i] / 2])
    const rl_counter* scratch;   // the plan's per-request counters
    const unsigned long long* rls_count;  // RLS: k_rls_plan's count
    const HttpScan* http_count;  // HTTP: k_http_plan's count
    uint8_t* txt;                // HTTP: the plan's unescape and skip-stack scratch
    uint8_t* bits;
    CvDict dict;
};

// The RLS request: its counters when it is a store request, and its decode (rl_wire.h) -> the bytes the entries point into.
struct CvWire {
    __device__ static uint32_t counters(const CvRecordArgs& a, uint64_t i) {
        const unsigned long long c = a.rls_count[i];
        return (c >> 32) ? (uint32_t)c : 0u;
    }
    __device__ static const uint8_t* decode(const CvRecordArgs& a, uint64_t i, rl_wire::EntrySink& sink) {
        const uint8_t* msg = a.buf + a.off[i];
        rl_rls_request q;
        return rl_wire::decode_request(msg, a.off[i + 1] - a.off[i], q, sink) ? msg : nullptr;
    }
};
// The HTTP body: the same over rl_json.h (the strings unescaped into txt at their source offsets).
struct CvJson {
    __device__ static uint32_t counters(const CvRecordArgs& a, uint64_t i) {
        const HttpScan& c = a.http_count[i];
        return c.n_store ? c.n_ctr : 0u;
    }
    __device__ static const uint8_t* decode(const CvRecordArgs& a, uint64_t i, rl_wire::EntrySink& sink) {
        uint8_t* txt = a.txt + a.off[i];
        rl_json::Info q;
        return rl_json::decode_info(a.buf + a.off[i], a.off[i + 1] - a.off[i], txt, a.bits + a.off[i] / 8 + i, q, sink) ? txt
                                                                                                                        : nullptr;
    }
};

template <class Dec>
__global__ void k_counter_vars_record(CvRecordArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const uint32_t n_ctr = Dec::counters(a, i);
    if (n_ctr == 0) return;
    const RlImage& I = a.img;
    const CvDict& D = a.dict;
    const rl_counter* C = a.scratch + i * a.per_req;
    rl_rls_entry* E = a.ent + a.off[i] / 2;
    const uint64_t len = a.off[i + 1] - a.off[i];
    rl_wire::EntrySink sink{E, (uint32_t)(len / 2 < 0xFFFFFFFFull ? len / 2 : 0xFFFFFFFFull), 0};
    const uint8_t* msg = nullptr;  // decoded and bound on the first miss
    for (uint32_t x = 0; x < n_ctr; x++) {
        const uint32_t* L = I.lims + 5ull * C[x].limit_id;
        const uint32_t vs = L[4];
        if (vs == 0) continue;
        bool seen = false;  // the first counter of each variable set carries its key
        for (uint32_t y = 0; y < x && !seen; y++) seen = I.lims[5ull * C[y].limit_id + 4] == vs;
        if (seen) continue;
        const unsigned long long fp = rl_cv_fp(vs, C[x].key_lo, C[x].key_hi);
        bool hit = false, free_seen = false;
        for (uint64_t k = 0, P = rl_cv_probe_len(D); k < P && !hit && !free_seen; k++) {
            const unsigned long long f = D.slots[(fp + k) & D.mask].fp;
            hit = f == fp;
            free_seen = f == 0;
        }
        if (hit) continue;
        if (!msg) {
            sink.n = 0;
            msg = Dec::decode(a, i, sink);
            if (!msg) return;  // (cannot happen: the plan decoded the same bytes)
            for (uint32_t k = 0; k < sink.n; k++)
                E[k].descriptor = rl_img_find_slot(I, E[k].descriptor, msg + E[k].key_off, E[k].key_len);
        }
        uint64_t bytes = 0;
        for (uint32_t v = L[2]; v < L[2] + L[3]; v++) bytes += 4 + rls_bound(E, sink.n, I.vars[3ull * v])->val_len;
        const uint64_t at = atomicAdd(&D.ctl[RL_CV_CURSOR], (unsigned long long)bytes);
        if (at + bytes > D.arena_bytes) {
            atomicAdd(&D.ctl[RL_CV_DROPPED], 1ull);
            continue;
        }
        uint8_t* o = D.arena + at;
        for (uint32_t v = L[2]; v < L[2] + L[3]; v++) {
            const rl_rls_entry* b = rls_bound(E, sink.n, I.vars[3ull * v]);
            for (int s = 0; s < 4; s++) *o++ = (uint8_t)(b->val_len >> (8 * s));
            for (uint32_t t = 0; t < b->val_len; t++) *o++ = msg[b->val_off + t];
        }
        if (!rl_cv_claim(D, vs, C[x].key_lo, C[x].key_hi, at, (uint32_t)bytes)) atomicAdd(&D.ctl[RL_CV_DROPPED], 1ull);
    }
}

struct CvLookupArgs {
    const uint32_t* limit_id;    // [n]: the counters asked for
    const uint64_t* key_lo;
    const uint64_t* key_hi;
    uint64_t n;
    RlImage img;
    CvDict dict;
    unsigned long long* len;     // [n + 1]: the blob's length (0 for an unqualified or unnamed counter); len[n] = 0
    uint64_t* src;               // [n]: the blob's arena offset, RL_CV_NONE for a qualified counter without an entry, 0 else
};

__global__ void k_counter_vars_lookup(CvLookupArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    if (i == a.n) {
        a.len[i] = 0;
        return;
    }
    const uint32_t vs = a.img.lims[5ull * a.limit_id[i] + 4];
    uint64_t src = 0;
    unsigned long long l = 0;
    if (vs) {
        const uint64_t p = rl_cv_find(a.dict, vs, a.key_lo[i], a.key_hi[i]);
        if (p == RL_CV_NONE) {
            src = RL_CV_NONE;
        } else {
            src = a.dict.slots[p].off;
            l = a.dict.slots[p].len;
        }
    }
    a.len[i] = l;
    a.src[i] = src;
}

struct CvGatherArgs {
    const unsigned long long* pos;  // [n + 1]: exclusive sum of the lengths
    const unsigned long long* len;
    const uint64_t* src;
    uint64_t n;
    const uint8_t* arena;
    uint8_t* out;                   // [pos[n]]
};

__global__ void k_counter_vars_gather(CvGatherArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    for (uint64_t t = 0; t < a.len[i]; t++) a.out[a.pos[i] + t] = a.arena[a.src[i] + t];
}

struct CvMarkArgs {
    const uint32_t* limit_id;    // [n]: the engine's live counters (rl_counters_export)
    const uint64_t* key_lo;
    const uint64_t* key_hi;
    uint64_t n;
    RlImage img;
    CvDict dict;
    uint8_t* mark;               // [slots]
};

__global__ void k_counter_vars_mark(CvMarkArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n || a.limit_id[i] >= a.img.n_limits) return;
    const uint32_t vs = a.img.lims[5ull * a.limit_id[i] + 4];
    if (vs == 0) return;
    const uint64_t p = rl_cv_find(a.dict, vs, a.key_lo[i], a.key_hi[i]);
    if (p != RL_CV_NONE) a.mark[p] = 1;
}

// the kept length of every old slot (0 when unmarked); len[slots] = 0
__global__ void k_counter_vars_kept(CvDict d, const uint8_t* mark, unsigned long long* len) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p > d.mask + 1) return;
    len[p] = p <= d.mask && mark[p] ? d.slots[p].len : 0;
}

struct CvRebuildArgs {
    CvDict from;
    const uint8_t* mark;
    const unsigned long long* pos;  // [slots + 1]: exclusive sum of the kept lengths
    CvDict to;                      // empty, same slot count
};

__global__ void k_counter_vars_rebuild(CvRebuildArgs a) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p > a.from.mask + 1) return;
    if (p == a.from.mask + 1) {
        a.to.ctl[RL_CV_CURSOR] = a.pos[p];
        return;
    }
    if (!a.mark[p]) return;
    const CvSlot& s = a.from.slots[p];
    const uint64_t at = a.pos[p];
    for (uint32_t t = 0; t < s.len; t++) a.to.arena[at + t] = a.from.arena[s.off + t];
    if (!rl_cv_claim(a.to, s.varset, s.key_lo, s.key_hi, at, s.len)) atomicAdd(&a.to.ctl[RL_CV_DROPPED], 1ull);
}

// ---- snapshots (include/rl_rls.h: rl_rls_counter_vars_export / _import) ---------------------------------------------
// Export: the GC's mark over the counters rl_counters_export selects, the kept lengths and their scan (each blob's
// position), a scan of the marks (each entry's index), then k_counter_vars_export lays the entries out for the host.
struct CvExportArgs {
    CvDict d;
    const uint8_t* mark;               // [slots]
    const unsigned long long* pos;     // [slots + 1]: exclusive sum of the kept lengths
    const unsigned long long* idx;     // [slots + 1]: exclusive sum of the marks
    uint32_t* varset;                  // [idx[slots]]
    uint64_t* key_lo;
    uint64_t* key_hi;
    uint64_t* blob_off;                // [idx[slots] + 1]
    uint8_t* blobs;                    // [pos[slots]]
};

__global__ void k_counter_vars_export(CvExportArgs a) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p > a.d.mask + 1) return;
    if (p == a.d.mask + 1) {
        a.blob_off[a.idx[p]] = a.pos[p];
        return;
    }
    if (!a.mark[p]) return;
    const CvSlot& s = a.d.slots[p];
    const uint64_t k = a.idx[p], at = a.pos[p];
    a.varset[k] = s.varset;
    a.key_lo[k] = s.key_lo;
    a.key_hi[k] = s.key_hi;
    a.blob_off[k] = at;
    for (uint32_t t = 0; t < s.len; t++) a.blobs[at + t] = a.d.arena[s.off + t];
}

// Why an imported entry is refused.  The call's word `bad` ends as the least (entry << 8 | reason), RL_CV_GOOD if none.
enum : uint32_t {
    RL_CV_BAD_VARSET = 1,     // not the variable set of a qualified limit of the image
    RL_CV_BAD_LENGTH = 2,     // a length prefix or a value runs past the blob (or the blob has too few values)
    RL_CV_BAD_TRAILING = 3,   // bytes after the set's last value
    RL_CV_BAD_VALUE = 4,      // a value that is not UTF-8 or holds a NUL: the recording never stores one
    RL_CV_BAD_DIGEST = 5,     // BLAKE2b-96 over (source, value) is not the key
    RL_CV_BAD_DUPLICATE = 6,  // the import names the key twice
};
#define RL_CV_GOOD 0xFFFFFFFFFFFFFFFFull

// One entry against the image: its variable set's sources (vs_vars[2 * vs] = first variable, [2 * vs + 1] = variables; 0
// variables: no qualified limit has the set) and its blob b[0 .. n), which must be exactly one (u32 LE length, bytes)
// per variable and digest to (lo, hi).  0 or an RL_CV_BAD_* reason.
RL_HD uint32_t rl_cv_check_entry(const RlImage& I, const uint32_t* vs_vars, uint32_t n_vs, uint32_t vs, uint64_t lo, uint64_t hi,
                                 const uint8_t* b, uint64_t n) {
    if (vs == 0 || vs >= n_vs || vs_vars[2ull * vs + 1] == 0) return RL_CV_BAD_VARSET;
    rl_b2::KeyDigest d;
    uint64_t at = 0;
    for (uint32_t v = vs_vars[2ull * vs], end = v + vs_vars[2ull * vs + 1]; v < end; v++) {
        if (n - at < 4) return RL_CV_BAD_LENGTH;
        const uint64_t len = (uint64_t)b[at] | (uint64_t)b[at + 1] << 8 | (uint64_t)b[at + 2] << 16 | (uint64_t)b[at + 3] << 24;
        at += 4;
        if (len > n - at) return RL_CV_BAD_LENGTH;
        const uint8_t* val = b + at;
        for (uint64_t t = 0; t < len; t++)
            if (val[t] == 0) return RL_CV_BAD_VALUE;
        if (!rl_wire::utf8_ok(val, val + len)) return RL_CV_BAD_VALUE;
        const uint32_t* V = I.vars + 3ull * v;
        d.str((const char*)I.arena + V[1], V[2]);
        d.str((const char*)val, len);
        at += len;
    }
    if (at != n) return RL_CV_BAD_TRAILING;
    uint64_t dlo, dhi;
    d.finish(dlo, dhi);
    return dlo == lo && dhi == hi ? 0 : RL_CV_BAD_DIGEST;
}

struct CvImportArgs {
    const uint32_t* varset;          // [n]
    const uint64_t* key_lo;
    const uint64_t* key_hi;
    const uint64_t* blob_off;        // [n + 1], non-decreasing (checked on the host)
    const uint8_t* blobs;
    uint64_t n;
    RlImage img;
    const uint32_t* vs_vars;         // [2 * n_vs] (rl_cv_check_entry)
    uint32_t n_vs;
    CvDict dict;                     // check: the dictionary as it stands; import: the fresh one
    unsigned long long* len;         // [n + 1]: the check's output, read by the import: the blob's length for a new key, 0
                                     // for a key already present (a valid blob has at least 4 bytes); len[n] = 0
    const unsigned long long* pos;   // import: [n + 1], exclusive sum of len
    uint64_t base;                   // import: the fresh arena's bytes before the first imported blob
    unsigned long long* bad;         // [1], RL_CV_GOOD before the check
};

// One thread per entry: refuse it, or leave its length for the import (0 when the dictionary has the key already: by
// the digest, with the same values).
__global__ void k_counter_vars_check(CvImportArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    a.len[i] = 0;
    if (i == a.n) return;
    const uint64_t o = a.blob_off[i], n = a.blob_off[i + 1] - o;
    const uint32_t why = rl_cv_check_entry(a.img, a.vs_vars, a.n_vs, a.varset[i], a.key_lo[i], a.key_hi[i], a.blobs + o, n);
    if (why) {
        atomicMin(a.bad, (unsigned long long)i << 8 | why);
        return;
    }
    if (rl_cv_find(a.dict, a.varset[i], a.key_lo[i], a.key_hi[i]) == RL_CV_NONE) a.len[i] = n;
}

// After k_counter_vars_rebuild copied every entry of the dictionary into the fresh one: one thread per new entry copies
// its blob to base + pos[i] and claims its slot.  No room counts in the fresh table's `dropped`; a slot that already
// holds the key means the import names it twice.
__global__ void k_counter_vars_import(CvImportArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > a.n) return;
    if (i == a.n) {
        a.dict.ctl[RL_CV_CURSOR] = a.base + a.pos[i];
        return;
    }
    const uint64_t n = a.len[i];
    if (n == 0) return;
    const uint64_t at = a.base + a.pos[i];
    const uint8_t* b = a.blobs + a.blob_off[i];
    for (uint64_t t = 0; t < n; t++) a.dict.arena[at + t] = b[t];
    const int r = rl_cv_claim_slot(a.dict, a.varset[i], a.key_lo[i], a.key_hi[i], at, (uint32_t)n);
    if (r == RL_CV_NO_ROOM) atomicAdd(&a.dict.ctl[RL_CV_DROPPED], 1ull);
    if (r == RL_CV_HELD) atomicMin(a.bad, (unsigned long long)i << 8 | RL_CV_BAD_DUPLICATE);
}

// every occupied slot (the import copies the whole dictionary into the fresh table)
__global__ void k_counter_vars_occupied(CvDict d, uint8_t* mark) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p <= d.mask) mark[p] = d.slots[p].fp != 0;
}

// Drains: the arena is append-only between a GC or an import (its cursor is an atomic add), so the entries recorded
// since a drain that read the cursor as `since` are exactly the slots whose blob starts at or past it.
__global__ void k_counter_vars_since(CvDict d, uint64_t since, uint8_t* mark) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p <= d.mask) mark[p] = d.slots[p].fp != 0 && d.slots[p].off >= since;
}
