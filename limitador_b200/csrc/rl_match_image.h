// rl_match_image.h — the matcher flattened for the device plan (library-internal; not part of include/).
//
// rl_matcher_image (rl_match.cpp) writes, under the matcher's shared lock, everything counters_that_apply reads into ONE
// array of 32-bit words: a header, then the sections below, then a byte arena holding every string.  The service
// uploads that array as it is and rebuilds it only when rl_matcher_generation changed (add_limit / _ex, delete_limit and
// set_counter_cap bump it).  rl_img_view turns it into pointers on either side; the lookups compile for host and device.
//
//   ns_tab     [ns_mask + 1]      open-addressed: namespace id or RL_IMG_EMPTY, probed from rl_img_hash(RL_IMG_NS_SEED, ns)
//   ns_str     [n_ns][2]          (arena offset, length) of namespace id's string
//   ns_lim_off [n_ns + 1]         namespace id's live limits are ns_lims[ns_lim_off[id] .. ns_lim_off[id + 1])
//   ns_lims    [...]              limit ids in the matcher's ns_limits order (the counter output order; deleted ones left out)
//   slot_tab   [slot_mask + 1]    open-addressed: slot or RL_IMG_EMPTY, probed from rl_img_hash(descriptor, key)
//   slot_key   [n_slots][3]       (descriptor, arena offset, length) of the slot's key
//   lims       [n_limits][5]      (first test, tests, first variable, variables, varset_id) by limit id
//   tests      [...][4]           (slot, first atom << 3 | atoms, truth table bits 0..31, bits 32..63): a limit applies iff
//                                 every one of its tests holds.  A test with 0 atoms is a presence test: it holds iff the
//                                 slot is bound.  Otherwise an unbound slot fails the test; atom j of a bound value gives
//                                 bit j of an index into the truth table, and the test holds iff that bit of the table is
//                                 set (at most RL_MATCH_MAX_ATOMS atoms: a table of at most 64 bits)
//   atoms      [...][3]           (RL_ATOM_* op, literal arena offset, literal length); for RL_ATOM_IN (op, arena offset of
//                                 the list, entries), the list being that many (u32 little-endian length, bytes) entries
//   vars       [...][3]           (slot, source arena offset, source length): the digest input, in the limit's `vars` order
#pragma once
#include <stdint.h>

#ifndef RL_HD
#if defined(__CUDACC__)
#define RL_HD __host__ __device__ __forceinline__
#else
#define RL_HD inline
#endif
#endif

#define RL_IMG_MAGIC 0x4D494C52u  // "RLIM"
#define RL_IMG_EMPTY 0xFFFFFFFFu
#define RL_IMG_NS_SEED 0x9E3779B9u
#define RL_MATCH_MAX_ATOMS 6u  // value atoms of one operand group: its truth table fits 64 bits

// what a value atom asks of the bound value v (bytes; every surface hands the matcher valid UTF-8, on which a byte-level
// prefix / suffix / substring match is the code-point one)
enum : uint32_t { RL_ATOM_EQ, RL_ATOM_PREFIX, RL_ATOM_SUFFIX, RL_ATOM_CONTAINS, RL_ATOM_IN };

// header word indices
enum : uint32_t {
    RL_IMG_H_MAGIC, RL_IMG_H_N_NS, RL_IMG_H_NS_MASK, RL_IMG_H_N_SLOTS, RL_IMG_H_SLOT_MASK, RL_IMG_H_N_LIMITS,
    RL_IMG_H_COUNTER_CAP, RL_IMG_H_NS_TAB, RL_IMG_H_NS_STR, RL_IMG_H_NS_LIM_OFF, RL_IMG_H_NS_LIMS, RL_IMG_H_SLOT_TAB,
    RL_IMG_H_SLOT_KEY, RL_IMG_H_LIMS, RL_IMG_H_TESTS, RL_IMG_H_ATOMS, RL_IMG_H_VARS, RL_IMG_H_ARENA, RL_IMG_H_ARENA_BYTES,
    RL_IMG_HDR_WORDS
};

struct RlImage {
    const uint32_t *ns_tab, *ns_str, *ns_lim_off, *ns_lims, *slot_tab, *slot_key, *lims, *tests, *atoms, *vars;
    const uint8_t* arena;
    uint32_t ns_mask, slot_mask, n_limits, counter_cap;
};

// hdr: the header as the host holds it; base: where the words live (host or device memory)
inline RlImage rl_img_view(const uint32_t* hdr, const uint32_t* base) {
    RlImage I;
    I.ns_tab = base + hdr[RL_IMG_H_NS_TAB];
    I.ns_str = base + hdr[RL_IMG_H_NS_STR];
    I.ns_lim_off = base + hdr[RL_IMG_H_NS_LIM_OFF];
    I.ns_lims = base + hdr[RL_IMG_H_NS_LIMS];
    I.slot_tab = base + hdr[RL_IMG_H_SLOT_TAB];
    I.slot_key = base + hdr[RL_IMG_H_SLOT_KEY];
    I.lims = base + hdr[RL_IMG_H_LIMS];
    I.tests = base + hdr[RL_IMG_H_TESTS];
    I.atoms = base + hdr[RL_IMG_H_ATOMS];
    I.vars = base + hdr[RL_IMG_H_VARS];
    I.arena = reinterpret_cast<const uint8_t*>(base + hdr[RL_IMG_H_ARENA]);
    I.ns_mask = hdr[RL_IMG_H_NS_MASK];
    I.slot_mask = hdr[RL_IMG_H_SLOT_MASK];
    I.n_limits = hdr[RL_IMG_H_N_LIMITS];
    I.counter_cap = hdr[RL_IMG_H_COUNTER_CAP];
    return I;
}

RL_HD uint64_t rl_img_hash(uint32_t seed, const uint8_t* p, uint32_t n) {
    uint64_t h = 0xcbf29ce484222325ULL ^ seed;
    h *= 0x100000001b3ULL;
    for (uint32_t i = 0; i < n; i++) {
        h ^= p[i];
        h *= 0x100000001b3ULL;
    }
    return h ^ (h >> 29);
}

RL_HD bool rl_img_bytes_eq(const uint8_t* a, const uint8_t* b, uint32_t n) {
    for (uint32_t i = 0; i < n; i++)
        if (a[i] != b[i]) return false;
    return true;
}

// RL_ATOM_EQ / _PREFIX / _SUFFIX / _CONTAINS of the literal l[0 .. ln) against the value v[0 .. n)
RL_HD bool rl_str_op(uint32_t op, const uint8_t* v, uint32_t n, const uint8_t* l, uint32_t ln) {
    if (ln > n || (op == RL_ATOM_EQ && ln != n)) return false;
    if (op == RL_ATOM_SUFFIX) return rl_img_bytes_eq(v + (n - ln), l, ln);
    if (op != RL_ATOM_CONTAINS) return rl_img_bytes_eq(v, l, ln);  // EQ (same length) and PREFIX
    for (uint32_t i = 0; i + ln <= n; i++)
        if (rl_img_bytes_eq(v + i, l, ln)) return true;
    return false;
}

// one atom row of the image (see the layout above) against the value v[0 .. n)
RL_HD bool rl_img_atom(const uint32_t* A, const uint8_t* arena, const uint8_t* v, uint32_t n) {
    if (A[0] != RL_ATOM_IN) return rl_str_op(A[0], v, n, arena + A[1], A[2]);
    const uint8_t* p = arena + A[1];
    for (uint32_t k = 0; k < A[2]; k++) {
        const uint32_t ln = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
        if (rl_str_op(RL_ATOM_EQ, v, n, p + 4, ln)) return true;
        p += 4 + ln;
    }
    return false;
}

// whether a bound value passes a test row of the image with k >= 1 atoms
RL_HD bool rl_img_test(const RlImage& I, const uint32_t* T, const uint8_t* v, uint32_t n) {
    const uint32_t k = T[1] & 7u;
    uint32_t bits = 0;
    for (uint32_t j = 0; j < k; j++) bits |= (uint32_t)rl_img_atom(I.atoms + 3ull * ((T[1] >> 3) + j), I.arena, v, n) << j;
    return ((bits < 32 ? T[2] >> bits : T[3] >> (bits - 32)) & 1u) != 0;
}

// namespace id of the string s[0 .. n), or RL_IMG_EMPTY
RL_HD uint32_t rl_img_find_ns(const RlImage& I, const uint8_t* s, uint32_t n) {
    for (uint64_t p = rl_img_hash(RL_IMG_NS_SEED, s, n) & I.ns_mask;; p = (p + 1) & I.ns_mask) {
        const uint32_t id = I.ns_tab[p];
        if (id == RL_IMG_EMPTY) return RL_IMG_EMPTY;
        if (I.ns_str[2 * id + 1] == n && rl_img_bytes_eq(I.arena + I.ns_str[2 * id], s, n)) return id;
    }
}

// slot of (descriptor, key), or RL_IMG_EMPTY when no limit refers to it
RL_HD uint32_t rl_img_find_slot(const RlImage& I, uint32_t desc, const uint8_t* k, uint32_t n) {
    for (uint64_t p = rl_img_hash(desc, k, n) & I.slot_mask;; p = (p + 1) & I.slot_mask) {
        const uint32_t s = I.slot_tab[p];
        if (s == RL_IMG_EMPTY) return RL_IMG_EMPTY;
        const uint32_t* sk = I.slot_key + 3 * (uint64_t)s;
        if (sk[0] == desc && sk[2] == n && rl_img_bytes_eq(I.arena + sk[1], k, n)) return s;
    }
}

struct rl_matcher;
extern "C" {
// The generation of the matcher's limits (bumped by every add_limit / _ex, delete_limit and set_counter_cap).
uint64_t rl_matcher_generation(rl_matcher* m);
// The image as one word array: RL_OK with *out_words written, or RL_FATAL with *out_words = the words needed when
// cap_words is too small.  *out_generation = the generation the image was taken at.
int rl_matcher_image(rl_matcher* m, uint32_t* out, uint64_t cap_words, uint64_t* out_words, uint64_t* out_generation);
}
