// rl_blake2b.h — BLAKE2b (RFC 7693, unkeyed, streaming) and the 96-bit counter key digest, one body for the host and the
// device.  rl_match.cpp digests counter keys with it (rl_matcher_counters*, rl_counter_key) and rl_rls_dev.cuh inside the
// device plan kernel, so both produce the same keys.  The IV and the message schedule are written out as literals in
// the rounds (no static tables), which both g++ and nvcc's device compiler accept, and which lets nvcc keep m[] and v[]
// in registers.
#pragma once
#include <stdint.h>
#include <string.h>

#ifndef RL_HD
#if defined(__CUDACC__)
#define RL_HD __host__ __device__ __forceinline__
#else
#define RL_HD inline
#endif
#endif

namespace rl_b2 {

#define RL_B2_IV0 0x6a09e667f3bcc908ULL
#define RL_B2_IV1 0xbb67ae8584caa73bULL
#define RL_B2_IV2 0x3c6ef372fe94f82bULL
#define RL_B2_IV3 0xa54ff53a5f1d36f1ULL
#define RL_B2_IV4 0x510e527fade682d1ULL
#define RL_B2_IV5 0x9b05688c2b3e6c1fULL
#define RL_B2_IV6 0x1f83d9abfb41bd6bULL
#define RL_B2_IV7 0x5be0cd19137e2179ULL

RL_HD uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
RL_HD uint64_t load64(const uint8_t* p) {
    uint64_t v;
    memcpy(&v, p, 8);  // little-endian hosts only (x86-64, aarch64) and the GPU
    return v;
}

struct Blake2b {
    uint64_t h[8];
    uint64_t t;
    uint8_t buf[128];
    uint32_t fill;
    uint32_t outlen;

    RL_HD explicit Blake2b(uint32_t out) : t(0), fill(0), outlen(out) {
        h[0] = RL_B2_IV0 ^ 0x01010000ULL ^ (uint64_t)out;
        h[1] = RL_B2_IV1;
        h[2] = RL_B2_IV2;
        h[3] = RL_B2_IV3;
        h[4] = RL_B2_IV4;
        h[5] = RL_B2_IV5;
        h[6] = RL_B2_IV6;
        h[7] = RL_B2_IV7;
    }
    RL_HD void compress(const uint8_t* block, bool last) {
        uint64_t m[16], v[16];
        for (int i = 0; i < 16; i++) m[i] = load64(block + 8 * i);
        for (int i = 0; i < 8; i++) v[i] = h[i];
        v[8] = RL_B2_IV0;
        v[9] = RL_B2_IV1;
        v[10] = RL_B2_IV2;
        v[11] = RL_B2_IV3;
        v[12] = RL_B2_IV4 ^ t;  // message lengths stay far below 2^64: the high counter word is 0
        v[13] = RL_B2_IV5;
        v[14] = last ? ~RL_B2_IV6 : RL_B2_IV6;
        v[15] = RL_B2_IV7;
#define RL_B2_G(a, b, c, d, x, y)          \
    v[a] = v[a] + v[b] + (x);              \
    v[d] = rotr(v[d] ^ v[a], 32);          \
    v[c] = v[c] + v[d];                    \
    v[b] = rotr(v[b] ^ v[c], 24);          \
    v[a] = v[a] + v[b] + (y);              \
    v[d] = rotr(v[d] ^ v[a], 16);          \
    v[c] = v[c] + v[d];                    \
    v[b] = rotr(v[b] ^ v[c], 63);
#define RL_B2_ROUND(s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15) \
    RL_B2_G(0, 4, 8, 12, m[s0], m[s1])                                                     \
    RL_B2_G(1, 5, 9, 13, m[s2], m[s3])                                                     \
    RL_B2_G(2, 6, 10, 14, m[s4], m[s5])                                                    \
    RL_B2_G(3, 7, 11, 15, m[s6], m[s7])                                                    \
    RL_B2_G(0, 5, 10, 15, m[s8], m[s9])                                                    \
    RL_B2_G(1, 6, 11, 12, m[s10], m[s11])                                                  \
    RL_B2_G(2, 7, 8, 13, m[s12], m[s13])                                                   \
    RL_B2_G(3, 4, 9, 14, m[s14], m[s15])
        // the twelve rounds: sigma[r % 10] (RFC 7693 §2.7)
        RL_B2_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
        RL_B2_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
        RL_B2_ROUND(11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4)
        RL_B2_ROUND(7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8)
        RL_B2_ROUND(9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13)
        RL_B2_ROUND(2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9)
        RL_B2_ROUND(12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11)
        RL_B2_ROUND(13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10)
        RL_B2_ROUND(6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5)
        RL_B2_ROUND(10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0)
        RL_B2_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
        RL_B2_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
#undef RL_B2_ROUND
#undef RL_B2_G
        for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
    }
    RL_HD void update(const void* data, uint64_t n) {
        const uint8_t* p = (const uint8_t*)data;
        while (n) {
            if (fill == 128) {  // a full buffer is only compressed once more input follows it
                t += 128;
                compress(buf, false);
                fill = 0;
            }
            const uint32_t k = n < (uint64_t)(128 - fill) ? (uint32_t)n : 128 - fill;
            memcpy(buf + fill, p, k);
            fill += k;
            p += k;
            n -= k;
        }
    }
    RL_HD void final(uint8_t* out) {
        t += fill;
        memset(buf + fill, 0, 128 - fill);
        compress(buf, true);
        uint8_t full[64];
        memcpy(full, h, 64);
        memcpy(out, full, outlen);
    }
};

// The counter key: BLAKE2b-96 over (source, value) pairs, each string length-prefixed (u32 LE); key_lo = digest bits
// 0..63, key_hi = bits 64..95 (include/rl_match.h: rl_counter_key).
struct KeyDigest {
    Blake2b b;
    RL_HD KeyDigest() : b(12) {}
    RL_HD void str(const char* s, uint64_t n) {
        const uint32_t len = (uint32_t)n;
        b.update(&len, 4);
        b.update(s, n);
    }
    RL_HD void finish(uint64_t& lo, uint64_t& hi) {
        uint8_t d[12];
        b.final(d);
        uint32_t hi32;
        memcpy(&lo, d, 8);
        memcpy(&hi32, d + 8, 4);
        hi = hi32;
    }
};

}  // namespace rl_b2
