// rl_wire.h — the protobuf reader of RateLimitRequest (include/rl_rls.h), one body for the host and the device.
//
// rl_rls.cpp decodes with it on the CPU workers (rl_rls_plan, rl_rls_decode_request) and rl_rls_dev.cuh inside the device
// plan kernel, so both plans run the same decoder.  Compiles as plain host C++ (g++, or nvcc on a .cpp) and as
// __host__ __device__ code under nvcc.  Nothing here recurses, allocates or calls the C library beyond memcpy: a group is
// skipped by a loop over an explicit stack of open group tags.
#pragma once
#include <stdint.h>

#include "../../include/rl_rls.h"

#ifndef RL_HD
#if defined(__CUDACC__)
#define RL_HD __host__ __device__ __forceinline__
#else
#define RL_HD inline
#endif
#endif

namespace rl_wire {

struct Rd {
    const uint8_t* p;
    const uint8_t* end;
};

// prost::encoding::decode_varint: at most 10 bytes, the 10th may only carry bit 63
RL_HD bool rd_varint(Rd& r, uint64_t& v) {
    v = 0;
    for (int i = 0; i < 10; i++) {
        if (r.p >= r.end) return false;
        const uint8_t b = *r.p++;
        if (i == 9 && b > 1) return false;
        v |= (uint64_t)(b & 0x7F) << (7 * i);
        if (!(b & 0x80)) return true;
    }
    return false;
}
RL_HD bool rd_key(Rd& r, uint32_t& tag, uint32_t& wt) {
    uint64_t k;
    if (!rd_varint(r, k) || k > 0xFFFFFFFFull) return false;  // "invalid key value"
    wt = (uint32_t)k & 7u;
    tag = (uint32_t)k >> 3;
    return tag != 0 && wt <= 5;  // "invalid tag value: 0", "invalid wire type value"
}
RL_HD bool rd_len(Rd& r, Rd& sub) {
    uint64_t n;
    if (!rd_varint(r, n) || n > (uint64_t)(r.end - r.p)) return false;
    sub.p = r.p;
    sub.end = r.p + n;
    r.p += n;
    return true;
}
// one value of wire type 0, 1, 2 or 5; false for a group marker
RL_HD bool rd_skip_value(Rd& r, uint32_t wt) {
    uint64_t v;
    Rd sub;
    switch (wt) {
        case 0: return rd_varint(r, v);
        case 1:
            if (r.end - r.p < 8) return false;
            r.p += 8;
            return true;
        case 2: return rd_len(r, sub);
        case 5:
            if (r.end - r.p < 4) return false;
            r.p += 4;
            return true;
        default: return false;
    }
}

#define RL_WIRE_MAX_GROUP_DEPTH 100

// prost::encoding::skip_field: a start group is skipped to its matching end group, at most 100 groups deep; a stray end
// group is an error
RL_HD bool rd_skip(Rd& r, uint32_t tag, uint32_t wt) {
    if (wt != 3) return rd_skip_value(r, wt);
    uint32_t open[RL_WIRE_MAX_GROUP_DEPTH];  // tags of the groups not yet closed, innermost last
    uint32_t depth = 0;
    open[depth++] = tag;
    for (;;) {
        uint32_t t2, w2;
        if (!rd_key(r, t2, w2)) return false;
        if (w2 == 4) {
            if (t2 != open[depth - 1]) return false;
            if (--depth == 0) return true;
        } else if (w2 == 3) {
            if (depth >= RL_WIRE_MAX_GROUP_DEPTH) return false;
            open[depth++] = t2;
        } else if (!rd_skip_value(r, w2)) {
            return false;
        }
    }
}

// str::from_utf8: no overlong forms, no surrogates, nothing above U+10FFFF
RL_HD bool utf8_ok(const uint8_t* p, const uint8_t* end) {
    while (p < end) {
        const uint8_t c = *p;
        if (c < 0x80) {
            p++;
            continue;
        }
        int n;
        uint32_t cp;
        if (c >= 0xC2 && c <= 0xDF) n = 1, cp = c & 0x1F;
        else if (c >= 0xE0 && c <= 0xEF) n = 2, cp = c & 0x0F;
        else if (c >= 0xF0 && c <= 0xF4) n = 3, cp = c & 0x07;
        else return false;
        if (end - p <= n) return false;
        for (int i = 1; i <= n; i++) {
            if ((p[i] & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (p[i] & 0x3F);
        }
        if (n == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) return false;
        if (n == 3 && (cp < 0x10000 || cp > 0x10FFFF)) return false;
        p += n + 1;
    }
    return true;
}

RL_HD bool rd_string(Rd& r, uint32_t wt, const uint8_t* base, uint32_t& off, uint32_t& len) {
    Rd s;
    if (wt != 2 || !rd_len(r, s) || !utf8_ok(s.p, s.end)) return false;
    off = (uint32_t)(s.p - base);
    len = (uint32_t)(s.end - s.p);
    return true;
}

// RateLimitDescriptor.RateLimitOverride {1: uint32, 2: enum}: only validated (the path ignores it)
RL_HD bool decode_override(Rd r) {
    while (r.p < r.end) {
        uint32_t tag, wt;
        uint64_t v;
        if (!rd_key(r, tag, wt)) return false;
        if (tag == 1 || tag == 2) {
            if (wt != 0 || !rd_varint(r, v)) return false;
        } else if (!rd_skip(r, tag, wt)) {
            return false;
        }
    }
    return true;
}

// Where the decoder puts a request's entries: a caller's range of `cap` entries (a worker's scratch vector, or the slice
// of a device scratch array a kernel thread owns).  n counts every entry decoded, also those past cap.
struct EntrySink {
    rl_rls_entry* out;
    uint32_t cap;
    uint32_t n;
};

RL_HD bool decode_entry(Rd r, const uint8_t* base, uint32_t descriptor, EntrySink& sink) {
    rl_rls_entry e{descriptor, 0, 0, 0, 0};
    while (r.p < r.end) {
        uint32_t tag, wt;
        if (!rd_key(r, tag, wt)) return false;
        if (tag == 1) {
            if (!rd_string(r, wt, base, e.key_off, e.key_len)) return false;
        } else if (tag == 2) {
            if (!rd_string(r, wt, base, e.val_off, e.val_len)) return false;
        } else if (!rd_skip(r, tag, wt)) {
            return false;
        }
    }
    if (sink.n < sink.cap) sink.out[sink.n] = e;
    sink.n++;
    return true;
}

RL_HD bool decode_descriptor(Rd r, const uint8_t* base, uint32_t descriptor, EntrySink& sink) {
    while (r.p < r.end) {
        uint32_t tag, wt;
        Rd sub;
        if (!rd_key(r, tag, wt)) return false;
        if (tag == 1) {
            if (wt != 2 || !rd_len(r, sub) || !decode_entry(sub, base, descriptor, sink)) return false;
        } else if (tag == 2) {
            if (wt != 2 || !rd_len(r, sub) || !decode_override(sub)) return false;
        } else if (!rd_skip(r, tag, wt)) {
            return false;
        }
    }
    return true;
}

// One RateLimitRequest.  Every entry takes at least two bytes of the message (its tag and its length), so a sink of
// len / 2 entries always holds all of them.
RL_HD bool decode_request(const uint8_t* buf, uint64_t len, rl_rls_request& q, EntrySink& sink) {
    if (len > 0xFFFFFFFFull) return false;
    Rd r{buf, buf + len};
    q = rl_rls_request{0, 0, 0, 0, 0};
    while (r.p < r.end) {
        uint32_t tag, wt;
        Rd sub;
        uint64_t v;
        if (!rd_key(r, tag, wt)) return false;
        if (tag == 1) {  // string domain = 1 (a repeated occurrence replaces the earlier one)
            if (!rd_string(r, wt, buf, q.domain_off, q.domain_len)) return false;
        } else if (tag == 2) {  // repeated RateLimitDescriptor descriptors = 2
            if (wt != 2 || !rd_len(r, sub) || !decode_descriptor(sub, buf, q.n_descriptors, sink)) return false;
            q.n_descriptors++;
        } else if (tag == 3) {  // uint32 hits_addend = 3
            if (wt != 0 || !rd_varint(r, v)) return false;
            q.hits_addend = (uint32_t)v;
        } else if (!rd_skip(r, tag, wt)) {
            return false;
        }
    }
    q.n_entries = sink.n;
    return true;
}

}  // namespace rl_wire
