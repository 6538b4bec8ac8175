// rl_json.h — the JSON reader of CheckAndReportInfo (include/rl_http.h), one body for the host and the device.
//
// The HTTP API takes `web::Json<CheckAndReportInfo>` (limitador-server/src/http_api/request_types.rs:10-16,
// server.rs:129-260): actix hands the body to `serde_json::from_slice`, and serde_derive's struct rules decide what the
// struct is.  This header accepts exactly those bodies; anything it refuses is what the extractor answers with 400.
// rl_rls.cpp decodes with it on the CPU workers (rl_http_plan, rl_http_decode_body) and rl_http_dev.cuh inside the
// device plan kernel.  Compiles as plain host C++ and as __host__ __device__ code under nvcc; nothing recurses,
// allocates or calls the C library.
//
// The rules, and the crate behaviour each restates:
//  - JSON text is RFC 8259, strictly (serde_json's parser).  Whitespace is space, \t, \n and \r only; a byte order mark
//    and an empty body are refused; only whitespace may follow the value (`Deserializer::end`, "trailing characters").
//    No comments, no trailing commas, no NaN / Infinity, no leading zeros in numbers.
//  - The top level is an object, or an array of exactly 4 elements in field order (serde_derive's `visit_seq`: a 4th
//    element that is missing is `invalid_length` even though the field is an Option; a 5th is refused by serde_json's
//    `end_seq`).
//  - Object fields are matched after unescaping (`"namespace"` is `namespace`).  An unknown field is skipped as
//    `IgnoredAny`, so it must still be valid JSON.  A repeated known field is `duplicate_field`, response_headers
//    included.  A missing namespace / values / delta is `missing_field`; a missing or null response_headers is None.
//  - namespace is a string.  values is an object of string values; a repeated key keeps the last value (the entries are
//    emitted in order, and the matcher binds the last one, as `HashMap::insert` keeps it).
//  - delta is `0|[1-9][0-9]*` and at most 2^64-1: serde_json reads a sign, a fraction or an exponent as i64 / f64 (`-0`
//    as f64) and a longer integer as f64, and serde's u64 visitor refuses all of those.
//  - Deserialized strings (field names, namespace, the keys and values of values, response_headers) are valid UTF-8
//    without a raw byte below 0x20; escapes are the RFC's, a surrogate pair combines, a lone surrogate is refused
//    (serde_json `parse_str`).  `\u0000` is accepted here; the service refuses it later (the matcher compares
//    NUL-terminated strings).
//  - Skipped values are skipped iteratively, as serde_json's `ignore_value` does (no 128-level recursion limit): the
//    nesting is bounded by the body only, and the open brackets live in a caller's bit stack of one bit per level.
//    Skipped strings are not checked for UTF-8 or for surrogates (`ignore_str`), but their escapes and control bytes are.
//
// Every deserialized string is written unescaped at its own source offset into `txt`, a buffer as long as the body (an
// unescaped string is never longer than its source), so each is an (offset, length) pair into `txt`.  The entries of
// values are rl_rls_entry with descriptor 0: the context is `descriptors[0]` (server.rs:140-141).
#pragma once
#include <stdint.h>

#include "../../include/rl_http.h"
#include "rl_wire.h"

namespace rl_json {

enum : uint32_t { HDR_NONE = 0, HDR_DRAFT03 = 1, HDR_OTHER = 2 };  // response_headers: None, "DraftVersion03", another

struct Info {
    uint32_t ns_off, ns_len;  // the namespace inside txt
    uint64_t delta;
    uint32_t n_entries;       // entries of values (may exceed the sink's cap: then only the first cap are written)
    uint32_t headers;         // HDR_*
};

struct Rd {
    const uint8_t* b;  // the body
    uint64_t p, n;
    uint8_t* txt;      // unescaped strings, at their source offsets
    uint8_t* bits;     // the skip stack: >= n / 8 + 1 bytes
};

RL_HD int peek(Rd& r) {
    while (r.p < r.n) {
        const uint8_t c = r.b[r.p];
        if (c != ' ' && c != '\t' && c != '\n' && c != '\r') return c;
        r.p++;
    }
    return -1;
}

RL_HD bool hex4(Rd& r, uint32_t& v) {
    if (r.n - r.p < 4) return false;
    v = 0;
    for (int k = 0; k < 4; k++) {
        const uint8_t c = r.b[r.p++];
        uint32_t d;
        if (c >= '0' && c <= '9') d = c - '0';
        else if (c >= 'a' && c <= 'f') d = c - 'a' + 10;
        else if (c >= 'A' && c <= 'F') d = c - 'A' + 10;
        else return false;
        v = (v << 4) | d;
    }
    return true;
}

// One string; r.p at its opening quote.  keep: a deserialized string (unescaped into txt at off, UTF-8 and surrogates
// checked); otherwise a skipped one (only escapes and control bytes checked, nothing written).
RL_HD bool string(Rd& r, bool keep, uint32_t& off, uint32_t& len) {
    r.p++;
    const uint64_t s = r.p;
    uint64_t k = s;  // write position in txt
    for (;;) {
        if (r.p >= r.n) return false;
        const uint8_t c = r.b[r.p++];
        if (c == '"') break;
        if (c < 0x20) return false;
        if (c != '\\') {
            if (keep) r.txt[k++] = c;
            continue;
        }
        if (r.p >= r.n) return false;
        const uint8_t e = r.b[r.p++];
        uint32_t cp;
        switch (e) {
            case '"': cp = '"'; break;
            case '\\': cp = '\\'; break;
            case '/': cp = '/'; break;
            case 'b': cp = 8; break;
            case 'f': cp = 12; break;
            case 'n': cp = 10; break;
            case 'r': cp = 13; break;
            case 't': cp = 9; break;
            case 'u': {
                if (!hex4(r, cp)) return false;
                if (!keep) continue;
                if (cp >= 0xDC00 && cp <= 0xDFFF) return false;  // a trailing surrogate first
                if (cp >= 0xD800 && cp <= 0xDBFF) {              // must be followed by \u and a trailing one
                    uint32_t lo;
                    if (r.n - r.p < 2 || r.b[r.p] != '\\' || r.b[r.p + 1] != 'u') return false;
                    r.p += 2;
                    if (!hex4(r, lo) || lo < 0xDC00 || lo > 0xDFFF) return false;
                    cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                }
                break;
            }
            default: return false;
        }
        if (!keep) continue;
        if (cp < 0x80) {
            r.txt[k++] = (uint8_t)cp;
        } else if (cp < 0x800) {
            r.txt[k++] = (uint8_t)(0xC0 | (cp >> 6));
            r.txt[k++] = (uint8_t)(0x80 | (cp & 0x3F));
        } else if (cp < 0x10000) {
            r.txt[k++] = (uint8_t)(0xE0 | (cp >> 12));
            r.txt[k++] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F));
            r.txt[k++] = (uint8_t)(0x80 | (cp & 0x3F));
        } else {
            r.txt[k++] = (uint8_t)(0xF0 | (cp >> 18));
            r.txt[k++] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F));
            r.txt[k++] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F));
            r.txt[k++] = (uint8_t)(0x80 | (cp & 0x3F));
        }
    }
    off = (uint32_t)s;
    len = (uint32_t)(k - s);
    return !keep || rl_wire::utf8_ok(r.txt + s, r.txt + k);
}

RL_HD bool literal(Rd& r, const char* w, uint32_t n) {
    if (r.n - r.p < n) return false;
    for (uint32_t k = 0; k < n; k++)
        if (r.b[r.p + k] != (uint8_t)w[k]) return false;
    r.p += n;
    return true;
}

RL_HD bool digits(Rd& r) {  // one or more
    if (r.p >= r.n || r.b[r.p] < '0' || r.b[r.p] > '9') return false;
    while (r.p < r.n && r.b[r.p] >= '0' && r.b[r.p] <= '9') r.p++;
    return true;
}

// -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?
RL_HD bool number(Rd& r) {
    if (r.b[r.p] == '-') r.p++;
    if (r.p >= r.n) return false;
    if (r.b[r.p] == '0') {
        r.p++;
        if (r.p < r.n && r.b[r.p] >= '0' && r.b[r.p] <= '9') return false;
    } else if (!digits(r)) {
        return false;
    }
    if (r.p < r.n && r.b[r.p] == '.') {
        r.p++;
        if (!digits(r)) return false;
    }
    if (r.p < r.n && (r.b[r.p] == 'e' || r.b[r.p] == 'E')) {
        r.p++;
        if (r.p < r.n && (r.b[r.p] == '+' || r.b[r.p] == '-')) r.p++;
        if (!digits(r)) return false;
    }
    return true;
}

RL_HD bool skip_key(Rd& r) {  // "key" :
    uint32_t o, l;
    if (peek(r) != '"' || !string(r, false, o, l) || peek(r) != ':') return false;
    r.p++;
    return true;
}

// One value of any shape (serde_json ignore_value), without recursion: bit d of r.bits is 1 when the d-th open bracket
// is an object.
RL_HD bool skip_value(Rd& r) {
    uint64_t depth = 0;
    for (;;) {
        const int c = peek(r);
        uint32_t o, l;
        if (c == '{' || c == '[') {
            r.p++;
            const uint8_t bit = (uint8_t)(1u << (depth & 7));
            if (c == '{') r.bits[depth >> 3] |= bit;
            else r.bits[depth >> 3] &= (uint8_t)~bit;
            depth++;
            const int d = peek(r);
            if (d == (c == '{' ? '}' : ']')) {
                r.p++;
                depth--;
            } else {
                if (c == '{' && !skip_key(r)) return false;
                continue;  // the container's first value
            }
        } else if (c == '"') {
            if (!string(r, false, o, l)) return false;
        } else if (c == '-' || (c >= '0' && c <= '9')) {
            if (!number(r)) return false;
        } else if (c == 't') {
            if (!literal(r, "true", 4)) return false;
        } else if (c == 'f') {
            if (!literal(r, "false", 5)) return false;
        } else if (c == 'n') {
            if (!literal(r, "null", 4)) return false;
        } else {
            return false;
        }
        // after a value: close what ends here, or move on to the next value of the innermost container
        for (;;) {
            if (depth == 0) return true;
            const bool obj = (r.bits[(depth - 1) >> 3] >> ((depth - 1) & 7)) & 1;
            const int d = peek(r);
            if (d == ',') {
                r.p++;
                if (obj && !skip_key(r)) return false;
                break;
            }
            if (d != (obj ? '}' : ']')) return false;
            r.p++;
            depth--;
        }
    }
}

RL_HD bool field_is(const Rd& r, uint32_t off, uint32_t len, const char* w, uint32_t n) {
    if (len != n) return false;
    for (uint32_t k = 0; k < n; k++)
        if (r.txt[off + k] != (uint8_t)w[k]) return false;
    return true;
}

enum : uint32_t { F_NAMESPACE = 0, F_VALUES = 1, F_DELTA = 2, F_HEADERS = 3, F_OTHER = 4 };

// The value of field f (serde's String / HashMap<String, String> / u64 / Option<String> visitors).
RL_HD bool field_value(Rd& r, uint32_t f, Info& q, rl_wire::EntrySink& sink) {
    const int c = peek(r);
    uint32_t o, l;
    switch (f) {
        case F_NAMESPACE: return c == '"' && string(r, true, q.ns_off, q.ns_len);
        case F_VALUES: {
            if (c != '{') return false;
            r.p++;
            if (peek(r) == '}') {
                r.p++;
                return true;
            }
            for (;;) {
                rl_rls_entry e{0, 0, 0, 0, 0};
                if (peek(r) != '"' || !string(r, true, e.key_off, e.key_len) || peek(r) != ':') return false;
                r.p++;
                if (peek(r) != '"' || !string(r, true, e.val_off, e.val_len)) return false;
                if (sink.n < sink.cap) sink.out[sink.n] = e;
                sink.n++;
                const int d = peek(r);
                r.p++;
                if (d == '}') return true;
                if (d != ',') return false;
            }
        }
        case F_DELTA: {
            if (c < '0' || c > '9') return false;  // a sign is i64 / f64 to serde_json
            uint64_t v = 0;
            if (c == '0') {
                r.p++;
                if (r.p < r.n && r.b[r.p] >= '0' && r.b[r.p] <= '9') return false;
            } else {
                while (r.p < r.n && r.b[r.p] >= '0' && r.b[r.p] <= '9') {
                    const uint64_t d = r.b[r.p++] - '0';
                    if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10) return false;  // past u64: f64 to serde_json
                    v = v * 10 + d;
                }
            }
            if (r.p < r.n && (r.b[r.p] == '.' || r.b[r.p] == 'e' || r.b[r.p] == 'E')) return false;  // f64
            q.delta = v;
            return true;
        }
        case F_HEADERS:
            if (c == 'n') {
                q.headers = HDR_NONE;
                return literal(r, "null", 4);
            }
            if (c != '"' || !string(r, true, o, l)) return false;
            q.headers = field_is(r, o, l, "DraftVersion03", 14) ? HDR_DRAFT03 : HDR_OTHER;
            return true;
        default: return skip_value(r);
    }
}

// One CheckAndReportInfo body.  txt: as long as the body; bits: body / 8 + 1 bytes.  Every entry takes at least six bytes
// of the body (`"":""` and a separator), so a sink of len / 2 entries always holds all of them.
RL_HD bool decode_info(const uint8_t* body, uint64_t len, uint8_t* txt, uint8_t* bits, Info& q, rl_wire::EntrySink& sink) {
    q = Info{0, 0, 0, 0, HDR_NONE};
    if (len > 0xFFFFFFFFull) return false;
    Rd r{body, 0, len, txt, bits};
    const int c = peek(r);
    if (c == '[') {  // visit_seq: the four fields in order
        r.p++;
        for (uint32_t f = F_NAMESPACE; f <= F_HEADERS; f++) {
            if (f != F_NAMESPACE) {
                if (peek(r) != ',') return false;
                r.p++;
            }
            if (!field_value(r, f, q, sink)) return false;
        }
        if (peek(r) != ']') return false;
        r.p++;
    } else if (c == '{') {  // visit_map
        r.p++;
        uint32_t seen = 0;
        if (peek(r) == '}') {
            r.p++;
        } else {
            for (;;) {
                uint32_t o, l;
                if (peek(r) != '"' || !string(r, true, o, l) || peek(r) != ':') return false;
                r.p++;
                const uint32_t f = field_is(r, o, l, "namespace", 9) ? F_NAMESPACE
                                   : field_is(r, o, l, "values", 6) ? F_VALUES
                                   : field_is(r, o, l, "delta", 5) ? F_DELTA
                                   : field_is(r, o, l, "response_headers", 16) ? F_HEADERS : F_OTHER;
                if (f != F_OTHER) {
                    if (seen & (1u << f)) return false;  // duplicate_field
                    seen |= 1u << f;
                }
                if (!field_value(r, f, q, sink)) return false;
                const int d = peek(r);
                r.p++;
                if (d == '}') break;
                if (d != ',') return false;
            }
        }
        if ((seen & 7u) != 7u) return false;  // missing_field (response_headers alone may be missing)
    } else {
        return false;
    }
    if (peek(r) != -1) return false;  // trailing characters
    q.n_entries = sink.n;
    return true;
}

// A deserialized string of a body that decoded, unescaped again from its source: the host's copy of the namespace when
// the device plan only reported where it starts (off: the first byte after its opening quote).  Writes txt[off ..
// off + length) as decode_info does; returns the length.
RL_HD uint32_t unescape(const uint8_t* body, uint64_t len, uint32_t off, uint8_t* txt) {
    Rd r{body, (uint64_t)off - 1, len, txt, nullptr};
    uint32_t o = 0, l = 0;
    string(r, true, o, l);
    return l;
}

// The store call's load_counters for a decoded body: check_and_report loads iff response_headers.is_some()
// (server.rs:206,210); /check and /report never do.
RL_HD uint8_t load_counters(int endpoint, uint32_t headers) {
    return endpoint == RL_HTTP_CHECK_AND_REPORT && headers != HDR_NONE ? 1 : 0;
}

}  // namespace rl_json
