// rl_rls.cpp — Envoy RLS v3 wire surface: RateLimitRequest bytes -> counters -> ONE engine call -> RateLimitResponse
// bytes (include/rl_rls.h; SURVEY.md §8 f2 with the f1 matcher inside the batching stage).
//
// Host-only code.  The reference serves one request per tonic task: prost decodes the message, a HashMap per
// descriptor is built and bound as `descriptors` (envoy_rls/server.rs:121-139), counters_that_apply walks the CEL
// ASTs, the store is called, the response is built (:183-205).  Here a batch of wire messages is decoded and
// matched — on the engine's device (rl_rls_dev.cu) in rl_rls_serve, by a pool of CPU workers in rl_rls_plan (each
// request is independent) —, the counters are laid out as one CSR, the store is called once for the whole batch, and
// the responses are encoded by the worker pool.  No protobuf runtime: the four message types on the path have a
// handful of fields, decoded by hand (rl_wire.h, shared with the device plan) and encoded below.
// The HTTP API (include/rl_http.h) is served by the same stages over JSON bodies (rl_json.h): both surfaces are a
// Batch and share the stage code around it; the decoding, how the store is called and the responses are each surface's
// own, and the HTTP API shares the RLS service's workers and metrics.
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "rl_error.h"
#include "rl_http.h"
#include "rl_json.h"
#include "rl_match_records.h"
#include "rl_rls.h"
#include "rl_rls_dev.h"
#include "rl_wire.h"

extern "C" uint32_t rl_matcher_counter_cap(rl_matcher* m);  // rl_match.cpp (library-internal)
// Weak: the wire surface is also linked without the engine and the CUDA units (the sanitizer build of tests/san); there
// every service plans on the CPU with the default engine's maximum.
extern "C" __attribute__((weak)) uint32_t rl_engine_max_counters_per_request(rl_engine* e);
extern "C" {
__attribute__((weak)) int rl_rls_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int method, uint64_t n, const uint8_t* buf,
                                          const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                                          const RlsDevReq** out_req);
__attribute__((weak)) int rl_rls_dev_copy_plan(rl_rls_dev* st, uint32_t* ctr_off, rl_counter* ctrs, uint64_t* delta, uint8_t* load);
__attribute__((weak)) int rl_rls_dev_decide(rl_rls_dev* st, rl_engine* e, int method, int load_counters, uint8_t* limited,
                                            uint32_t* first_limited, uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off,
                                            rl_counter* ctrs);
__attribute__((weak)) int rl_http_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int endpoint, uint64_t n, const uint8_t* buf,
                                           const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                                           const HttpDevReq** out_req, const HttpRun** out_runs, uint32_t* out_n_runs);
__attribute__((weak)) int rl_http_dev_decide(rl_rls_dev* st, rl_engine* e, int endpoint, int* run_status, uint8_t* limited,
                                             uint32_t* first_limited, uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off,
                                             rl_counter* ctrs);
__attribute__((weak)) int rl_rls_dev_wait(rl_rls_dev* st);
__attribute__((weak)) int rl_rls_dev_shard_send(rl_rls_dev* st, rl_shard_batch* sb, int empty, int http, int method, int load_counters,
                                                int* out_failed);
__attribute__((weak)) int rl_rls_dev_shard_collect(rl_rls_dev* st, rl_shard_batch* sb, int load_counters, uint8_t* limited,
                                                   uint32_t* first_limited, uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off,
                                                   rl_counter* ctrs);
__attribute__((weak)) int rl_shard_batch_decide(rl_shard_batch* s);
__attribute__((weak)) rl_engine* rl_shard_batch_engine(rl_shard_batch* s);
__attribute__((weak)) int rl_cv_dev_configure(rl_rls_dev** st, rl_engine* e, uint64_t max_keys, uint64_t arena_bytes);
__attribute__((weak)) int rl_cv_dev_stats(rl_rls_dev* st, uint64_t* out_slots, uint64_t* out_keys, uint64_t* out_arena_used,
                                          uint64_t* out_dropped);
__attribute__((weak)) int rl_cv_dev_lookup(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* limit_id,
                                           const uint64_t* key_lo, const uint64_t* key_hi, const uint8_t** out_blobs,
                                           const uint64_t** out_blob_off, const uint8_t** out_unnamed);
__attribute__((weak)) int rl_cv_dev_gc(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t now_us, uint64_t* out_kept,
                                       uint64_t* out_freed);
__attribute__((weak)) int rl_cv_dev_export(rl_rls_dev** st, rl_engine* e, rl_matcher* m, const uint32_t* ns_ids, uint32_t n_ns,
                                           uint64_t now_us, uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset,
                                           uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_blob_off, uint8_t* out_blobs,
                                           uint64_t* out_count, uint64_t* out_bytes);
__attribute__((weak)) int rl_cv_dev_import(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* varset,
                                           const uint64_t* key_lo, const uint64_t* key_hi, const uint64_t* blob_off,
                                           const uint8_t* blobs, uint64_t* out_added);
__attribute__((weak)) int rl_cv_dev_drain(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t cap, uint64_t bytes_cap,
                                          uint32_t* out_varset, uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_blob_off,
                                          uint8_t* out_blobs, uint64_t* out_count, uint64_t* out_bytes, int* out_full);
__attribute__((weak)) int rl_get_counters(rl_engine* e, const uint32_t* limit_ids, uint32_t n, uint64_t now_us, uint64_t cap,
                                          uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi,
                                          uint64_t* out_remaining, uint64_t* out_ttl_us, uint64_t* out_count);
__attribute__((weak)) int rl_limits_set(rl_engine* e, const rl_limit_desc* limits, uint32_t n);
__attribute__((weak)) int rl_limits_delete(rl_engine* e, const uint32_t* limit_ids, uint32_t n);
__attribute__((weak)) int rl_fence(rl_engine* e);
__attribute__((weak)) const char* rl_rls_dev_error(rl_rls_dev* st);
__attribute__((weak)) void rl_rls_dev_destroy(rl_rls_dev* st);
}

namespace {

// the protobuf reader (rl_wire.h) is shared with the device plan
using rl_wire::decode_request;
using rl_wire::EntrySink;

// ---- encoding ----------------------------------------------------------------------------------------------------
void put_varint(std::vector<uint8_t>& o, uint64_t v) {
    while (v >= 0x80) {
        o.push_back((uint8_t)(v | 0x80));
        v >>= 7;
    }
    o.push_back((uint8_t)v);
}
size_t varint_size(uint64_t v) {
    size_t n = 1;
    while (v >= 0x80) {
        v >>= 7;
        n++;
    }
    return n;
}
void put_string_field(std::vector<uint8_t>& o, uint32_t tag, const char* s, size_t n) {
    if (n == 0) return;  // proto3: an empty string is not written
    put_varint(o, ((uint64_t)tag << 3) | 2);
    put_varint(o, n);
    o.insert(o.end(), (const uint8_t*)s, (const uint8_t*)s + n);
}
void encode_response(std::vector<uint8_t>& o, uint32_t code, const char* const* keys, const char* const* values, uint32_t nh) {
    if (code) {  // Code overall_code = 1
        o.push_back(0x08);
        put_varint(o, code);
    }
    for (uint32_t h = 0; h < nh; h++) {  // repeated HeaderValue response_headers_to_add = 3 {string key = 1; string value = 2}
        const size_t kn = strlen(keys[h]), vn = strlen(values[h]);
        size_t body = 0;
        if (kn) body += 1 + varint_size(kn) + kn;
        if (vn) body += 1 + varint_size(vn) + vn;
        o.push_back(0x1A);
        put_varint(o, body);
        put_string_field(o, 1, keys[h], kn);
        put_string_field(o, 2, values[h], vn);
    }
}

uint64_t wall_us() {
    return (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
}
double mono_us() {
    return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---- a small fork-join pool ----------------------------------------------------------------------------------------
struct Pool {
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_go, cv_done;
    std::function<void(uint32_t)> job;
    uint64_t gen = 0;
    uint32_t pending = 0;
    bool stop = false;
    uint32_t n = 1;

    explicit Pool(uint32_t threads) : n(std::max<uint32_t>(threads, 1)) {
        for (uint32_t w = 1; w < n; w++) workers.emplace_back([this, w] { loop(w); });
    }
    ~Pool() {
        {
            std::lock_guard<std::mutex> g(mu);
            stop = true;
        }
        cv_go.notify_all();
        for (auto& t : workers) t.join();
    }
    void loop(uint32_t w) {
        uint64_t seen = 0;
        for (;;) {
            std::function<void(uint32_t)> f;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv_go.wait(lk, [&] { return stop || gen != seen; });
                if (stop) return;
                seen = gen;
                f = job;
            }
            f(w);
            {
                std::lock_guard<std::mutex> g(mu);
                if (--pending == 0) cv_done.notify_all();
            }
        }
    }
    // f(w) runs once for every w in [0, n): worker 0 is the calling thread
    void run(const std::function<void(uint32_t)>& f) {
        if (n == 1) {
            f(0);
            return;
        }
        {
            std::lock_guard<std::mutex> g(mu);
            job = f;
            pending = n - 1;
            gen++;
        }
        cv_go.notify_all();
        f(0);
        std::unique_lock<std::mutex> lk(mu);
        cv_done.wait(lk, [&] { return pending == 0; });
    }
};

// A per-batch buffer that is NOT value-initialised when it is sized (std::vector::resize would zero megabytes per batch);
// its contents do not survive ensure().
template <class T>
struct RawBuf {
    std::unique_ptr<T[]> p;
    size_t cap = 0, n = 0;
    void ensure(size_t want) {
        if (want > cap) {
            cap = want + want / 2 + 16;
            p.reset(new T[cap]);
        }
        n = want;
    }
    T* data() { return p.get(); }
    const T* data() const { return p.get(); }
    size_t size() const { return n; }
};

struct NsCounts {
    uint64_t authorized_calls = 0, authorized_hits = 0, limited_calls = 0;
};

struct ReqPlan {
    uint8_t kind = 0;
    uint8_t hdr = 0;     // HTTP: response_headers (RL_HTTP_HEADERS_*)
    uint32_t hits = 1;   // RLS: hits_addend, 0 -> 1
    uint32_t n_ctr = 0;
    uint32_t store = RL_RLS_NO_STORE;
    uint64_t delta = 0;  // HTTP: the body's delta
};

struct WorkerOut {
    // plan: the requests of the range that go to the matcher, as rl_matcher_counters_batch_ns takes them
    RawBuf<rl_counter> ctrs;            // the range's counters, request after request (ctr_off)
    std::vector<rl_rls_entry> entries;
    RawBuf<char> arena;                 // NUL-terminated copies of the keys and values (the bindings point into it)
    RawBuf<uint8_t> txt, bits;          // HTTP: one body's unescaped strings and skip stack (rl_json.h)
    uint64_t n_store = 0;               // requests of the range that reach the store
    std::vector<rl_binding> binds;
    std::vector<uint32_t> bind_off, ctr_off;
    std::vector<const char*> ns;
    std::vector<uint64_t> req_of;       // matcher request k = batch request req_of[k]
    std::vector<uint8_t> status;
    // finish
    std::vector<uint8_t> resp;          // this worker's responses, concatenated
    std::vector<uint64_t> resp_len;     // one per request of the worker's range
    std::vector<char> hdr;              // header values of the range's store requests (rl_matcher_response_headers_batch)
    std::vector<uint64_t> hdr_off;
    std::vector<uint8_t> hval;          // HTTP: the range's X-RateLimit-* values, three per request (hval_len)
    std::vector<uint64_t> hval_len;
    std::unordered_map<std::string, NsCounts> by_ns;  // the range's metrics, merged into the service's after the workers
    std::map<std::pair<std::string, std::string>, uint64_t> limited_by_name;
};

// One batch of either surface as the stages below take it: the plan, the store call's CSR, the engine's outputs and the
// stage times.  The RLS service and the HTTP API each derive from it and add what is their own.
struct Batch {
    rl_matcher* m = nullptr;
    rl_engine* engine = nullptr;
    Pool* pool = nullptr;
    std::string last_error;

    int method = 0;  // RLS: the method; HTTP: the endpoint
    uint64_t n = 0;
    const uint8_t* buf = nullptr;  // only dereferenced during plan
    bool planned = false, finished = false;
    std::vector<ReqPlan> plan;
    std::vector<std::string> domains;  // every request's domain / namespace (the metrics outlive the input buffer)
    std::vector<WorkerOut> wout;
    std::vector<uint32_t> store_index;
    // store requests
    uint64_t n_store = 0;
    std::vector<uint32_t> ctr_off;
    RawBuf<rl_counter> ctrs;
    std::vector<uint64_t> delta, now;
    // engine outputs (serve)
    std::vector<uint8_t> o_limited;
    std::vector<uint32_t> o_first;
    std::vector<uint64_t> o_rem, o_ttl;
    double t_plan = 0, t_store = 0, t_finish = 0;
    // a sharded step between its send and its collect: the plan's status, the collect's load flag, the send's and the
    // decide's status and message, the stage clocks
    bool sh_pending = false, sh_load = false;
    int sh_plan = RL_OK, sh_status = RL_OK;
    std::string sh_error;
    double sh_t0 = 0, sh_t1 = 0;
};

}  // namespace

struct rl_rls : Batch {
    int header_mode = RL_RLS_HEADERS_NONE;
    bool use_limit_name = false;
    rl_rls_dev* dev = nullptr;  // the device plan's state (rl_rls_dev.cu), created by the first device plan
    int load_counters = 0;
    rl_shard_batch* shard = nullptr;          // rl_rls_attach_shard: store calls go through the sharded exchange
    const uint8_t* report_verdicts = nullptr;  // sharded Report: error verdicts mark the requests that were not decided
    // responses
    RawBuf<uint8_t> resp;
    std::vector<uint64_t> resp_off;
    std::vector<uint8_t> grpc, code;
    // metrics
    std::map<std::string, NsCounts> by_ns;
    std::map<std::pair<std::string, std::string>, uint64_t> limited_by_name;
    // rl_rls_configure outcomes (Status::config_success / config_failure)
    uint64_t config_version = 0, config_err_since = 0;
};

// The HTTP API (include/rl_http.h) over an RLS service: its own batch, the service's matcher, engine, workers, device
// state and metrics.
struct rl_http : Batch {
    rl_rls* rls = nullptr;
    std::vector<uint8_t> load;  // one load_counters flag per store request
    std::vector<int> run_status;
    std::vector<int32_t> o_status;
    // responses
    std::vector<uint16_t> status;
    RawBuf<uint8_t> body, hval;
    std::vector<uint64_t> body_off, hval_off;
    uint32_t store_calls = 0;
    // the last GET response
    uint16_t get_status = 0;
    std::string get_body;
    uint64_t get_unnamed = 0;
};

namespace {

template <class... A>
int sfail(Batch* s, const char* fmt, A... a) {
    s->last_error = rl_format(fmt, a...);
    return RL_FATAL;
}

// requests [lo, hi) of worker w
void range_of(uint64_t n, uint32_t workers, uint32_t w, uint64_t& lo, uint64_t& hi) {
    const uint64_t per = (n + workers - 1) / workers;
    lo = std::min<uint64_t>(n, (uint64_t)w * per);
    hi = std::min<uint64_t>(n, lo + per);
}

// Decode request i of an RLS batch (one wire message) into the worker's entries.  false: the request never reaches the
// matcher (its kind is set); true: its context is `sink`'s entries and its namespace base[ns_off .. ns_off + ns_len).
bool decode_one(rl_rls* s, const uint64_t* off, uint64_t i, WorkerOut& W, ReqPlan& P, EntrySink& sink, const uint8_t*& base,
                uint32_t& ns_off, uint32_t& ns_len) {
    const uint8_t* msg = s->buf + off[i];
    const uint64_t len = off[i + 1] - off[i];
    rl_rls_request q;
    if (W.entries.size() < 16) W.entries.resize(16);
    sink = EntrySink{W.entries.data(), (uint32_t)W.entries.size(), 0};
    if (!decode_request(msg, len, q, sink)) {
        P.kind = REQ_BAD_WIRE;
        return false;
    }
    if (sink.n > sink.cap) {  // rare: more entries than the scratch holds — decode again into a larger one
        W.entries.resize(sink.n);
        sink = EntrySink{W.entries.data(), (uint32_t)W.entries.size(), 0};
        decode_request(msg, len, q, sink);
    }
    P.hits = q.hits_addend ? q.hits_addend : 1;  // server.rs:131-135
    s->domains[i].assign((const char*)msg + q.domain_off, q.domain_len);
    if (q.domain_len == 0) {  // server.rs:106-116
        P.kind = REQ_UNKNOWN_DOMAIN;
        return false;
    }
    base = msg;
    ns_off = q.domain_off;
    ns_len = q.domain_len;
    return true;
}

// The same for body i of an HTTP batch (rl_json.h): the strings are unescaped into the worker's txt, which `base` is.
bool decode_one(rl_http* h, const uint64_t* off, uint64_t i, WorkerOut& W, ReqPlan& P, EntrySink& sink, const uint8_t*& base,
                uint32_t& ns_off, uint32_t& ns_len) {
    const uint8_t* body = h->buf + off[i];
    const uint64_t len = off[i + 1] - off[i];
    W.txt.ensure(len + 1);
    W.bits.ensure(len / 8 + 1);
    rl_json::Info q;
    if (W.entries.size() < 16) W.entries.resize(16);
    sink = EntrySink{W.entries.data(), (uint32_t)W.entries.size(), 0};
    if (!rl_json::decode_info(body, len, W.txt.data(), W.bits.data(), q, sink)) {
        P.kind = REQ_BAD_WIRE;
        return false;
    }
    if (sink.n > sink.cap) {
        W.entries.resize(sink.n);
        sink = EntrySink{W.entries.data(), (uint32_t)W.entries.size(), 0};
        rl_json::decode_info(body, len, W.txt.data(), W.bits.data(), q, sink);
    }
    P.delta = q.delta;
    P.hdr = (uint8_t)q.headers;
    h->domains[i].assign((const char*)W.txt.data() + q.ns_off, q.ns_len);
    base = W.txt.data();
    ns_off = q.ns_off;
    ns_len = q.ns_len;
    return true;
}

// Requests [lo, hi) of worker w: decode every message and lay its CEL context out (pass 1), then ONE matcher call for
// the whole range (pass 2) — a reader section per range, not per request: eight workers taking the matcher's
// reader/writer lock twice per request spent their time passing its cache line around and did not scale at all.  The
// same body for both surfaces: only decode_one differs.
template <class Svc>
void plan_range(Svc* s, const uint64_t* off, uint32_t w) {
    uint64_t lo, hi;
    range_of(s->n, s->pool->n, w, lo, hi);
    WorkerOut& W = s->wout[w];
    W.n_store = 0;
    W.binds.clear();
    W.bind_off.assign(1, 0);
    W.ns.clear();
    W.req_of.clear();
    // every string gets a NUL behind it: an entry is at least two bytes on the wire, so twice the range's bytes is enough
    // — sized up front, because the bindings point into it
    W.arena.ensure(2 * (size_t)(off[hi] - off[lo]) + 16);
    char* a = W.arena.data();
    for (uint64_t i = lo; i < hi; i++) {
        ReqPlan& P = s->plan[i];
        P = ReqPlan();
        EntrySink sink{nullptr, 0, 0};
        const uint8_t* msg = nullptr;
        uint32_t ns_off = 0, ns_len = 0;
        if (!decode_one(s, off, i, W, P, sink, msg, ns_off, ns_len)) continue;
        if (memchr(msg + ns_off, 0, ns_len) != nullptr) {
            P.kind = REQ_NO_LIMITS;  // no namespace the matcher knows holds a NUL: nothing applies (lib.rs:434-440)
            continue;
        }
        // the CEL context: descriptors[d] = map of the d-th descriptor's entries (server.rs:121-127, 137-139)
        bool nul = false;
        const size_t first_bind = W.binds.size();
        for (uint32_t k = 0; k < sink.n; k++) {
            const rl_rls_entry& e = W.entries[k];
            nul = nul || memchr(msg + e.key_off, 0, e.key_len) || memchr(msg + e.val_off, 0, e.val_len);
            rl_binding b;
            b.descriptor = e.descriptor;
            b._pad = 0;
            b.key = a;
            memcpy(a, msg + e.key_off, e.key_len);
            a[e.key_len] = 0;
            a += e.key_len + 1;
            b.value = a;
            memcpy(a, msg + e.val_off, e.val_len);
            a[e.val_len] = 0;
            a += e.val_len + 1;
            W.binds.push_back(b);
        }
        if (nul) {  // the matcher compares NUL-terminated strings: an embedded NUL would be cut, not compared
            W.binds.resize(first_bind);
            P.kind = REQ_UNSUPPORTED;
            continue;
        }
        W.bind_off.push_back((uint32_t)W.binds.size());
        W.ns.push_back(s->domains[i].c_str());  // (s->domains was sized before the workers started: the pointer stays)
        W.req_of.push_back(i);
    }
    const uint64_t k_req = W.req_of.size();
    W.ctr_off.assign(k_req + 1, 0);
    W.status.assign(k_req, 0);
    // room per request: the matcher's cap, but not more than the engine takes (a service without an engine: 16)
    const uint32_t engine_max = (s->engine && rl_engine_max_counters_per_request)
                                    ? rl_engine_max_counters_per_request(s->engine) : RL_MAX_COUNTERS_PER_REQUEST;
    const uint32_t per_req = std::min(rl_matcher_counter_cap(s->m), engine_max);
    W.ctrs.ensure((k_req + 1) * (size_t)per_req);
    if (rl_matcher_counters_batch_ns(s->m, k_req, W.ns.data(), W.bind_off.data(), W.binds.data(), W.ctr_off.data(), W.ctrs.data(),
                                     W.ctrs.size(), W.status.data()) != RL_OK) {
        for (const uint64_t i : W.req_of) s->plan[i].kind = REQ_UNSUPPORTED;  // (the matcher's cap was raised past the engine's)
        W.ctr_off.assign(k_req + 1, 0);
        return;
    }
    for (uint64_t k = 0; k < k_req; k++) {
        ReqPlan& P = s->plan[W.req_of[k]];
        P.n_ctr = W.ctr_off[k + 1] - W.ctr_off[k];
        // 2 = more counters than the engine takes per request; 1 = a namespace without limits (lib.rs:434-440)
        P.kind = W.status[k] == 2 ? REQ_UNSUPPORTED : (P.n_ctr ? REQ_STORE : REQ_NO_LIMITS);
        W.n_store += P.kind == REQ_STORE;
    }
}

// the delta of a store request: CheckRateLimit asks with delta 1 whatever hits_addend says (kuadrant_service.rs:62-65);
// HTTP sends the body's own delta, also for /check (server.rs:144)
uint64_t store_delta(const rl_rls* s, const ReqPlan& P) { return s->method == RL_RLS_CHECK_RATE_LIMIT ? 1 : P.hits; }
uint64_t store_delta(const rl_http*, const ReqPlan& P) { return P.delta; }

// Second pass of the plan: worker w copies its counters into the batch's CSR at the offsets the prefix over the workers
// gave it (store requests in batch order: worker ranges are consecutive).
template <class Svc>
void plan_scatter(Svc* s, uint32_t w, uint64_t store_base, uint64_t ctr_base) {
    WorkerOut& W = s->wout[w];
    uint64_t j = store_base, c = ctr_base;
    for (uint64_t k = 0; k < W.req_of.size(); k++) {
        const uint64_t i = W.req_of[k];
        ReqPlan& P = s->plan[i];
        if (P.kind != REQ_STORE) continue;
        P.store = (uint32_t)j;
        s->store_index[i] = (uint32_t)j;
        s->ctr_off[j] = (uint32_t)c;
        memcpy(s->ctrs.data() + c, W.ctrs.data() + W.ctr_off[k], (size_t)P.n_ctr * sizeof(rl_counter));
        s->delta[j] = store_delta(s, P);
        c += P.n_ctr;
        j++;
    }
}

// Second pass of the finish: worker w copies its responses behind those of the workers before it.
void finish_scatter(rl_rls* s, uint32_t w, uint64_t byte_base) {
    uint64_t lo, hi;
    range_of(s->n, s->pool->n, w, lo, hi);
    const WorkerOut& W = s->wout[w];
    if (!W.resp.empty()) memcpy(s->resp.data() + byte_base, W.resp.data(), W.resp.size());
    uint64_t at = byte_base;
    for (uint64_t i = lo; i < hi; i++) {
        at += W.resp_len[i - lo];
        s->resp_off[i + 1] = at;
    }
}

// Worker w's range [lo, hi) of the batch, with its finish outputs emptied.
WorkerOut& finish_worker(Batch* s, uint32_t w, uint64_t& lo, uint64_t& hi) {
    range_of(s->n, s->pool->n, w, lo, hi);
    WorkerOut& W = s->wout[w];
    W.resp.clear();
    W.resp_len.assign(hi - lo, 0);
    W.by_ns.clear();
    W.limited_by_name.clear();
    return W;
}

// The header values of the store requests in [lo, hi), which are one run of store indices from j0: ONE matcher call into
// W.hdr, made when `all` is set, or with `by_body` when one of the requests asks for draft-03 headers (HTTP).  Returns
// whether the values are there.
bool range_headers(const Batch* s, WorkerOut& W, uint64_t lo, uint64_t hi, bool all, bool by_body, const uint64_t* rem,
                   const uint64_t* ttl, uint64_t& j0) {
    j0 = RL_RLS_NO_STORE;
    uint64_t j1 = 0;
    bool want = all;
    for (uint64_t i = lo; i < hi; i++)
        if (s->plan[i].kind == REQ_STORE) {
            if (j0 == RL_RLS_NO_STORE) j0 = s->plan[i].store;
            j1 = (uint64_t)s->plan[i].store + 1;
            want = want || (by_body && s->plan[i].hdr == RL_HTTP_HEADERS_DRAFT_VERSION_03);
        }
    if (!want || j0 == RL_RLS_NO_STORE) return false;
    W.hdr_off.assign(j1 - j0 + 1, 0);
    uint64_t need = 0;
    W.hdr.resize(std::max<size_t>(W.hdr.size(), (size_t)(j1 - j0) * 96));
    int r = rl_matcher_response_headers_batch(s->m, j1 - j0, s->ctr_off.data() + j0, s->ctrs.data(), rem, ttl, W.hdr.data(), W.hdr.size(),
                                              W.hdr_off.data(), &need);
    if (r != RL_OK && need > W.hdr.size()) {
        W.hdr.resize(need);
        r = rl_matcher_response_headers_batch(s->m, j1 - j0, s->ctr_off.data() + j0, s->ctrs.data(), rem, ttl, W.hdr.data(), W.hdr.size(),
                                              W.hdr_off.data(), &need);
    }
    return r == RL_OK;
}

// The three X-RateLimit-* values range_headers fetched for store request j.
void header_values(const WorkerOut& W, uint64_t j, uint64_t j0, const char* vals[3]) {
    vals[0] = W.hdr.data() + W.hdr_off[j - j0];
    vals[1] = vals[0] + strlen(vals[0]) + 1;
    vals[2] = vals[1] + strlen(vals[1]) + 1;
}

// The worker's metrics entry of the namespace last counted: consecutive requests of one namespace share it.
struct NsCache {
    const std::string* ns = nullptr;
    NsCounts* counts = nullptr;
};

// Count decided request i into the worker's metrics: a limited one also under the name of its first limited limit when
// the service labels by name; an authorized one with `calls` calls and `hits` hits.
void count_decided(const Batch* s, WorkerOut& W, NsCache& at, uint64_t i, bool limited, bool by_name, const uint32_t* first,
                   uint64_t calls, uint64_t hits) {
    if (!at.ns || *at.ns != s->domains[i]) {
        at.ns = &s->domains[i];
        at.counts = &W.by_ns[s->domains[i]];
    }
    if (!limited) {
        at.counts->authorized_calls += calls;
        at.counts->authorized_hits += hits;
        return;
    }
    at.counts->limited_calls++;
    if (!by_name) return;
    std::string name;
    const uint32_t lid = first ? first[s->plan[i].store] : RL_NONE;
    if (lid != RL_NONE) {
        char nb[512];
        int has = 0;
        if (rl_matcher_limit_name_copy(s->m, lid, nb, sizeof nb, &has) == RL_OK && has) name = nb;
    }
    W.limited_by_name[{s->domains[i], name}]++;
}

// The workers' metrics into the RLS service's tables, which both surfaces count into.
void merge_metrics(rl_rls* s, const std::vector<WorkerOut>& wout) {
    for (const WorkerOut& W : wout) {
        for (const auto& kv : W.by_ns) {
            NsCounts& c = s->by_ns[kv.first];
            c.authorized_calls += kv.second.authorized_calls;
            c.authorized_hits += kv.second.authorized_hits;
            c.limited_calls += kv.second.limited_calls;
        }
        for (const auto& kv : W.limited_by_name) s->limited_by_name[kv.first] += kv.second;
    }
}

void finish_range(rl_rls* s, int store_status, const uint8_t* limited, const uint32_t* first, const uint64_t* rem, const uint64_t* ttl,
                  uint32_t w) {
    uint64_t lo, hi, j0;
    WorkerOut& W = finish_worker(s, w, lo, hi);
    static const char* const kKeys[3] = {"X-RateLimit-Limit", "X-RateLimit-Remaining", "X-RateLimit-Reset"};  // sorted by key (server.rs:55)
    const bool with_headers = store_status == RL_OK && s->method == RL_RLS_SHOULD_RATE_LIMIT && s->load_counters;
    const bool headers_ok = range_headers(s, W, lo, hi, with_headers, false, rem, ttl, j0);
    NsCache at;
    for (uint64_t i = lo; i < hi; i++) {
        const ReqPlan& P = s->plan[i];
        uint8_t grpc = RL_GRPC_OK, code = RL_RLS_CODE_UNKNOWN;
        uint32_t nh = 0;
        const char* vals[3] = {"", "", ""};
        switch (P.kind) {
            case REQ_BAD_WIRE: grpc = RL_GRPC_INTERNAL; break;
            case REQ_UNSUPPORTED: grpc = RL_GRPC_UNAVAILABLE; break;
            case REQ_UNKNOWN_DOMAIN: code = RL_RLS_CODE_UNKNOWN; break;
            case REQ_NO_LIMITS: code = RL_RLS_CODE_OK; break;
            case REQ_STORE: {
                if (store_status != RL_OK) {  // server.rs:160-172
                    grpc = RL_GRPC_UNAVAILABLE;
                    break;
                }
                const uint32_t j = P.store;
                if (s->method == RL_RLS_REPORT) {
                    if (s->report_verdicts && s->report_verdicts[j] == RL_VERDICT_ERROR) grpc = RL_GRPC_UNAVAILABLE;
                    else code = RL_RLS_CODE_OK;  // kuadrant_service.rs:176-178
                    break;
                }
                if (limited[j] == RL_VERDICT_ERROR) {
                    grpc = RL_GRPC_UNAVAILABLE;
                    break;
                }
                code = limited[j] ? RL_RLS_CODE_OVER_LIMIT : RL_RLS_CODE_OK;
                if (with_headers) {
                    if (!headers_ok) {
                        grpc = RL_GRPC_UNAVAILABLE;
                        break;
                    }
                    header_values(W, j, j0, vals);
                    nh = 3;
                }
                break;
            }
            default: grpc = RL_GRPC_INTERNAL; break;
        }
        s->grpc[i] = grpc;
        s->code[i] = grpc == RL_GRPC_OK ? code : 0;
        if (grpc != RL_GRPC_OK) continue;
        const size_t before = W.resp.size();
        encode_response(W.resp, code, kKeys, vals, nh);
        W.resp_len[i - lo] = W.resp.size() - before;
        // metrics, once per request after the decision (server.rs:183-195, kuadrant_service.rs:81-92,173-174), into the
        // worker's own table (merged after the workers are done)
        if (P.kind == REQ_UNKNOWN_DOMAIN) continue;
        const bool report = s->method == RL_RLS_REPORT;
        count_decided(s, W, at, i, !report && code == RL_RLS_CODE_OVER_LIMIT, s->use_limit_name, first, report ? 0 : 1,
                      s->method == RL_RLS_CHECK_RATE_LIMIT ? 0 : P.hits);
    }
}

// requests (RLS) or bodies (HTTP) are byte ranges [off[i], off[i + 1]) of the batch
int check_offsets(Batch* s, const char* what, uint64_t n, const uint64_t* off) {
    for (uint64_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) return sfail(s, "%s offsets must be non-decreasing (%s %llu)", what, what, (unsigned long long)i);
    return RL_OK;
}

int check_batch(rl_rls* s, int method, uint64_t n, const uint64_t* off) {
    if (method != RL_RLS_SHOULD_RATE_LIMIT && method != RL_RLS_CHECK_RATE_LIMIT && method != RL_RLS_REPORT)
        return sfail(s, "unknown method %d", method);
    return check_offsets(s, "request", n, off);
}

int check_batch(rl_http* h, int endpoint, uint64_t n, const uint64_t* off) {
    if (endpoint != RL_HTTP_CHECK && endpoint != RL_HTTP_REPORT && endpoint != RL_HTTP_CHECK_AND_REPORT)
        return sfail(h, "unknown endpoint %d", endpoint);
    return check_offsets(h, "body", n, off);
}

// What a device plan of either surface starts with: the checks (rl_rls_dev.cu's plans are linked together or not at all)
// and the new batch; now_us is set to the clock the plan runs at.
template <class Svc>
int device_plan_begin(Svc* s, int method, uint64_t n, const uint64_t* off, uint64_t& now_us) {
    if (!s->engine) return sfail(s, "the device plan needs a service created with an engine");
    if (!rl_rls_dev_plan) return sfail(s, "this build of the library has no device plan");
    const int r = check_batch(s, method, n, off);
    if (r) return r;
    s->planned = s->finished = false;
    s->method = method;
    s->n = n;
    if (!now_us) now_us = wall_us();
    return RL_OK;
}

// r, with the device state's reason in last_error when it is not RL_OK
int dev_fail(Batch* s, rl_rls_dev* dev, int r) {
    if (r) s->last_error = std::string("device plan: ") + rl_rls_dev_error(dev);
    return r;
}

// What a device plan of either surface ends with, given the status r of its rl_*_dev_plan call: the store request count
// and, with copy_csr, host copies of the CSR (and of HTTP's load flags, when `load` is given).
int device_plan_end(Batch* s, rl_rls_dev* dev, int r, uint64_t n_store, uint64_t n_ctr, uint64_t now_us, bool copy_csr,
                    std::vector<uint8_t>* load) {
    s->n_store = n_store;
    if (r || !copy_csr) return dev_fail(s, dev, r);
    s->ctr_off.resize(n_store + 1);
    s->ctrs.ensure(n_ctr);
    s->delta.resize(n_store);
    s->now.assign(n_store, now_us);
    if (load) load->resize(n_store);
    return dev_fail(s, dev,
                    rl_rls_dev_copy_plan(dev, s->ctr_off.data(), s->ctrs.data(), s->delta.data(), load ? load->data() : nullptr));
}

// The host arrays a served batch's store calls return into: the verdicts, and with `load` the remaining / ttl of the
// counters and the CSR their headers are formatted from.
void size_outputs(Batch* s, bool load, uint64_t n_ctr) {
    const uint64_t m = s->n_store;
    s->o_limited.resize(m);
    s->o_first.resize(m);
    if (load) {
        s->o_rem.resize(n_ctr);
        s->o_ttl.resize(n_ctr);
        s->ctr_off.resize(m + 1);
        s->ctrs.ensure(n_ctr);
    }
}

// rl_rls_plan_view / rl_http_plan_view but for load_counters, which each surface keeps its own way
int plan_view(Batch* s, uint64_t* out_n_store, const uint32_t** out_ctr_off, const rl_counter** out_ctrs, const uint64_t** out_delta,
              const uint64_t** out_now_us, const uint32_t** out_store_index) {
    if (!s->planned) return sfail(s, "no planned batch");
    if (out_n_store) *out_n_store = s->n_store;
    if (out_ctr_off) *out_ctr_off = s->ctr_off.data();
    if (out_ctrs) *out_ctrs = s->ctrs.data();
    if (out_delta) *out_delta = s->delta.data();
    if (out_now_us) *out_now_us = s->now.data();
    if (out_store_index) *out_store_index = s->store_index.data();
    return RL_OK;
}

// A served batch's stage times, from the clock at its start, after its plan, after its store calls and after the take of
// its plan; the finish ends now.
void stage_times(Batch* s, double t0, double t1, double t2, double t3) {
    const double t4 = mono_us();
    s->t_plan = (t1 - t0) + (t3 - t2);
    s->t_store = t2 - t1;
    s->t_finish = t4 - t3;
}

// Stage 1 on the engine's device (rl_rls_dev.cu).  Leaves the service as rl_rls_plan does, except for what the kernels
// wrote: the per-request outcomes are taken in by take_device_plan, and the CSR is copied to the host only with copy_csr
// (rl_rls_plan_device; rl_rls_serve keeps it on the device).
int plan_on_device(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us, bool copy_csr,
                   const RlsDevReq*& req, uint64_t& n_ctr) {
    int r = device_plan_begin(s, method, n, off, now_us);
    if (r) return r;
    uint64_t n_store = 0;
    r = rl_rls_dev_plan(&s->dev, s->engine, s->m, method, n, buf, off, now_us, &n_store, &n_ctr, &req);
    s->load_counters = (method == RL_RLS_SHOULD_RATE_LIMIT && s->header_mode != RL_RLS_HEADERS_NONE) ? 1 : 0;  // server.rs:146
    return device_plan_end(s, s->dev, r, n_store, n_ctr, now_us, copy_csr, nullptr);
}

// What the take of a device plan starts with, for either surface: the plan, domains and store index sized for the batch.
void size_plan(Batch* s) {
    s->plan.resize(s->n);
    s->domains.resize(s->n);
    s->store_index.resize(s->n);
}

// The per-request outcomes of a device plan (in host memory once rl_rls_dev_copy_plan / _wait returned) into the
// service's plan, store index and domains, on the worker pool.
void take_device_plan(rl_rls* s, const RlsDevReq* req, const uint8_t* buf, const uint64_t* off) {
    size_plan(s);
    s->pool->run([&](uint32_t w) {
        uint64_t lo, hi;
        range_of(s->n, s->pool->n, w, lo, hi);
        for (uint64_t i = lo; i < hi; i++) {
            const RlsDevReq& R = req[i];
            ReqPlan& P = s->plan[i];
            P.kind = (uint8_t)R.kind;
            P.hits = R.hits;
            P.n_ctr = 0;  // (read by the CPU plan's scatter only)
            P.store = R.store;
            s->store_index[i] = R.store;
            if (R.kind == REQ_BAD_WIRE) s->domains[i].clear();
            else s->domains[i].assign((const char*)buf + off[i] + R.dom_off, R.dom_len);
        }
    });
    s->planned = true;
}

// Stage 1 on the CPU workers, for both surfaces (the caller has checked the batch and sets what is its own after it).
template <class Svc>
int plan_cpu(Svc* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    s->planned = s->finished = false;
    s->method = method;
    s->n = n;
    s->buf = buf;
    s->plan.resize(n);
    s->domains.resize(n);
    s->pool->run([&](uint32_t w) { plan_range(s, off, w); });
    s->buf = nullptr;
    // lay the workers' counters out as one CSR, requests in batch order: a prefix over the workers, then every worker
    // copies its own slice
    std::vector<uint64_t> store_base(s->pool->n + 1, 0), ctr_base(s->pool->n + 1, 0);
    for (uint32_t w = 0; w < s->pool->n; w++) {
        const WorkerOut& W = s->wout[w];
        store_base[w + 1] = store_base[w] + W.n_store;
        ctr_base[w + 1] = ctr_base[w] + (W.ctr_off.empty() ? 0 : W.ctr_off.back());
    }
    const uint64_t n_store = store_base[s->pool->n], n_ctr = ctr_base[s->pool->n];
    if (n_ctr > 0xFFFFFFFFull) return sfail(s, "more than 2^32 counters in one batch");
    s->store_index.assign(n, RL_RLS_NO_STORE);
    s->ctr_off.assign(n_store + 1, 0);
    s->ctr_off[n_store] = (uint32_t)n_ctr;
    s->ctrs.ensure(n_ctr);
    s->delta.assign(n_store, 0);
    s->pool->run([&](uint32_t w) { plan_scatter(s, w, store_base[w], ctr_base[w]); });
    s->n_store = n_store;
    s->now.assign(s->n_store, now_us ? now_us : wall_us());
    return RL_OK;
}


// ---- the HTTP API (include/rl_http.h) ------------------------------------------------------------------------------
// Responses [lo, hi) of worker w (server.rs:129-260): status, body, X-RateLimit-* values, and the metrics of
// /check_and_report (server.rs:217-242).
void finish_range_http(rl_http* h, const int32_t* store_status, const uint8_t* limited, const uint32_t* first, const uint64_t* rem,
                       const uint64_t* ttl, uint32_t w) {
    uint64_t lo, hi, j0;
    WorkerOut& W = finish_worker(h, w, lo, hi);
    W.hval.clear();
    W.hval_len.assign(3 * (hi - lo), 0);
    const bool car = h->method == RL_HTTP_CHECK_AND_REPORT;
    const bool headers_ok = range_headers(h, W, lo, hi, false, car, rem, ttl, j0);
    NsCache at;
    for (uint64_t i = lo; i < hi; i++) {
        const ReqPlan& P = h->plan[i];
        uint16_t status = 500;
        bool decided = false, lim = false;
        const char* vals[3] = {"", "", ""};
        if (P.kind == REQ_BAD_WIRE) {
            status = 400;  // what the Json extractor answers
        } else if (P.kind == REQ_NO_LIMITS) {
            status = 200;  // lib.rs:434-440: nothing applies, nothing is limited
            decided = true;
        } else if (P.kind == REQ_STORE) {
            const uint32_t j = P.store;
            const bool failed = (store_status && store_status[j] != RL_OK) || (h->method != RL_HTTP_REPORT && limited[j] == RL_VERDICT_ERROR);
            if (!failed && h->method == RL_HTTP_REPORT) {
                status = 200;
            } else if (!failed) {
                lim = limited[j] != 0;
                status = lim ? 429 : 200;
                decided = true;
                if (car && P.hdr == RL_HTTP_HEADERS_DRAFT_VERSION_03) {  // server.rs:262-280
                    if (headers_ok) {
                        header_values(W, j, j0, vals);
                    } else {
                        status = 500;
                        decided = false;
                    }
                }
            }
        }  // REQ_UNSUPPORTED: 500
        h->status[i] = status;
        const char* body = "null";  // Json(()) and HttpResponse::...().json(())
        if (status == 500 && !car) body = "Internal server error";  // ErrorResponse's Display
        else if (status == 429 && !car) body = "Too many requests";
        else if (status == 400) body = "";
        const size_t bl = strlen(body);
        W.resp.insert(W.resp.end(), (const uint8_t*)body, (const uint8_t*)body + bl);
        W.resp_len[i - lo] = bl;
        for (int k = 0; k < 3; k++) {
            const size_t vl = strlen(vals[k]);
            W.hval.insert(W.hval.end(), (const uint8_t*)vals[k], (const uint8_t*)vals[k] + vl);
            W.hval_len[3 * (i - lo) + k] = vl;
        }
        if (car && decided) count_decided(h, W, at, i, lim, h->rls->use_limit_name, first, 1, P.delta);
    }
}

// Stage 1 of an HTTP batch on the engine's device, through the RLS service's device state (rl_rls_dev.cu).
int http_plan_on_device(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us, bool copy_csr,
                        const HttpDevReq*& req, uint64_t& n_ctr, const HttpRun*& runs, uint32_t& n_runs) {
    int r = device_plan_begin(h, endpoint, n, off, now_us);
    if (r) return r;
    uint64_t n_store = 0;
    rl_rls* s = h->rls;
    r = rl_http_dev_plan(&s->dev, h->engine, h->m, endpoint, n, buf, off, now_us, &n_store, &n_ctr, &req, &runs, &n_runs);
    return device_plan_end(h, s->dev, r, n_store, n_ctr, now_us, copy_csr, &h->load);
}

// The per-body outcomes of a device plan into the service's plan, store index and namespaces.  The namespace comes from
// the host's copy of the body, unescaped again (rl_json.h) when its source holds a backslash.
void take_http_device_plan(rl_http* h, const HttpDevReq* req, const uint8_t* buf, const uint64_t* off) {
    size_plan(h);
    h->pool->run([&](uint32_t w) {
        uint64_t lo, hi;
        range_of(h->n, h->pool->n, w, lo, hi);
        WorkerOut& W = h->wout[w];
        for (uint64_t i = lo; i < hi; i++) {
            const HttpDevReq& R = req[i];
            ReqPlan& P = h->plan[i];
            P = ReqPlan();
            P.kind = (uint8_t)R.kind;
            P.hdr = (uint8_t)R.headers;
            P.delta = R.delta;
            P.store = R.store;
            h->store_index[i] = R.store;
            const uint8_t* src = buf + off[i] + R.dom_off;
            if (R.kind == REQ_BAD_WIRE) {
                h->domains[i].clear();
            } else if (memchr(src, '\\', R.dom_len) == nullptr) {  // (an escape makes the source longer than the string)
                h->domains[i].assign((const char*)src, R.dom_len);
            } else {
                const uint64_t len = off[i + 1] - off[i];
                W.txt.ensure(len + 1);
                const uint32_t l = rl_json::unescape(buf + off[i], len, R.dom_off, W.txt.data());
                h->domains[i].assign((const char*)W.txt.data() + R.dom_off, l);
            }
        }
    });
    h->planned = true;
}

// ---- GET /limits and GET /counters (include/rl_http.h) -----------------------------------------------------------
// A string as serde_json writes it (ser.rs format_escaped_str): the short escapes, \u00XX (lower-case hex) for the other
// control characters, every other byte as it is (the strings are UTF-8 already).
void json_str(std::string& o, const char* p, size_t n) {
    static const char kHex[] = "0123456789abcdef";
    o.push_back('"');
    for (size_t i = 0; i < n; i++) {
        const unsigned char c = (unsigned char)p[i];
        switch (c) {
            case '"': o += "\\\""; break;
            case '\\': o += "\\\\"; break;
            case '\b': o += "\\b"; break;
            case '\f': o += "\\f"; break;
            case '\n': o += "\\n"; break;
            case '\r': o += "\\r"; break;
            case '\t': o += "\\t"; break;
            default:
                if (c < 0x20) {
                    o += "\\u00";
                    o.push_back(kHex[c >> 4]);
                    o.push_back(kHex[c & 15]);
                } else {
                    o.push_back((char)c);
                }
        }
    }
    o.push_back('"');
}
void json_str(std::string& o, const std::string& s) { json_str(o, s.data(), s.size()); }

void json_str_list(std::string& o, const std::vector<std::string>& v) {
    o.push_back('[');
    for (size_t i = 0; i < v.size(); i++) {
        if (i) o.push_back(',');
        json_str(o, v[i]);
    }
    o.push_back(']');
}

// request_types.rs Limit; id is null for limits added without one (rl_matcher_add_limit)
void json_limit(std::string& o, const std::string& ns, const RlLimitRecord& L) {
    o += "{\"id\":";
    if (L.has_id) json_str(o, L.id);
    else o += "null";
    o += ",\"namespace\":";
    json_str(o, ns);
    o += ",\"max_value\":" + std::to_string(L.max_value) + ",\"seconds\":" + std::to_string(L.seconds) + ",\"name\":";
    if (L.has_name) json_str(o, L.name);
    else o += "null";
    o += ",\"conditions\":";
    json_str_list(o, L.conditions);
    o += ",\"variables\":";
    json_str_list(o, L.variables);
    o.push_back('}');
}

void get_answer(rl_http* h, uint16_t status, std::string body, uint64_t unnamed) {
    h->get_status = status;
    h->get_body = std::move(body);
    h->get_unnamed = unnamed;
}

// Counter i's set_variables from its blob, or false when the blob does not hold exactly one value per variable.
bool blob_values(const uint8_t* b, uint64_t len, size_t n_vars, std::vector<std::pair<const char*, uint32_t>>& out) {
    out.clear();
    uint64_t at = 0;
    while (at < len) {
        if (len - at < 4) return false;
        const uint32_t l = (uint32_t)b[at] | (uint32_t)b[at + 1] << 8 | (uint32_t)b[at + 2] << 16 | (uint32_t)b[at + 3] << 24;
        at += 4;
        if (len - at < l) return false;
        out.emplace_back((const char*)b + at, l);
        at += l;
    }
    return out.size() == n_vars;
}

// The /counters body of namespace ns over the given counters (the rendering stage of rl_http_get_counters).
void render_counters(rl_http* h, const std::string& ns, uint64_t n, const rl_counter* ctrs, const uint64_t* rem, const uint64_t* ttl,
                     const uint8_t* blobs, const uint64_t* blob_off, const uint8_t* unnamed) {
    std::vector<RlLimitRecord> lims;
    if (!rl_matcher_ns_limit_records(h->m, ns, lims)) return get_answer(h, 200, "[]", 0);
    std::unordered_map<uint32_t, uint32_t> pos;  // limit id -> position among the namespace's live limits
    for (uint32_t k = 0; k < lims.size(); k++) pos[lims[k].limit_id] = k;
    struct Row {
        uint32_t pos;
        uint64_t lo, hi, i;
    };
    std::vector<Row> rows;
    for (uint64_t i = 0; i < n; i++) {
        const auto it = pos.find(ctrs[i].limit_id);
        if (it != pos.end()) rows.push_back({it->second, ctrs[i].key_lo, ctrs[i].key_hi, i});
    }
    std::sort(rows.begin(), rows.end(), [](const Row& a, const Row& b) {
        return a.pos != b.pos ? a.pos < b.pos : a.lo != b.lo ? a.lo < b.lo : a.hi != b.hi ? a.hi < b.hi : a.i < b.i;
    });
    std::string o = "[";
    uint64_t bad = 0;
    std::vector<std::pair<const char*, uint32_t>> vals;
    for (const Row& r : rows) {
        const RlLimitRecord& L = lims[r.pos];
        const uint64_t i = r.i;
        if (!L.variables.empty() &&
            ((unnamed && unnamed[i]) || !blob_values(blobs + blob_off[i], blob_off[i + 1] - blob_off[i], L.variables.size(), vals))) {
            bad++;
            continue;
        }
        if (o.size() > 1) o.push_back(',');
        o += "{\"limit\":";
        json_limit(o, ns, L);
        o += ",\"set_variables\":{";
        for (size_t v = 0; v < L.variables.size(); v++) {  // sorted by source, as a BTreeMap
            if (v) o.push_back(',');
            json_str(o, L.variables[v]);
            o.push_back(':');
            json_str(o, vals[v].first, vals[v].second);
        }
        o += "},\"remaining\":" + std::to_string(rem[i]) + ",\"expires_in_seconds\":" + std::to_string(ttl[i] / 1000000ull) + "}";
    }
    o.push_back(']');
    if (bad) {
        h->last_error = std::to_string(bad) + " qualified counter(s) of namespace have no recorded variables";
        return get_answer(h, 500, "Internal server error", bad);
    }
    get_answer(h, 200, std::move(o), 0);
}

}  // namespace

extern "C" {

int rl_rls_decode_request(const uint8_t* buf, uint64_t len, rl_rls_request* out, rl_rls_entry* entries, uint32_t cap_entries) {
    if (!out || (len && !buf) || (cap_entries && !entries)) return RL_FATAL;
    EntrySink sink{entries, cap_entries};
    return decode_request(buf, len, *out, sink) ? RL_OK : RL_FATAL;
}

int rl_rls_encode_response(uint32_t overall_code, const char* const* keys, const char* const* values, uint32_t n_headers,
                           uint8_t* out, uint64_t cap, uint64_t* out_len) {
    if (!out_len || (n_headers && (!keys || !values))) return RL_FATAL;
    std::vector<uint8_t> o;
    encode_response(o, overall_code, keys, values, n_headers);
    *out_len = o.size();
    if (o.size() > cap || (!out && !o.empty())) return RL_FATAL;
    if (!o.empty()) memcpy(out, o.data(), o.size());
    return RL_OK;
}

int rl_rls_create(rl_matcher* m, rl_engine* engine, int header_mode, uint32_t threads, int use_limit_name_label, rl_rls** out) {
    if (!m || !out) return RL_FATAL;
    if (header_mode != RL_RLS_HEADERS_NONE && header_mode != RL_RLS_HEADERS_DRAFT_VERSION_03) return RL_FATAL;
    rl_rls* s = new rl_rls();
    s->m = m;
    s->engine = engine;
    s->header_mode = header_mode;
    s->use_limit_name = use_limit_name_label != 0;
    if (threads == 0) threads = std::max(1u, std::thread::hardware_concurrency());
    threads = std::min<uint32_t>(threads, 64);
    s->pool = new Pool(threads);
    s->wout.resize(threads);
    *out = s;
    return RL_OK;
}

void rl_rls_destroy(rl_rls* s) {
    if (!s) return;
    if (s->dev && rl_rls_dev_destroy) rl_rls_dev_destroy(s->dev);
    delete s->pool;
    delete s;
}

const char* rl_rls_last_error(rl_rls* s) { return s ? s->last_error.c_str() : "null service"; }

int rl_rls_plan(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!s || (n && (!off || !buf))) return RL_FATAL;
    int r = check_batch(s, method, n, off);
    if (r) return r;
    if ((r = plan_cpu(s, method, n, buf, off, now_us))) return r;
    s->load_counters = (method == RL_RLS_SHOULD_RATE_LIMIT && s->header_mode != RL_RLS_HEADERS_NONE) ? 1 : 0;  // server.rs:146
    s->planned = true;
    return RL_OK;
}

int rl_rls_plan_device(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!s || (n && (!off || !buf))) return RL_FATAL;
    const RlsDevReq* req = nullptr;
    uint64_t n_ctr = 0;
    const int r = plan_on_device(s, method, n, buf, off, now_us, true, req, n_ctr);
    if (r) return r;
    take_device_plan(s, req, buf, off);
    return RL_OK;
}

int rl_rls_plan_view(rl_rls* s, uint64_t* out_n_store, const uint32_t** out_ctr_off, const rl_counter** out_ctrs,
                     const uint64_t** out_delta, const uint64_t** out_now_us, int* out_load_counters,
                     const uint32_t** out_store_index) {
    if (!s) return RL_FATAL;
    const int r = plan_view(s, out_n_store, out_ctr_off, out_ctrs, out_delta, out_now_us, out_store_index);
    if (r == RL_OK && out_load_counters) *out_load_counters = s->load_counters;
    return r;
}

int rl_rls_finish(rl_rls* s, int store_status, const uint8_t* limited, const uint32_t* first_limited,
                  const uint64_t* remaining, const uint64_t* ttl_us) {
    if (!s) return RL_FATAL;
    if (!s->planned) return sfail(s, "no planned batch");
    const bool need_verdicts = s->n_store && store_status == RL_OK && s->method != RL_RLS_REPORT;
    if (need_verdicts && !limited) return sfail(s, "finish needs the verdicts of the store call");
    if (need_verdicts && s->load_counters && (!remaining || !ttl_us))
        return sfail(s, "finish needs remaining / ttl of the store call (draft-03 headers)");
    s->grpc.assign(s->n, 0);
    s->code.assign(s->n, 0);
    s->pool->run([&](uint32_t w) { finish_range(s, store_status, limited, first_limited, remaining, ttl_us, w); });
    // the workers' responses behind one another (a prefix over the workers, then every worker copies its own), their
    // metrics merged
    std::vector<uint64_t> byte_base(s->pool->n + 1, 0);
    for (uint32_t w = 0; w < s->pool->n; w++) byte_base[w + 1] = byte_base[w] + s->wout[w].resp.size();
    s->resp.ensure(byte_base[s->pool->n]);
    s->resp_off.assign(s->n + 1, 0);
    s->pool->run([&](uint32_t w) { finish_scatter(s, w, byte_base[w]); });
    merge_metrics(s, s->wout);
    s->finished = true;
    s->planned = false;  // a batch is finished once: its metrics are counted once
    return RL_OK;
}

int rl_rls_responses(rl_rls* s, const uint8_t** out_buf, const uint64_t** out_off, const uint8_t** out_grpc, const uint8_t** out_code) {
    if (!s) return RL_FATAL;
    if (!s->finished) return sfail(s, "no finished batch");
    static const uint8_t kEmpty = 0;
    if (out_buf) *out_buf = s->resp.size() ? s->resp.data() : &kEmpty;
    if (out_off) *out_off = s->resp_off.data();
    if (out_grpc) *out_grpc = s->grpc.empty() ? &kEmpty : s->grpc.data();
    if (out_code) *out_code = s->code.empty() ? &kEmpty : s->code.data();
    return RL_OK;
}

int rl_rls_serve(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!s) return RL_FATAL;
    if (s->shard) return rl_rls_serve_sharded(s, method, n, buf, off, now_us);
    if (!s->engine) return sfail(s, "the service was created without an engine: there is no CPU store to fall back to");
    if (n && (!off || !buf)) return RL_FATAL;
    // plan on the device: the store call's CSR stays there
    const double t0 = mono_us();
    const RlsDevReq* req = nullptr;
    uint64_t n_ctr = 0;
    int r = plan_on_device(s, method, n, buf, off, now_us, false, req, n_ctr);
    if (r) return r;
    const double t1 = mono_us();
    // the store call on the device arrays; only what the finish reads comes back
    size_outputs(s, s->load_counters, n_ctr);
    const int st = rl_rls_dev_decide(s->dev, s->engine, method, s->load_counters, s->o_limited.data(), s->o_first.data(),
                                     s->o_rem.data(), s->o_ttl.data(), s->ctr_off.data(), s->ctrs.data());
    if (st != RL_OK) s->last_error = std::string("store call failed: ") + rl_last_error(s->engine);
    if ((r = dev_fail(s, s->dev, rl_rls_dev_wait(s->dev)))) return r;
    const double t2 = mono_us();
    take_device_plan(s, req, buf, off);
    const double t3 = mono_us();
    r = rl_rls_finish(s, st, s->o_limited.data(), s->o_first.data(), s->o_rem.data(), s->o_ttl.data());
    stage_times(s, t0, t1, t2, t3);
    return r;
}

// The engine's half of rl_rls_configure, on the matcher's staged plan: register the added limits and the new maxima, then
// delete the removed limits in one call.  On a refusal, what was set is undone, so that the engine is as it was.
static int configure_engine(rl_engine* e, RlConfigurePlan& plan) {
    if (!rl_limits_set || !rl_limits_delete || !rl_fence) {
        plan.error = "this build of the library has no engine";
        return RL_FATAL;
    }
    int r = rl_fence(e);  // pipelined record calls still read the limit tables that rl_limits_set marks for upload
    if (r) {
        plan.error = std::string("fencing the pipelined calls: ") + rl_last_error(e);
        return r;
    }
    const auto undo = [&](size_t upto) {
        std::vector<uint32_t> drop;
        for (size_t k = 0; k < upto; k++) {
            if (plan.set_added[k]) {
                drop.push_back(plan.set[k].limit_id);
                continue;
            }
            rl_limit_desc d = plan.set[k];
            d.max_value = plan.old_max[k];
            rl_limits_set(e, &d, 1);
        }
        if (!drop.empty()) rl_limits_delete(e, drop.data(), (uint32_t)drop.size());
    };
    for (size_t k = 0; k < plan.set.size(); k++) {
        if ((r = rl_limits_set(e, &plan.set[k], 1)) == RL_OK) continue;
        const std::string why = rl_last_error(e);
        undo(k);
        plan.refused = plan.set_entry[k];
        plan.error = rl_format("entry %u: the engine refused the limit: %s", plan.set_entry[k], why.c_str());
        return r;
    }
    if (!plan.deleted.empty() && (r = rl_limits_delete(e, plan.deleted.data(), (uint32_t)plan.deleted.size())) != RL_OK) {
        const std::string why = rl_last_error(e);
        undo(plan.set.size());
        plan.error = "deleting the removed limits: " + why;
        return r;
    }
    return RL_OK;
}

int rl_rls_metrics_render(rl_rls* s, char* out, uint64_t cap, uint64_t* out_len) {
    if (!s || !out_len) return RL_FATAL;
    std::string t;
    auto esc = [](const std::string& v) {  // label values: backslash, quote and newline are escaped
        std::string o;
        for (const char c : v) {
            if (c == '\\') o += "\\\\";
            else if (c == '"') o += "\\\"";
            else if (c == '\n') o += "\\n";
            else o.push_back(c);
        }
        return o;
    };
    t += "# TYPE authorized_calls counter\n";
    for (const auto& kv : s->by_ns)
        if (kv.second.authorized_calls)
            t += "authorized_calls{limitador_namespace=\"" + esc(kv.first) + "\"} " + std::to_string(kv.second.authorized_calls) + "\n";
    t += "# TYPE authorized_hits counter\n";
    for (const auto& kv : s->by_ns)
        if (kv.second.authorized_hits)
            t += "authorized_hits{limitador_namespace=\"" + esc(kv.first) + "\"} " + std::to_string(kv.second.authorized_hits) + "\n";
    t += "# TYPE limited_calls counter\n";
    if (s->use_limit_name) {
        for (const auto& kv : s->limited_by_name)
            t += "limited_calls{limitador_namespace=\"" + esc(kv.first.first) + "\",limit_name=\"" + esc(kv.first.second) + "\"} " +
                 std::to_string(kv.second) + "\n";
    } else {
        for (const auto& kv : s->by_ns)
            if (kv.second.limited_calls)
                t += "limited_calls{limitador_namespace=\"" + esc(kv.first) + "\"} " + std::to_string(kv.second.limited_calls) + "\n";
    }
    t += "# TYPE limitador_up gauge\nlimitador_up 1\n";
    *out_len = t.size() + 1;
    if (!out || cap < t.size() + 1) return RL_FATAL;
    memcpy(out, t.c_str(), t.size() + 1);
    return RL_OK;
}

int rl_rls_last_timings(rl_rls* s, double* out_plan_us, double* out_store_us, double* out_finish_us) {
    if (!s) return RL_FATAL;
    if (out_plan_us) *out_plan_us = s->t_plan;
    if (out_store_us) *out_store_us = s->t_store;
    if (out_finish_us) *out_finish_us = s->t_finish;
    return RL_OK;
}

int rl_rls_configure(rl_rls* s, const rl_limit_spec* limits, uint32_t n, int dry_run, rl_configure_report* out_report) {
    if (!s || (n && !limits)) return RL_FATAL;
    if (out_report) *out_report = rl_configure_report{0, 0, 0, 0, RL_NONE, 0};
    const uint32_t engine_max = (s->engine && rl_engine_max_counters_per_request)
                                    ? rl_engine_max_counters_per_request(s->engine) : RL_MAX_COUNTERS_PER_REQUEST;
    RlConfigurePlan plan;
    std::function<int(RlConfigurePlan&)> apply;
    if (s->engine) apply = [s](RlConfigurePlan& p) { return configure_engine(s->engine, p); };
    const int r = rl_matcher_configure(s->m, limits, n, engine_max, dry_run != 0, plan, apply);
    if (out_report) {
        *out_report = rl_configure_report{plan.kept, plan.added, plan.updated, (uint32_t)plan.deleted.size(), plan.refused, 0};
        if (r != RL_OK) out_report->kept = out_report->added = out_report->updated = out_report->deleted = 0;
    }
    if (r != RL_OK) s->last_error = plan.error.empty() ? "configure: invalid arguments" : plan.error;
    if (!dry_run) {
        if (r == RL_OK) {
            s->config_version++;
            s->config_err_since = 0;
        } else {
            s->config_err_since++;
        }
    }
    return r;
}

int rl_rls_config_status(rl_rls* s, uint64_t* out_version, uint64_t* out_err_since) {
    if (!s) return RL_FATAL;
    if (out_version) *out_version = s->config_version;
    if (out_err_since) *out_err_since = s->config_err_since;
    return RL_OK;
}

// ---- the HTTP API --------------------------------------------------------------------------------------------------
int rl_http_decode_body(const uint8_t* body, uint64_t len, uint8_t* txt, rl_http_info* out, rl_rls_entry* entries,
                        uint32_t cap_entries) {
    if (!out || (len && (!body || !txt)) || (cap_entries && !entries)) return RL_FATAL;
    std::vector<uint8_t> bits(len / 8 + 1);
    EntrySink sink{entries, cap_entries, 0};
    rl_json::Info q;
    if (!rl_json::decode_info(body, len, txt, bits.data(), q, sink)) return RL_FATAL;
    *out = rl_http_info{q.ns_off, q.ns_len, q.delta, q.n_entries, q.headers};
    return RL_OK;
}

int rl_http_create(rl_rls* rls, rl_http** out) {
    if (!rls || !out) return RL_FATAL;
    rl_http* h = new rl_http();
    h->rls = rls;
    h->m = rls->m;
    h->engine = rls->engine;
    h->pool = rls->pool;
    h->wout.resize(rls->pool->n);
    *out = h;
    return RL_OK;
}

void rl_http_destroy(rl_http* h) { delete h; }

const char* rl_http_last_error(rl_http* h) { return h ? h->last_error.c_str() : "null service"; }

int rl_http_plan(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!h || (n && (!off || !buf))) return RL_FATAL;
    int r = check_batch(h, endpoint, n, off);
    if (r) return r;
    if ((r = plan_cpu(h, endpoint, n, buf, off, now_us))) return r;
    h->load.assign(h->n_store, 0);
    for (uint64_t i = 0; i < n; i++)
        if (h->plan[i].kind == REQ_STORE) h->load[h->plan[i].store] = rl_json::load_counters(endpoint, h->plan[i].hdr);
    h->planned = true;
    return RL_OK;
}

int rl_http_plan_device(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!h || (n && (!off || !buf))) return RL_FATAL;
    const HttpDevReq* req = nullptr;
    const HttpRun* runs = nullptr;
    uint64_t n_ctr = 0;
    uint32_t n_runs = 0;
    const int r = http_plan_on_device(h, endpoint, n, buf, off, now_us, true, req, n_ctr, runs, n_runs);
    if (r) return r;
    take_http_device_plan(h, req, buf, off);
    return RL_OK;
}

int rl_http_plan_view(rl_http* h, uint64_t* out_n_store, const uint32_t** out_ctr_off, const rl_counter** out_ctrs,
                      const uint64_t** out_delta, const uint64_t** out_now_us, const uint8_t** out_load_counters,
                      const uint32_t** out_store_index) {
    if (!h) return RL_FATAL;
    const int r = plan_view(h, out_n_store, out_ctr_off, out_ctrs, out_delta, out_now_us, out_store_index);
    if (r == RL_OK && out_load_counters) *out_load_counters = h->load.data();
    return r;
}

int rl_http_finish(rl_http* h, const int32_t* store_status, const uint8_t* limited, const uint32_t* first_limited,
                   const uint64_t* remaining, const uint64_t* ttl_us) {
    if (!h) return RL_FATAL;
    if (!h->planned) return sfail(h, "no planned batch");
    if (h->n_store && h->method != RL_HTTP_REPORT && !limited) return sfail(h, "finish needs the verdicts of the store calls");
    bool headers = false;
    for (uint64_t i = 0; i < h->n && !headers; i++)
        headers = h->plan[i].kind == REQ_STORE && h->method == RL_HTTP_CHECK_AND_REPORT && h->plan[i].hdr == RL_HTTP_HEADERS_DRAFT_VERSION_03;
    if (headers && (!remaining || !ttl_us)) return sfail(h, "finish needs remaining / ttl of the store calls (draft-03 headers)");
    h->status.assign(h->n, 0);
    h->pool->run([&](uint32_t w) { finish_range_http(h, store_status, limited, first_limited, remaining, ttl_us, w); });
    // the workers' bodies and header values behind one another, their metrics merged into the RLS service's
    const uint32_t nw = h->pool->n;
    std::vector<uint64_t> bb(nw + 1, 0), hb(nw + 1, 0);
    for (uint32_t w = 0; w < nw; w++) {
        bb[w + 1] = bb[w] + h->wout[w].resp.size();
        hb[w + 1] = hb[w] + h->wout[w].hval.size();
    }
    h->body.ensure(bb[nw]);
    h->hval.ensure(hb[nw]);
    h->body_off.assign(h->n + 1, 0);
    h->hval_off.assign(3 * h->n + 1, 0);
    h->pool->run([&](uint32_t w) {
        uint64_t lo, hi;
        range_of(h->n, nw, w, lo, hi);
        const WorkerOut& W = h->wout[w];
        if (!W.resp.empty()) memcpy(h->body.data() + bb[w], W.resp.data(), W.resp.size());
        if (!W.hval.empty()) memcpy(h->hval.data() + hb[w], W.hval.data(), W.hval.size());
        uint64_t at = bb[w], hat = hb[w];
        for (uint64_t i = lo; i < hi; i++) {
            at += W.resp_len[i - lo];
            h->body_off[i + 1] = at;
            for (int k = 0; k < 3; k++) {
                hat += W.hval_len[3 * (i - lo) + k];
                h->hval_off[3 * i + k + 1] = hat;
            }
        }
    });
    merge_metrics(h->rls, h->wout);
    h->finished = true;
    h->planned = false;  // a batch is finished once: its metrics are counted once
    return RL_OK;
}

int rl_http_responses(rl_http* h, const uint16_t** out_status, const uint8_t** out_body, const uint64_t** out_body_off,
                      const uint8_t** out_hdr, const uint64_t** out_hdr_off) {
    if (!h) return RL_FATAL;
    if (!h->finished) return sfail(h, "no finished batch");
    static const uint8_t kEmpty = 0;
    static const uint16_t kNone = 0;
    if (out_status) *out_status = h->status.empty() ? &kNone : h->status.data();
    if (out_body) *out_body = h->body.size() ? h->body.data() : &kEmpty;
    if (out_body_off) *out_body_off = h->body_off.data();
    if (out_hdr) *out_hdr = h->hval.size() ? h->hval.data() : &kEmpty;
    if (out_hdr_off) *out_hdr_off = h->hval_off.data();
    return RL_OK;
}

int rl_http_serve(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!h) return RL_FATAL;
    if (h->rls->shard) return rl_http_serve_sharded(h, endpoint, n, buf, off, now_us);
    if (!h->engine) return sfail(h, "the service was created without an engine: there is no CPU store to fall back to");
    if (n && (!off || !buf)) return RL_FATAL;
    const double t0 = mono_us();
    const HttpDevReq* req = nullptr;
    const HttpRun* runs = nullptr;
    uint64_t n_ctr = 0;
    uint32_t n_runs = 0;
    int r = http_plan_on_device(h, endpoint, n, buf, off, now_us, false, req, n_ctr, runs, n_runs);
    if (r) return r;
    const double t1 = mono_us();
    // one store call per run on the device arrays; only what the finish reads comes back
    const uint64_t m = h->n_store;
    bool any_load = false;
    for (uint32_t k = 0; k < n_runs; k++) any_load = any_load || runs[k].load;
    size_outputs(h, any_load, n_ctr);
    h->run_status.assign(n_runs, RL_OK);
    const int st = rl_http_dev_decide(h->rls->dev, h->engine, endpoint, h->run_status.data(), h->o_limited.data(), h->o_first.data(),
                                      h->o_rem.data(), h->o_ttl.data(), h->ctr_off.data(), h->ctrs.data());
    if (st != RL_OK) h->run_status.assign(n_runs, st);
    for (uint32_t k = 0; k < n_runs; k++)
        if (h->run_status[k] != RL_OK) h->last_error = std::string("store call failed: ") + rl_last_error(h->engine);
    if ((r = dev_fail(h, h->rls->dev, rl_rls_dev_wait(h->rls->dev)))) return r;
    h->o_status.resize(m);
    for (uint32_t k = 0; k < n_runs; k++) {
        const uint64_t j1 = k + 1 < n_runs ? runs[k + 1].store : m;
        for (uint64_t j = runs[k].store; j < j1; j++) h->o_status[j] = h->run_status[k];
    }
    h->store_calls = n_runs;
    const double t2 = mono_us();
    take_http_device_plan(h, req, buf, off);
    const double t3 = mono_us();
    r = rl_http_finish(h, h->o_status.data(), h->o_limited.data(), h->o_first.data(), h->o_rem.data(), h->o_ttl.data());
    stage_times(h, t0, t1, t2, t3);
    return r;
}

int rl_http_last_timings(rl_http* h, double* out_plan_us, double* out_store_us, double* out_finish_us, uint32_t* out_store_calls) {
    if (!h) return RL_FATAL;
    if (out_plan_us) *out_plan_us = h->t_plan;
    if (out_store_us) *out_store_us = h->t_store;
    if (out_finish_us) *out_finish_us = h->t_finish;
    if (out_store_calls) *out_store_calls = h->store_calls;
    return RL_OK;
}

// ---- serving on a namespace-sharded store (rl_shard_batch, include/rl_engine.h) ------------------------------------
static const char* const kShardedNoCvars =
    "counter variables are kept by one engine's service: a service with a sharded store does not keep, export, import or drain them";

namespace {

// The send half of a sharded step for either surface, after its device plan returned r: the plan's store requests (or,
// when the plan failed, an empty batch: every rank takes part in every step) go to their owners.
int sharded_send(Batch* s, rl_rls_dev* dev, rl_shard_batch* sb, bool http, int method, int r, bool load, double t0) {
    s->sh_plan = r;
    s->sh_load = load;
    s->sh_status = RL_OK;
    s->sh_error.clear();
    s->sh_t0 = t0;
    int failed = RL_OK;
    const int st = rl_rls_dev_shard_send(r ? nullptr : dev, sb, r != 0, http, method, load, &failed);
    if (st) {  // refused before anything went out (a protocol error of the caller): there is nothing to collect
        s->sh_pending = false;
        if (!r) s->last_error = std::string("sharded store: ") + rl_last_error(s->engine);
        return r ? r : st;
    }
    if (failed) s->sh_plan = dev_fail(s, dev, failed);  // the batch went out empty
    s->sh_pending = true;
    s->sh_t1 = mono_us();
    return RL_OK;
}

int sharded_decide(Batch* s, rl_shard_batch* sb) {
    if (!s->sh_pending) return sfail(s, "no sharded step sent");
    const int st = rl_shard_batch_decide(sb);
    if (st != RL_OK && s->sh_status == RL_OK) {
        s->sh_error = std::string("sharded store: ") + rl_last_error(s->engine);
        s->sh_status = st;
    }
    return RL_OK;
}

// The collect of a sharded step into the batch's output arrays; its status, or the plan's when that failed
int sharded_collect(Batch* s, rl_rls_dev* dev, rl_shard_batch* sb, int& store_status) {
    if (!s->sh_pending) return sfail(s, "no sharded step sent");
    s->sh_pending = false;
    store_status = rl_rls_dev_shard_collect(s->sh_plan ? nullptr : dev, sb, s->sh_load, s->o_limited.data(), s->o_first.data(),
                                            s->o_rem.data(), s->o_ttl.data(), s->ctr_off.data(), s->ctrs.data());
    if (store_status != RL_OK && store_status != RL_TRANSIENT) s->last_error = std::string("store call failed: ") + rl_last_error(s->engine);
    return s->sh_plan;
}

// the step's status once the batch is finished: a failed finish, else what the decide reported (the digest check)
int sharded_status(Batch* s, int r) {
    if (r) return r;
    if (s->sh_status == RL_FATAL) {
        s->last_error = s->sh_error;
        return RL_FATAL;
    }
    return RL_OK;
}

}  // namespace

int rl_rls_attach_shard(rl_rls* s, rl_shard_batch* shard) {
    if (!s) return RL_FATAL;
    if (shard) {
        if (!s->engine) return sfail(s, "a sharded store needs a service created with an engine");
        if (!rl_rls_dev_shard_send) return sfail(s, "this build of the library has no device plan");
        if (rl_shard_batch_engine(shard) != s->engine) return sfail(s, "the sharded store was created on another engine than the service's");
        uint64_t slots = 0;
        if (s->dev && rl_cv_dev_stats && rl_cv_dev_stats(s->dev, &slots, nullptr, nullptr, nullptr) == RL_OK && slots)
            return sfail(s, "%s (turn keeping off first)", kShardedNoCvars);
    }
    s->shard = shard;
    return RL_OK;
}

int rl_rls_send(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!s) return RL_FATAL;
    if (!s->shard) return sfail(s, "no sharded store attached (rl_rls_attach_shard)");
    if (s->sh_pending) return sfail(s, "the previous sharded step is not collected");
    const double t0 = mono_us();
    const RlsDevReq* req = nullptr;
    uint64_t n_ctr = 0;
    int r = n && (!off || !buf) ? sfail(s, "null request buffer or offsets") : plan_on_device(s, method, n, buf, off, now_us, false, req, n_ctr);
    if (r == RL_OK) size_outputs(s, s->load_counters, n_ctr);
    if ((r = sharded_send(s, s->dev, s->shard, false, method, r, r == RL_OK && s->load_counters, t0))) return r;
    if (s->sh_plan) return RL_OK;
    // the per-request outcomes now (the wire bytes need not outlive this call)
    if ((r = dev_fail(s, s->dev, rl_rls_dev_wait(s->dev)))) {
        s->sh_plan = r;
        return RL_OK;
    }
    take_device_plan(s, req, buf, off);
    return RL_OK;
}

int rl_rls_decide(rl_rls* s) {
    if (!s) return RL_FATAL;
    return sharded_decide(s, s->shard);
}

int rl_rls_collect(rl_rls* s) {
    if (!s) return RL_FATAL;
    int st = RL_OK;
    const std::string plan_error = s->last_error;
    int r = sharded_collect(s, s->dev, s->shard, st);
    if (r) {
        s->last_error = plan_error;
        return r;
    }
    const double t2 = mono_us();
    s->report_verdicts = s->method == RL_RLS_REPORT ? s->o_limited.data() : nullptr;
    r = rl_rls_finish(s, st == RL_TRANSIENT && s->n_store ? RL_OK : st, s->o_limited.data(), s->o_first.data(), s->o_rem.data(),
                      s->o_ttl.data());
    s->report_verdicts = nullptr;
    s->t_plan = s->sh_t1 - s->sh_t0;
    s->t_store = t2 - s->sh_t1;
    s->t_finish = mono_us() - t2;
    return sharded_status(s, r);
}

int rl_rls_serve_sharded(rl_rls* s, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    int r = rl_rls_send(s, method, n, buf, off, now_us);
    if (r) return r;
    rl_rls_decide(s);
    return rl_rls_collect(s);
}

int rl_http_send(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    if (!h) return RL_FATAL;
    rl_shard_batch* sb = h->rls->shard;
    if (!sb) return sfail(h, "no sharded store attached to the RLS service (rl_rls_attach_shard)");
    if (h->sh_pending) return sfail(h, "the previous sharded step is not collected");
    const double t0 = mono_us();
    const HttpDevReq* req = nullptr;
    const HttpRun* runs = nullptr;
    uint64_t n_ctr = 0;
    uint32_t n_runs = 0;
    int r = n && (!off || !buf) ? sfail(h, "null body buffer or offsets")
                                : http_plan_on_device(h, endpoint, n, buf, off, now_us, false, req, n_ctr, runs, n_runs);
    bool any_load = false;
    if (r == RL_OK) {
        for (uint32_t k = 0; k < n_runs; k++) any_load = any_load || runs[k].load;
        size_outputs(h, any_load, n_ctr);
        h->store_calls = n_runs ? 1 : 0;  // one step, however many load_counters runs
    }
    if ((r = sharded_send(h, h->rls->dev, sb, true, endpoint, r, any_load, t0))) return r;
    if (h->sh_plan) return RL_OK;
    if ((r = dev_fail(h, h->rls->dev, rl_rls_dev_wait(h->rls->dev)))) {
        h->sh_plan = r;
        return RL_OK;
    }
    take_http_device_plan(h, req, buf, off);
    return RL_OK;
}

int rl_http_decide(rl_http* h) {
    if (!h) return RL_FATAL;
    return sharded_decide(h, h->rls->shard);
}

int rl_http_collect(rl_http* h) {
    if (!h) return RL_FATAL;
    int st = RL_OK;
    const std::string plan_error = h->last_error;
    int r = sharded_collect(h, h->rls->dev, h->rls->shard, st);
    if (r) {
        h->last_error = plan_error;
        return r;
    }
    const double t2 = mono_us();
    // per store request: the collect's status, or the error verdict of a request that was not decided
    h->o_status.resize(h->n_store);
    for (uint64_t j = 0; j < h->n_store; j++)
        h->o_status[j] = (st != RL_OK && st != RL_TRANSIENT) ? st : h->o_limited[j] == RL_VERDICT_ERROR ? RL_TRANSIENT : RL_OK;
    r = rl_http_finish(h, h->o_status.data(), h->o_limited.data(), h->o_first.data(), h->o_rem.data(), h->o_ttl.data());
    h->t_plan = h->sh_t1 - h->sh_t0;
    h->t_store = t2 - h->sh_t1;
    h->t_finish = mono_us() - t2;
    return sharded_status(h, r);
}

int rl_http_serve_sharded(rl_http* h, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us) {
    int r = rl_http_send(h, endpoint, n, buf, off, now_us);
    if (r) return r;
    rl_http_decide(h);
    return rl_http_collect(h);
}

// ---- counter variables and the GET endpoints -------------------------------------------------------------------
int rl_rls_keep_counter_vars(rl_rls* s, uint64_t max_keys, uint64_t arena_bytes) {
    if (!s) return RL_FATAL;
    if (s->shard) return sfail(s, "%s", kShardedNoCvars);
    if (!s->engine) return sfail(s, "keeping counter variables needs a service created with an engine");
    if (!rl_cv_dev_configure) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_configure(&s->dev, s->engine, max_keys, arena_bytes);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_rls_counter_vars_stats(rl_rls* s, uint64_t* out_keys, uint64_t* out_arena_used, uint64_t* out_dropped) {
    if (!s) return RL_FATAL;
    if (!rl_cv_dev_stats) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_stats(s->dev, nullptr, out_keys, out_arena_used, out_dropped);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_rls_counter_vars_gc(rl_rls* s, uint64_t now_us, uint64_t* out_kept, uint64_t* out_freed) {
    if (!s) return RL_FATAL;
    if (!s->engine) return sfail(s, "keeping counter variables needs a service created with an engine");
    if (!rl_cv_dev_gc) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_gc(&s->dev, s->engine, s->m, now_us ? now_us : wall_us(), out_kept, out_freed);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_rls_counter_vars_export(rl_rls* s, const uint32_t* ns_ids, uint32_t n_ns, uint64_t now_us, uint64_t cap, uint64_t bytes_cap,
                               uint32_t* out_varset, uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_blob_off,
                               uint8_t* out_blobs, uint64_t* out_count, uint64_t* out_bytes) {
    if (!s || !out_count || !out_bytes) return RL_FATAL;
    if (s->shard) return sfail(s, "%s", kShardedNoCvars);
    if (!s->engine) return sfail(s, "keeping counter variables needs a service created with an engine");
    if (!rl_cv_dev_export) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_export(&s->dev, s->engine, s->m, ns_ids, n_ns, now_us, cap, bytes_cap, out_varset, out_key_lo, out_key_hi,
                                   out_blob_off, out_blobs, out_count, out_bytes);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_rls_counter_vars_import(rl_rls* s, uint64_t n, const uint32_t* varset, const uint64_t* key_lo, const uint64_t* key_hi,
                               const uint64_t* blob_off, const uint8_t* blobs, uint64_t* out_added) {
    if (!s) return RL_FATAL;
    if (s->shard) return sfail(s, "%s", kShardedNoCvars);
    if (!s->engine) return sfail(s, "keeping counter variables needs a service created with an engine");
    if (!rl_cv_dev_import) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_import(&s->dev, s->engine, s->m, n, varset, key_lo, key_hi, blob_off, blobs, out_added);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_rls_counter_vars_drain(rl_rls* s, uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset, uint64_t* out_key_lo,
                              uint64_t* out_key_hi, uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count,
                              uint64_t* out_bytes, int* out_full) {
    if (!s || !out_count || !out_bytes || !out_full) return RL_FATAL;
    if (s->shard) return sfail(s, "%s", kShardedNoCvars);
    if (!s->engine) return sfail(s, "keeping counter variables needs a service created with an engine");
    if (!rl_cv_dev_drain) return sfail(s, "this build of the library has no device plan");
    const int r = rl_cv_dev_drain(&s->dev, s->engine, s->m, cap, bytes_cap, out_varset, out_key_lo, out_key_hi, out_blob_off,
                                  out_blobs, out_count, out_bytes, out_full);
    if (r) s->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
    return r;
}

int rl_http_get_limits(rl_http* h, const char* ns, uint32_t ns_len) {
    if (!h || (ns_len && !ns)) return RL_FATAL;
    const std::string name(ns ? ns : "", ns_len);
    std::vector<RlLimitRecord> lims;
    rl_matcher_ns_limit_records(h->m, name, lims);  // an unknown namespace has none: 200 []
    std::string o = "[";
    for (size_t k = 0; k < lims.size(); k++) {
        if (k) o.push_back(',');
        json_limit(o, name, lims[k]);
    }
    o.push_back(']');
    get_answer(h, 200, std::move(o), 0);
    return RL_OK;
}

int rl_http_get_counters(rl_http* h, const char* ns, uint32_t ns_len, uint64_t now_us) {
    if (!h || (ns_len && !ns)) return RL_FATAL;
    if (h->rls->shard) return sfail(h, "GET /counters reads one engine's table: a sharded service does not serve it");
    if (!h->engine || !rl_get_counters || !rl_cv_dev_lookup) return sfail(h, "GET /counters needs a service created with an engine");
    const std::string name(ns ? ns : "", ns_len);
    std::vector<RlLimitRecord> lims;
    if (!rl_matcher_ns_limit_records(h->m, name, lims) || lims.empty()) {
        get_answer(h, 200, "[]", 0);
        return RL_OK;
    }
    const uint64_t now = now_us ? now_us : wall_us();
    std::vector<uint32_t> ids;
    for (const auto& L : lims) ids.push_back(L.limit_id);
    // every counter of the namespace with ttl > 0 (in_memory.rs:158-187); it may hold deleted limits' counters too
    std::vector<uint32_t> lid;
    std::vector<uint64_t> lo, hi, rem, ttl;
    uint64_t cap = 4096, found = 0;
    for (;;) {
        lid.resize(cap);
        lo.resize(cap);
        hi.resize(cap);
        rem.resize(cap);
        ttl.resize(cap);
        if (rl_get_counters(h->engine, ids.data(), (uint32_t)ids.size(), now, cap, lid.data(), lo.data(), hi.data(), rem.data(),
                            ttl.data(), &found) != RL_OK) {
            h->last_error = std::string("get_counters failed: ") + rl_last_error(h->engine);
            get_answer(h, 500, "Internal server error", 0);
            return RL_OK;
        }
        if (found <= cap) break;
        cap = found + found / 8;
    }
    // the live limits' counters only, then their variables from the device dictionary
    std::vector<uint8_t> live(1, 0);
    for (const uint32_t x : ids) {
        if (x >= live.size()) live.resize(x + 1, 0);
        live[x] = 1;
    }
    uint64_t k = 0;
    for (uint64_t i = 0; i < found; i++)
        if (lid[i] < live.size() && live[lid[i]]) {
            lid[k] = lid[i];
            lo[k] = lo[i];
            hi[k] = hi[i];
            rem[k] = rem[i];
            ttl[k] = ttl[i];
            k++;
        }
    const uint8_t *blobs = nullptr, *unnamed = nullptr;
    const uint64_t* blob_off = nullptr;
    rl_rls* s = h->rls;
    if (rl_cv_dev_lookup(&s->dev, h->engine, h->m, k, lid.data(), lo.data(), hi.data(), &blobs, &blob_off, &unnamed) != RL_OK) {
        h->last_error = std::string("counter variables: ") + rl_rls_dev_error(s->dev);
        get_answer(h, 500, "Internal server error", 0);
        return RL_OK;
    }
    std::vector<rl_counter> ctrs(k);
    for (uint64_t i = 0; i < k; i++) ctrs[i] = rl_counter{lid[i], 0, lo[i], hi[i]};
    render_counters(h, name, k, ctrs.data(), rem.data(), ttl.data(), blobs, blob_off, unnamed);
    return RL_OK;
}

int rl_http_render_counters(rl_http* h, const char* ns, uint32_t ns_len, uint64_t n, const rl_counter* ctrs, const uint64_t* remaining,
                            const uint64_t* ttl_us, const uint8_t* blobs, const uint64_t* blob_off, const uint8_t* unnamed) {
    if (!h || (ns_len && !ns) || (n && (!ctrs || !remaining || !ttl_us || !blob_off))) return RL_FATAL;
    static const uint8_t kNone = 0;
    render_counters(h, std::string(ns ? ns : "", ns_len), n, ctrs, remaining, ttl_us, blobs ? blobs : &kNone, blob_off, unnamed);
    return RL_OK;
}

int rl_http_get_response(rl_http* h, uint16_t* out_status, const uint8_t** out_body, uint64_t* out_len, uint64_t* out_unnamed) {
    if (!h) return RL_FATAL;
    if (!h->get_status) return sfail(h, "no GET response");
    if (out_status) *out_status = h->get_status;
    if (out_body) *out_body = (const uint8_t*)h->get_body.data();
    if (out_len) *out_len = h->get_body.size();
    if (out_unnamed) *out_unnamed = h->get_unnamed;
    return RL_OK;
}

}  // extern "C"
