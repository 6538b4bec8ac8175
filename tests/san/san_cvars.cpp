// ASan/UBSan driver of the counter variable dictionary's kernels (limitador_b200/csrc/rl_cvars_dev.cuh) under the host
// shim: random and mutated JSON bodies and RLS messages go through the plan kernels and k_counter_vars_record into a small
// dictionary (so that the table and the arena fill up), then every entry is looked up, rendered by
// rl_http_render_counters and collected by a GC that keeps half of them.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../emu/emu_cvars.cpp"
#include "rl_http.h"

// the engine entry points the CPU stages would call: never reached here (the service is created without an engine)
extern "C" {
const char* rl_last_error(rl_engine*) { return "no engine in the sanitizer build"; }
int rl_check_and_update_batch(rl_engine*, uint64_t, const uint32_t*, const rl_counter*, const uint64_t*, const uint64_t*, int, int,
                              uint8_t*, uint32_t*, uint64_t*, uint64_t*) { return RL_FATAL; }
int rl_is_within_limits_batch(rl_engine*, uint64_t, const uint32_t*, const rl_counter*, const uint64_t*, const uint64_t*, int, uint8_t*,
                              uint32_t*) { return RL_FATAL; }
int rl_update_batch(rl_engine*, uint64_t, const uint32_t*, const rl_counter*, const uint64_t*, const uint64_t*, int) { return RL_FATAL; }
int rl_front_check_and_update(rl_front*, const rl_counter*, uint32_t, uint64_t, uint64_t, int, uint8_t*, uint32_t*, uint64_t*, uint64_t*,
                              uint64_t*) { return RL_FATAL; }
}

static void put_str(std::string& o, uint32_t tag, const std::string& s) {
    o.push_back((char)(tag << 3 | 2));
    o.push_back((char)s.size());
    o += s;
}

int main() {
    std::mt19937_64 rng(11);
    rl_matcher* m = nullptr;
    if (rl_matcher_create(&m) != RL_OK) return 2;
    rl_limit_desc d;
    const char* c1[] = {"descriptors[0]['req.method'] == 'GET'"};
    const char* v1[] = {"descriptors[0]['app.id']"};
    const char* v2[] = {"descriptors[0]['app.id']", "descriptors[0].y"};
    if (rl_matcher_add_limit(m, "test_namespace", 1, 60, c1, 1, v1, 1, "a", &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 100, 3600, nullptr, 0, v2, 2, "q\"\x01", &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 9, 10, nullptr, 0, nullptr, 0, nullptr, &d) != RL_OK) return 3;
    uint64_t words = 0;
    rl_matcher_image(m, nullptr, 0, &words, nullptr);
    std::vector<uint32_t> image(words);
    if (rl_matcher_image(m, image.data(), words, &words, nullptr) != RL_OK) return 4;
    rl_rls* s = nullptr;
    rl_http* h = nullptr;
    if (rl_rls_create(m, nullptr, RL_RLS_HEADERS_NONE, 1, 0, &s) != RL_OK || rl_http_create(s, &h) != RL_OK) return 5;
    const std::string base =
        "{\"namespace\":\"test_\\u006eamespace\",\"values\":{\"req.method\":\"GET\",\"app.id\":\"\\ud83d\\ude00\",\"y\":\"\xc3\xbc\"},"
        "\"delta\":1,\"response_headers\":\"DraftVersion03\"}";
    void* dict = emu_cv_create(64, 2048);
    uint64_t total = 0;
    for (int batch = 0; batch < 40; batch++) {
        const int http = batch % 2;
        std::string buf;
        std::vector<uint64_t> off{0};
        const int n = 1 + (int)(rng() % 200);
        for (int i = 0; i < n; i++) {
            std::string body;
            const std::string id = std::to_string(rng() % 500), y(rng() % 9, (char)('a' + rng() % 26));
            if (http) {
                body = rng() % 4 ? "{\"namespace\":\"test_namespace\",\"values\":{\"req.method\":\"GET\",\"app.id\":\"" + id +
                                       "\",\"y\":\"" + y + "\",\"app.id\":\"" + id + "x\"},\"delta\":1}"
                                 : base;
                if (rng() % 5 == 0) body[rng() % body.size()] = "{}[]\",:\\u0123 \x01\xff"[rng() % 16];
            } else {
                std::string e1, e2, e3, desc;
                put_str(e1, 1, "app.id");
                put_str(e1, 2, id);
                put_str(e2, 1, "y");
                put_str(e2, 2, y);
                put_str(e3, 1, "req.method");
                put_str(e3, 2, "GET");
                put_str(desc, 1, e1);
                put_str(desc, 1, e2);
                put_str(desc, 1, e3);
                put_str(body, 1, "test_namespace");
                put_str(body, 2, desc);
                if (rng() % 5 == 0) body[rng() % body.size()] = (char)rng();
            }
            buf += body;
            off.push_back(buf.size());
        }
        emu_cv_plan_record(dict, http, image.data(), RL_HTTP_CHECK_AND_REPORT, n, (const uint8_t*)buf.data(), off.data(), 16);
        // every entry: lookup, render, then a GC that keeps every other one
        std::vector<uint32_t> vs(64), blen(64), lid;
        std::vector<uint64_t> lo(64), hi(64), boff(64);
        const uint64_t k = emu_cv_dump(dict, vs.data(), lo.data(), hi.data(), boff.data(), blen.data(), 64);
        std::vector<rl_counter> ctrs;
        for (uint64_t i = 0; i < k; i++) {
            lid.push_back(vs[i] == d.varset_id ? 1u : 0u);  // limit 1 has the two-variable set, limit 0 the one-variable set
            ctrs.push_back(rl_counter{lid.back(), 0, lo[i], hi[i]});
        }
        std::vector<uint64_t> pos(k + 1), rem(k + 1, 7), ttl(k + 1, 5000000);
        std::vector<uint8_t> unnamed(k + 1), out(1 << 16);
        emu_cv_lookup(dict, image.data(), k, lid.data(), lo.data(), hi.data(), pos.data(), unnamed.data(), out.data(), out.size());
        if (rl_http_render_counters(h, "test_namespace", 14, k, ctrs.data(), rem.data(), ttl.data(), out.data(), pos.data(),
                                    unnamed.data()) != RL_OK)
            return 6;
        uint16_t st = 0;
        const uint8_t* body = nullptr;
        uint64_t len = 0, un = 0;
        if (rl_http_get_response(h, &st, &body, &len, &un) != RL_OK || (st != 200 && st != 500)) return 7;
        std::vector<uint32_t> klid;
        std::vector<uint64_t> klo, khi;
        for (uint64_t i = 0; i < k; i += 2) {
            klid.push_back(lid[i]);
            klo.push_back(lo[i]);
            khi.push_back(hi[i]);
        }
        uint64_t kept = 0, freed = 0;
        emu_cv_gc(dict, image.data(), klid.size(), klid.data(), klo.data(), khi.data(), &kept, &freed);
        if (kept + freed != k) return 8;
        total += k;
    }
    if (rl_http_get_limits(h, "test_namespace", 14) != RL_OK) return 9;
    emu_cv_destroy(dict);
    rl_http_destroy(h);
    rl_rls_destroy(s);
    rl_matcher_destroy(m);
    printf("ok entries=%llu\n", (unsigned long long)total);
    return 0;
}
