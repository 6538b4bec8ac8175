// ASan/UBSan driver of the HTTP device plan kernels (limitador_b200/csrc/rl_http_dev.cuh) under the host shim: they read
// bodies from the network, so random and mutated JSON goes through them, and every batch is compared with the CPU plan
// (rl_http_plan) on the same bytes: store index, CSR, delta, load_counters and the outcome of every body must agree.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../emu/emu_http.cpp"
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

int main() {
    std::mt19937_64 rng(7);
    rl_matcher* m = nullptr;
    if (rl_matcher_create(&m) != RL_OK) return 2;
    rl_limit_desc d;
    const char* c1[] = {"descriptors[0]['req.method'] == 'GET'"};
    const char* v1[] = {"descriptors[0]['app.id']"};
    const char* v2[] = {"descriptors[0]['app.id']", "descriptors[0].y"};
    if (rl_matcher_add_limit(m, "test_namespace", 1, 60, c1, 1, v1, 1, "a", &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 100, 3600, nullptr, 0, v2, 2, nullptr, &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 9, 10, nullptr, 0, nullptr, 0, nullptr, &d) != RL_OK) return 3;
    uint64_t words = 0;
    rl_matcher_image(m, nullptr, 0, &words, nullptr);
    std::vector<uint32_t> image(words);
    if (rl_matcher_image(m, image.data(), words, &words, nullptr) != RL_OK) return 4;
    const std::string base =
        "{\"namespace\":\"test_\\u006eamespace\",\"values\":{\"req.method\":\"GET\",\"app.id\":\"\\ud83d\\ude00\",\"y\":\"\xc3\xbc\"},"
        "\"x\":[{\"a\":[1.5e3,-0,true,null,\"\\ud800\"]}],\"delta\":18446744073709551615,\"response_headers\":\"DraftVersion03\"}";
    uint64_t compared = 0, stored = 0;
    for (int threads = 1; threads <= 3; threads += 2) {
        rl_rls* s = nullptr;
        rl_http* h = nullptr;
        if (rl_rls_create(m, nullptr, RL_RLS_HEADERS_NONE, threads, 0, &s) != RL_OK || rl_http_create(s, &h) != RL_OK) return 5;
        for (int batch = 0; batch < 60; batch++) {
            const int endpoint = batch % 3;
            std::string buf;
            std::vector<uint64_t> off{0};
            const int n = 1 + (int)(rng() % 300);
            for (int i = 0; i < n; i++) {
                std::string body;
                switch (rng() % 6) {
                    case 0: body = base.substr(0, rng() % (base.size() + 1)); break;
                    case 1:
                        body = base;
                        for (int k = 0; k < 1 + (int)(rng() % 3); k++) body[rng() % body.size()] = "{}[]\",:\\u0123456789-.eE \x01\xff"[rng() % 24];
                        break;
                    case 2:
                        body = "{\"x\":";
                        for (int k = 0; k < (int)(rng() % 200); k++) body += rng() % 2 ? "[" : "{\"k\":";
                        break;
                    default:
                        body = std::string("{\"namespace\":\"") + (rng() % 5 ? "test_namespace" : "nobody") + "\",\"values\":{\"req.method\":\"" +
                               (rng() % 2 ? "GET" : "POST") + "\",\"app.id\":\"" + std::to_string(rng() % 5) + "\"},\"delta\":" +
                               std::to_string(rng() % 3) + (rng() % 2 ? ",\"response_headers\":\"DraftVersion03\"}" : "}");
                        break;
                }
                buf += body;
                off.push_back(buf.size());
            }
            const uint8_t* bp = (const uint8_t*)buf.data();
            if (rl_http_plan(h, endpoint, n, bp, off.data(), 1700000000000000ull) != RL_OK) return 6;
            uint64_t n_store = 0;
            const uint32_t *ctr_off = nullptr, *store_index = nullptr;
            const rl_counter* ctrs = nullptr;
            const uint64_t* delta = nullptr;
            const uint8_t* load = nullptr;
            if (rl_http_plan_view(h, &n_store, &ctr_off, &ctrs, &delta, nullptr, &load, &store_index) != RL_OK) return 7;
            std::vector<HttpDevReq> req(n);
            std::vector<uint32_t> e_off(n + 1), runs(3 * n + 3), ctr_run(2 * n + 2);
            std::vector<rl_counter> e_ctrs(16 * (size_t)n + 1);
            std::vector<uint64_t> e_delta(n), e_now(n);
            std::vector<uint8_t> e_load(n);
            uint64_t e_nctr = 0;
            uint32_t e_runs = 0;
            const uint64_t e_store = emu_http_plan(image.data(), endpoint, n, bp, off.data(), 1700000000000000ull, RL_MAX_COUNTERS_PER_REQUEST,
                                                   req.data(), e_off.data(), e_ctrs.data(), e_ctrs.size(), e_delta.data(), e_now.data(),
                                                   e_load.data(), runs.data(), ctr_run.data(), &e_nctr, &e_runs);
            if (e_store != n_store) return 8;
            for (int i = 0; i < n; i++)
                if (req[i].store != store_index[i]) return 9;
            for (uint64_t j = 0; j <= n_store; j++)
                if (e_off[j] != ctr_off[j]) return 10;
            for (uint64_t j = 0; j < n_store; j++)
                if (e_delta[j] != delta[j] || e_load[j] != load[j]) return 11;
            for (uint64_t c = 0; c < e_nctr; c++)
                if (memcmp(&e_ctrs[c], &ctrs[c], sizeof(rl_counter)) != 0) return 12;
            std::vector<uint8_t> lim(n_store + 1, 0);
            std::vector<uint32_t> first(n_store + 1, RL_NONE);
            std::vector<uint64_t> zero(e_nctr + 1, 0);
            if (rl_http_finish(h, nullptr, lim.data(), first.data(), zero.data(), zero.data()) != RL_OK) return 13;
            const uint16_t* status = nullptr;
            if (rl_http_responses(h, &status, nullptr, nullptr, nullptr, nullptr) != RL_OK) return 14;
            for (int i = 0; i < n; i++) {
                const uint16_t want = req[i].kind == REQ_BAD_WIRE ? 400 : req[i].kind == REQ_UNSUPPORTED ? 500 : 200;
                if (status[i] != want) return 15;
            }
            compared += n;
            stored += n_store;
        }
        rl_http_destroy(h);
        rl_rls_destroy(s);
    }
    rl_matcher_destroy(m);
    printf("ok compared=%llu stored=%llu\n", (unsigned long long)compared, (unsigned long long)stored);
    return stored > 1000 ? 0 : 16;
}
