// ASan/UBSan driver of the RLS device plan kernels (limitador_b200/csrc/rl_rls_dev.cuh) under the host shim: they read
// bytes from the network, so random and mutated messages go through them, and every batch is compared with the CPU plan
// (rl_rls_plan) on the same bytes: store index, CSR, delta and request kind must agree.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../emu/emu_rls.cpp"
#include "rl_rls.h"

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

static void put_varint(std::string& o, uint64_t v) {
    while (v >= 0x80) {
        o.push_back((char)(v | 0x80));
        v >>= 7;
    }
    o.push_back((char)v);
}
static void put_len(std::string& o, uint32_t tag, const std::string& body) {
    put_varint(o, (tag << 3) | 2);
    put_varint(o, body.size());
    o += body;
}
static std::string request(const std::string& domain, const std::vector<std::vector<std::pair<std::string, std::string>>>& descs, uint32_t hits) {
    std::string o;
    if (!domain.empty()) put_len(o, 1, domain);
    for (const auto& d : descs) {
        std::string body;
        for (const auto& kv : d) {
            std::string e;
            if (!kv.first.empty()) put_len(e, 1, kv.first);
            if (!kv.second.empty()) put_len(e, 2, kv.second);
            put_len(body, 1, e);
        }
        put_len(o, 2, body);
    }
    if (hits) {
        put_varint(o, 3 << 3);
        put_varint(o, hits);
    }
    return o;
}

int main() {
    std::mt19937_64 rng(7);
    rl_matcher* m = nullptr;
    if (rl_matcher_create(&m) != RL_OK) return 2;
    rl_limit_desc d;
    const char* c1[] = {"descriptors[0]['req.method'] == 'GET'"};
    const char* c2[] = {"descriptors[1].y != '2'"};
    const char* v1[] = {"descriptors[0]['app.id']"};
    const char* v2[] = {"descriptors[0]['app.id']", "descriptors[1].y"};
    if (rl_matcher_add_limit(m, "test_namespace", 1, 60, c1, 1, v1, 1, "a", &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 100, 3600, nullptr, 0, v1, 1, nullptr, &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 5, 10, c2, 1, v2, 2, nullptr, &d) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "test_namespace", 9, 10, nullptr, 0, nullptr, 0, nullptr, &d) != RL_OK) return 3;
    uint64_t words = 0;
    rl_matcher_image(m, nullptr, 0, &words, nullptr);
    std::vector<uint32_t> image(words);
    if (rl_matcher_image(m, image.data(), words, &words, nullptr) != RL_OK) return 4;
    const std::string base = request("test_namespace", {{{"req.method", "GET"}, {"app.id", "1"}, {"ü", "日本"}}, {{"y", "3"}}, {}}, 6) +
                             std::string("\x7a\x01\x66\x81\x01\x01\x02\x03\x04\x05\x06\x07\x08\x8d\x01\x01\x02\x03\x04\x7b\x08\x01\x7c", 23);
    uint64_t compared = 0, stored = 0;
    for (int threads = 1; threads <= 3; threads += 2) {
        rl_rls* s = nullptr;
        if (rl_rls_create(m, nullptr, RL_RLS_HEADERS_NONE, threads, 0, &s) != RL_OK) return 5;
        for (int batch = 0; batch < 60; batch++) {
            const int method = batch % 3;
            std::string buf;
            std::vector<uint64_t> off{0};
            const int n = 1 + (int)(rng() % 400);
            for (int i = 0; i < n; i++) {
                std::string msg;
                switch (rng() % 7) {
                    case 0: msg = base.substr(0, rng() % (base.size() + 1)); break;
                    case 1:
                        msg = base;
                        for (int k = 0; k < 1 + (int)(rng() % 3); k++) msg[rng() % msg.size()] = (char)rng();
                        break;
                    case 2:
                        msg.resize(rng() % 48);
                        for (auto& c : msg) c = (char)rng();
                        break;
                    case 3: msg = request("test_namespace", {{{"req.method", "GET"}, {"app.id", std::string("a\0b", 3)}}}, 1); break;
                    default:
                        msg = request(rng() % 5 ? "test_namespace" : "nobody",
                                      {{{"req.method", rng() % 2 ? "GET" : "POST"}, {"app.id", std::to_string(rng() % 5)}},
                                       {{"y", std::to_string(rng() % 4)}}},
                                      (uint32_t)(rng() % 3));
                        break;
                }
                buf += msg;
                off.push_back(buf.size());
            }
            const uint8_t* bp = (const uint8_t*)buf.data();
            if (rl_rls_plan(s, method, n, bp, off.data(), 1700000000000000ull) != RL_OK) return 6;
            uint64_t n_store = 0;
            const uint32_t *ctr_off = nullptr, *store_index = nullptr;
            const rl_counter* ctrs = nullptr;
            const uint64_t* delta = nullptr;
            if (rl_rls_plan_view(s, &n_store, &ctr_off, &ctrs, &delta, nullptr, nullptr, &store_index) != RL_OK) return 7;
            std::vector<RlsDevReq> req(n);
            std::vector<uint32_t> e_off(n + 1);
            std::vector<rl_counter> e_ctrs(16 * (size_t)n + 1);
            std::vector<uint64_t> e_delta(n), e_now(n);
            uint64_t e_nctr = 0;
            const uint64_t e_store = emu_rls_plan(image.data(), method, n, bp, off.data(), 1700000000000000ull, RL_MAX_COUNTERS_PER_REQUEST,
                                                  req.data(), e_off.data(), e_ctrs.data(), e_ctrs.size(), e_delta.data(), e_now.data(), &e_nctr);
            if (e_store != n_store) return 8;
            for (int i = 0; i < n; i++)
                if (req[i].store != store_index[i]) return 9;
            for (uint64_t j = 0; j <= n_store; j++)
                if (e_off[j] != ctr_off[j]) return 10;
            for (uint64_t j = 0; j < n_store; j++)
                if (e_delta[j] != delta[j]) return 11;
            for (uint64_t c = 0; c < e_nctr; c++)
                if (memcmp(&e_ctrs[c], &ctrs[c], sizeof(rl_counter)) != 0) return 12;
            // the request kinds, through the finish's gRPC statuses
            std::vector<uint8_t> lim(n_store + 1, 0);
            std::vector<uint32_t> first(n_store + 1, RL_NONE);
            if (rl_rls_finish(s, RL_OK, lim.data(), first.data(), nullptr, nullptr) != RL_OK) return 13;
            const uint8_t* grpc = nullptr;
            if (rl_rls_responses(s, nullptr, nullptr, &grpc, nullptr) != RL_OK) return 14;
            for (int i = 0; i < n; i++) {
                const uint8_t want = req[i].kind == REQ_BAD_WIRE ? RL_GRPC_INTERNAL : req[i].kind == REQ_UNSUPPORTED ? RL_GRPC_UNAVAILABLE : RL_GRPC_OK;
                if (grpc[i] != want) return 15;
            }
            compared += n;
            stored += n_store;
        }
        rl_rls_destroy(s);
    }
    rl_matcher_destroy(m);
    printf("ok compared=%llu stored=%llu\n", (unsigned long long)compared, (unsigned long long)stored);
    return stored > 1000 ? 0 : 16;
}
