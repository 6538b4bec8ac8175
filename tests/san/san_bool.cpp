// ASan/UBSan driver of the matcher's boolean dialect: the RLS device plan kernels (limitador_b200/csrc/rl_rls_dev.cuh)
// under the host shim over limits with `in` lists, startsWith / endsWith / contains groups, presence tests and a group of
// six atoms, every batch compared with the CPU plan (rl_rls_plan) on the same bytes; then random and mutated expressions
// through the boolean parser (rl_matcher_add_limit), which must accept or refuse without any sanitizer report.
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

static const char* const kConds[] = {
    "descriptors[0].method in ['GET', 'HEAD']",
    "descriptors[0]['req.path'].startsWith('/api/') && descriptors[0]['req.path'] != '/api/health'",
    "has(descriptors[0].user)",
    "'tier' in descriptors[1]",
    "descriptors[1].tier.endsWith('-gold') || descriptors[1].tier == 'free' && !descriptors[1].tier.contains('\xc3\xa9')",
    "descriptors[0].method == 'PUT' || descriptors[0].method == 'PATCH' || descriptors[0].method.startsWith('DEL') || "
    "descriptors[0].method.endsWith('ST') && !descriptors[0].method.contains('O') || descriptors[0].method in []",
    "!(descriptors[0].method in ['OPTIONS'])",
};

int main() {
    std::mt19937_64 rng(11);
    rl_matcher* m = nullptr;
    if (rl_matcher_create(&m) != RL_OK || rl_matcher_set_dialect(m, RL_MATCH_DIALECT_BOOLEAN) != RL_OK) return 2;
    rl_limit_desc d;
    const char* v1[] = {"descriptors[0].user"};
    const char* v2[] = {"descriptors[1].tier"};
    for (int i = 0; i < 7; i++) {
        const char* c[] = {kConds[i], kConds[(i + 3) % 7]};
        if (rl_matcher_add_limit(m, "api", 1 + i, 60 + i, c, 1 + (i % 2), i % 3 == 1 ? v2 : v1, i % 3 ? 1 : 0, nullptr, &d) != RL_OK) return 3;
    }
    uint64_t words = 0;
    rl_matcher_image(m, nullptr, 0, &words, nullptr);
    std::vector<uint32_t> image(words);
    if (rl_matcher_image(m, image.data(), words, &words, nullptr) != RL_OK) return 4;
    const char* methods[] = {"GET", "HEAD", "PUT", "PATCH", "DELETE", "POST", "CAST", "OPTIONS"};
    const char* paths[] = {"/api/", "/api/health", "/api/v1", "/ap", "/\xe6\x97\xa5", ""};
    const char* tiers[] = {"gold", "x-gold", "free", "free-\xc3\xa9", "", "-gold"};
    uint64_t compared = 0, stored = 0;
    for (int threads = 1; threads <= 3; threads += 2) {
        rl_rls* s = nullptr;
        if (rl_rls_create(m, nullptr, RL_RLS_HEADERS_NONE, threads, 0, &s) != RL_OK) return 5;
        for (int batch = 0; batch < 40; batch++) {
            const int method = batch % 3;
            std::string buf;
            std::vector<uint64_t> off{0};
            const int n = 1 + (int)(rng() % 400);
            for (int i = 0; i < n; i++) {
                std::vector<std::pair<std::string, std::string>> d0;
                if (rng() % 8) d0.push_back({"method", methods[rng() % 8]});
                if (rng() % 4) d0.push_back({"user", "u" + std::to_string(rng() % 5)});
                if (rng() % 3) d0.push_back({"req.path", paths[rng() % 6]});
                std::vector<std::vector<std::pair<std::string, std::string>>> descs{d0};
                if (rng() % 2) descs.push_back({{"tier", tiers[rng() % 6]}});
                std::string msg = request(rng() % 6 ? "api" : "nobody", descs, (uint32_t)(rng() % 3));
                if (rng() % 10 == 0) msg[rng() % msg.size()] = (char)rng();  // a mutated message now and then
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
            std::vector<uint8_t> lim(n_store + 1, 0);
            std::vector<uint32_t> first(n_store + 1, RL_NONE);
            if (rl_rls_finish(s, RL_OK, lim.data(), first.data(), nullptr, nullptr) != RL_OK) return 13;
            compared += n;
            stored += n_store;
        }
        rl_rls_destroy(s);
    }
    // the parser: random token soup and accepted expressions with a byte changed, dropped or inserted
    static const char* const kPieces[] = {"x", "descriptors", "[", "]", "0", "7", ".", "u", "'a'", "\"b\"", "==", "!=", "&&", "||", "!",
                                          "(", ")", " in ", "has", "startsWith", "endsWith", "contains", ",", " ", "'\xc3\xa9'", "''",
                                          "\\", "'", "\"", "'''", "r'a'", "\xff", "9999999999"};
    uint64_t parsed = 0, accepted = 0;
    for (int i = 0; i < 20000; i++) {
        std::string e;
        if (rng() % 2) {
            e = kConds[rng() % 7];
            const size_t k = rng() % (e.size() + 1);
            switch (rng() % 3) {
                case 0: e.insert(k, kPieces[rng() % (sizeof kPieces / sizeof *kPieces)]); break;
                case 1: if (k < e.size()) e.erase(k, 1); break;
                default: if (k < e.size()) e[k] = (char)(rng() % 255 + 1);
            }
        } else {
            const int n = 1 + (int)(rng() % 14);
            for (int t = 0; t < n; t++) e += kPieces[rng() % (sizeof kPieces / sizeof *kPieces)];
        }
        if (rng() % 50 == 0) e = std::string(1 + rng() % 80, '(') + "x == 'a'" + std::string(1 + rng() % 80, ')');
        const char* c[] = {e.c_str()};
        if (rl_matcher_add_limit(m, "fuzz", 1, 1 + (uint64_t)i, c, 1, nullptr, 0, nullptr, &d) == RL_OK) accepted++;
        parsed++;
    }
    rl_matcher_destroy(m);
    printf("ok compared=%llu stored=%llu parsed=%llu accepted=%llu\n", (unsigned long long)compared, (unsigned long long)stored,
           (unsigned long long)parsed, (unsigned long long)accepted);
    return stored > 1000 && accepted > 1000 ? 0 : 16;
}
