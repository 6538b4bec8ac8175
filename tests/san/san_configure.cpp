// ASan/UBSan driver of rl_rls_configure on a service without an engine (limitador_b200/csrc/rl_rls.cpp, rl_match.cpp): random
// sets of limits in both dialects, with refused expressions, duplicates, empty namespaces and null names / ids, applied one
// after the other (and as dry runs) while CPU plans match requests against the result.  Test infrastructure.
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "rl_match_dialect.h"
#include "rl_rls.h"

// the engine entry points rl_rls_serve would call: never reached here (the service is created without an engine)
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

static unsigned long long rnd(unsigned long long& s) {
    s ^= s << 13;
    s ^= s >> 7;
    s ^= s << 17;
    return s;
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

int main() {
    static const char* const kNs[] = {"a", "b", "c\"d", ""};
    static const char* const kConds[] = {"descriptors[0].k == 'v'", "descriptors[0].k != 'w'", "x == 'y'", "descriptors[0].k.startsWith('v')",
                                         "descriptors[0].k in ['v', 'w'] || descriptors[0].k == 'z'", "bad(", "descriptors[0]['u'] == \"1\"",
                                         "has(descriptors[0].u)", "a.b == 'c'", "!(x == 'q')"};
    static const char* const kVars[] = {"descriptors[0].u", "descriptors[0]['k']", "x", "9bad", "descriptors[1].z"};
    static const char* const kText[] = {"n1", "n\"2", "é"};
    unsigned long long s = 0x2545F4914F6CDD1DULL;
    unsigned long long ok = 0, refused = 0, planned = 0;
    for (int dialect = 0; dialect < 2; dialect++) {
        rl_matcher* m = nullptr;
        rl_rls* svc = nullptr;
        if (rl_matcher_create(&m) || rl_matcher_set_dialect(m, dialect ? RL_MATCH_DIALECT_BOOLEAN : RL_MATCH_DIALECT_TABLE) ||
            rl_rls_create(m, nullptr, RL_RLS_HEADERS_DRAFT_VERSION_03, 2, 1, &svc))
            return 1;
        for (int round = 0; round < 400; round++) {
            const uint32_t n = (uint32_t)(rnd(s) % 24);
            std::vector<std::vector<const char*>> conds(n), vars(n);
            std::vector<rl_limit_spec> specs(n);
            for (uint32_t i = 0; i < n; i++) {
                for (unsigned k = rnd(s) % 3; k > 0; k--) conds[i].push_back(kConds[rnd(s) % 10]);
                for (unsigned k = rnd(s) % 3; k > 0; k--) vars[i].push_back(kVars[rnd(s) % 5]);
                rl_limit_spec& x = specs[i];
                x = rl_limit_spec{};
                x.ns = kNs[rnd(s) % 4];
                x.max_value = rnd(s) % 5;
                x.seconds = 1 + rnd(s) % 3;
                x.conditions = conds[i].data();
                x.n_cond = (uint32_t)conds[i].size();
                x.variables = vars[i].data();
                x.n_var = (uint32_t)vars[i].size();
                x.name = rnd(s) % 2 ? kText[rnd(s) % 3] : nullptr;
                x.id = rnd(s) % 2 ? kText[rnd(s) % 3] : nullptr;
            }
            rl_configure_report rep;
            const int r = rl_rls_configure(svc, specs.data(), n, (int)(rnd(s) % 5 == 0), &rep);
            if (r == RL_OK) ok++;
            else refused++;
            if (r != RL_OK && rep.first_refused >= n) {
                fprintf(stderr, "refusal without an entry index: %s\n", rl_rls_last_error(svc));
                return 1;
            }
            // a batch against whatever the service now holds
            std::string buf;
            std::vector<uint64_t> off(1, 0);
            for (int q = 0; q < 32; q++) {
                std::string e, d, msg;
                put_len(e, 1, rnd(s) % 2 ? "k" : "u");
                put_len(e, 2, rnd(s) % 2 ? "v" : "1");
                put_len(d, 1, e);
                put_len(msg, 1, kNs[rnd(s) % 3]);
                put_len(msg, 2, d);
                buf += msg;
                off.push_back(buf.size());
            }
            if (rl_rls_plan(svc, RL_RLS_SHOULD_RATE_LIMIT, 32, (const uint8_t*)buf.data(), off.data(), 1700000000000000ull)) return 1;
            uint64_t n_store = 0;
            const uint32_t* ctr_off = nullptr;
            if (rl_rls_plan_view(svc, &n_store, &ctr_off, nullptr, nullptr, nullptr, nullptr, nullptr)) return 1;
            std::vector<uint8_t> lim(n_store + 1, 0);
            std::vector<uint32_t> first(n_store + 1, RL_NONE);
            std::vector<uint64_t> rem(ctr_off[n_store] + 1, 1), ttl(ctr_off[n_store] + 1, 1000000);
            if (rl_rls_finish(svc, RL_OK, lim.data(), first.data(), rem.data(), ttl.data())) return 1;
            planned += n_store;
        }
        uint64_t version = 0, err_since = 0;
        rl_rls_config_status(svc, &version, &err_since);
        rl_rls_destroy(svc);
        rl_matcher_destroy(m);
    }
    printf("ok configured=%llu refused=%llu store_requests=%llu\n", ok, refused, planned);
    return 0;
}
