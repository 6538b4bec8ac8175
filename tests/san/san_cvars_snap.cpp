// ASan/UBSan driver of the dictionary's snapshot kernels (limitador_b200/csrc/rl_cvars_dev.cuh) under the host shim:
// valid entries of a one- and a two-variable set, random blobs, and adversarial mutations of valid ones (bytes flipped,
// cut, appended, length prefixes near 2^32, NUL and invalid UTF-8) through rl_cv_check_entry, each in an array of exactly
// its size; then imports of valid and mutated entry sets into a small dictionary and an export of what it holds.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../emu/emu_cvars_snap.cpp"

// the engine entry points the CPU stages would call: never reached here (no service is created)
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

struct Entry {
    uint32_t vs;
    uint64_t lo, hi;
    std::vector<uint8_t> b;
};

static uint32_t check(const uint32_t* image, const Entry& e) {
    std::vector<uint8_t> exact(e.b);  // exactly the blob's size: ASan sees any read past it
    return emu_cvs_check_entry(image, e.vs, e.lo, e.hi, exact.empty() ? nullptr : exact.data(), exact.size());
}

static void put(std::vector<uint8_t>& b, const std::string& v) {
    const uint32_t n = (uint32_t)v.size();
    for (int s = 0; s < 4; s++) b.push_back((uint8_t)(n >> (8 * s)));
    b.insert(b.end(), v.begin(), v.end());
}

static int import(void* d, const uint32_t* image, const std::vector<Entry>& es, uint64_t* added, uint64_t* bad) {
    std::vector<uint32_t> vs;
    std::vector<uint64_t> lo, hi, off{0};
    std::vector<uint8_t> blobs;
    for (const Entry& e : es) {
        vs.push_back(e.vs);
        lo.push_back(e.lo);
        hi.push_back(e.hi);
        blobs.insert(blobs.end(), e.b.begin(), e.b.end());
        off.push_back(blobs.size());
    }
    return emu_cvs_import(d, image, es.size(), vs.data(), lo.data(), hi.data(), off.data(), blobs.empty() ? nullptr : blobs.data(), added,
                          bad);
}

int main() {
    std::mt19937_64 rng(17);
    rl_matcher* m = nullptr;
    if (rl_matcher_create(&m) != RL_OK) return 2;
    rl_limit_desc d1, d2;
    const char* v1[] = {"descriptors[0].user"};
    const char* v2[] = {"descriptors[0].user", "descriptors[0].app"};
    if (rl_matcher_add_limit(m, "a", 5, 60, nullptr, 0, v1, 1, nullptr, &d1) != RL_OK) return 3;
    if (rl_matcher_add_limit(m, "b", 5, 60, nullptr, 0, v2, 2, nullptr, &d2) != RL_OK) return 3;
    uint64_t words = 0;
    rl_matcher_image(m, nullptr, 0, &words, nullptr);
    std::vector<uint32_t> image(words);
    if (rl_matcher_image(m, image.data(), words, &words, nullptr) != RL_OK) return 4;
    const char* pieces[] = {"u", "é", "😀", "\x7f", "x y", "\xe2\x82\xac", ""};
    std::vector<Entry> valid;
    for (int k = 0; valid.size() < 200; k++) {
        std::string a, b;
        for (int j = (int)(rng() % 4); j > 0; j--) a += pieces[rng() % 7];
        for (int j = (int)(rng() % 4); j > 0; j--) b += pieces[rng() % 7];
        Entry e;
        const bool two = k % 2;
        e.vs = two ? d2.varset_id : d1.varset_id;
        const char* src[] = {"descriptors[0].app", "descriptors[0].user"};  // sorted: the digest order
        const char* val[] = {b.c_str(), a.c_str()};
        if (two) {
            rl_counter_key(src, val, 2, &e.lo, &e.hi);
            put(e.b, b);
            put(e.b, a);
        } else {
            rl_counter_key(src + 1, val + 1, 1, &e.lo, &e.hi);
            put(e.b, a);
        }
        if (check(image.data(), e) != 0) return 10;
        bool seen = false;  // one entry per key: an import refuses a key named twice
        for (const Entry& x : valid) seen = seen || (x.vs == e.vs && x.lo == e.lo && x.hi == e.hi);
        if (!seen) valid.push_back(e);
    }
    uint64_t refused = 0;
    for (int k = 0; k < 20000; k++) {
        Entry e = valid[rng() % valid.size()];
        switch (rng() % 8) {
            case 0:  // random bytes
                e.b.resize(rng() % 40);
                for (auto& x : e.b) x = (uint8_t)rng();
                break;
            case 1:  // a byte flipped
                if (!e.b.empty()) e.b[rng() % e.b.size()] ^= (uint8_t)(1 + rng() % 255);
                break;
            case 2:  // cut
                e.b.resize(rng() % (e.b.size() + 1));
                break;
            case 3:  // bytes appended
                for (int j = 1 + (int)(rng() % 5); j > 0; j--) e.b.push_back((uint8_t)rng());
                break;
            case 4: {  // a length prefix near 2^32
                const uint32_t n = 0xFFFFFFFFu - (uint32_t)(rng() % 8);
                memcpy(e.b.data(), &n, 4);
                break;
            }
            case 5:  // NUL or a byte that is never UTF-8
                if (e.b.size() > 4) e.b[4 + rng() % (e.b.size() - 4)] = rng() % 2 ? 0 : 0xFF;
                break;
            case 6:  // another or an unknown variable set
                e.vs = (uint32_t)(rng() % 5);
                break;
            default:  // another key
                e.lo ^= 1ull << (rng() % 64);
                break;
        }
        refused += check(image.data(), e) != 0;
    }
    // imports: the valid entries, then sets with one mutated entry; the dictionary holds the valid ones throughout
    void* dict = emu_cv_create(64, 1 << 12);
    uint64_t added = 0, bad = 0;
    std::vector<Entry> first(valid.begin(), valid.begin() + 40);
    if (import(dict, image.data(), first, &added, &bad) != RL_OK || added != 40) return 11;
    for (int k = 0; k < 300; k++) {
        std::vector<Entry> es(valid.begin() + 40 + rng() % 100, valid.begin() + 150);
        Entry& e = es[rng() % es.size()];
        if (rng() % 2) e.b.resize(e.b.size() - 1);
        else e.b.push_back('x');
        if (import(dict, image.data(), es, &added, &bad) != RL_FATAL || added != 0) return 12;
    }
    std::vector<Entry> many(valid.begin(), valid.end());
    const int big = import(dict, image.data(), many, &added, &bad);  // 200 keys into 64 slots: no room
    if (big != RL_TRANSIENT) return 13;
    uint64_t slots, keys, used, dropped;
    emu_cv_stats(dict, &slots, &keys, &used, &dropped);
    if (keys != 40 || dropped != 0) return 14;
    // export what the first 40 keys' counters reference
    std::vector<uint32_t> lid;
    std::vector<uint64_t> lo, hi;
    for (const Entry& e : first) {
        lid.push_back(e.vs == d2.varset_id ? d2.limit_id : d1.limit_id);
        lo.push_back(e.lo);
        hi.push_back(e.hi);
    }
    uint64_t bytes = 0;
    const uint64_t n = emu_cvs_export(dict, image.data(), lid.size(), lid.data(), lo.data(), hi.data(), 0, 0, nullptr, nullptr, nullptr,
                                      nullptr, nullptr, &bytes);
    std::vector<uint32_t> ovs(n);
    std::vector<uint64_t> olo(n), ohi(n), ooff(n + 1);
    std::vector<uint8_t> ob(bytes);
    if (emu_cvs_export(dict, image.data(), lid.size(), lid.data(), lo.data(), hi.data(), n, bytes, ovs.data(), olo.data(), ohi.data(),
                       ooff.data(), ob.data(), &bytes) != 40)
        return 15;
    for (uint64_t i = 0; i < n; i++) {
        Entry e{ovs[i], olo[i], ohi[i], std::vector<uint8_t>(ob.begin() + ooff[i], ob.begin() + ooff[i + 1])};
        if (check(image.data(), e) != 0) return 16;
    }
    emu_cv_destroy(dict);
    rl_matcher_destroy(m);
    printf("ok valid=%zu refused=%llu exported=%llu\n", valid.size(), (unsigned long long)refused, (unsigned long long)n);
    return 0;
}
