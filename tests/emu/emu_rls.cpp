// emu_rls.cpp — TEST-ONLY host driver of the RLS device plan kernels (limitador_b200/csrc/rl_rls_dev.cuh) under
// tests/emu/cuda_shim.h: the SAME kernel source the GPU runs, one CUDA thread after the other in a shuffled order.  Not
// shipped, not a fallback.  The call sequence follows rl_rls_dev.cu's rl_rls_dev_plan, with a host loop in place of the
// CUB scan.  Also compiled into tests/san/san_rls_dev.cpp for the ASan + UBSan run.
#include "cuda_shim.h"
// (the shim must come first: it defines __global__ & co. away)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../limitador_b200/csrc/rl_rls_dev.cuh"

extern "C" {

void emu_rls_seed(uint64_t s) { shim_seed = s; }

// One device plan.  image: rl_matcher_image's words.  Outputs as rl_rls_plan_view gives them: req [n], ctr_off
// [n_store + 1] (n + 1 room), ctrs (cap_ctrs room), delta / now [n_store] (n room).  Returns n_store (or ~0 when
// cap_ctrs is too small); *out_n_ctr = counters.
uint64_t emu_rls_plan(const uint32_t* image, int method, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us,
                      uint32_t engine_max, RlsDevReq* req, uint32_t* ctr_off, rl_counter* ctrs, uint64_t cap_ctrs, uint64_t* delta,
                      uint64_t* now, uint64_t* out_n_ctr) {
    const uint32_t per_req = std::min(image[RL_IMG_H_COUNTER_CAP], engine_max);
    const uint64_t bytes = n ? off[n] : 0;
    // the device buffers (exact sizes, so that ASan sees any access past them)
    std::vector<rl_rls_entry> ent(bytes / 2 + 1);
    std::vector<rl_counter> scratch(n * (uint64_t)per_req + 1);
    std::vector<unsigned long long> count(n + 1), start(n + 1);
    RlsPlanArgs a;
    a.buf = buf;
    a.off = off;
    a.n = n;
    a.img = rl_img_view(image, image);
    a.per_req = per_req;
    a.ent = ent.data();
    a.scratch = scratch.data();
    a.req = req;
    a.count = count.data();
    const uint32_t threads = 128;
    shim_launch((uint32_t)((n + threads) / threads), threads, [&] { k_rls_plan(a); });
    unsigned long long acc = 0;
    for (uint64_t i = 0; i <= n; i++) {
        start[i] = acc;
        acc += count[i];
    }
    const uint64_t n_store = start[n] >> 32, n_ctr = start[n] & 0xFFFFFFFFull;
    *out_n_ctr = n_ctr;
    if (n_ctr > cap_ctrs) return ~0ull;
    RlsScatterArgs b;
    b.req = req;
    b.scratch = scratch.data();
    b.start = start.data();
    b.n = n;
    b.per_req = per_req;
    b.method = method;
    b.now_us = now_us;
    b.ctr_off = ctr_off;
    b.ctrs = ctrs;
    b.delta = delta;
    b.now = now;
    shim_launch((uint32_t)((n + threads) / threads), threads, [&] { k_rls_scatter(b); });
    return n_store;
}

// The shared BLAKE2b-96 counter key of (source, value) pairs in the given order (the matcher sorts them first).
void emu_key_digest(const char* const* sources, const char* const* values, uint32_t n, uint64_t* lo, uint64_t* hi) {
    rl_b2::KeyDigest d;
    for (uint32_t i = 0; i < n; i++) {
        d.str(sources[i], strlen(sources[i]));
        d.str(values[i], strlen(values[i]));
    }
    d.finish(*lo, *hi);
}

// Plain BLAKE2b of any output length (1..64 bytes) over one message.
void emu_blake2b(const uint8_t* msg, uint64_t len, uint32_t outlen, uint8_t* out) {
    rl_b2::Blake2b b(outlen);
    b.update(msg, len);
    b.final(out);
}

}  // extern "C"
