// emu_http.cpp — TEST-ONLY host driver of the HTTP device plan kernels (limitador_b200/csrc/rl_http_dev.cuh) under
// tests/emu/cuda_shim.h: the SAME kernel source the GPU runs, one CUDA thread after the other in a shuffled order.  Not
// shipped, not a fallback.  The call sequence follows rl_rls_dev.cu's rl_http_dev_plan, with a host loop in place of the
// CUB scan.  Also compiled into tests/san/san_http_dev.cpp for the ASan + UBSan run.
#include "cuda_shim.h"
// (the shim must come first: it defines __global__ & co. away)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../limitador_b200/csrc/rl_http_dev.cuh"

extern "C" {

void emu_http_seed(uint64_t s) { shim_seed = s; }

// One device plan.  image: rl_matcher_image's words.  Outputs as rl_http_plan_view gives them: req [n], ctr_off
// [n_store + 1] (n + 1 room), ctrs (cap_ctrs room), delta / now / load [n_store] (n room); runs [3 * n_runs] (3n room)
// and ctr_run [n_store + n_runs] (2n + 1 room), the per-call CSR the store calls read.  Returns n_store (or ~0 when
// cap_ctrs is too small); *out_n_ctr = counters, *out_n_runs = store calls.
uint64_t emu_http_plan(const uint32_t* image, int endpoint, uint64_t n, const uint8_t* buf, const uint64_t* off, uint64_t now_us,
                       uint32_t engine_max, HttpDevReq* req, uint32_t* ctr_off, rl_counter* ctrs, uint64_t cap_ctrs, uint64_t* delta,
                       uint64_t* now, uint8_t* load, uint32_t* runs, uint32_t* ctr_run, uint64_t* out_n_ctr, uint32_t* out_n_runs) {
    const uint32_t per_req = std::min(image[RL_IMG_H_COUNTER_CAP], engine_max);
    const uint64_t bytes = n ? off[n] : 0;
    // the device buffers (exact sizes, so that ASan sees any access past them)
    std::vector<uint8_t> txt(bytes + 1), bits(bytes / 8 + n + 1);
    std::vector<rl_rls_entry> ent(bytes / 2 + 1);
    std::vector<rl_counter> scratch(n * (uint64_t)per_req + 1);
    std::vector<HttpScan> count(n + 1), start(n + 1);
    std::vector<uint32_t> block(RL_HTTP_RUNS_HEAD + 3 * (n + 1));
    HttpPlanArgs a;
    a.buf = buf;
    a.off = off;
    a.n = n;
    a.img = rl_img_view(image, image);
    a.per_req = per_req;
    a.endpoint = endpoint;
    a.txt = txt.data();
    a.bits = bits.data();
    a.ent = ent.data();
    a.scratch = scratch.data();
    a.req = req;
    a.count = count.data();
    const uint32_t threads = 128;
    shim_launch((uint32_t)((n + threads) / threads), threads, [&] { k_http_plan(a); });
    HttpScan acc{0, 0, 0, 0, 0, {0, 0}};
    for (uint64_t i = 0; i <= n; i++) {
        start[i] = acc;
        acc = HttpScanOp()(acc, count[i]);
    }
    HttpRunsArgs ra{count.data(), start.data(), n, block.data()};
    shim_launch((uint32_t)((n + threads) / threads), threads, [&] { k_http_runs(ra); });
    const uint64_t n_store = block[0], n_ctr = block[1], n_runs = block[2];
    *out_n_ctr = n_ctr;
    *out_n_runs = (uint32_t)n_runs;
    if (n_ctr > cap_ctrs) return ~0ull;
    HttpScatterArgs b;
    b.req = req;
    b.scratch = scratch.data();
    b.start = start.data();
    b.runs = block.data() + RL_HTTP_RUNS_HEAD;
    b.n = n;
    b.per_req = per_req;
    b.endpoint = endpoint;
    b.now_us = now_us;
    b.ctr_off = ctr_off;
    b.ctr_run = ctr_run;
    b.ctrs = ctrs;
    b.delta = delta;
    b.now = now;
    b.load = load;
    shim_launch((uint32_t)((n + threads) / threads), threads, [&] { k_http_scatter(b); });
    memcpy(runs, block.data() + RL_HTTP_RUNS_HEAD, 3 * n_runs * sizeof(uint32_t));
    return n_store;
}

}  // extern "C"
