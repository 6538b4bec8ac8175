// emu_cvars.cpp — TEST-ONLY host driver of the counter variable dictionary's kernels (limitador_b200/csrc/rl_cvars_dev.cuh)
// under tests/emu/cuda_shim.h: the SAME kernel source the GPU runs, one CUDA thread after the other in a shuffled order.
// Not shipped, not a fallback.  The call sequences follow rl_rls_dev.cu: a plan kernel (RLS or HTTP) and the recording
// kernel over its scratch (the scatter writes nothing the recording reads, so it is left out); the lookup with its
// scan and gather; the GC's mark, kept lengths, scan and rebuild, with host loops in place of the CUB scans.  Also
// compiled into tests/san/san_cvars.cpp for the ASan + UBSan run.
// Built a second time with -DEMU_SIMT under tests/emu/cuda_simt.h, whose interleaving mode lets the recording threads of a
// block race for the same new keys; there the recording kernel runs in 256-thread blocks (the GPU uses 128), so that all
// 256 requests of a block can collide.
#ifdef EMU_SIMT
#include "cuda_simt.h"
#define shim_launch simt_launch
static uint64_t shim_seed = 0;
#else
#include "cuda_shim.h"
#endif
// (the shim must come first: it defines __global__ & co. away)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../limitador_b200/csrc/rl_cvars_dev.cuh"

namespace {

struct EmuDict {
    std::vector<CvSlot> slots;
    std::vector<uint8_t> arena;
    std::vector<unsigned long long> ctl;
    CvDict view() { return CvDict{slots.data(), slots.size() - 1, arena.data(), arena.size(), ctl.data()}; }
};

const uint32_t kThreads = 128;
uint32_t grid(uint64_t n) { return (uint32_t)((n + kThreads - 1) / kThreads); }
#ifdef EMU_SIMT
const uint32_t kRecordThreads = 256;
#else
const uint32_t kRecordThreads = kThreads;
#endif

// the scratch a plan leaves and the recording reads (exact sizes, so that ASan sees any access past them)
struct Scratch {
    std::vector<rl_rls_entry> ent;
    std::vector<rl_counter> ctrs;
    std::vector<uint8_t> txt, bits;
    std::vector<unsigned long long> rls_count;
    std::vector<HttpScan> http_count;
};

void record(EmuDict* d, const RlImage& img, uint32_t per_req, uint64_t n, const uint8_t* buf, const uint64_t* off, Scratch& s) {
    CvRecordArgs a;
    a.buf = buf;
    a.off = off;
    a.n = n;
    a.img = img;
    a.per_req = per_req;
    a.ent = s.ent.data();
    a.scratch = s.ctrs.data();
    a.rls_count = s.rls_count.data();
    a.http_count = s.http_count.data();
    a.txt = s.txt.data();
    a.bits = s.bits.data();
    a.dict = d->view();
    const uint32_t blocks = (uint32_t)((n + kRecordThreads - 1) / kRecordThreads);
    if (!s.rls_count.empty()) shim_launch(blocks, kRecordThreads, [&] { k_counter_vars_record<CvWire>(a); });
    else shim_launch(blocks, kRecordThreads, [&] { k_counter_vars_record<CvJson>(a); });
}

}  // namespace

extern "C" {

void emu_cv_seed(uint64_t s) { shim_seed = s; }
#ifdef EMU_SIMT
// cuda_simt.h's interleaving mode for the launches that follow (on = 0: off, the default)
void emu_cv_interleave(int on, uint64_t seed, double p) { simt_interleave(on != 0, seed, p); }
#endif

// max_keys rounded up to a power of two (at least 16) slots, as rl_cv_dev_configure sizes them
void* emu_cv_create(uint64_t max_keys, uint64_t arena_bytes) {
    uint64_t slots = 16;
    while (slots < max_keys) slots *= 2;
    EmuDict* d = new EmuDict();
    d->slots.assign(slots, CvSlot{});
    d->arena.assign(arena_bytes, 0);
    d->ctl.assign(RL_CV_CTL_WORDS, 0);
    return d;
}
void emu_cv_destroy(void* d) { delete static_cast<EmuDict*>(d); }

void emu_cv_stats(void* h, uint64_t* slots, uint64_t* keys, uint64_t* arena_used, uint64_t* dropped) {
    EmuDict* d = static_cast<EmuDict*>(h);
    *slots = d->slots.size();
    *keys = d->ctl[RL_CV_KEYS];
    *arena_used = std::min<uint64_t>(d->ctl[RL_CV_CURSOR], d->arena.size());
    *dropped = d->ctl[RL_CV_DROPPED];
}

// k_rls_plan (method 0..2) or k_http_plan (endpoint 0..2) over the batch, then the recording kernel.  Returns the store
// requests of the batch.
uint64_t emu_cv_plan_record(void* h, int http, const uint32_t* image, int endpoint, uint64_t n, const uint8_t* buf,
                            const uint64_t* off, uint32_t engine_max) {
    EmuDict* d = static_cast<EmuDict*>(h);
    const uint32_t per_req = std::min(image[RL_IMG_H_COUNTER_CAP], engine_max);
    const uint64_t bytes = n ? off[n] : 0;
    const RlImage img = rl_img_view(image, image);
    Scratch s;
    s.ent.resize(bytes / 2 + 1);
    s.ctrs.resize(n * (uint64_t)per_req + 1);
    uint64_t n_store = 0;
    if (!http) {
        std::vector<RlsDevReq> req(n + 1);
        s.rls_count.resize(n + 1);
        RlsPlanArgs a;
        a.buf = buf;
        a.off = off;
        a.n = n;
        a.img = img;
        a.per_req = per_req;
        a.ent = s.ent.data();
        a.scratch = s.ctrs.data();
        a.req = req.data();
        a.count = s.rls_count.data();
        shim_launch(grid(n + 1), kThreads, [&] { k_rls_plan(a); });
        for (uint64_t i = 0; i < n; i++) n_store += s.rls_count[i] >> 32;
    } else {
        std::vector<HttpDevReq> req(n + 1);
        s.txt.resize(bytes + 1);
        s.bits.resize(bytes / 8 + n + 1);
        s.http_count.resize(n + 1);
        HttpPlanArgs a;
        a.buf = buf;
        a.off = off;
        a.n = n;
        a.img = img;
        a.per_req = per_req;
        a.endpoint = endpoint;
        a.txt = s.txt.data();
        a.bits = s.bits.data();
        a.ent = s.ent.data();
        a.scratch = s.ctrs.data();
        a.req = req.data();
        a.count = s.http_count.data();
        shim_launch(grid(n + 1), kThreads, [&] { k_http_plan(a); });
        for (uint64_t i = 0; i < n; i++) n_store += s.http_count[i].n_store;
    }
    record(d, img, per_req, n, buf, off, s);
    return n_store;
}

// Every entry: (varset, key_lo, key_hi, blob offset, blob length) in slot order.  Returns the entries (at most cap written).
uint64_t emu_cv_dump(void* h, uint32_t* varset, uint64_t* lo, uint64_t* hi, uint64_t* boff, uint32_t* blen, uint64_t cap) {
    EmuDict* d = static_cast<EmuDict*>(h);
    uint64_t k = 0;
    for (const CvSlot& s : d->slots) {
        if (!s.fp) continue;
        if (k < cap) {
            varset[k] = s.varset;
            lo[k] = s.key_lo;
            hi[k] = s.key_hi;
            boff[k] = s.off;
            blen[k] = s.len;
        }
        k++;
    }
    return k;
}
const uint8_t* emu_cv_arena(void* h) { return static_cast<EmuDict*>(h)->arena.data(); }

// The lookup of n counters: pos [n + 1], unnamed [n], the packed blobs into out (cap bytes).  Returns the blobs' bytes.
uint64_t emu_cv_lookup(void* h, const uint32_t* image, uint64_t n, const uint32_t* lid, const uint64_t* lo, const uint64_t* hi,
                       uint64_t* pos, uint8_t* unnamed, uint8_t* out, uint64_t cap) {
    EmuDict* d = static_cast<EmuDict*>(h);
    std::vector<unsigned long long> len(n + 1), p(n + 1);
    std::vector<uint64_t> src(n + 1);
    CvLookupArgs a{lid, lo, hi, n, rl_img_view(image, image), d->view(), len.data(), src.data()};
    shim_launch(grid(n + 1), kThreads, [&] { k_counter_vars_lookup(a); });
    unsigned long long acc = 0;
    for (uint64_t i = 0; i <= n; i++) {
        p[i] = acc;
        acc += len[i];
    }
    if (acc > cap) return acc;
    CvGatherArgs g{p.data(), len.data(), src.data(), n, d->arena.data(), out};
    shim_launch(grid(n), kThreads, [&] { k_counter_vars_gather(g); });
    for (uint64_t i = 0; i <= n; i++) pos[i] = p[i];
    for (uint64_t i = 0; i < n; i++) unnamed[i] = src[i] == RL_CV_NONE;
    return acc;
}

// The GC over the given live counters.
void emu_cv_gc(void* h, const uint32_t* image, uint64_t n, const uint32_t* lid, const uint64_t* lo, const uint64_t* hi,
               uint64_t* kept, uint64_t* freed) {
    EmuDict* d = static_cast<EmuDict*>(h);
    const uint64_t slots = d->slots.size(), before = d->ctl[RL_CV_KEYS];
    std::vector<uint8_t> mark(slots, 0);
    std::vector<unsigned long long> len(slots + 1), pos(slots + 1);
    CvMarkArgs a{lid, lo, hi, n, rl_img_view(image, image), d->view(), mark.data()};
    shim_launch(grid(n), kThreads, [&] { k_counter_vars_mark(a); });
    const CvDict from = d->view();
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_kept(from, mark.data(), len.data()); });
    unsigned long long acc = 0;
    for (uint64_t p = 0; p <= slots; p++) {
        pos[p] = acc;
        acc += len[p];
    }
    EmuDict* to = new EmuDict();
    to->slots.assign(slots, CvSlot{});
    to->arena.assign(d->arena.size(), 0);
    to->ctl.assign(RL_CV_CTL_WORDS, 0);
    to->ctl[RL_CV_DROPPED] = d->ctl[RL_CV_DROPPED];
    CvRebuildArgs b{from, mark.data(), pos.data(), to->view()};
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_rebuild(b); });
    std::swap(d->slots, to->slots);
    std::swap(d->arena, to->arena);
    std::swap(d->ctl, to->ctl);
    delete to;
    *kept = d->ctl[RL_CV_KEYS];
    *freed = before - std::min<uint64_t>(before, *kept);
}

}  // extern "C"
