// emu_shard_csr.cpp — TEST-ONLY host driver of the general (CSR) form of the sharded exchange
// (limitador_b200/csrc/rl_shard_csr.cuh: k_ccount .. k_cgather, with rl_shard.cuh's k_xwait / k_xwaitv) under
// tests/emu/cuda_simt.h, over `world` emulated engines (emu_engine.cpp) and host slabs laid out as rl_shard_batch_create
// lays out the device ones.  The call sequence follows rl_shard_host.inc (rl_shard_batch_send / _decide / _collect):
// the same kernels, the same run loop over the owner's inbox with one general-form engine call per run, the same error
// verdicts.  Every step poisons what a step must overwrite: the source's inbox blocks at every owner, its return blocks,
// dest / cpos, and the owner's CSR arrays and output mirror.
#include "emu_engine.cpp"
// (emu_engine.cpp brings the emulator, the decision kernels and rl_shard.cuh)
#include "../../limitador_b200/csrc/rl_shard_csr.cuh"

namespace {
constexpr uint8_t kPoisonC = 0xA5;
size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

template <class T>
void poison(std::vector<T>& v) {
    memset(v.data(), kPoisonC, v.size() * sizeof(T));
}
}  // namespace

struct emu_cshard_rank {
    emu_engine* e = nullptr;
    std::vector<uint8_t> slab;
    RlCXchg X{};
    std::vector<uint32_t> dest, cpos, totals, ctrs, errv, seg, cseg, head, off, roff;
    std::vector<rl_counter> csr;
    std::vector<uint64_t> delta, now, rem, ttl;
    std::vector<uint8_t> op, lim;
    std::vector<uint32_t> first;
    uint64_t sent = 0, decided = 0, collected = 0;
    uint32_t n = 0, s_op = 0, s_load_all = 0;
    bool refused = false;
    const uint32_t* s_off = nullptr;
    const uint8_t* s_load = nullptr;
};
struct emu_cshard {
    uint32_t world = 1, cap_req = 0, cap_ctr = 0;
    std::vector<emu_cshard_rank> r;
};

extern "C" {

emu_cshard* emu_cshard_create(emu_engine** engines, uint32_t world, uint32_t cap_req, uint32_t cap_ctr) {
    if (world == 0 || world > RL_XCHG_MAX_WORLD || !cap_req || (cap_req & 15u) || !cap_ctr || (cap_ctr & 15u)) return nullptr;
    emu_cshard* S = new emu_cshard();
    S->world = world;
    S->cap_req = cap_req;
    S->cap_ctr = cap_ctr;
    const size_t hdr = al256((size_t)world * cap_req * sizeof(RlCHdr)), ctr = al256((size_t)world * cap_ctr * sizeof(rl_counter));
    const size_t blk = al256((size_t)world * sizeof(RlCBlk)), ret = al256((size_t)5 * cap_req + (size_t)16 * cap_ctr);
    const size_t ctl = al256((size_t)world * sizeof(RlXCtl));
    const size_t n_max = (size_t)world * cap_req, c_max = (size_t)world * cap_ctr;
    S->r.resize(world);
    for (uint32_t k = 0; k < world; k++) {
        emu_cshard_rank& R = S->r[k];
        R.e = engines[k];
        R.slab.assign(hdr + ctr + blk + world * ret + ctl, 0);
        R.dest.assign(cap_req, 0);
        R.cpos.assign(cap_req, 0);
        R.totals.assign(96, 0);
        R.ctrs.assign(4, 0);
        R.errv.assign(8, 0);
        R.seg.assign(40, 0);
        R.cseg.assign(RL_XCHG_MAX_WORLD + 1, 0);
        R.head.assign(12 + 3 * n_max, 0);
        R.off.assign(n_max + 1, 0);
        R.roff.assign(2 * n_max + 1, 0);
        R.csr.resize(c_max);
        R.delta.assign(n_max, 0);
        R.now.assign(n_max, 0);
        R.op.assign(n_max, 0);
        R.lim.assign(n_max, 0);
        R.first.assign(n_max, 0);
        R.rem.assign(c_max, 0);
        R.ttl.assign(c_max, 0);
    }
    for (uint32_t k = 0; k < world; k++) {
        RlCXchg& X = S->r[k].X;
        for (auto& b : X.x.base) b = nullptr;
        for (uint32_t j = 0; j < world; j++) X.x.base[j] = S->r[j].slab.data();
        X.x.trace = nullptr;
        X.x.trace_pos = nullptr;
        X.x.off_recs = X.x.off_vin = 0;
        X.off_hdr = 0;
        X.off_ctr = hdr;
        X.off_blk = hdr + ctr;
        X.off_ret = hdr + ctr + blk;
        X.ret_stride = ret;
        X.x.off_ctl = hdr + ctr + blk + world * ret;
        X.x.world = world;
        X.x.rank = k;
        X.x.cap = cap_req;
        X.x.depth = 1;
        X.cap_ctr = cap_ctr;
    }
    return S;
}
void emu_cshard_destroy(emu_cshard* S) { delete S; }

// rl_shard_batch_send.  digest = this rank's registry digest (the engine's is computed on the host from its registry)
int emu_cshard_send(emu_cshard* S, uint32_t rank, uint32_t n, uint32_t n_ctr, const uint32_t* off, const rl_counter* ctrs,
                    const uint64_t* delta, const uint64_t* now, uint32_t op, const uint8_t* load, uint32_t load_all,
                    unsigned long long digest) {
    emu_cshard_rank& R = S->r[rank];
    if (R.sent != R.collected || op > 2) return -1;
    const uint32_t step = (uint32_t)R.sent, world = S->world;
    for (uint32_t o = 0; o < world; o++) {
        memset(R.X.hdr(o, rank), kPoisonC, (size_t)S->cap_req * sizeof(RlCHdr));
        memset(R.X.ctr(o, rank), kPoisonC, (size_t)S->cap_ctr * sizeof(rl_counter));
        memset(R.X.ret(rank, o), kPoisonC, R.X.ret_stride);
    }
    poison(R.dest);
    poison(R.cpos);
    poison(R.totals);
    std::fill(R.errv.begin(), R.errv.end(), 0u);
    std::fill(R.head.begin() + 4, R.head.begin() + 12, 0u);
    R.refused = n > S->cap_req || n_ctr > S->cap_ctr;
    const uint32_t nn = R.refused ? 0 : n;
    emu_engine* e = R.e;
    const RlDev D = make_dev(e);
    interleave_on(e, 11);
    simt_launch(1, 1024, [&] {
        k_ccount(D.limits, D.limits_cap, nn, off, ctrs, op, load, load_all, world, rank, R.dest.data(), R.cpos.data(), R.totals.data());
    });
    const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>(rl_ceil_div(nn, 256), 4));
    simt_launch(grid, 256, [&] {
        k_cscatter(R.X, nn, off, ctrs, delta, now, op, load, load_all, R.dest.data(), R.cpos.data(), R.totals.data(), digest, step,
                   R.ctrs.data() + 0);
    });
    interleave_off();
    R.n = n;
    R.s_off = off;
    R.s_load = load;
    R.s_op = op;
    R.s_load_all = load_all;
    R.sent++;
    return 0;
}

// rl_shard_batch_decide.  Returns a bit set: 1 an exchange error, 2 a source with another digest, 4 a failed engine call;
// head_out[4] = requests, counters, runs, digest mask of the step.
int emu_cshard_decide(emu_cshard* S, uint32_t rank, unsigned long long digest, uint32_t* head_out) {
    emu_cshard_rank& R = S->r[rank];
    if (R.decided >= R.sent) return -1;
    emu_engine* e = R.e;
    const uint32_t step = (uint32_t)R.decided, world = S->world, n_max = world * S->cap_req;
    poison(R.seg);
    poison(R.cseg);
    poison(R.off);
    poison(R.roff);
    poison(R.csr);
    poison(R.delta);
    poison(R.now);
    poison(R.op);
    poison(R.lim);
    poison(R.first);
    poison(R.rem);
    poison(R.ttl);
    uint32_t* head = R.head.data();
    simt_launch(1, 32, [&] { k_xwait(R.X.x, 0, step, R.seg.data(), R.seg.data() + 36, n_max, head + 4); });
    simt_launch(1, 32, [&] { k_cprep(R.X, R.seg.data(), digest, R.cseg.data(), head); });
    interleave_on(e, 12);
    simt_launch(4, 256, [&] {
        k_cunpack(R.X, R.seg.data(), R.cseg.data(), head, R.off.data(), R.csr.data(), R.delta.data(), R.now.data(), R.op.data());
    });
    simt_launch(1, 1024, [&] { k_cruns(R.off.data(), R.op.data(), head, head + 12); });
    simt_launch(4, 256, [&] { k_crebase(R.off.data(), head, head + 12, R.roff.data()); });
    interleave_off();
    const uint32_t n = head[0], nc = head[1], nr = head[2], bad = head[3];
    for (int k = 0; k < 4; k++) head_out[k] = head[k];
    std::fill(R.rem.begin(), R.rem.begin() + nc, 0ull);
    std::fill(R.ttl.begin(), R.ttl.begin() + nc, 0ull);
    int status = 0;
    const uint32_t* runs = head + 12;
    for (uint32_t k = 0; k < nr; k++) {  // shard_batch_runs
        const uint32_t j0 = runs[3 * k], c0 = runs[3 * k + 1], rop = runs[3 * k + 2];
        const uint32_t m = (k + 1 < nr ? runs[3 * (k + 1)] : n) - j0;
        uint8_t* lim = R.lim.data() + j0;
        uint32_t* first = R.first.data() + j0;
        int st = 0;
        if (rop != RL_COP_REFUSED) {
            const uint32_t* ro = R.roff.data() + j0 + k;
            const rl_counter* c = R.csr.data() + c0;
            const uint64_t *d = R.delta.data() + j0, *nw = R.now.data() + j0;
            const uint32_t base = rop & 0x0Fu;
            const bool lc = (rop & RL_COP_LOAD) != 0;
            if (base == RL_COP_IS_WITHIN) {
                begin_call(e);
                RlDev D = make_dev(e);
                rl_with_cells(e->cells, [&](auto cl) {
                    simt_launch(rl_ceil_div(m, 128), 128, [&] { k_query_csr<decltype(cl)::value>(D, m, ro, c, d, nw, lim, first); });
                });
                st = (int)e->err[0];
            } else {
                st = emu_engine_csr(e, base == RL_COP_UPDATE ? 2 : 0, m, ro, c, d, nw, lc, lim, first, lc ? R.rem.data() + c0 : nullptr,
                                    lc ? R.ttl.data() + c0 : nullptr);
            }
            if (st == 0 && base == RL_COP_UPDATE) {
                memset(lim, 0, m);
                memset(first, 0xFF, m * sizeof(uint32_t));
            }
            if (st) status |= 4;
        }
        if (rop == RL_COP_REFUSED || st) {
            memset(lim, 0xFF, m);
            memset(first, 0xFF, m * sizeof(uint32_t));
        }
    }
    interleave_on(e, 13);
    simt_launch(world * RL_CRET_SLICES, 256, [&] {
        k_creturn(R.X, R.seg.data(), R.cseg.data(), R.lim.data(), R.first.data(), R.rem.data(), R.ttl.data(), step, R.ctrs.data() + 2);
    });
    interleave_off();
    R.decided++;
    if (head[4]) status |= 1;
    if (bad) status |= 2;
    return status;
}

// rl_shard_batch_collect.  Returns 0, 1 on an exchange error, 2 for a batch over its caps (error verdicts)
int emu_cshard_collect(emu_cshard* S, uint32_t rank, uint8_t* lim, uint32_t* first, uint64_t* rem, uint64_t* ttl) {
    emu_cshard_rank& R = S->r[rank];
    if (R.collected >= R.decided) return -1;
    const uint32_t step = (uint32_t)R.collected, nn = R.refused ? 0 : R.n;
    simt_launch(1, 32, [&] { k_xwaitv(R.X.x, 0, step, R.errv.data()); });
    if (nn) {
        interleave_on(R.e, 14);
        simt_launch(std::max<uint32_t>(1, std::min<uint32_t>(rl_ceil_div(nn, 256), 4)), 256, [&] {
            k_cgather(R.X, nn, R.s_off, R.s_op, R.s_load, R.s_load_all, R.dest.data(), R.cpos.data(), lim, first, rem, ttl);
        });
        interleave_off();
    }
    if (R.refused && R.n) {
        memset(lim, 0xFF, R.n);
        memset(first, 0xFF, (size_t)R.n * sizeof(uint32_t));
    }
    R.collected++;
    if (R.errv[0]) return 1;
    return R.refused ? 2 : 0;
}

}  // extern "C"
