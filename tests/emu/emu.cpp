// emu.cpp — TEST-ONLY sequential host driver of the batching algorithm (not shipped, not a
// fallback).  It runs the same rl_core.h functions the sm_90a kernels run — request
// resolution into row accesses, per-row stream-order replay, and the fixed-point rounds
// for multi-row requests — so the algorithm can be checked against the oracle on a
// machine without a GPU.  The kernels' own mechanics (partition, smem grouping, CAS inserts,
// the chained commit) run on the host in emu_engine.cpp, and on the GPU in the -m gpu tests.  Both position encodings of rl_core.h run through the one
// driver: narrow (up to 16 counters per request) and wide (up to 64).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../limitador_b200/csrc/rl_core.h"
#include "../../limitador_b200/csrc/rl_registry.h"

struct emu_counter {
    uint32_t limit_id, _pad;
    uint64_t key_lo, key_hi;
};

struct emu {
    int cells;
    RlRegistry reg;
    std::vector<RlLimitDev> limits;  // reg's device tables
    std::vector<RlCellDesc> desc;    // [groups][8]
    std::map<std::pair<uint64_t, uint64_t>, RlRow<RL_MAX_CELLS>> table;
    uint64_t steps = 0;  // replay steps (one run or one request alone each) of the last batch's committing pass
};

// mode 0: check_and_update, 2: update.  Returns 0 or a positive RL_DEV_* code.
// WIDE: the walkers write remaining / ttl in processing order into scratch, and the resolve's permutation scatters
// them into the caller's order, as k_wide_scatter does.
template <bool WIDE>
static int batch_csr(emu* e, int mode, uint32_t n, const uint32_t* off, const emu_counter* ctrs, const uint64_t* delta,
                     const uint64_t* now, int lc, uint8_t* out_limited, uint32_t* out_first, uint64_t* out_rem_user,
                     uint64_t* out_ttl_user, int* rounds_out) {
    constexpr uint32_t MAXC = WIDE ? RL_MAX_CTRS_PER_REQ_WIDE : RL_MAX_CTRS_PER_REQ;
    std::vector<uint64_t> scr_rem(WIDE ? off[n] + 1 : 0), scr_ttl(WIDE ? off[n] + 1 : 0);
    std::vector<uint8_t> perm(WIDE ? off[n] + 1 : 0);
    uint64_t* out_rem = WIDE ? (out_rem_user ? scr_rem.data() : nullptr) : out_rem_user;
    uint64_t* out_ttl = WIDE ? (out_ttl_user ? scr_ttl.data() : nullptr) : out_ttl_user;
    std::vector<RlAccess> acc(off[n]);
    bool any_multi = false;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t o0 = off[i], m = off[i + 1] - o0;
        if (m == 0) {
            if (out_limited) out_limited[i] = 0;
            if (out_first) out_first[i] = RL_NONE_U32;
            continue;
        }
        auto get = [&](uint32_t j) {
            RlCtrIn r;
            r.limit_id = ctrs[o0 + j].limit_id;
            r.key_lo = ctrs[o0 + j].key_lo;
            r.key_hi = ctrs[o0 + j].key_hi;
            return r;
        };
        RlAccess tmp[MAXC];
        const int nacc = rl_resolve_request<WIDE>(i, m, get, e->limits.data(), (uint32_t)e->limits.size(), true, tmp,
                                                  WIDE ? perm.data() + o0 : nullptr);
        if (nacc < 0) return -nacc;
        for (uint32_t x = 0; x < m; x++) acc[o0 + x] = tmp[x];
        if (nacc > 1) any_multi = true;
    }
    // group accesses by row, keeping stream order (what k_part + the smem grouping produce)
    std::map<std::pair<uint64_t, uint64_t>, std::vector<uint32_t>> by_row;
    for (uint32_t a = 0; a < acc.size(); a++)
        if (acc[a].hdr_hi != 0) by_row[{acc[a].key_lo, acc[a].hdr_hi}].push_back(a);

    std::vector<uint32_t> fl_prev(n, RL_NONE_U32), fl_next(n, RL_NONE_U32);
    e->steps = 0;
    auto pass = [&](bool commit) {
        // where the walkers write request req's remaining / ttl: only in the committing pass
        auto lc_out = [&](uint32_t req) {
            const bool on = lc && commit;
            return std::make_pair(on && out_rem ? out_rem + off[req] : nullptr, on && out_ttl ? out_ttl + off[req] : nullptr);
        };
        for (auto& kv : by_row) {
            RlRow<RL_MAX_CELLS> st;
            auto it = e->table.find(kv.first);
            if (it != e->table.end()) st = it->second;
            else memset(&st, 0, sizeof st);
            const uint32_t group = (uint32_t)(kv.first.second >> 32);
            const RlCellDesc* desc = e->desc.data() + (size_t)group * 8;
            // run-length replay, exactly as k_main's lock-step rounds do it (rl_core.h hypotheses)
            const std::vector<uint32_t>& mem = kv.second;
            const uint32_t n = (uint32_t)mem.size();
            std::vector<uint64_t> P(n);
            uint64_t run = 0;
            for (uint32_t i = 0; i < n; i++) {
                run += delta[acc[mem[i]].req];
                P[i] = run;
            }
            const uint32_t lead_cells = acc[mem[0]].cells;
            bool uniform = true;  // k_main: runs of allowed requests are closed-form only for equal deltas
            for (uint32_t i = 1; i < n; i++)
                if (delta[acc[mem[i]].req] != delta[acc[mem[0]].req] || acc[mem[i]].cells != lead_cells) uniform = false;
            uint32_t pos = 0;
            uint64_t pbase = 0;
            auto outputs = [&](const RlAccess& A, uint32_t fl) {
                const uint32_t req = A.req;
                out_limited[req] = fl != RL_NONE_U32;
                if (!out_first) return;
                if (fl == RL_NONE_U32) {
                    out_first[req] = RL_NONE_U32;
                    return;
                }
                for (uint32_t k = 0; k < rl_cells_n(A.cells); k++)
                    if (rl_pos_of<WIDE>(A.posorig, k) == fl) out_first[req] = desc[rl_cells_at(A.cells, k)].limit_id;
            };
            while (pos < n) {
                uint32_t mA = n, mB = n;
                for (uint32_t i = pos; i < n && (mA == n || mB == n); i++) {
                    const RlAccess& A = acc[mem[i]];
                    const bool multi = mode == 0 && rl_cells_multi(A.cells);
                    bool aok = false, bok = false;
                    if (!multi) {
                        if (mode == 0) {
                            aok = rl_eval_deny_noeffect<RL_MAX_CELLS, WIDE>(st, desc, A.cells, A.posorig, delta[A.req], now[A.req], lc != 0);
                            bok = uniform && rl_eval_allow_run<RL_MAX_CELLS>(st, desc, A.cells, P[i] - pbase, now[A.req]);
                        } else {
                            bok = uniform && rl_eval_update_run<RL_MAX_CELLS>(st, A.cells, now[A.req]);
                        }
                    }
                    if (!aok && mA == n) mA = i;
                    if (!bok && mB == n) mB = i;
                }
                uint32_t newpos;
                if (mA > pos) {
                    newpos = mA;
                    for (uint32_t i = pos; i < mA; i++) {
                        const RlAccess& A = acc[mem[i]];
                        RlRow<RL_MAX_CELLS> loc = st;
                        uint32_t dd = 0;
                        const auto [rem, ttl] = lc_out(A.req);
                        const uint32_t fl = rl_walk_check_single<RL_MAX_CELLS, WIDE>(loc, dd, desc, A.cells, A.posorig, delta[A.req],
                                                                                     now[A.req], lc != 0, rem, ttl);
                        if (commit) outputs(A, fl);
                    }
                } else if (mB > pos) {
                    newpos = mB;
                    for (uint32_t i = pos; i < mB; i++) {
                        const RlAccess& A = acc[mem[i]];
                        RlRow<RL_MAX_CELLS> loc = st;
                        uint32_t dd = 0;
                        rl_advance_run<RL_MAX_CELLS>(loc, A.cells, (P[i] - delta[A.req]) - pbase);
                        if (mode == 0) {
                            const auto [rem, ttl] = lc_out(A.req);
                            const uint32_t fl = rl_walk_check_single<RL_MAX_CELLS, WIDE>(loc, dd, desc, A.cells, A.posorig,
                                                                                         delta[A.req], now[A.req], lc != 0, rem, ttl);
                            if (commit) outputs(A, fl);
                        } else {
                            rl_walk_update<RL_MAX_CELLS>(loc, dd, desc, A.cells, delta[A.req], now[A.req]);
                        }
                        if (i == mB - 1) st = loc;
                    }
                } else {
                    newpos = pos + 1;
                    const RlAccess& A = acc[mem[pos]];
                    const uint32_t req = A.req;
                    uint32_t dd = 0;
                    if (mode == 2) {
                        rl_walk_update<RL_MAX_CELLS>(st, dd, desc, A.cells, delta[req], now[req]);
                    } else {
                        const auto [rem, ttl] = lc_out(req);
                        if (!rl_cells_multi(A.cells)) {
                            const uint32_t fl = rl_walk_check_single<RL_MAX_CELLS, WIDE>(st, dd, desc, A.cells, A.posorig, delta[req],
                                                                                         now[req], lc != 0, rem, ttl);
                            if (commit) outputs(A, fl);
                        } else {
                            const uint32_t fl_in = fl_prev[req];
                            const uint32_t local = rl_walk_check_multi<RL_MAX_CELLS, WIDE>(st, dd, desc, A.cells, A.posorig, delta[req],
                                                                                          now[req], lc != 0, fl_in, rem, ttl);
                            if (!commit) {
                                if (local < fl_next[req]) fl_next[req] = local;
                            } else {
                                outputs(A, fl_in);
                            }
                        }
                    }
                }
                pbase = P[newpos - 1];
                pos = newpos;
                if (commit) e->steps++;
            }
            if (commit) e->table[kv.first] = st;  // physical row exists once probed (cells may be absent)
        }
    };
    int rounds = 0;
    if (mode == 0 && any_multi) {
        for (;;) {
            pass(false);
            rounds++;
            bool changed = false;
            for (uint32_t i = 0; i < n; i++) {
                if (fl_prev[i] != fl_next[i]) {
                    fl_prev[i] = fl_next[i];
                    changed = true;
                }
                fl_next[i] = RL_NONE_U32;
            }
            if (!changed) break;
            if (rounds > (int)n + 2) return 99;
        }
    }
    pass(true);
    if (WIDE && lc)
        for (uint32_t i = 0; i < n; i++)
            for (uint32_t p = off[i]; p < off[i + 1]; p++) {
                if (out_rem_user) out_rem_user[off[i] + perm[p]] = scr_rem[p];
                if (out_ttl_user) out_ttl_user[off[i] + perm[p]] = scr_ttl[p];
            }
    if (rounds_out) *rounds_out = rounds;
    return 0;
}

extern "C" {

emu* emu_create(int cells) {
    emu* e = new emu();
    e->cells = cells;
    e->reg.cells = cells;
    return e;
}
void emu_destroy(emu* e) { delete e; }

// rl_limits_set: RL_OK, or RL_FATAL and the refusal in err[err_cap] (the limits before the refused one stay set)
int emu_limits_set(emu* e, const rl_limit_desc* d, uint32_t n, char* err, uint32_t err_cap) {
    std::string msg;
    const int r = e->reg.set(d, n, &msg);
    RlTableImage t = e->reg.image();
    e->limits = std::move(t.lim);
    e->desc = std::move(t.desc);
    if (err_cap) snprintf(err, err_cap, "%s", msg.c_str());
    return r;
}

// the row group of a limit (0: not defined)
uint32_t emu_limit_group(emu* e, uint32_t limit_id) {
    const HostLimit* l = e->reg.find(limit_id);
    return l ? l->group : 0;
}

// batch_csr in the narrow (wide = 0) or the wide position encoding.
int emu_batch_csr(emu* e, int wide, int mode, uint32_t n, const uint32_t* off, const emu_counter* ctrs,
                  const uint64_t* delta, const uint64_t* now, int lc, uint8_t* out_limited, uint32_t* out_first,
                  uint64_t* out_rem, uint64_t* out_ttl, int* rounds_out) {
    return (wide ? batch_csr<true> : batch_csr<false>)(e, mode, n, off, ctrs, delta, now, lc, out_limited, out_first,
                                                       out_rem, out_ttl, rounds_out);
}

uint64_t emu_steps(emu* e) { return e->steps; }

// rl_resolve_request alone, for request index `req` of m counters: out_acc[0..m) and (wide) out_perm[0..m).  Returns the
// number of accesses or a negative RL_DEV_* code.
int emu_resolve(emu* e, int wide, uint32_t req, uint32_t m, const emu_counter* ctrs, uint32_t max_ctrs,
                RlAccess* out_acc, uint8_t* out_perm) {
    auto get = [&](uint32_t j) {
        RlCtrIn r;
        r.limit_id = ctrs[j].limit_id;
        r.key_lo = ctrs[j].key_lo;
        r.key_hi = ctrs[j].key_hi;
        return r;
    };
    if (wide)
        return rl_resolve_request<true>(req, m, get, e->limits.data(), (uint32_t)e->limits.size(), true, out_acc, out_perm,
                                        max_ctrs);
    return rl_resolve_request(req, m, get, e->limits.data(), (uint32_t)e->limits.size(), true, out_acc);
}

// every present cell -> (limit_id, key_lo, key_hi, value, expiry); unqualified cells always
uint64_t emu_dump(emu* e, uint64_t cap, uint32_t* lid, uint64_t* klo, uint64_t* khi, uint64_t* val, uint64_t* exp) {
    uint64_t cnt = 0;
    for (auto& kv : e->table) {
        const uint32_t group = (uint32_t)(kv.first.second >> 32);
        const RlCellDesc* desc = e->desc.data() + (size_t)group * 8;
        for (int c = 0; c < e->cells; c++) {
            if (desc[c].limit_id == RL_NONE_U32) continue;
            if (desc[c].qualified && kv.second.expiry[c] == 0) continue;
            if (cnt < cap) {
                lid[cnt] = desc[c].limit_id;
                klo[cnt] = kv.first.first;
                khi[cnt] = kv.first.second & 0xFFFFFFFFull;
                val[cnt] = kv.second.value[c];
                exp[cnt] = kv.second.expiry[c];
            }
            cnt++;
        }
    }
    return cnt;
}

}  // extern "C"
