"""Micro-benchmark of the native CPU front (rl_matcher_counters_batch) on the reference's own bench scenarios
(limitador/benches/bench.rs:65-90,521-568: N namespaces x L limits, each with C conditions `cond_i == '1'` and
V variables `var_j`, every limit applies to every request of its namespace).

    python -m limitador_b200.bench_matcher [--requests 20000] [--threads 1]

Prints one JSON line per scenario: requests/s and counters/s of ONE call over a prebuilt binding array (the
ctypes marshalling is outside the timed region: a server builds `rl_binding`s straight from the decoded RLS
request).  The reference's Criterion bench of the same scenarios times the whole check_rate_limited_and_update
(CEL matching + moka); it cannot be run here (no Rust toolchain), so no ratio is claimed.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import threading
import time

import numpy as np

from . import engine as _eng
from . import matcher as MT

SCENARIOS = [(10, 50, 10, 0), (1, 1, 1, 1), (10, 10, 10, 10), (10, 50, 10, 10)]  # bench.rs:65-90


def build(n_ns, n_lim, n_cond, n_var):
    m = MT.Matcher()
    m.set_counter_cap(max(16, n_lim))  # a default engine takes 16 counters per request; tools/reference_scenarios.py decides these on a wide one
    conds = [f"cond_{i} == '1'" for i in range(n_cond)]
    vars_ = [f"var_{j}" for j in range(n_var)]
    for ns in range(n_ns):
        for l in range(n_lim):
            m.add_limit(str(ns), 2 ** 64 - 1, l * 60 + 10, conds, vars_)
    values = {f"cond_{i}": "1" for i in range(n_cond)}
    values.update({f"var_{j}": "1" for j in range(n_var)})
    return m, values


def run(scn, n_req, threads):
    n_ns, n_lim, n_cond, n_var = scn
    m, values = build(*scn)
    keep = [(k.encode(), v.encode()) for k, v in values.items()]
    nb = len(keep)
    binds = (MT.RlBinding * (n_req * nb))()
    for i in range(n_req):
        for j, (k, v) in enumerate(keep):
            binds[i * nb + j] = MT.RlBinding(MT.BIND_ROOT, 0, k, v)
    off = (np.arange(n_req + 1, dtype=np.uint32) * nb).astype(np.uint32)
    ns_ids = (np.arange(n_req, dtype=np.uint32) % n_ns).astype(np.uint32)
    cap = n_req * n_lim
    lib = m._lib

    def work(out):
        ctr_off = np.zeros(n_req + 1, dtype=np.uint32)
        ctrs = np.zeros(cap, dtype=_eng.COUNTER_DTYPE)
        lib.rl_matcher_counters_batch(m._h, n_req, ns_ids.ctypes.data, off.ctypes.data, binds, ctr_off.ctypes.data,
                                      ctrs.ctypes.data, cap)  # warm-up (page faults of the outputs)
        t0 = time.perf_counter()
        st = lib.rl_matcher_counters_batch(m._h, n_req, ns_ids.ctypes.data, off.ctypes.data, binds, ctr_off.ctypes.data,
                                           ctrs.ctypes.data, cap)
        out.append((time.perf_counter() - t0, st, int(ctr_off[-1])))

    outs = [[] for _ in range(threads)]
    ts = [threading.Thread(target=work, args=(o,)) for o in outs]
    t0 = time.perf_counter()
    [t.start() for t in ts]
    [t.join() for t in ts]
    wall = time.perf_counter() - t0
    assert all(o[0][1] == 0 for o in outs)
    per_call = max(o[0][0] for o in outs)
    n_ctr = outs[0][0][2]
    assert n_ctr == n_req * n_lim
    return {"scenario": f"{n_ns} namespaces with {n_lim} limits each with {n_cond} conditions and {n_var} variables",
            "threads": threads, "requests_per_s": threads * n_req / per_call, "counters_per_s": threads * n_ctr / per_call,
            "ns_per_request": per_call / n_req * 1e9, "counters_per_request": n_lim, "wall_s": wall,
            "fits_one_engine_request": n_lim <= 16}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=20000)
    ap.add_argument("--threads", type=int, default=1)
    a = ap.parse_args()
    for scn in SCENARIOS:
        print(json.dumps(run(scn, a.requests, a.threads)))


if __name__ == "__main__":
    main()
