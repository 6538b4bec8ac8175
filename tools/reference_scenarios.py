"""The reference's own benchmark on one wide engine: its four TestScenarios (limitador/benches/bench.rs:65-90) and its
three benchmarked calls (is_rate_limited, update_counters, check_rate_limited_and_update with load_counters = false),
with every limit of a namespace applying to every request (50 counters per request in two of the scenarios).

    python tools/reference_scenarios.py [--batch 65536] [--steps 20] [--verify-batches 2] [--seed 0] [--cpu-only]

Limits are built through the native matcher as bench.rs:526-568 builds them: conditions `cond_k == '1'`, variables
`var_k` (root bindings), max u64::MAX, window 60*l + 10 s.  Each request picks a namespace from a seeded RNG.  One
engine with max_counters_per_request = 64 and max_counters sized for 50 counters per request runs every scenario.

Per (scenario, call) it first replays --verify-batches batches through the engine and the CPU oracle and compares the
verdicts, the first-limited ids and the whole table; then it times --steps batches (host clock around calls that end
in a device synchronise: the CSR calls read their counter count and resolve status back).  One JSON line each, with
the card's name and power limit read in the same run; the exit status is 1 if anything differed.  --cpu-only runs the
matcher and the oracle arm alone (a rehearsal on a machine without a GPU; no rate is printed).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import engine as _eng  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from oracle import binding as ob  # noqa: E402

SCENARIOS = [(10, 50, 10, 0), (1, 1, 1, 1), (10, 10, 10, 10), (10, 50, 10, 10)]  # bench.rs:65-90
CALLS = [("is_rate_limited", 1), ("update_counters", 2), ("check_rate_limited_and_update", 0)]  # oracle batch modes
T0 = 1_700_000_000_000_000


def scenario_name(s):
    return f"{s[0]} namespaces with {s[1]} limits each with {s[2]} conditions and {s[3]} variables"


def build(scn):
    n_ns, n_lim, n_cond, n_var = scn
    m = MT.Matcher()
    m.set_counter_cap(max(16, n_lim))
    conds = [f"cond_{i} == '1'" for i in range(n_cond)]
    vars_ = [f"var_{j}" for j in range(n_var)]
    descs = [m.add_limit(str(ns), 2 ** 64 - 1, l * 60 + 10, conds, vars_) for ns in range(n_ns) for l in range(n_lim)]
    values = {f"cond_{i}": "1" for i in range(n_cond)}
    values.update({f"var_{j}": "1" for j in range(n_var)})
    return m, np.array(descs, dtype=_eng.LIMIT_DESC_DTYPE), values


def match_batch(m, values, n_ns, n_lim, n, rng):
    """CSR counters of n requests, each of a namespace drawn from rng, through rl_matcher_counters_batch."""
    keep = [(k.encode(), v.encode()) for k, v in values.items()]
    nb = len(keep)
    binds = (MT.RlBinding * max(1, n * nb))()
    for i in range(n):
        for j, (k, v) in enumerate(keep):
            binds[i * nb + j] = MT.RlBinding(MT.BIND_ROOT, 0, k, v)
    bind_off = (np.arange(n + 1, dtype=np.uint32) * nb).astype(np.uint32)
    ns_ids = np.array([m.namespace_id(str(int(x))) for x in rng.integers(0, n_ns, size=n)], dtype=np.uint32)
    cap = n * n_lim
    off = np.zeros(n + 1, dtype=np.uint32)
    ctrs = np.zeros(cap, dtype=_eng.COUNTER_DTYPE)
    st = m._lib.rl_matcher_counters_batch(m._h, n, ns_ids.ctypes.data, bind_off.ctypes.data, binds, off.ctypes.data,
                                          ctrs.ctypes.data, cap)
    if st != 0 or int(off[-1]) != cap:
        raise RuntimeError(f"matching failed ({st}, {int(off[-1])} counters)")
    return off, ctrs


def normalised(dump, descs):
    unq = {int(d["limit_id"]) for d in descs if not d["qualified"]}
    return sorted(t for t in dump if not (t[0] in unq and t[3] == 0 and t[4] == 0))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return name, power
    except Exception as ex:  # the rate is still stated with the device name torch reports
        import torch
        return torch.cuda.get_device_name(0), f"unknown ({type(ex).__name__})"


def engine_call(e, call, off, ctrs, delta, now):
    if call == 0:
        return e.check_and_update_batch(off, ctrs, delta, now, False)[:2]
    if call == 1:
        return e.is_within_limits_batch(off, ctrs, delta, now)
    e.update_batch(off, ctrs, delta, now)
    return None


class DeviceBatch:
    """A batch staged once in device memory (torch tensors), so that a timed call moves no counters over PCIe."""

    def __init__(self, off, ctrs, delta, now):
        import torch
        dev = torch.device("cuda")
        self.n = len(delta)
        self.off = torch.from_numpy(off.view(np.int32).copy()).to(dev)
        self.ctrs = torch.from_numpy(ctrs.view(np.uint8).copy()).to(dev)
        self.delta = torch.from_numpy(delta.view(np.int64).copy()).to(dev)
        self.now = torch.from_numpy(now.view(np.int64).copy()).to(dev)
        self.lim = torch.zeros(self.n, dtype=torch.uint8, device=dev)
        self.first = torch.zeros(self.n, dtype=torch.int32, device=dev)

    def run(self, e, call):
        L, h, p = e._lib, e._h, lambda t: C.c_void_p(t.data_ptr())
        if call == 0:
            st = L.rl_check_and_update_batch(h, self.n, p(self.off), p(self.ctrs), p(self.delta), p(self.now), 0,
                                             _eng.MEM_DEVICE, p(self.lim), p(self.first), None, None)
        elif call == 1:
            st = L.rl_is_within_limits_batch(h, self.n, p(self.off), p(self.ctrs), p(self.delta), p(self.now),
                                             _eng.MEM_DEVICE, p(self.lim), p(self.first))
        else:
            st = L.rl_update_batch(h, self.n, p(self.off), p(self.ctrs), p(self.delta), p(self.now), _eng.MEM_DEVICE)
        e._check(st)


def run(scn, call_name, call, a, rng_seed, cpu_only):
    n_ns, n_lim, _, _ = scn
    m, descs, values = build(scn)
    rng = np.random.default_rng(rng_seed)
    o = ob.Oracle(1 << 12)
    for d in descs:
        o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    e = None
    if not cpu_only:
        e = _eng.Engine(capacity_rows=1 << 14, cells_per_row=7, max_batch=a.batch, max_counters=a.batch * 50,
                        max_counters_per_request=64)
        e.limits_set(descs)
    out = {"scenario": scenario_name(scn), "call": call_name, "batch": a.batch, "counters_per_request": n_lim}
    mism = 0
    t = T0
    delta = np.ones(a.batch, dtype=np.uint64)
    for b in range(a.verify_batches):
        off, ctrs = match_batch(m, values, n_ns, n_lim, a.batch, rng)
        now = np.full(a.batch, t, dtype=np.uint64)
        t += 1_000
        want = o.batch_csr(call, off, ctrs, delta, now, False)
        if e is not None:
            got = engine_call(e, call, off, ctrs, delta, now)
            if got is not None:
                mism += int(np.count_nonzero(got[0] != want[0])) + int(np.count_nonzero(got[1] != want[1]))
            if normalised(e.dump(), descs) != normalised(o.dump(), descs):
                mism += 1
                out["table_differs_after_batch"] = b
    out["verified_batches"] = a.verify_batches
    out["mismatches"] = mism
    if e is None:
        out["note"] = "cpu-only: oracle arm only, no rate"
        return out
    off, ctrs = match_batch(m, values, n_ns, n_lim, a.batch, rng)
    db = DeviceBatch(off, ctrs, delta, np.full(a.batch, t, dtype=np.uint64))
    for _ in range(a.warmup):
        db.run(e, call)
    e.sync()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        db.run(e, call)
    e.sync()
    dt = (time.perf_counter() - t0) / a.steps
    st = e.stats()
    out.update({"ms_per_batch": dt * 1e3, "decisions_per_s": a.batch / dt, "counters_per_s": a.batch * n_lim / dt,
                "fixed_point_rounds_last_batch": st["fixed_point_rounds"]})
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--verify-batches", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--cpu-only", action="store_true")
    a = ap.parse_args()
    name, power = ("none", "none") if a.cpu_only else card()
    bad = 0
    for si, scn in enumerate(SCENARIOS):
        for call_name, call in CALLS:
            r = run(scn, call_name, call, a, a.seed * 1000 + si * 10 + call, a.cpu_only)
            r.update({"device": name, "power_limit": power})
            bad += r["mismatches"]
            print(json.dumps(r), flush=True)
    print(json.dumps({"total_mismatches": bad, "device": name, "power_limit": power}), flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
