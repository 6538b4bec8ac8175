"""Time the RLS wire path with the plan on the GPU against the old composition with the plan on the CPU.

The stream is bench.py's `extra.rls` shape: 32 namespaces of three limits (GET per user, hourly per user, a global one),
one descriptor (method, user) per request, users drawn Zipf(1.1), ShouldRateLimit with draft-03 headers.  For each batch
size, alternating batch by batch in one process on two engines that see the same requests:
  new  rl_rls_serve: device plan -> ONE store call on the device arrays -> CPU finish (stage times from the service);
  old  the CPU plan (rl_rls_plan) -> rl_check_and_update_batch from host arrays -> the CPU finish.
Wall time per batch is the median over the timed batches; the response bytes of the two paths are compared for every
batch.  Prints one JSON object (with the card's name and power limit, read in the same run).
Usage: python tools/rls_time.py [--batches 64,4096,32768,65536] [--steps 20] [--threads 0]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import Engine  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from limitador_b200 import rls as R  # noqa: E402

T0 = 1_700_000_000_000_000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:  # noqa: BLE001
        return {"name": "unknown", "power_limit": "unknown", "error": str(ex)}


def stream(batch, steps, seed=42):
    rng = np.random.default_rng(seed)
    n_ns, n_users = 32, 200_000
    limits = []
    for ns in range(n_ns):
        limits.append((f"ns{ns}", 100, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"))
        limits.append((f"ns{ns}", 1000, 3600, [], ["descriptors[0].user"], "hourly-per-user"))
        limits.append((f"ns{ns}", 1 << 40, 60, ["descriptors[0].method != 'OPTIONS'"], [], None))
    methods = ["GET", "GET", "GET", "POST", "OPTIONS"]
    zipf = rng.zipf(1.1, size=steps * batch) % n_users
    batches = []
    for s in range(steps):
        u = zipf[s * batch:(s + 1) * batch]
        ns = rng.integers(0, n_ns, size=batch)
        me = rng.integers(0, len(methods), size=batch)
        batches.append(R.pack_requests([R.encode_request(f"ns{ns[i]}", [[("method", methods[me[i]]), ("user", f"u{u[i]}")]], 1)
                                        for i in range(batch)]))
    return limits, batches


def one_size(batch, steps, warmup, threads):
    limits, batches = stream(batch, steps + warmup)
    sides = []
    for _ in range(2):
        m = MT.Matcher()
        e = Engine(capacity_rows=1 << 20, cells_per_row=3, max_batch=batch, max_counters=4 * batch)
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
        sides.append((m, e, R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, threads)))
    (_, _, new), (_, e_old, old) = sides
    t_new, t_old, st_new, st_old, mism = [], [], [], [], 0
    for s, (buf, off) in enumerate(batches):
        now = T0 + s * 1_000_000
        a = time.perf_counter()
        new.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        b = time.perf_counter()
        got = new.responses()
        c = time.perf_counter()
        p = old.plan(R.SHOULD_RATE_LIMIT, buf, off, now)
        d = time.perf_counter()
        outs = e_old.check_and_update_batch(p["ctr_off"], p["ctrs"], p["delta"], p["now_us"], True)
        f = time.perf_counter()
        old._check(old._lib.rl_rls_finish(old._h, 0, *[np.ascontiguousarray(x).ctypes.data for x in outs]))
        g = time.perf_counter()
        want = old.responses()
        mism += sum(1 for x, y in zip(got, want) if x != y)
        if s >= warmup:
            t_new.append(b - a)
            t_old.append(g - c)
            st_new.append(new.timings())
            st_old.append({"plan_us": (d - c) * 1e6, "store_us": (f - d) * 1e6, "finish_us": (g - f) * 1e6})
    med = lambda xs: float(np.median(xs))  # noqa: E731
    row = {
        "batch": batch, "steps": steps, "threads": threads,
        "new_ms_per_batch": round(med(t_new) * 1e3, 3),
        "new_stage_ms": {k[:-3]: round(med([t[k] for t in st_new]) / 1e3, 3) for k in ("plan_us", "store_us", "finish_us")},
        "old_ms_per_batch": round(med(t_old) * 1e3, 3),
        "old_stage_ms": {k[:-3]: round(med([t[k] for t in st_old]) / 1e3, 3) for k in ("plan_us", "store_us", "finish_us")},
        "new_requests_per_s": round(batch / med(t_new)),
        "old_requests_per_s": round(batch / med(t_old)),
        "responses_compared": batch * len(batches), "response_mismatches": mism,
    }
    for _, e, svc in sides:
        svc.close()
        e.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,4096,32768,65536")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--threads", type=int, default=0, help="CPU workers of plan / finish (0 = one per CPU, at most 64)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    threads = a.threads or min(os.cpu_count() or 1, 64)
    rows = [one_size(int(b), a.steps, a.warmup, threads) for b in a.batches.split(",")]
    res = {"card": card(), "nproc": os.cpu_count(), "rows": rows,
           "note": "old = CPU plan -> rl_check_and_update_batch (RL_MEM_HOST, called through the Python binding) -> CPU finish"}
    text = json.dumps(res)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
