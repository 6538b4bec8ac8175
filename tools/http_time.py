"""Time the HTTP API path (rl_http_serve: device plan -> store calls on the device arrays -> CPU finish) against the CPU
composition (rl_http_plan -> rl_check_and_update_batch from host arrays, one call per run -> rl_http_finish).

The stream is tools/rls_time.py's: 32 namespaces of three limits, `values` = {method, user}, users drawn Zipf(1.1), as
/check_and_report bodies; response_headers is absent ("off") or "DraftVersion03" ("on") for every body.  For each batch
size and header setting, alternating batch by batch in one process on two engines that see the same bodies; the status,
body and headers of every response of the two paths are compared.  Prints one JSON object with the card's name and power
limit, read in the same run.
Usage: python tools/http_time.py [--batches 64,4096,32768,65536] [--steps 20] [--threads 16]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from limitador_b200 import Engine  # noqa: E402
from limitador_b200 import http_api as HA  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from limitador_b200 import rls as R  # noqa: E402
from rls_time import T0, card  # noqa: E402


def stream(batch, steps, headers, seed=42):
    rng = np.random.default_rng(seed)
    n_ns, n_users = 32, 200_000
    limits = []
    for ns in range(n_ns):
        limits.append((f"ns{ns}", 100, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"))
        limits.append((f"ns{ns}", 1000, 3600, [], ["descriptors[0].user"], "hourly-per-user"))
        limits.append((f"ns{ns}", 1 << 40, 60, ["descriptors[0].method != 'OPTIONS'"], [], None))
    methods = ["GET", "GET", "GET", "POST", "OPTIONS"]
    zipf = rng.zipf(1.1, size=steps * batch) % n_users
    hdr = "DraftVersion03" if headers == "on" else None
    batches = []
    for s in range(steps):
        u = zipf[s * batch:(s + 1) * batch]
        ns = rng.integers(0, n_ns, size=batch)
        me = rng.integers(0, len(methods), size=batch)
        batches.append(HA.pack_bodies([HA.encode_info(f"ns{ns[i]}", {"method": methods[me[i]], "user": f"u{u[i]}"}, 1, hdr)
                                       for i in range(batch)]))
    return limits, batches


def one_size(batch, steps, warmup, threads, headers):
    limits, batches = stream(batch, steps + warmup, headers)
    sides = []
    for _ in range(2):
        m = MT.Matcher()
        e = Engine(capacity_rows=1 << 20, cells_per_row=3, max_batch=batch, max_counters=4 * batch)
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
        svc = R.RlsService(m, e, R.HEADERS_NONE, threads)
        sides.append((m, e, svc, HA.HttpApi(svc)))
    (_, _, _, new), (_, e_old, _, old) = sides
    t_new, t_old, st_new, st_old, mism = [], [], [], [], 0
    for s, (buf, off) in enumerate(batches):
        now = T0 + s * 1_000_000
        a = time.perf_counter()
        new.serve(HA.CHECK_AND_REPORT, buf, off, now)
        b = time.perf_counter()
        got = new.responses()
        c = time.perf_counter()
        p = old.plan(HA.CHECK_AND_REPORT, buf, off, now)
        d = time.perf_counter()
        k, co = p["n_store"], p["ctr_off"]
        nc = int(co[-1]) if k else 0
        lim, fl = np.zeros(k, np.uint8), np.full(k, 0xFFFFFFFF, np.uint32)
        rem, ttl = np.zeros(nc, np.uint64), np.zeros(nc, np.uint64)
        for j0, j1 in HA.store_runs(p["load_counters"]):
            c0, c1 = int(co[j0]), int(co[j1])
            lim[j0:j1], fl[j0:j1], rem[c0:c1], ttl[c0:c1] = e_old.check_and_update_batch(
                co[j0:j1 + 1] - c0, p["ctrs"][c0:c1], p["delta"][j0:j1], p["now_us"][j0:j1], bool(p["load_counters"][j0]))
        f = time.perf_counter()
        old._check(old._lib.rl_http_finish(old._h, None, *[np.ascontiguousarray(x).ctypes.data for x in (lim, fl, rem, ttl)]))
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
        "batch": batch, "headers": headers, "steps": steps, "threads": threads,
        "new_ms_per_batch": round(med(t_new) * 1e3, 3),
        "new_stage_ms": {k[:-3]: round(med([t[k] for t in st_new]) / 1e3, 3) for k in ("plan_us", "store_us", "finish_us")},
        "old_ms_per_batch": round(med(t_old) * 1e3, 3),
        "old_stage_ms": {k[:-3]: round(med([t[k] for t in st_old]) / 1e3, 3) for k in ("plan_us", "store_us", "finish_us")},
        "new_requests_per_s": round(batch / med(t_new)),
        "old_requests_per_s": round(batch / med(t_old)),
        "responses_compared": batch * len(batches), "response_mismatches": mism,
    }
    for _, e, svc, api in sides:
        api.close()
        svc.close()
        e.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,4096,32768,65536")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16, help="CPU workers of plan / finish")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rows = [one_size(int(b), a.steps, a.warmup, a.threads, h) for b in a.batches.split(",") for h in ("off", "on")]
    res = {"card": card(), "nproc": os.cpu_count(), "rows": rows,
           "note": "old = CPU plan -> rl_check_and_update_batch per run (RL_MEM_HOST, through the Python binding) -> CPU finish"}
    text = json.dumps(res)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    assert all(r["response_mismatches"] == 0 for r in rows), "the two paths answered differently"


if __name__ == "__main__":
    main()
