"""Time rl_rls_serve and rl_http_serve with limits in the matcher's boolean dialect against the same namespaces with
==-only conditions.

Two limit sets over rls_time.py's stream shape (32 namespaces, one descriptor (method, user, path) per request, users
drawn Zipf(1.1)):
  eq       rls_time.py's set: GET per user, hourly per user, a global limit with != OPTIONS;
  boolean  the same namespaces with `method in ['GET', 'HEAD']` per user, a `path.startsWith('/api/') && path !=
           '/api/health'` group per user, and a global limit on `has(descriptors[0].user)`.
For each set and batch size, the device path (rl_rls_serve / rl_http_serve: device plan -> one store call -> CPU finish,
stage times from the service) and the CPU composition (CPU plan -> rl_check_and_update_batch from host arrays -> CPU finish)
run alternately, batch by batch, on two engines that see the same requests, and their responses are compared for every
batch.  Times are medians over the timed batches.  Prints one JSON object with the card's name and power limit.
Usage: python tools/conditions_time.py [--batches 64,4096,65536] [--sets eq,boolean] [--steps 20] [--threads 0]
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

N_NS, N_USERS = 32, 200_000


def limit_set(name):
    limits = []
    for ns in range(N_NS):
        if name == "eq":
            limits.append((f"ns{ns}", 100, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"))
            limits.append((f"ns{ns}", 1000, 3600, [], ["descriptors[0].user"], "hourly-per-user"))
            limits.append((f"ns{ns}", 1 << 40, 60, ["descriptors[0].method != 'OPTIONS'"], [], None))
        else:
            limits.append((f"ns{ns}", 100, 60, ["descriptors[0].method in ['GET', 'HEAD']"], ["descriptors[0].user"], "read-per-user"))
            limits.append((f"ns{ns}", 1000, 3600, ["descriptors[0].path.startsWith('/api/') && descriptors[0].path != '/api/health'"],
                           ["descriptors[0].user"], "api-per-user"))
            limits.append((f"ns{ns}", 1 << 40, 60, ["has(descriptors[0].user)"], [], None))
    return limits


def stream(batch, steps, seed=42):
    """-> per step, (namespace, [(key, value)]) of every request"""
    rng = np.random.default_rng(seed)
    methods = ["GET", "GET", "GET", "HEAD", "POST", "OPTIONS"]
    paths = ["/api/v1/items", "/api/health", "/static/a.css", "/api/", "/"]
    zipf = rng.zipf(1.1, size=steps * batch) % N_USERS
    out = []
    for s in range(steps):
        u = zipf[s * batch:(s + 1) * batch]
        ns = rng.integers(0, N_NS, size=batch)
        me = rng.integers(0, len(methods), size=batch)
        pa = rng.integers(0, len(paths), size=batch)
        out.append([(f"ns{ns[i]}", [("method", methods[me[i]]), ("user", f"u{u[i]}"), ("path", paths[pa[i]])]) for i in range(batch)])
    return out


def _sides(limits, dialect, batch, threads):
    sides = []
    for _ in range(2):
        m = MT.Matcher() if dialect == "table" else MT.Matcher(dialect=dialect)
        e = Engine(capacity_rows=1 << 20, cells_per_row=3, max_batch=batch, max_counters=4 * batch)
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
        svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, threads)
        sides.append((e, svc, HA.HttpApi(svc)))
    return sides


def _row(surface, set_name, batch, steps, t_new, t_old, st_new, st_old, mism, n):
    med = lambda xs: float(np.median(xs))  # noqa: E731
    keys = ("plan_us", "store_us", "finish_us")
    return {"surface": surface, "limits": set_name, "batch": batch, "steps": steps,
            "new_ms_per_batch": round(med(t_new) * 1e3, 3),
            "new_stage_ms": {k[:-3]: round(med([t[k] for t in st_new]) / 1e3, 3) for k in keys},
            "cpu_ms_per_batch": round(med(t_old) * 1e3, 3),
            "cpu_stage_ms": {k[:-3]: round(med([t[k] for t in st_old]) / 1e3, 3) for k in keys},
            "responses_compared": n, "response_mismatches": mism}


def one(set_name, batch, steps, warmup, threads, dialect):
    limits = limit_set(set_name)
    reqs = stream(batch, steps + warmup)
    rows = []
    # RLS: ShouldRateLimit with draft-03 headers
    (_, new, _), (e_old, old, _) = _sides(limits, dialect, batch, threads)
    t_new, t_old, st_new, st_old, mism = [], [], [], [], 0
    for s, rq in enumerate(reqs):
        buf, off = R.pack_requests([R.encode_request(ns, [d], 1) for ns, d in rq])
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
        mism += sum(1 for x, y in zip(got, old.responses()) if x != y)
        if s >= warmup:
            t_new.append(b - a)
            t_old.append(g - c)
            st_new.append(new.timings())
            st_old.append({"plan_us": (d - c) * 1e6, "store_us": (f - d) * 1e6, "finish_us": (g - f) * 1e6})
    rows.append(_row("rls", set_name, batch, steps, t_new, t_old, st_new, st_old, mism, batch * len(reqs)))
    # HTTP: /check_and_report with draft-03 headers (one store call per batch)
    (_, _, new), (e_old, _, old) = _sides(limits, dialect, batch, threads)
    t_new, t_old, st_new, st_old, mism = [], [], [], [], 0
    for s, rq in enumerate(reqs):
        buf, off = HA.pack_bodies([HA.encode_info(ns, dict(d), 1, "DraftVersion03") for ns, d in rq])
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
        mism += sum(1 for x, y in zip(got, old.responses()) if x != y)
        if s >= warmup:
            t_new.append(b - a)
            t_old.append(g - c)
            st_new.append(new.timings())
            st_old.append({"plan_us": (d - c) * 1e6, "store_us": (f - d) * 1e6, "finish_us": (g - f) * 1e6})
    rows.append(_row("http", set_name, batch, steps, t_new, t_old, st_new, st_old, mism, batch * len(reqs)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,4096,65536")
    ap.add_argument("--sets", default="eq,boolean")
    ap.add_argument("--dialect", default="boolean", help="dialect of the matchers (the eq set also parses in 'table')")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--threads", type=int, default=0, help="CPU workers of plan / finish (0 = one per CPU, at most 64)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    threads = a.threads or min(os.cpu_count() or 1, 64)
    rows = []
    for s in a.sets.split(","):
        for b in a.batches.split(","):
            for r in one(s, int(b), a.steps, a.warmup, threads, a.dialect):
                print(json.dumps(r), file=sys.stderr, flush=True)  # progress: a row as soon as it is measured
                rows.append(r)
    res = {"card": card(), "nproc": os.cpu_count(), "threads": threads, "dialect": a.dialect, "rows": rows,
           "note": "new = rl_*_serve (device plan); cpu = CPU plan -> rl_check_and_update_batch (host arrays) -> CPU finish"}
    text = json.dumps(res)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
