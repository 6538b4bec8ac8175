"""What keeping counter variables costs (RlsService.keep_counter_vars) and what GET /counters takes.

  python tools/counter_vars_time.py [--reps 20]

Serve: rl_http_serve and rl_rls_serve at 4 096 and 65 536 requests, keeping off and on, on two services of their own
engines that are called alternately (off, on, off, on, ...), each in the steady state (every key already recorded) and
with a cold batch (every key new).  GET /counters: one namespace with about 10^4 and about 10^6 counters.  Prints the
card and its power limit beside the numbers, and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import Engine  # noqa: E402
from limitador_b200 import http_api as HA  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from limitador_b200 import rls as R  # noqa: E402

T0 = 1_700_000_000_000_000
LIMITS = [("api", 10 ** 9, 3600, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"),
          ("api", 10 ** 9, 3600, [], ["descriptors[0].user", "descriptors[0].path"], None),
          ("api", 10 ** 12, 60, [], [], "global")]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        watts = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0]
    except Exception:  # noqa: BLE001
        watts = "unknown"
    return name, watts.strip()


def service(keep, rows=1 << 21):
    m = MT.Matcher()
    e = Engine(capacity_rows=rows, cells_per_row=3, max_batch=1 << 17)
    e.limits_set(np.array([m.add_limit(*l) for l in LIMITS]))
    s = R.RlsService(m, e, R.HEADERS_NONE, 0)
    if keep:
        s.keep_counter_vars(1 << 22, 1 << 28)
    return m, e, s, HA.HttpApi(s)


def http_batch(n, tag):
    return HA.pack_bodies([HA.encode_info("api", {"method": "GET", "user": f"{tag}u{k}", "path": f"/p{k % 7}"}, 1) for k in range(n)])


def rls_batch(n, tag):
    return R.pack_requests([R.encode_request("api", [[("method", "GET"), ("user", f"{tag}u{k}"), ("path", f"/p{k % 7}")]])
                            for k in range(n)])


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    name, watts = card()
    print(f"# {name}, power limit {watts}")
    svc = {False: service(False), True: service(True)}
    out = {"card": name, "power_limit": watts, "serve_ms": {}, "get_counters_ms": {}}
    now = T0
    for surface in ("http", "rls"):
        for n in (4096, 65536):
            for mode in ("steady", "cold"):
                ts = {False: [], True: []}
                warm = (http_batch if surface == "http" else rls_batch)(n, f"w{n}")
                for keep in (False, True):  # the steady batch's keys recorded once before timing
                    _, _, s, api = svc[keep]
                    (api.serve(HA.CHECK_AND_REPORT, *warm, now) if surface == "http" else s.serve(R.SHOULD_RATE_LIMIT, *warm, now))
                for rep in range(a.reps):
                    batch = warm if mode == "steady" else (http_batch if surface == "http" else rls_batch)(n, f"c{n}{surface}{rep}")
                    now += 1000
                    for keep in (False, True):
                        _, _, s, api = svc[keep]
                        if surface == "http":
                            ts[keep].append(timed(lambda: api.serve(HA.CHECK_AND_REPORT, *batch, now)))
                        else:
                            ts[keep].append(timed(lambda: s.serve(R.SHOULD_RATE_LIMIT, *batch, now)))
                off, on = float(np.median(ts[False][2:])), float(np.median(ts[True][2:]))
                key = f"{surface}_{n}_{mode}"
                out["serve_ms"][key] = {"off": round(off, 3), "on": round(on, 3), "overhead_pct": round(100 * (on - off) / off, 1)}
                print(f"serve {surface:4s} {n:6d} {mode:6s}  off {off:8.3f} ms  on {on:8.3f} ms  ({100 * (on - off) / off:+.1f}%)")
    # GET /counters over ~10^4 and ~10^6 counters (two qualified limits per user + one global)
    for users in (5_000, 500_000):
        m, e, s, api = service(True)
        for k in range(0, users, 65536):
            s.serve(R.SHOULD_RATE_LIMIT, *rls_batch(min(65536, users - k), f"g{k}"), T0)
        ts = []
        for _ in range(max(3, a.reps // 4)):
            ts.append(timed(lambda: api.get_counters("api", T0 + 1)))
        status, body = api.get_counters("api", T0 + 1)
        n_ctr = body.count(b'"limit":')
        med = float(np.median(ts))
        out["get_counters_ms"][str(n_ctr)] = {"ms": round(med, 3), "status": status, "body_bytes": len(body)}
        print(f"GET /counters  {n_ctr:8d} counters  {med:9.3f} ms  (status {status}, {len(body) / 1e6:.1f} MB)")
        del api, s, e, m
    print(json.dumps(out))


if __name__ == "__main__":
    main()
