"""What a reload costs: RlsService.configure_with (rl_rls_configure) keeping 90 % of 1 000 limits and replacing the other
100, on an engine holding about 1 M live counters, and the first serve after it (which uploads the new match image).

  python tools/configure_time.py [--reps 5]

1 000 qualified limits in 100 namespaces (10 each, one variable, no condition).  HTTP /report batches of 65 536 bodies
(one new user per body) fill the table until it holds 1 M counters.  Each rep then alternates between the two sets of
limits (set A, and A with 100 limits replaced), so every reload deletes 100 limits with their counters, adds 100 and keeps
900, and serves one RLS batch of 65 536 requests right after it and a second one for comparison.  Every timing is a host
clock around a call that ends in a device synchronise.  Prints the card and its power limit beside the numbers, and one
JSON line.
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
N_NS, PER_NS, BATCH, COUNTERS = 100, 10, 65536, 1 << 20


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        watts = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0]
    except Exception:  # noqa: BLE001
        watts = "unknown"
    return name, watts.strip()


def limits(shift):
    """1 000 limits; the last limit of every namespace has another window when shift is set (100 replaced)."""
    out = []
    for k in range(N_NS):
        for j in range(PER_NS):
            secs = 3600 + j + (1000 if shift and j == PER_NS - 1 else 0)
            out.append({"namespace": f"ns{k}", "max_value": 10 ** 9, "seconds": secs, "conditions": [],
                        "variables": ["descriptors[0].user"], "name": None, "id": None})
    return out


def synced(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("configure_time needs a GPU: there is nothing to measure on the CPU")
    m = MT.Matcher()
    e = Engine(capacity_rows=1 << 21, cells_per_row=3, max_batch=BATCH, max_counters=BATCH * PER_NS)
    s = R.RlsService(m, e, R.HEADERS_NONE, 0)
    api = HA.HttpApi(s)
    sets = [limits(False), limits(True)]
    s.configure_with(sets[0])
    print("engine ready, filling the table", flush=True)
    rng = np.random.default_rng(0)
    users, now = 0, T0
    t0 = time.perf_counter()
    live = 0
    for _ in range(8):  # each batch adds about 655 360 counters
        ns = rng.integers(0, N_NS, BATCH)
        bodies = [HA.encode_info(f"ns{k}", {"user": f"u{users + i}"}, 1) for i, k in enumerate(ns)]
        api.serve(HA.REPORT, *HA.pack_bodies(bodies), now)
        assert all(st == 200 for st, _, _ in api.responses()), "a /report batch was refused"
        users += BATCH
        live = len(e.export_counters()[0])
        print(f"filled: {live} counters after {time.perf_counter() - t0:.1f} s", flush=True)
        if live >= COUNTERS:
            break
    reqs = R.pack_requests([R.encode_request(f"ns{k}", [[("user", f"u{int(u)}")]], 1)
                            for k, u in zip(rng.integers(0, N_NS, BATCH), rng.integers(0, users, BATCH))])
    def serve():
        s.serve(R.SHOULD_RATE_LIMIT, *reqs, now)
        assert not s.grpc_status().any(), "a ShouldRateLimit batch was refused"

    serve()  # warm the serve path
    rows = []
    for rep in range(2 * args.reps):
        target = sets[(rep + 1) % 2]
        ms_cfg, report = synced(lambda: s.configure_with(target))
        assert (report["kept"], report["added"], report["deleted"]) == (900, 100, 100), report
        ms_first, _ = synced(serve)
        ms_next, _ = synced(serve)
        rows.append((ms_cfg, ms_first, ms_next, len(e.export_counters()[0])))
        print(f"reload {rep}: configure {ms_cfg:.2f} ms, first serve {ms_first:.2f} ms, next {ms_next:.2f} ms", flush=True)
    name, watts = card()
    cfg, first, nxt = (np.array([r[i] for r in rows]) for i in range(3))
    print(f"{name}, power limit {watts}; {live} live counters before the first reload, {len(rows)} reloads")
    print(f"configure_with (900 kept, 100 added, 100 deleted): median {np.median(cfg):.2f} ms, min {cfg.min():.2f}, max {cfg.max():.2f}")
    print(f"first serve after it ({BATCH} RLS requests): median {np.median(first):.2f} ms; the serve after that: "
          f"median {np.median(nxt):.2f} ms")
    print(json.dumps({"card": name, "power_limit": watts, "live_counters": live, "reloads": len(rows),
                      "configure_ms": [round(x, 3) for x in cfg], "first_serve_ms": [round(x, 3) for x in first],
                      "next_serve_ms": [round(x, 3) for x in nxt], "counters_after": [r[3] for r in rows]}))


if __name__ == "__main__":
    main()
