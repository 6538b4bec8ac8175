"""What carrying the counter variables through a snapshot costs: RlsService.export_counter_vars and
import_counter_vars (rl_rls_counter_vars_export / _import) at 64 K and 1 M qualified keys.

  python tools/counter_vars_snapshot_time.py [--reps 5]

One service records the keys (HTTP /report batches of 65 536 bodies, one variable per key), then each rep exports the
dictionary, and imports that export into an empty dictionary of a second service (a fresh one per rep, so that every key
is new).  Each call is timed with CUDA events on the current stream around it, after a final device synchronise, and
with the host clock; both calls synchronise before they return.  Prints the card and its power limit beside the numbers,
and one JSON line.
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
LIMIT = ("big", 10 ** 9, 3600, [], ["descriptors[0].user"], None)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        watts = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).split("\n")[0]
    except Exception:  # noqa: BLE001
        watts = "unknown"
    return name, watts.strip()


def service(keys):
    m = MT.Matcher()
    d = m.add_limit(*LIMIT)
    e = Engine(capacity_rows=2 * keys, cells_per_row=1, max_batch=1 << 17)  # a row per key, half the rows free
    e.limits_set(np.array([d]))
    s = R.RlsService(m, e, R.HEADERS_NONE, 0)
    s.keep_counter_vars(2 * keys, 32 * keys)
    return m, e, s


def timed(fn):
    import torch
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = time.perf_counter()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b), (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    name, watts = card()
    print(f"card: {name}, power limit {watts}")
    res = {"card": name, "power_limit": watts}
    for keys in (1 << 16, 1 << 20):
        m, e, s = service(keys)
        api = HA.HttpApi(s)
        for lo in range(0, keys, 1 << 16):
            bodies = [b'{"namespace":"big","values":{"user":"u%07d"},"delta":1}' % k for k in range(lo, min(keys, lo + (1 << 16)))]
            api.serve(HA.REPORT, *HA.pack_bodies(bodies), T0)
        assert s.counter_vars_stats()["keys"] == keys
        exp, imp = [], []
        for _ in range(args.reps + 1):  # the first rep warms up
            cv, ev, host = timed(lambda: s.export_counter_vars(T0 + 1))
            assert len(cv[0]) == keys
            exp.append((ev, host))
            _, _, t = service(keys)
            added, ev, host = timed(lambda: t.import_counter_vars(*cv))
            assert added == keys
            imp.append((ev, host))
            t.close()
        for label, xs in (("export", exp[1:]), ("import", imp[1:])):
            ev = sorted(x[0] for x in xs)
            host = sorted(x[1] for x in xs)
            print(f"{keys:>8} keys {label}: median {ev[len(ev) // 2]:.2f} ms (events), {host[len(host) // 2]:.2f} ms (host); "
                  f"min {ev[0]:.2f} max {ev[-1]:.2f}")
            res[f"{label}_{keys}_ms"] = ev[len(ev) // 2]
        s.close()
        del api, e, m
    print(json.dumps(res))


if __name__ == "__main__":
    main()
