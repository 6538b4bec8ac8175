"""Time counter snapshots (rl_counters_export / rl_counters_import) on C2's and C3's tables.

For each table: fill an engine with the workload's counters (by an import), then time, with CUDA events around the
call and a final synchronise,
  export  RL_MEM_DEVICE (the scan writes the caller's device arrays) and RL_MEM_HOST (staged, copied to numpy),
  import  RL_MEM_DEVICE and RL_MEM_HOST into a fresh engine with twice the capacity.
Each call is timed `--reps` times (best and median reported) and one JSON line per measurement is printed, with
counters/s.  Usage: python tools/snapshot_time.py [--tables C2,C3] [--reps 3]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import Engine, streams  # noqa: E402
from limitador_b200.engine import MEM_DEVICE, MEM_HOST  # noqa: E402

T0 = streams.T0_US


def table_counters(name):
    """(workload, the five counter columns) of a full C2 (1M rows x 4 counters) or C3 (16M counters) table."""
    if name == "C2":
        w = streams.WORKLOADS["C2"]()
        n_rows, n_ns = 1_000_000, 64
        rank = np.repeat(np.arange(n_rows, dtype=np.uint64), 4)
        k = np.tile(np.arange(4, dtype=np.uint64), n_rows)
        lid = ((rank % np.uint64(n_ns)) * np.uint64(4) + k).astype(np.uint32)
        key_lo = streams._mix(rank + np.uint64(1))
    else:
        w = streams.WORKLOADS["C3"]()
        n = 16_000_000
        lid = np.zeros(n, dtype=np.uint32)
        key_lo = streams._mix(np.arange(1, n + 1, dtype=np.uint64))
    n = len(lid)
    win = w.limits["window_us"][lid].astype(np.uint64)
    return w, [lid, key_lo, np.zeros(n, np.uint64), (np.arange(n, dtype=np.uint64) % np.uint64(5)) + np.uint64(1),
               np.uint64(T0) + win]


def timed(fn, reps):
    import time

    import torch
    ms, wall = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t) * 1e3)
        ms.append(a.elapsed_time(b))
    return min(ms), float(np.median(ms)), float(np.median(wall))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", default="C2,C3")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
    for name in args.tables.split(","):
        w, cols = table_counters(name)
        n = len(cols[0])
        src = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=65536)
        src.limits_set(w.limits)
        src.import_counters(*cols)
        L, h = src._lib, src._h
        cnt = C.c_uint64(0)
        d_out = [torch.empty(n, dtype=torch.int32, device=dev)] + [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(4)]
        h_out = [np.zeros(n, np.uint32)] + [np.zeros(n, np.uint64) for _ in range(4)]

        def export(mem, outs):
            ptrs = [C.c_void_p(o.data_ptr()) if mem == MEM_DEVICE else o.ctypes.data_as(C.c_void_p) for o in outs]
            src._check(L.rl_counters_export(h, None, 0, 0, n, mem, *ptrs, C.byref(cnt)))
            assert cnt.value == n, (cnt.value, n)

        results = []
        for label, mem, outs in (("export device", MEM_DEVICE, d_out), ("export host", MEM_HOST, h_out)):
            results.append((label, timed(lambda: export(mem, outs), args.reps)))
        for label, data in (("import device", d_out), ("import host", h_out)):
            dsts = []

            def imp():
                dst = Engine(capacity_rows=2 * w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=65536)
                dst.limits_set(w.limits)
                dsts.append(dst)
                torch.cuda.synchronize()
                return dst

            ms = []
            for _ in range(args.reps):  # a fresh target per repetition; its creation is not timed
                dst = imp()
                ms.append(timed(lambda: dst.import_counters(*data), 1))
                del dsts[:]
                dst.close()
            results.append((label, (min(m[0] for m in ms), float(np.median([m[1] for m in ms])), float(np.median([m[2] for m in ms])))))
        for label, (best, med, wall) in results:
            print(json.dumps({"table": name, "counters": n, "call": label, "best_ms": round(best, 3),
                              "median_ms": round(med, 3), "median_wall_ms": round(wall, 3),
                              "counters_per_s_best": round(n / (best / 1e3)), "target_capacity_rows": 2 * w.capacity_rows
                              if label.startswith("import") else w.capacity_rows}))
        src.close()


if __name__ == "__main__":
    main()
