"""Time the counter journal (limitador_b200/journal.py) on C2's table: about 1 M live rows (4 M counters) under C2's
Zipf(1.1) traffic in batches of 65536.

  full     a checkpoint: the full drain and the base written (fsynced)
  every N  drains after every N = 1, 8 and 64 batches: time per drain (the device scan, the host copy and the fsynced
           record) and bytes per drain
  recover  recover() of a journal of one base and 64 records into a fresh engine
  serve    per-batch time of check_and_update_records with tracking off, and with tracking on and a drain after every
           batch (serve and drain timed apart), in alternating blocks of 8 batches
Host clocks around calls that end in a device synchronise.  One JSON line per measurement, then the card.  Usage:
python tools/journal_time.py [--dir DIR] [--blocks 3]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import Engine, streams  # noqa: E402
from limitador_b200 import journal as J  # noqa: E402

T0 = streams.T0_US


def c2_engine(w):
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch)
    e.limits_set(w.limits)
    # every one of the 1 M rows present, as after a long run of the stream
    n_rows, n_ns = 1_000_000, 64
    rank = np.repeat(np.arange(n_rows, dtype=np.uint64), 4)
    k = np.tile(np.arange(4, dtype=np.uint64), n_rows)
    lid = ((rank % np.uint64(n_ns)) * np.uint64(4) + k).astype(np.uint32)
    n = len(lid)
    win = w.limits["window_us"][lid].astype(np.uint64)
    e.import_counters(lid, streams._mix(rank + np.uint64(1)), np.zeros(n, np.uint64),
                      (np.arange(n, dtype=np.uint64) % np.uint64(5)) + np.uint64(1), np.uint64(T0) + win)
    return e


def clock(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="journal directory (default: a temporary one)")
    ap.add_argument("--blocks", type=int, default=3)
    args = ap.parse_args()
    root = args.dir or tempfile.mkdtemp(prefix="rl_journal_")
    w = streams.WORKLOADS["C2"]()
    e = c2_engine(w)
    batches = iter(range(10 ** 9))

    def serve():
        e.check_and_update_records(w.batch_records(next(batches)), want_first=False)

    for _ in range(3):
        serve()
    live = len(e.export_counters()[0])
    jdir = os.path.join(root, "j")
    jr = J.CounterJournal(e, jdir)
    ms, r = clock(jr.checkpoint)
    emit(what="full", ms=round(ms, 2), counters=live, bytes=r["bytes"])
    for every in (1, 8, 64):
        rounds = max(2, 16 // every)
        times, sizes, entries = [], [], []
        for _ in range(rounds):
            for _ in range(every):
                serve()
            ms, r = clock(jr.drain)
            assert not r["full"]
            times.append(ms)
            sizes.append(r["bytes"])
            entries.append(r["counters"])
        emit(what="drain", every_batches=every, drains=rounds, ms_median=round(float(np.median(times)), 3),
             ms_min=round(min(times), 3), bytes_median=int(np.median(sizes)), counters_median=int(np.median(entries)))
    # a journal of one base and 64 records
    jr.checkpoint()
    for _ in range(64):
        serve()
        jr.drain()
    copy = os.path.join(root, "copy")
    shutil.copytree(jdir, copy)
    f = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch)
    f.limits_set(w.limits)
    ms, info = clock(lambda: J.recover(copy, f))
    emit(what="recover", ms=round(ms, 1), records=info["records"], counters=info["counters"],
         bytes=sum(os.path.getsize(os.path.join(copy, x)) for x in os.listdir(copy)))
    f.close()
    jr.close()
    # serve time: tracking off, then on with a drain after every batch, alternating
    off, on, dr = [], [], []
    for _ in range(args.blocks):
        e.track_changes(False)
        for _ in range(8):
            off.append(clock(serve)[0])
        jr = J.CounterJournal(e, jdir)
        jr.checkpoint()
        for _ in range(8):
            on.append(clock(serve)[0])
            dr.append(clock(jr.drain)[0])
        jr.close()
    emit(what="serve", batch=w.batch, off_ms_median=round(float(np.median(off)), 3),
         on_ms_median=round(float(np.median(on)), 3), drain_ms_median=round(float(np.median(dr)), 3), batches_each=len(off))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    emit(what="card", card=card)
    if args.dir is None:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
