#!/usr/bin/env python
"""Device-side breakdown of bench.py's C2 step: where the ~30 us of a 65536-request step go.

Runs C2 the way bench.py does (same generator and seed, 64 namespaces x 4 limits, 1 M keys Zipf(1.1), a 2^21-row
table of 7-cell rows, RL_FLAG_PIPELINE, the batch resident in HBM, one dedicated stream), three passes over the same
number of steps after the same warm-up:
  plain   no accounting: step time from CUDA events (what bench.py's `value` measures);
  trace   RL_FLAG_TRACE: per step the start / end of k_front and k_main on the GPU's nanosecond timer, whether
          k_front(s+1) overlaps k_main(s) and for how long, and the distribution of k_main's duration;
  kstats  RL_FLAG_KERNEL_STATS: k_main's chunks, replay rounds, chained and ordered chunks per batch, and the SM
          cycles of its phases per chunk (thread 0's clock64, summed over chunks).
Writes <out>/step_breakdown.json (with the card's name and power limit, read in the same run) and prints a summary.
The library is the in-tree build, or RL_ENGINE_LIB.
Usage: python tools/step_breakdown.py --out DIR [--steps 200] [--warmup 20] [--tag NAME]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")  # as bench.py
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BATCH = 65536
FLAG_PIPELINE, FLAG_KERNEL_STATS, FLAG_TRACE = 2, 4, 8
# k_main's RL_PHASE_TICK boundaries (rl_kernels.cuh); the rep's row-state staging is counted in the first
PHASES = ["item+gather+grouping", "(unused)", "ordinals", "replay rounds", "chained protocol", "write-back"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:  # no nvidia-smi: say so rather than guess
        return {"name": "unknown", "power_limit": "unknown", "error": str(ex)}


def pct(v, qs=(0, 10, 50, 90, 99, 100)):
    v = np.asarray(v, dtype=np.float64)
    return {f"p{q}": round(float(np.percentile(v, q)), 3) for q in qs} | {"mean": round(float(v.mean()), 3)}


def run_pass(flags, recs, steps, warmup, dev):
    """One engine over warmup + steps batches; returns (ms per step, stats delta, trace events or None)."""
    import torch
    from limitador_b200 import Engine, streams
    from limitador_b200.engine import MEM_DEVICE

    limits = streams.c2_zipf_4limits(batch=1, n_rows=1000, n_ns=64).limits
    eng = Engine(capacity_rows=1 << 21, cells_per_row=7, max_batch=BATCH, max_counters=BATCH, device=dev.index or 0,
                 flags=FLAG_PIPELINE | flags)
    try:
        eng.limits_set(limits)
        torch.cuda.synchronize()
        stream = torch.cuda.Stream(device=dev)
        torch.cuda.set_stream(stream)
        eng.set_stream(stream.cuda_stream)
        out_lim = torch.zeros((warmup + steps, BATCH), dtype=torch.uint8, device=dev)
        out_first = torch.zeros((warmup + steps, BATCH), dtype=torch.int32, device=dev)

        def step(s):
            eng.check_and_update_records_ptr(BATCH, recs[s].data_ptr(), out_lim[s].data_ptr(), MEM_DEVICE,
                                             out_first_ptr=out_first[s].data_ptr(), stride=7)

        for s in range(warmup):
            step(s)
        eng.sync()
        torch.cuda.synchronize()
        if flags & FLAG_TRACE:
            eng.trace_dump()  # clear the ring
        st0 = eng.stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for s in range(warmup, warmup + steps):
            step(s)
        eng.fence()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        st1 = eng.stats()
        delta = {k: (st1[k] - st0[k]) if not isinstance(st1[k], list) else [a - b for a, b in zip(st1[k], st0[k])]
                 for k in ("batches", "chunks", "replay_rounds", "chained_chunks", "ordered_chunks", "phase_cycles")}
        ev = eng.trace_dump() if flags & FLAG_TRACE else None
        torch.cuda.set_stream(torch.cuda.default_stream(dev))
        return ms, delta, ev
    finally:
        eng.close()


def trace_summary(ev):
    steps = {}
    for name, end, seq, ns in ev:
        steps.setdefault(seq, {})[(name, end)] = ns
    seqs = sorted(s for s in steps if all(k in steps[s] for k in (("front", 0), ("front", 1), ("main", 0), ("main", 1))))
    t0 = steps[seqs[0]][("front", 0)]
    per_step, main_us, front_us, overlap_us, gap_us = [], [], [], [], []
    for s in seqs:
        d = steps[s]
        row = {"seq": s, **{f"{n}_{'end' if e else 'start'}_us": round((d[(n, e)] - t0) / 1e3, 3)
                            for n in ("front", "main") for e in (0, 1)}}
        main_us.append((d[("main", 1)] - d[("main", 0)]) / 1e3)
        front_us.append((d[("front", 1)] - d[("front", 0)]) / 1e3)
        nxt = steps.get(s + 1)
        if nxt is not None and s + 1 in seqs:
            # k_front(s+1) against k_main(s): the length of the intersection of the two intervals
            ov = min(d[("main", 1)], nxt[("front", 1)]) - max(d[("main", 0)], nxt[("front", 0)])
            row["next_front_overlap_us"] = round(max(ov, 0) / 1e3, 3)
            overlap_us.append(max(ov, 0) / 1e3)
            gap_us.append((nxt[("main", 0)] - d[("main", 1)]) / 1e3)
        per_step.append(row)
    return {
        "steps": len(seqs),
        "k_main_us": pct(main_us),
        "k_front_us": pct(front_us),
        "next_front_overlaps_main": {"steps": int(sum(1 for o in overlap_us if o > 0)), "of": len(overlap_us),
                                     "overlap_us": pct(overlap_us) if overlap_us else None},
        "main_end_to_next_main_start_us": pct(gap_us) if gap_us else None,
        "per_step": per_step,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for step_breakdown.json")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--tag", default="", help="name of the build under test (written into the JSON)")
    args = ap.parse_args()
    if args.steps < 200:
        ap.error("--steps: at least 200 timed steps")

    import torch
    from limitador_b200 import engine as _eng, streams

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = args.warmup + args.steps
    recs = streams.c2_device_stream(n, BATCH, dev, n_rows=1_000_000, n_ns=64, first_batch=0, seed=streams.SEED)
    torch.cuda.synchronize()
    res = {"tag": args.tag, "library": os.environ.get("RL_ENGINE_LIB") or _eng._build.LIB_PATH, "card": card(),
           "batch": BATCH, "steps": args.steps, "warmup": args.warmup,
           "sm_count": torch.cuda.get_device_properties(dev).multi_processor_count}

    ms, _, _ = run_pass(0, recs, args.steps, args.warmup, dev)
    res["plain"] = {"us_per_step": round(ms * 1e3, 3), "decisions_per_s": round(BATCH / (ms * 1e-3))}

    ms, _, ev = run_pass(FLAG_TRACE, recs, args.steps, args.warmup, dev)
    res["trace"] = {"us_per_step": round(ms * 1e3, 3), **trace_summary(ev)}

    ms, st, _ = run_pass(FLAG_KERNEL_STATS, recs, args.steps, args.warmup, dev)
    nb = max(st["batches"], 1)
    ch = max(st["chunks"], 1)
    res["kstats"] = {
        "us_per_step": round(ms * 1e3, 3),
        "batches": st["batches"],
        "per_batch": {k: round(st[k] / nb, 2) for k in ("chunks", "replay_rounds", "chained_chunks", "ordered_chunks")},
        "phase_cycles_per_chunk": {PHASES[i]: round(c / ch, 1) for i, c in enumerate(st["phase_cycles"]) if i != 1},
    }

    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "step_breakdown.json"), "w") as f:
        json.dump(res, f, indent=1)
    t = res["trace"]
    ov = t["next_front_overlaps_main"]
    print(f"[{args.tag or 'build'}] {res['card']['name']} @ {res['card']['power_limit']}: "
          f"plain {res['plain']['us_per_step']} us/step | k_main p10/p50/p90 {t['k_main_us']['p10']}/"
          f"{t['k_main_us']['p50']}/{t['k_main_us']['p90']} us, k_front p50 {t['k_front_us']['p50']} us | "
          f"front(s+1) overlaps main(s) in {ov['steps']}/{ov['of']} steps"
          + (f", p50 {ov['overlap_us']['p50']} us" if ov["overlap_us"] else "")
          + f" | chunks/batch {res['kstats']['per_batch']['chunks']}, chained {res['kstats']['per_batch']['chained_chunks']},"
          f" ordered {res['kstats']['per_batch']['ordered_chunks']} | cycles/chunk {res['kstats']['phase_cycles_per_chunk']}")


if __name__ == "__main__":
    main()
