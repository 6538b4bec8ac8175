"""Requests per second of RLS serving on a namespace-sharded store (rl_shard_batch + rl_rls_serve_sharded's phases), at
world 1, 2 and 4 on one GPU: `world` engines and services in this process, every step = every rank's send, then every
decide, then every collect.  Each rank serves a batch of --batch ShouldRateLimit requests (draft-03 headers) over
--namespaces namespaces.  Prints one line per world and the device it ran on.  Across GPUs the deployment is one process
per GPU joined by CUDA IPC (tests/test_zzh_shard_serve_gpu.py runs it); this tool does not time that case.

    python tools/shard_serve_time.py [--batch 512] [--steps 50] [--warmup 5]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from limitador_b200 import Engine, ShardBatch  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from limitador_b200 import rls as R  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--namespaces", type=int, default=64)
    ap.add_argument("--worlds", default="1,2,4")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("shard_serve_time: no GPU: nothing measured")
    print(f"device: {torch.cuda.get_device_name(0)}")
    limits = [l for k in range(a.namespaces) for l in (
        (f"ns{k}", 50, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], f"get-{k}"),
        (f"ns{k}", 500, 60, [], [], None))]
    rng = np.random.default_rng(1)
    cap = (a.batch + 15) // 16 * 16
    for world in [int(w) for w in a.worlds.split(",")]:
        ranks = []
        for r in range(world):
            m = MT.Matcher()
            e = Engine(capacity_rows=1 << 16, cells_per_row=3, max_batch=world * cap, max_counters=world * cap * 4)
            e.limits_set(np.array([m.add_limit(*l) for l in limits]))
            svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 4)
            ranks.append((m, e, svc, ShardBatch(e, r, world, cap, cap * 4)))
        for _, _, svc, sb in ranks:
            sb.connect_ptrs([x[3].slab for x in ranks])
            svc.attach_shard(sb)
        batches = []
        for _ in range(4):
            msgs = [R.encode_request(f"ns{int(rng.integers(0, a.namespaces))}",
                                     [[("method", "GET"), ("user", f"u{int(rng.integers(0, 1000))}")]], 1) for _ in range(a.batch)]
            batches.append(R.pack_requests(msgs))
        t0 = 0.0
        for step in range(a.warmup + a.steps):
            if step == a.warmup:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            now = 1_700_000_000_000_000 + step * 1000
            for r, (_, _, svc, _) in enumerate(ranks):
                svc.send(R.SHOULD_RATE_LIMIT, *batches[(step + r) % 4], now)
            for _, _, svc, _ in ranks:
                svc.decide()
            for _, _, svc, _ in ranks:
                svc.collect()
        dt = time.perf_counter() - t0
        n = a.steps * world * a.batch
        print(f"world {world}: {n / dt:,.0f} requests/s ({a.steps} steps of {world} x {a.batch} requests, "
              f"{1e3 * dt / a.steps:.2f} ms per step, one GPU, one host thread)")
        for _, _, svc, sb in ranks:
            svc.attach_shard(None)
            sb.close()


if __name__ == "__main__":
    main()
