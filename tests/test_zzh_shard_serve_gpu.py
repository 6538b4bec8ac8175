"""RLS and HTTP serving on a namespace-sharded store (rl_shard_batch, rl_rls_serve_sharded / rl_http_serve_sharded) on
the GPU: world engines on one H100, joined with connect_ptrs, each with its own matcher and service.  Every step is
checked against the same rank batches served one after another, in rank order, through one unsharded service on one
engine: byte-identical responses, equal metric sums, and the union of the owners' tables equal to the one table."""
import re
import subprocess

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R

T0 = 1_700_000_000_000_000
N_NS = 8
CAP_REQ, CAP_CTR = 512, 2048
LIMITS = [l for k in range(N_NS) for l in (
    (f"ns{k}", 4 + k, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], f"get-{k}"),
    (f"ns{k}", 30, 3600, [], ["descriptors[0].user"], None),
    (f"ns{k}", 60 + 5 * k, 60, ["descriptors[0].method != 'OPTIONS'"], [], f"global-{k}"),
    (f"ns{k}", 3, 10, ["descriptors[0].method == 'POST'"], ["descriptors[0].user", "descriptors[0].path"], None))]


def _stack(limits=LIMITS, headers=R.HEADERS_DRAFT_VERSION_03, device=0):
    from limitador_b200 import Engine
    m = MT.Matcher()
    e = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=4096, device=device)
    e.limits_set(np.array([m.add_limit(*l) for l in limits]))
    svc = R.RlsService(m, e, headers, 2, True)
    return m, e, svc, HA.HttpApi(svc)


def _sharded(world, limits_of=lambda r: LIMITS):
    from limitador_b200 import ShardBatch
    ranks = [_stack(limits_of(r)) for r in range(world)]
    shards = [ShardBatch(e, r, world, CAP_REQ, CAP_CTR) for r, (_, e, _, _) in enumerate(ranks)]
    for sb in shards:
        sb.connect_ptrs([s.slab for s in shards])
    for (_, _, svc, _), sb in zip(ranks, shards):
        svc.attach_shard(sb)
    return ranks, shards


def _values(rng):
    v = {"method": str(rng.choice(["GET", "GET", "POST", "OPTIONS"])), "user": f"u{int(rng.integers(0, 5))}"}
    if rng.random() < 0.6:
        v["path"] = str(rng.choice(["/a", "/b"]))
    return v


def _rls_batch(rng, n, names=None):
    """n RLS requests; names (a list, optional) receives each request's domain."""
    msgs = []
    for _ in range(n):
        ns = f"ns{int(rng.integers(0, N_NS))}" if rng.random() < 0.95 else str(rng.choice(["", "other"]))
        if names is not None:
            names.append(ns)
        msgs.append(R.encode_request(ns, [list(_values(rng).items())], int(rng.choice([0, 1, 1, 2]))))
    return R.pack_requests(msgs) if msgs else (np.zeros(0, np.uint8), np.zeros(1, np.uint64))


def _ns_ids():
    """namespace -> ns_id as every rank's matcher interns them (the same limits in the same order)"""
    m = MT.Matcher()
    return {l[0]: int(m.add_limit(*l)["ns_id"]) for l in LIMITS}


def _http_batch(rng, n):
    bodies = [HA.encode_info(f"ns{int(rng.integers(0, N_NS))}", _values(rng), int(rng.choice([0, 1, 2])),
                             [None, "DraftVersion03"][int(rng.integers(0, 2))]) for _ in range(n)]
    return HA.pack_bodies(bodies) if bodies else (np.zeros(0, np.uint8), np.zeros(1, np.uint64))


def _sizes(rng, world):
    s = [int(rng.integers(0, 300)) for _ in range(world)]
    s[int(rng.integers(0, world))] = 0  # an empty batch every step
    return s


def _metric_sums(texts):
    out = {}
    for t in texts:
        for line in t.splitlines():
            mm = re.match(r"^(\S+) (\d+)$", line)
            if mm and not line.startswith("limitador_up"):
                out[mm.group(1)] = out.get(mm.group(1), 0) + int(mm.group(2))
    return out


def _table(engines):
    """The union of the owners' tables: each engine's counters of the namespaces it owns (every rank registers every
    limit, so a rank also lists the untouched unqualified counters of namespaces it does not own)."""
    from limitador_b200 import owner_of
    rows = []
    for r, e in enumerate(engines):
        ns = [int(n) for n in np.unique(e.limits_get()["ns_id"]) if owner_of(int(n), len(engines)) == r]
        lid, lo, hi, val, exp = e.export_counters(0, ns_ids=ns)
        rows += list(zip(lid.tolist(), lo.tolist(), hi.tolist(), val.tolist(), exp.tolist()))
    return sorted(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_serving_equals_one_engine_in_rank_order(world):
    rng = np.random.default_rng(world)
    ranks, shards = _sharded(world)
    _, ref_e, ref, ref_http = _stack()
    rls_methods = [R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT]
    http_eps = [HA.CHECK_AND_REPORT, HA.CHECK, HA.REPORT]
    for step in range(12):
        http = step % 3 == 2
        sizes = _sizes(rng, world)
        batches = [(_http_batch if http else _rls_batch)(rng, n) for n in sizes]
        ops = [int(rng.integers(0, 3)) for _ in range(world)]  # RLS methods / HTTP endpoints mixed across ranks
        ops = [(http_eps if http else rls_methods)[o] for o in ops]
        # per-rank clocks, not monotone in rank order
        nows = [T0 + step * 3_000_000 + ((world - r) * 700_000 if r % 2 else r * 50_000) for r in range(world)]
        surf = [(h if http else svc) for _, _, svc, h in ranks]
        for s, op, (buf, off), now in zip(surf, ops, batches, nows):
            s.send(op, buf, off, now)
        for s in surf:
            s.decide()
        got = [s.collect() for s in surf]
        want = []
        for op, (buf, off), now in zip(ops, batches, nows):
            (ref_http if http else ref).serve(op, buf, off, now)
            want.append((ref_http if http else ref).responses())
        for r in range(world):
            assert got[r] == want[r], (step, r, http)
        t = ranks[0][3 if http else 2].timings()
        if http:
            assert t["store_calls"] <= 1  # one step per batch, however many load_counters runs
    assert _metric_sums([svc.metrics() for _, _, svc, _ in ranks]) == _metric_sums([ref.metrics()])
    assert _table([e for _, e, _, _ in ranks]) == _table([ref_e])
    for sb in shards:
        sb.close()


@pytest.mark.gpu
def test_refusals_caps_and_registry_digest():
    from limitador_b200 import Engine, EngineError, ShardBatch
    e = Engine(capacity_rows=1 << 10, cells_per_row=3, max_batch=1024)
    with pytest.raises(EngineError, match="max_batch"):
        ShardBatch(e, 0, 4, 512, 512)
    with pytest.raises(EngineError, match="max_counters"):
        ShardBatch(e, 0, 2, 512, 4096)
    rng = np.random.default_rng(5)
    world = 2
    # a source over its caps: its store requests are answered UNAVAILABLE, the other rank's are decided normally
    ranks, shards = _sharded(world)
    _, ref_e, ref, _ = _stack()
    big, small = _rls_batch(rng, CAP_REQ + 40), _rls_batch(rng, 100)
    for (_, _, svc, _), (buf, off) in zip(ranks, [big, small]):
        svc.send(R.SHOULD_RATE_LIMIT, buf, off, T0)
    for _, _, svc, _ in ranks:
        svc.decide()
    got = [svc.collect() for _, _, svc, _ in ranks]
    ref.serve(R.SHOULD_RATE_LIMIT, *small, T0)
    assert got[1] == ref.responses()
    plan = ranks[0][2].plan(R.SHOULD_RATE_LIMIT, *big, T0)
    stored = plan["store_index"] != 0xFFFFFFFF
    assert stored.any() and all(g[0] == 14 for g, s in zip(got[0], stored) if s)
    assert _table([e for _, e, _, _ in ranks]) == _table([ref_e])
    # counter variables and GET /counters are one engine's: refused on a sharded service
    with pytest.raises(R.RlsError, match="sharded"):
        ranks[0][2].keep_counter_vars(1024, 1 << 16)
    for sb in shards:
        sb.close()
    # ranks with different limits never decide each other's requests
    changed = [tuple(l) for l in LIMITS]
    changed[0] = (changed[0][0], 99) + changed[0][2:]
    ranks, shards = _sharded(world, lambda r: LIMITS if r == 0 else changed)
    names = [[] for _ in range(world)]
    batches = [_rls_batch(rng, 200, names[r]) for r in range(world)]
    for (_, _, svc, _), (buf, off) in zip(ranks, batches):
        svc.send(R.SHOULD_RATE_LIMIT, buf, off, T0)
    for _, _, svc, _ in ranks:
        svc.decide()
    errors = []
    for _, _, svc, _ in ranks:
        try:
            svc.collect()
        except R.RlsError as ex:
            errors.append(str(ex))
    assert len(errors) == world and all("limit registry of rank" in m for m in errors), errors
    # a request owned by the other rank crossed between registries that differ: UNAVAILABLE, never decided.  A request
    # owned by its own rank was decided there: answered as one engine with that rank's limits answers it.
    from limitador_b200 import owner_of
    ids = _ns_ids()
    for r, (_, _, svc, _) in enumerate(ranks):
        _, _, ref, _ = _stack(LIMITS if r == 0 else changed)
        got = svc.responses()
        own = [n in ids and owner_of(ids[n], world) == r for n in names[r]]
        crossed = [n in ids and not o for n, o in zip(names[r], own)]
        assert any(crossed) and any(own)
        keep = [i for i, c in enumerate(crossed) if not c]
        msgs = [bytes(batches[r][0][int(batches[r][1][i]):int(batches[r][1][i + 1])]) for i in keep]
        ref.serve(R.SHOULD_RATE_LIMIT, *R.pack_requests(msgs), T0)
        want = ref.responses()
        for i, c in enumerate(crossed):
            if c:
                assert got[i][0] == 14, (r, i)
        assert [got[i] for i in keep] == want
    for sb in shards:
        sb.close()


def _ipc_rank(rank, world, device, steps, seed, conn):
    """One process of the one-process-per-GPU deployment: its own service and exchange, IPC handles through the parent,
    then serve (the one call) on every step."""
    from limitador_b200 import ShardBatch
    _, e, svc, _ = _stack(device=device)
    sb = ShardBatch(e, rank, world, CAP_REQ, CAP_CTR)
    conn.send(sb.ipc_handle())
    sb.connect_ipc(conn.recv())
    svc.attach_shard(sb)
    rng = np.random.default_rng(seed)
    out = []
    for step in range(steps):
        batches = [_rls_batch(rng, int(rng.integers(0, 200))) for _ in range(world)]
        buf, off = batches[rank]
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, T0 + step * 1_000_000 + rank)
        out.append(svc.responses())
    conn.send(out)
    sb.close()
    conn.close()


def _device_count():
    import torch
    return torch.cuda.device_count()


@pytest.mark.gpu
@pytest.mark.parametrize("devices", [(0, 0), (0, 1)], ids=["one-gpu", "two-gpus"])
def test_two_processes_over_cuda_ipc(devices):
    """Two processes, one rank each, joined by CUDA IPC; each serves with the one call.  (0, 1): engines on distinct
    GPUs, skipped with one visible device."""
    import multiprocessing as mp
    import os
    if max(devices) >= _device_count():
        pytest.skip("needs two visible GPUs")
    world, steps, seed = 2, 6, 21
    os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")  # no lazy load while a peer spins (INTEGRATION.md §5)
    ctx = mp.get_context("spawn")
    pipes = [ctx.Pipe() for _ in range(world)]
    procs = [ctx.Process(target=_ipc_rank, args=(r, world, devices[r], steps, seed, pipes[r][1])) for r in range(world)]
    for p in procs:
        p.start()
    def recv(r):
        assert pipes[r][0].poll(300), f"rank {r} sent nothing in 300 s"
        return pipes[r][0].recv()

    try:
        handles = b"".join(recv(r) for r in range(world))
        for r in range(world):
            pipes[r][0].send(handles)
        got = [recv(r) for r in range(world)]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    _, _, ref, _ = _stack()
    rng = np.random.default_rng(seed)
    for step in range(steps):
        batches = [_rls_batch(rng, int(rng.integers(0, 200))) for _ in range(world)]
        for r in range(world):
            ref.serve(R.SHOULD_RATE_LIMIT, *batches[r], T0 + step * 1_000_000 + r)
            assert got[r][step] == ref.responses(), (step, r)


@pytest.mark.gpu
def test_kernel_resources():
    """ptxas registers, stack and spills of the exchange's general-form kernels (cuobjdump -res-usage of the library)."""
    from limitador_b200 import build as B
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", B.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    budget = {"k_ccount": 64, "k_cscatter": 40, "k_cprep": 32, "k_cunpack": 40, "k_cruns": 32, "k_crebase": 32,
              "k_creturn": 40, "k_cgather": 40}
    seen = {}
    for fn, reg, stack, local in re.findall(r"Function _Z\d+(k_c[a-z]+)\S*:\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out):
        if fn in budget:
            seen[fn] = (int(reg), int(stack), int(local))
    assert set(seen) == set(budget), seen
    for fn, (reg, stack, local) in seen.items():
        assert reg <= budget[fn] and stack == 0 and local == 0, (fn, reg, stack, local)
