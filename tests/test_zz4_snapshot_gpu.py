"""Counter snapshots on the GPU through the C-ABI: rl_counters_export / rl_counters_import / rl_limits_get and the
Python file form (Engine.save_counters / load_counters).  A stream runs on engine A and the oracle, A's counters move
to engine B of another geometry, and the stream goes on on B and the oracle with identical verdicts.  The import
kernels' logic is also run on the host under tests/emu/cuda_shim.h (tests/test_snapshot_emu.py).  Sorted last on
purpose: these entry points are new."""
import numpy as np
import pytest

from limitador_b200 import Engine, EngineError, exchange, streams
from limitador_b200.engine import RL_FATAL, RL_TRANSIENT, Shard
from tests import helpers as H
from tests.test_snapshot_emu import oracle_restore

pytestmark = pytest.mark.gpu
S = 1_000_000


def _import_from(dst, src, device, **kw):
    cols = src.export_counters(device=device, **kw)
    dst.import_counters(*cols)
    return cols


def _same_records(e, o, recs, stride, load=True):
    got = e.check_and_update_records(recs, load, stride=stride)
    want = o.batch_records(0, recs, load, stride)
    for k in range(4 if load else 2):
        assert got[k].tolist() == want[k].tolist(), f"output {k} differs"


def _same_csr(e, o, stream, load=True):
    off, ctrs, delta, now = stream
    got = e.check_and_update_batch(off, ctrs, delta, now, load)
    want = o.batch_csr(0, off, ctrs, delta, now, load)
    for k in range(4 if load else 2):
        assert got[k].tolist() == want[k].tolist(), f"output {k} differs"


@pytest.mark.parametrize("device", [False, True], ids=["host-arrays", "device-tensors"])
def test_round_trip_into_another_geometry_goes_on_with_identical_verdicts(device):
    # a reduced C2 stream: 4 qualified limits per namespace, one row per key on 7 cells, two rows on 3 cells
    w = streams.WORKLOADS["C2"](batch=4096, n_rows=3000, n_ns=8)
    a = Engine(capacity_rows=1 << 13, cells_per_row=7, max_batch=8192)
    b = Engine(capacity_rows=1 << 14, cells_per_row=3, max_batch=8192, regions=16)
    for e in (a, b):
        e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, 1 << 16)
    for s in range(3):
        _same_records(a, o, w.batch_records(s), 4)
    _import_from(b, a, device)
    assert H.normalise_dump(b.dump(), w.limits) == H.normalise_dump(a.dump(), w.limits)
    for s in range(3, 6):
        _same_records(b, o, w.batch_records(s), 4)
    assert H.normalise_dump(b.dump(), w.limits) == H.normalise_dump(o.dump(), w.limits)

    # unqualified and coupled (multi-row) counters, 3 <-> 7 cells per row
    descs = H.mixed_limits(12, seed=3)
    a = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    b = Engine(capacity_rows=1 << 13, cells_per_row=7, max_batch=8192, regions=8)
    for e in (a, b):
        e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    for s in range(3):
        _same_csr(a, o, H.random_csr_stream(descs, 3000, seed=10 + s, n_keys=40))
    _import_from(b, a, device)
    assert H.normalise_dump(b.dump(), descs) == H.normalise_dump(a.dump(), descs)
    for s in range(3, 6):
        _same_csr(b, o, H.random_csr_stream(descs, 3000, seed=10 + s, n_keys=40))
    assert H.normalise_dump(b.dump(), descs) == H.normalise_dump(o.dump(), descs)


def test_export_at_a_time_is_the_state_a_sweep_would_leave():
    descs = H.mixed_limits(12, seed=4)
    a = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    a.limits_set(descs)
    o = H.oracle_with_limits(descs)
    stream = H.random_csr_stream(descs, 4000, seed=21, n_keys=60)
    _same_csr(a, o, stream)
    before = a.dump()
    t = int(stream[3][len(stream[3]) // 2])
    got = a.export_counters(now_us=t)
    assert a.dump() == before, "an export changed the table"
    o.invalidate_expired(t)
    rows = sorted(zip(*[c.tolist() for c in got]))
    assert len(rows) == len(set(rows))
    assert H.normalise_dump(rows, descs) == H.normalise_dump(o.dump(), descs)
    # a namespace selection: exactly those namespaces' counters
    ns_of = {int(d["limit_id"]): int(d["ns_id"]) for d in descs}
    sel = [1, 4, 5]
    part = sorted(zip(*[c.tolist() for c in a.export_counters(ns_ids=sel)]))
    full = sorted(zip(*[c.tolist() for c in a.export_counters()]))
    assert full == before  # now_us = 0: exactly the dump
    assert part == [r for r in full if ns_of[r[0]] in sel] and part


def test_import_over_live_counters_replaces_them():
    descs = H.mixed_limits(12, seed=5)
    a = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    b = Engine(capacity_rows=1 << 12, cells_per_row=7, max_batch=8192)
    for e in (a, b):
        e.limits_set(descs)
    oa, ob_ = H.oracle_with_limits(descs), H.oracle_with_limits(descs)
    _same_csr(a, oa, H.random_csr_stream(descs, 3000, seed=31, n_keys=30))
    _same_csr(b, ob_, H.random_csr_stream(descs, 3000, seed=32, n_keys=30))
    cols = a.export_counters()
    keep = np.arange(len(cols[0])) % 3 != 0  # two thirds of A's counters, many of which B holds too
    cols = [c[keep] for c in cols]
    b.import_counters(*cols)
    oracle_restore(ob_, descs, *cols)
    assert H.normalise_dump(b.dump(), descs) == H.normalise_dump(ob_.dump(), descs)
    for s in range(2):
        _same_csr(b, ob_, H.random_csr_stream(descs, 3000, seed=33 + s, n_keys=30))
    assert H.normalise_dump(b.dump(), descs) == H.normalise_dump(ob_.dump(), descs)


def test_refused_imports_change_nothing():
    descs = H.mixed_limits(12, seed=6)
    e = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    _same_csr(e, o, H.random_csr_stream(descs, 2000, seed=41, n_keys=30))
    q = int(np.flatnonzero(descs["qualified"] == 1)[0])
    fresh = [np.array([q, q, q], dtype=np.uint32), np.array([1000, 1001, 1002], dtype=np.uint64),
             np.array([0, 1, 2], dtype=np.uint64), np.array([1, 2, 3], dtype=np.uint64),
             np.array([H.T0 + 5 * S] * 3, dtype=np.uint64)]

    def variant(col, idx, val):
        c = [x.copy() for x in fresh]
        c[col][idx] = val
        return c

    dup = variant(1, 2, 1000)
    dup[2][2] = 0  # entry 2 names entry 0's counter (key 1000, key_hi 0)
    cases = [(dup, RL_FATAL, "twice"),
             (variant(0, 1, 50_000), RL_FATAL, "not registered"),
             (variant(2, 1, 1 << 32), RL_FATAL, "key_hi"),
             (variant(4, 0, 0), RL_FATAL, "expiry 0")]
    before = e.dump()
    for cols, status, words in cases:
        with pytest.raises(EngineError, match=words) as ei:
            e.import_counters(*cols)
        assert ei.value.status == status
        assert e.dump() == before
    # a full region: more distinct rows than the table holds
    n = 1 << 13
    full = [np.full(n, q, np.uint32), np.arange(1, n + 1, dtype=np.uint64), np.zeros(n, np.uint64),
            np.ones(n, np.uint64), np.full(n, H.T0 + 5 * S, np.uint64)]
    with pytest.raises(EngineError, match="full") as ei:
        e.import_counters(*full)
    assert ei.value.status == RL_TRANSIENT
    assert e.dump() == before
    e.compact(0)
    assert e.dump() == before
    _same_csr(e, o, H.random_csr_stream(descs, 2000, seed=42, n_keys=30))


def _shard_steps(engines, w, recs_steps, oracle, batch, lag=1):
    import torch
    world = len(engines)
    shards = [Shard(engines[r], r, world, batch, lag) for r in range(world)]
    for s in shards:
        s.connect_ptrs([x.slab for x in shards])
    for recs in recs_steps:
        d = [torch.from_numpy(x.view(np.int64).reshape(-1, 4).copy()).cuda() for x in recs]
        out = [torch.full((batch,), 7, dtype=torch.uint8, device="cuda") for _ in range(world)]
        for r in range(world):
            shards[r].send(batch, d[r].data_ptr(), out[r].data_ptr())
        for r in range(world):
            shards[r].decide()
        for r in range(world):
            shards[r].collect()
        for s in shards:
            s.flush()
        for e in engines:
            e.sync()
        for r in range(world):
            assert np.array_equal(out[r].cpu().numpy(), oracle.batch_records(0, recs[r])[0])
    for s in shards:
        s.close()


def test_reshard_two_ranks_into_three():
    batch = 2048
    w = streams.WORKLOADS["C2"](batch=batch, n_rows=3000, n_ns=16)
    mk = lambda: Engine(capacity_rows=w.capacity_rows, cells_per_row=7, max_batch=3 * batch, flags=2)  # noqa: E731
    old = [mk() for _ in range(2)]
    for e in old:
        e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, 1 << 16)

    def step(st, world):
        recs = [w.batch_records(100 * st + r) for r in range(world)]
        for r in range(world):
            recs[r]["now_us"] = recs[0]["now_us"]
        return recs

    _shard_steps(old, w, [step(s, 2) for s in range(3)], o, batch)
    all_ns = np.unique(w.limits["ns_id"])
    new = [mk() for _ in range(3)]
    for r, e in enumerate(new):
        e.limits_set(w.limits)
        mine = exchange.namespaces_owned(all_ns, r, 3)
        parts = [x.export_counters(ns_ids=mine) for x in old]
        e.import_counters(*[np.concatenate([p[k] for p in parts]) for k in range(5)])
    union = [row for e in new for row in e.dump()]
    assert H.normalise_dump(union, w.limits) == H.normalise_dump(o.dump(), w.limits)
    _shard_steps(new, w, [step(s, 3) for s in range(3, 6)], o, batch)
    ns_of = {int(d["limit_id"]): int(d["ns_id"]) for d in w.limits}
    union = []
    for r, e in enumerate(new):
        d = e.dump()
        assert all(exchange.owner_of(ns_of[row[0]], 3) == r for row in d)
        union.extend(d)
    assert H.normalise_dump(union, w.limits) == H.normalise_dump(o.dump(), w.limits)


def test_save_and_load_counters_file(tmp_path):
    descs = H.mixed_limits(12, seed=7)
    a = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    a.limits_set(descs)
    o = H.oracle_with_limits(descs)
    _same_csr(a, o, H.random_csr_stream(descs, 3000, seed=51, n_keys=30))
    path, again = str(tmp_path / "counters.npz"), str(tmp_path / "again.npz")
    a.save_counters(path)
    a.save_counters(again)
    with np.load(path) as x, np.load(again) as y:
        assert sorted(x.files) == sorted(y.files)
        for k in x.files:
            assert x[k].tobytes() == y[k].tobytes(), f"the same table gave another '{k}'"
        assert np.array_equal(np.lexsort((x["key_hi"], x["key_lo"], x["limit_id"])), np.arange(len(x["limit_id"])))
    lims = a.limits_get()
    assert lims.tolist() == np.sort(descs, order="limit_id").tolist()
    b = Engine(capacity_rows=1 << 13, cells_per_row=7, max_batch=8192)
    b.limits_set(descs)
    b.load_counters(path)
    assert H.normalise_dump(b.dump(), descs) == H.normalise_dump(a.dump(), descs)
    stream = H.random_csr_stream(descs, 3000, seed=52, n_keys=30)
    _same_csr(b, o, stream)  # remaining / ttl included
    # a target whose limit 2 has another window: refused, naming the limit, nothing imported
    other = descs.copy()
    q = int(np.flatnonzero(other["qualified"] == 1)[1])
    other[q]["window_us"] += S
    c = Engine(capacity_rows=1 << 12, cells_per_row=3, max_batch=8192)
    c.limits_set(other)
    with pytest.raises(ValueError, match=rf"\[{q}\]"):
        c.load_counters(path)
    assert H.normalise_dump(c.dump(), other) == []
