"""GPU parity: the sm_90a kernels, called through the C-ABI, against the CPU oracle on the
same seeded request streams — verdicts, named limit, remaining/ttl and the full table."""
import numpy as np
import pytest

from limitador_b200 import Engine, EngineError
from limitador_b200 import engine as engine_module
from limitador_b200 import streams
from limitador_b200.engine import LIMIT_DESC_DTYPE, NONE, RECORD_DTYPE, COUNTER_DTYPE
from tests import helpers as H

pytestmark = pytest.mark.gpu
S = 1_000_000


def engine_with_limits(descs, cells, capacity=1 << 14, max_batch=1 << 16, regions=0, flags=0):
    e = Engine(capacity_rows=capacity, cells_per_row=cells, max_batch=max_batch, regions=regions, flags=flags)
    e.limits_set(descs)
    return e


def assert_tables_equal(e, o, descs):
    assert H.normalise_dump(e.dump(), descs) == H.normalise_dump(o.dump(), descs)


def single_row_limits(cells, n_ns=9, seed=0):
    """Every namespace maps to one row (fast record path): 1..cells limits on one varset, or
    1..cells unqualified limits."""
    rng = np.random.default_rng(seed)
    descs, lid = [], 0
    for ns in range(n_ns):
        k = int(rng.integers(1, cells + 1))
        q = 0 if ns % 4 == 3 else 1
        for _ in range(k):
            mx = int(rng.choice([0, 1, 2, 3, 5, 8, 20, 1 << 40]))
            win = int(rng.choice([1, 2, 10, 60, 3600])) * S
            descs.append((lid, ns, 1 if q else 0, q, mx, win))
            lid += 1
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
def test_records_fast_path(cells, load_counters):
    descs = single_row_limits(cells, seed=cells)
    e = engine_with_limits(descs, cells, regions=16)
    o = H.oracle_with_limits(descs)
    for b in range(6):
        recs = H.random_records(descs, 3000, 10 * cells + b, n_keys=40, monotone=(b % 2 == 0))
        got = e.check_and_update_records(recs, load_counters, stride=cells)
        want = o.batch_records(0, recs, load_counters, cells)
        assert got[0].tolist() == want[0].tolist()
        assert got[1].tolist() == want[1].tolist()
        if load_counters:
            assert got[2].tolist() == want[2].tolist()
            assert got[3].tolist() == want[3].tolist()
        assert_tables_equal(e, o, descs)
    assert e.stats()["kernel_launches"] > 0


@pytest.mark.parametrize("cells", [1, 3, 7])
def test_records_with_multi_row_namespaces(cells):
    descs = H.mixed_limits(n_ns=12, seed=4)
    e = engine_with_limits(descs, cells, regions=8)
    o = H.oracle_with_limits(descs)
    stride = 5
    for b in range(4):
        recs = H.random_records(descs, 1500, 77 + b, n_keys=6)
        got = e.check_and_update_records(recs, True, stride=stride)
        want = o.batch_records(0, recs, True, stride)
        for k in range(4):
            assert got[k].tolist() == want[k].tolist(), f"output {k} differs in batch {b}"
        assert_tables_equal(e, o, descs)


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
def test_csr_general_path_with_coupled_requests(cells, load_counters):
    descs = H.mixed_limits(n_ns=12, seed=cells)
    e = engine_with_limits(descs, cells, regions=8)
    o = H.oracle_with_limits(descs)
    for b in range(5):
        off, ctrs, delta, now = H.random_csr_stream(descs, 2000, 1000 * cells + b, n_keys=4, monotone=(b != 3))
        got = e.check_and_update_batch(off, ctrs, delta, now, load_counters)
        want = o.batch_csr(0, off, ctrs, delta, now, load_counters)
        assert got[0].tolist() == want[0].tolist()
        assert got[1].tolist() == want[1].tolist()
        if load_counters:
            assert got[2].tolist() == want[2].tolist()
            assert got[3].tolist() == want[3].tolist()
        assert_tables_equal(e, o, descs)
    assert e.stats()["fixed_point_rounds"] >= 1


@pytest.mark.parametrize("cells", [1, 7])
def test_grouping_tag_collisions(cells):
    """RL_FLAG_DEBUG_WEAK_TAGS: only 16 distinct grouping tags per salt level, so distinct keys
    collide inside a chunk and take the salted re-insertion path; results must not change."""
    descs = H.mixed_limits(n_ns=12, seed=3)
    e = Engine(capacity_rows=1 << 14, cells_per_row=cells, max_batch=1 << 16, regions=2, flags=1)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    for b in range(3):
        off, ctrs, delta, now = H.random_csr_stream(descs, 2500, 31 + b, n_keys=60)
        got = e.check_and_update_batch(off, ctrs, delta, now, True)
        want = o.batch_csr(0, off, ctrs, delta, now, True)
        for k in range(4):
            assert got[k].tolist() == want[k].tolist()
        assert_tables_equal(e, o, descs)


def test_long_dependency_chain():
    descs = np.array([(0, 0, 1, 1, 1, 3600 * S), (1, 0, 2, 1, 1, 3600 * S)], dtype=LIMIT_DESC_DTYPE)
    n = 40
    off = np.arange(0, 2 * n + 1, 2, dtype=np.uint32)
    ctrs = np.zeros(2 * n, dtype=COUNTER_DTYPE)
    for i in range(n):
        ctrs[2 * i] = (0, 0, 1 + i // 2, 0)
        ctrs[2 * i + 1] = (1, 0, 1 + (i + 1) // 2, 0)
    delta = np.ones(n, dtype=np.uint64)
    now = np.full(n, H.T0, dtype=np.uint64)
    e = engine_with_limits(descs, 1)
    o = H.oracle_with_limits(descs)
    got = e.check_and_update_batch(off, ctrs, delta, now)
    want = o.batch_csr(0, off, ctrs, delta, now)
    assert got[0].tolist() == want[0].tolist()
    assert_tables_equal(e, o, descs)
    assert e.stats()["fixed_point_rounds"] > 2


def test_update_and_is_within_limits_batches():
    descs = H.mixed_limits(n_ns=12, seed=9)
    e = engine_with_limits(descs, 3, regions=4)
    o = H.oracle_with_limits(descs)
    for b in range(4):
        off, ctrs, delta, now = H.random_csr_stream(descs, 1500, 500 + b, n_keys=4)
        e.update_batch(off, ctrs, delta, now)
        o.batch_csr(2, off, ctrs, delta, now)
        assert_tables_equal(e, o, descs)
        off, ctrs, delta, now = H.random_csr_stream(descs, 1500, 600 + b, n_keys=4)
        now = now + np.uint64(int(now[-1] - now[0]))
        lim, fl = e.is_within_limits_batch(off, ctrs, delta, now)
        wl, wf, _, _ = o.batch_csr(1, off, ctrs, delta, now)
        assert lim.tolist() == wl.tolist() and fl.tolist() == wf.tolist()
        assert_tables_equal(e, o, descs)  # read-only
    recs = H.random_records(descs, 2000, 5, n_keys=4)
    e.update_records(recs)
    o.batch_records(2, recs)
    assert_tables_equal(e, o, descs)
    lim, fl = e.is_within_limits_records(recs)
    wl, wf, _, _ = o.batch_records(1, recs)
    assert lim.tolist() == wl.tolist() and fl.tolist() == wf.tolist()


@pytest.mark.parametrize("flags", [0, 2])
def test_host_async_mem_acts_as_host_where_a_call_cannot_take_it(flags, monkeypatch):
    """RL_MEM_HOST_ASYNC behaves like RL_MEM_HOST outside the record check calls (rl_engine.h): the query calls
    and the CSR check write their outputs to host memory before they return."""
    descs = H.mixed_limits(n_ns=12, seed=9)
    e_host = engine_with_limits(descs, 3, regions=4, flags=flags)
    e_async = engine_with_limits(descs, 3, regions=4, flags=flags)
    for b in range(3):
        off, ctrs, delta, now = H.random_csr_stream(descs, 1500, 700 + b, n_keys=4)
        recs = H.random_records(descs, 1500, 800 + b, n_keys=4)
        want = [e_host.check_and_update_batch(off, ctrs, delta, now, True),
                e_host.is_within_limits_batch(off, ctrs, delta, now), e_host.is_within_limits_records(recs)]
        with monkeypatch.context() as m:
            m.setattr(engine_module, "MEM_HOST", engine_module.MEM_HOST_ASYNC)  # what the Engine methods pass as mem
            got = [e_async.check_and_update_batch(off, ctrs, delta, now, True),
                   e_async.is_within_limits_batch(off, ctrs, delta, now), e_async.is_within_limits_records(recs)]
        for w, g in zip(want, got):
            for k in range(len(w)):
                assert g[k].tolist() == w[k].tolist(), f"output {k} differs in batch {b}"
        assert int(want[0][0].sum()) > 0  # some request was limited: the outputs differ from their initial values
    assert_tables_equal(e_async, e_host, descs)


def test_hot_key_spanning_many_chunks():
    """One key takes 5000 requests of a batch (20 chunks of the owning CTA) interleaved with
    other keys; max 1000 so the verdict flips inside the batch; deltas vary (greedy, not a
    prefix sum)."""
    descs = np.array([(0, 0, 1, 1, 1000, 60 * S), (1, 0, 1, 1, 100000, 3600 * S)], dtype=LIMIT_DESC_DTYPE)
    rng = np.random.default_rng(0)
    n = 12000
    recs = np.zeros(n, dtype=RECORD_DTYPE)
    recs["ns_id"] = 0
    recs["hits_addend"] = rng.choice([1, 1, 2, 5, 400], size=n)
    hot = rng.random(n) < 0.45
    recs["key_lo"] = np.where(hot, 7, rng.integers(8, 3000, size=n))
    recs["now_us"] = H.T0 + np.arange(n) * 7000  # 84 s: the 60 s window rolls over once
    e = engine_with_limits(descs, 3, regions=4)
    o = H.oracle_with_limits(descs)
    got = e.check_and_update_records(recs, True, stride=3)
    want = o.batch_records(0, recs, True, 3)
    for k in range(4):
        assert got[k].tolist() == want[k].tolist()
    assert 0 < int(got[0].sum()) < n
    assert_tables_equal(e, o, descs)


def test_maintenance_get_delete_clear_sweep():
    descs = H.mixed_limits(n_ns=12, seed=2)
    e = engine_with_limits(descs, 7, regions=4)
    o = H.oracle_with_limits(descs)
    off, ctrs, delta, now = H.random_csr_stream(descs, 3000, 42, n_keys=30)
    e.update_batch(off, ctrs, delta, now)
    o.batch_csr(2, off, ctrs, delta, now)
    t = int(now[-1])
    ids = descs["limit_id"][descs["ns_id"] < 5]
    assert e.get_counters(ids, t) == o.get_counters(ids, t)
    assert e.get_counters(ids, t + 30 * S) == o.get_counters(ids, t + 30 * S)
    # sweep == oracle invalidate event; a later denied check must agree (SURVEY §7 hard part 3c)
    n_gpu = e.sweep(t + 5 * S)
    n_cpu = o.invalidate_expired(t + 5 * S)
    assert n_gpu == n_cpu and n_gpu > 0
    assert_tables_equal(e, o, descs)
    off, ctrs, delta, now2 = H.random_csr_stream(descs, 3000, 43, n_keys=30)
    now2 = now2 + np.uint64(t + 6 * S - H.T0)
    got = e.check_and_update_batch(off, ctrs, delta, now2, True)
    want = o.batch_csr(0, off, ctrs, delta, now2, True)
    for k in range(4):
        assert got[k].tolist() == want[k].tolist()
    assert_tables_equal(e, o, descs)
    # delete by limit, clear
    kill = descs["limit_id"][::3]
    e.delete_counters(kill)
    o.delete_counters(kill)
    assert_tables_equal(e, o, descs)
    e.clear()
    o.clear()
    assert_tables_equal(e, o, descs)
    # Storage::clear also forgets the limits (storage/mod.rs:137-140); the front re-adds them,
    # which re-creates the unqualified counters (add_counter, in_memory.rs:38-44)
    e.limits_set(descs)
    for d in descs:
        o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    # limits_delete + max_value update
    e.limits_delete(kill[:2])
    for k in kill[:2]:
        o.limit_delete(int(k))
    d = descs[5].copy()
    d["max_value"] = 1 << 20
    e.limits_set(np.array([d], dtype=LIMIT_DESC_DTYPE))
    o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    live = np.array([x for x in descs if int(x["limit_id"]) not in set(kill[:2].tolist())], dtype=LIMIT_DESC_DTYPE)
    off, ctrs, delta, now3 = H.random_csr_stream(live, 2000, 44, n_keys=30)
    now3 = now3 + np.uint64(int(now2[-1]) - H.T0)
    got = e.check_and_update_batch(off, ctrs, delta, now3)
    want = o.batch_csr(0, off, ctrs, delta, now3)
    assert got[0].tolist() == want[0].tolist() and got[1].tolist() == want[1].tolist()
    assert_tables_equal(e, o, live)


def test_errors_are_loud():
    descs = np.array([(0, 0, 1, 1, 10, 60 * S)], dtype=LIMIT_DESC_DTYPE)
    e = engine_with_limits(descs, 1, capacity=64, regions=1)
    recs = np.zeros(200, dtype=RECORD_DTYPE)
    recs["hits_addend"] = 1
    recs["key_lo"] = np.arange(1, 201)
    recs["now_us"] = H.T0
    with pytest.raises(EngineError) as ei:
        e.check_and_update_records(recs)
    assert ei.value.transient  # table full: RL_TRANSIENT, never a silent allow
    e2 = engine_with_limits(descs, 1)
    off = np.array([0, 1], dtype=np.uint32)
    bad = np.array([(5, 0, 1, 0)], dtype=COUNTER_DTYPE)
    with pytest.raises(EngineError) as ei:
        e2.check_and_update_batch(off, bad, [1], [H.T0])
    assert not ei.value.transient
    hi = np.array([(0, 0, 1, 1 << 32)], dtype=COUNTER_DTYPE)
    with pytest.raises(EngineError):
        e2.check_and_update_batch(off, hi, [1], [H.T0])
    with pytest.raises(EngineError):
        e2.check_and_update_records(np.zeros((1 << 16) + 1, dtype=RECORD_DTYPE))


@pytest.mark.parametrize("cells", [1, 7])
def test_compact_16_byte_records_match_the_32_byte_form(cells):
    """rl_record16 (include/rl_engine.h): ns_id:24 | hits:8 | key_hi:32 | key_lo:64, the whole batch stamped with one
    clock reading — the same decisions and table as the 32-byte records carrying that timestamp; host, device
    (pipelined) and async-host calls."""
    import torch
    from limitador_b200.engine import pack_records16, RECORD16_DTYPE
    descs = single_row_limits(cells, seed=50 + cells)
    o = H.oracle_with_limits(descs)
    e = engine_with_limits(descs, cells, regions=8, flags=2)
    t = H.T0
    for b in range(6):
        recs = H.random_records(descs, 5000, 900 + b, n_keys=60)
        recs["key_hi"] = (recs["key_lo"] * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)  # exercise the key_hi bits
        recs["hits_addend"] = 1 + (recs["key_lo"] % np.uint64(3)).astype(np.uint32)
        t += 700_000 * (1 + b % 3)
        recs["now_us"] = t
        r16 = pack_records16(recs)
        want = o.batch_records(0, recs)
        if b % 3 == 0:
            lim, fl = e.check_and_update_compact(r16, t)
        else:
            mem = 1 if b % 3 == 1 else 2
            if mem == 1:
                d = torch.from_numpy(r16.view(np.int64).reshape(-1, 2).copy()).cuda()
                out = torch.zeros(len(r16), dtype=torch.uint8, device="cuda")
                first = torch.zeros(len(r16), dtype=torch.int32, device="cuda")
            else:
                d = torch.from_numpy(r16.view(np.int64).reshape(-1, 2).copy()).pin_memory()
                out = torch.zeros(len(r16), dtype=torch.uint8).pin_memory()
                first = torch.zeros(len(r16), dtype=torch.int32).pin_memory()
            e.check_and_update_compact_ptr(len(r16), d.data_ptr(), t, out.data_ptr(), mem, first.data_ptr())
            e.fence()
            e.sync()
            lim, fl = out.cpu().numpy(), first.cpu().numpy().astype(np.uint32)
        assert np.array_equal(lim, want[0]) and np.array_equal(fl, want[1]), f"batch {b}"
        assert_tables_equal(e, o, descs)
    with pytest.raises(ValueError):
        bad = recs[:2].copy()
        bad["hits_addend"] = 256
        pack_records16(bad)


def test_unevaluated_requests_never_read_as_allowed():
    """ADVICE r1: a request the engine cannot evaluate gets RL_VERDICT_ERROR (0xFF), not 0 = allowed, and a
    general-form call with an unresolvable request is refused BEFORE the table is touched (a retry of the
    corrected batch must not double count the other requests)."""
    import torch
    descs = np.array([(0, 0, 1, 1, 3, 60 * S), (1, 1, 1, 1, 3, 60 * S)], dtype=LIMIT_DESC_DTYPE)
    e = engine_with_limits(descs, 1, flags=2)
    o = H.oracle_with_limits(descs)
    recs = np.zeros(64, dtype=RECORD_DTYPE)
    recs["ns_id"] = np.arange(64) % 2
    recs["hits_addend"] = 1
    recs["key_lo"] = 1 + np.arange(64) % 5
    recs["now_us"] = H.T0
    bad = recs.copy()
    bad["key_hi"][[3, 17]] = np.uint64(1 << 40)  # bits 32..55 set: malformed
    d = torch.from_numpy(bad.view(np.int64).reshape(-1, 4).copy()).cuda()
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    e.check_and_update_records_ptr(64, d.data_ptr(), out.data_ptr(), 1, stride=1)
    with pytest.raises(EngineError):
        e.sync()
    got = out.cpu().numpy()
    assert got[3] == 0xFF and got[17] == 0xFF
    good = np.ones(64, dtype=bool)
    good[[3, 17]] = False
    want = o.batch_records(0, recs[good])[0]
    assert np.array_equal(got[good], want)  # the well-formed requests were decided as if the bad ones were absent
    assert_tables_equal(e, o, descs)
    # general form: unknown limit in request 2 of 3 -> the whole call is refused, nothing is counted
    e2 = engine_with_limits(descs, 1)
    off = np.array([0, 1, 2, 3], dtype=np.uint32)
    ctrs = np.array([(0, 0, 7, 0), (9, 0, 7, 0), (1, 0, 7, 0)], dtype=COUNTER_DTYPE)
    with pytest.raises(EngineError) as ei:
        e2.check_and_update_batch(off, ctrs, [1, 1, 1], [H.T0] * 3)
    assert "before the table was touched" in str(ei.value)
    assert e2.dump() == []
    ctrs["limit_id"][1] = 0
    lim = e2.check_and_update_batch(off, ctrs, [1, 1, 1], [H.T0] * 3)[0]
    assert lim.tolist() == [0, 0, 0] and len(e2.dump()) == 2
    # 17 counters in one request (the engine takes 16)
    many = np.zeros(17, dtype=COUNTER_DTYPE)
    many["key_lo"] = 1
    with pytest.raises(EngineError):
        e2.check_and_update_batch(np.array([0, 17], dtype=np.uint32), many, [1], [H.T0])
    assert len(e2.dump()) == 2


@pytest.mark.parametrize("name,kw,nb", [
    ("C1", dict(batch=65536), 3),
    ("C2", dict(batch=65536, n_rows=100_000), 4),
    ("C3", dict(batch=1 << 18, n_keys=1_000_000), 3),
    ("C5", dict(batch=1 << 17, n_keys=1_000_000, n_ns=500), 2),
])
def test_baseline_configs_reduced_size(name, kw, nb):
    """BASELINE.json's configs at sizes the oracle replays in seconds: full verdict + table parity."""
    w = streams.WORKLOADS[name](**kw)
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch)
    e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, capacity_hint=1 << 20)
    for b in range(nb):
        recs = w.batch_records(b)
        got = e.check_and_update_records(recs, False, stride=w.cells_per_row)
        want = o.batch_records(0, recs)
        assert np.array_equal(got[0], want[0]), f"{name} batch {b}: {int((got[0] != want[0]).sum())} verdicts differ"
        assert np.array_equal(got[1], want[1])
    ge, go = e.dump_arrays(), o.dump_arrays()
    assert len(ge[0]) == len(go[0])
    def canon(d):
        order = np.lexsort((d[2], d[1], d[0]))
        return [x[order] for x in d]
    for a, b_ in zip(canon(ge), canon(go)):
        assert np.array_equal(a, b_)


def _table_rows(lid, lo, hi, val, exp):
    """A counter dump as one sorted structured array (order-independent comparison of millions of rows)."""
    n = len(lid)
    rows = np.empty(n, dtype=[("lid", "<u8"), ("lo", "<u8"), ("hi", "<u8"), ("val", "<u8"), ("exp", "<u8")])
    rows["lid"], rows["lo"], rows["hi"], rows["val"], rows["exp"] = lid, lo, hi, val, exp
    rows.sort(order=["lid", "lo", "hi"])
    return rows


@pytest.mark.parametrize("name,nb,pipelined,hot", [("C2", 40, False, 0), ("C2", 40, True, 0), ("C2", 40, True, 1), ("C3", 4, True, 0)])
def test_full_size_configs_match_the_oracle_state(name, nb, pipelined, hot, monkeypatch):
    """BASELINE.json configs[1] / configs[2] at FULL size (C2: 1 M rows, batch 65 536, Zipf(1.1), a 1-s window
    rollover inside the run; C3: 16 M keys, batch 1 M): every verdict AND the final counter table (every value and
    expiry, millions of rows) equal the oracle's — not invariants (VERDICT r1, item 7).  C2 also through the
    pipelined device path (front of batch s+1 overlapping the replay of batch s, hot rows learnt on the way)."""
    import torch
    monkeypatch.setenv("RL_HOT", str(hot))
    w = streams.WORKLOADS[name]()
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch, flags=2 if pipelined else 0)
    e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, capacity_hint=1 << 22)
    # C2: batches 0..nb-1 except that the second half starts after the stream's 1-s jump (batch 64), so that the
    # 1-s windows of the hot keys roll over inside the test
    ids = list(range(nb)) if name == "C3" else list(range(nb // 2)) + list(range(64, 64 + nb - nb // 2))
    recs = [w.batch_records(b) for b in ids]
    if pipelined:
        d_recs = [torch.from_numpy(r.view(np.int64).reshape(-1, 4).copy()).cuda() for r in recs]
        d_lim = [torch.full((w.batch,), 9, dtype=torch.uint8, device="cuda") for _ in recs]
        torch.cuda.synchronize()
        for i in range(len(recs)):
            e.check_and_update_records_ptr(w.batch, d_recs[i].data_ptr(), d_lim[i].data_ptr(), 1, stride=w.cells_per_row)
        e.fence()
        e.sync()
        got = [t.cpu().numpy() for t in d_lim]
    else:
        got = [e.check_and_update_records(r, False, stride=w.cells_per_row)[0] for r in recs]
    for i, r in enumerate(recs):
        want = o.batch_records(0, r)[0]
        assert np.array_equal(got[i], want), f"{name} batch {ids[i]}: {int((got[i] != want).sum())} verdicts differ"
    g, x = _table_rows(*e.dump_arrays(cap=1 << 23)), _table_rows(*o.dump_arrays())
    assert len(g) == len(x) and len(g) > 100_000
    assert np.array_equal(g, x), "counter tables differ"
    if name == "C2" and hot:
        assert e.stats()["hot_rows"] > 0  # the Zipf head was learnt


def test_bucket_by_owner_is_stable_and_matches_host_function():
    """Multi-GPU exchange helpers: rl_bucket_by_owner == a stable sort by rl_owner_of(ns_id)."""
    import torch
    from limitador_b200 import exchange, owner_of
    descs = np.array([(0, 0, 1, 1, 10, 60 * S)], dtype=LIMIT_DESC_DTYPE)
    e = engine_with_limits(descs, 1)
    rng = np.random.default_rng(7)
    n = 50000
    recs = np.zeros(n, dtype=RECORD_DTYPE)
    recs["ns_id"] = rng.integers(0, 300, size=n)
    recs["key_lo"] = np.arange(n)
    for world in (2, 8):
        d_in = torch.from_numpy(recs.view(np.int64).reshape(-1, 4).copy()).cuda()
        d_out = torch.empty_like(d_in)
        d_src = torch.empty(n, dtype=torch.int32, device="cuda")
        counts = e.bucket_by_owner_ptr(n, d_in.data_ptr(), world, d_out.data_ptr(), d_src.data_ptr())
        e.sync()
        owners = np.array([owner_of(int(ns), world) for ns in recs["ns_id"]])
        perm, src, want_counts = exchange.stable_bucket_numpy(recs.view(np.int64).reshape(-1, 4), owners, world)
        assert counts.tolist() == want_counts
        assert np.array_equal(d_src.cpu().numpy(), src)
        assert np.array_equal(d_out.cpu().numpy(), perm)
        v_in = torch.from_numpy((np.arange(n) % 251).astype(np.uint8)).cuda()
        v_out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        e.unpermute_u8_ptr(n, v_in.data_ptr(), d_src.data_ptr(), v_out.data_ptr())
        e.sync()
        want = np.zeros(n, dtype=np.uint8)
        want[src] = (np.arange(n) % 251).astype(np.uint8)
        assert np.array_equal(v_out.cpu().numpy(), want)


def test_padded_bucket_exchange_roundtrip_single_process():
    """The sync-free exchange used by bench.py at N>1, folded onto one GPU: bucket into fixed
    blocks (no-op padding), run the engine over ALL blocks in (owner, slot) order, gather back —
    equals running the oracle over the same permuted stream."""
    import torch
    descs = single_row_limits(3, n_ns=40, seed=5)
    e = engine_with_limits(descs, 3, max_batch=1 << 17)
    o = H.oracle_with_limits(descs)
    world, n = 4, 20000
    slot_cap = 8192
    recs = H.random_records(descs, n, 99, n_keys=50)
    d_in = torch.from_numpy(recs.view(np.int64).reshape(-1, 4).copy()).cuda()
    send = torch.full((world * slot_cap, 4), -1, dtype=torch.int64, device="cuda")
    pos = torch.empty(n, dtype=torch.int32, device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.bucket_by_owner_padded_ptr(n, d_in.data_ptr(), world, slot_cap, send.data_ptr(), pos.data_ptr(), ovf.data_ptr())
    verdict = torch.zeros(world * slot_cap, dtype=torch.uint8, device="cuda")
    e.check_and_update_records_ptr(world * slot_cap, send.data_ptr(), verdict.data_ptr(), 1, stride=3)
    out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    e.gather_u8_ptr(n, verdict.data_ptr(), pos.data_ptr(), out.data_ptr())
    e.sync()
    assert int(ovf.item()) == 0
    from limitador_b200 import owner_of
    owners = np.array([owner_of(int(ns), world) for ns in recs["ns_id"]])
    order = np.argsort(owners, kind="stable")
    lim, _, _, _ = o.batch_records(0, recs[order])
    want = np.zeros(n, dtype=np.uint8)
    want[order] = lim
    assert np.array_equal(out.cpu().numpy(), want)
    assert_tables_equal(e, o, descs)


def test_record_lane_byte_is_opaque_and_round_trips():
    """rl_record_lane_put/_gather (the one-collective exchange): the lane byte travels in the records,
    the decision calls ignore it, and gathering through the bucket positions restores request order."""
    import torch
    descs = single_row_limits(3, n_ns=40, seed=6)
    e = engine_with_limits(descs, 3, max_batch=1 << 17)
    o = H.oracle_with_limits(descs)
    world, n, slot_cap = 4, 20000, 8192
    recs = H.random_records(descs, n, 77, n_keys=50)
    d_in = torch.from_numpy(recs.view(np.int64).reshape(-1, 4).copy()).cuda()
    send = torch.empty((world * slot_cap, 4), dtype=torch.int64, device="cuda")
    pos = torch.empty(n, dtype=torch.int32, device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    lane = torch.randint(0, 256, (world * slot_cap,), dtype=torch.uint8, device="cuda")
    e.bucket_by_owner_padded_ptr(n, d_in.data_ptr(), world, slot_cap, send.data_ptr(), pos.data_ptr(), ovf.data_ptr())
    e.record_lane_put_ptr(world * slot_cap, send.data_ptr(), lane.data_ptr())
    verdict = torch.zeros(world * slot_cap, dtype=torch.uint8, device="cuda")
    e.check_and_update_records_ptr(world * slot_cap, send.data_ptr(), verdict.data_ptr(), 1, stride=3)
    back = torch.zeros(n, dtype=torch.uint8, device="cuda")
    e.record_lane_gather_ptr(n, send.data_ptr(), pos.data_ptr(), back.data_ptr())
    e.sync()
    assert int(ovf.item()) == 0
    # the lane bytes came back in request order ...
    assert np.array_equal(back.cpu().numpy(), lane.cpu().numpy()[pos.cpu().numpy().astype(np.int64)])
    # ... and did not change a single decision: same verdicts and table as the oracle on the clean records
    from limitador_b200 import owner_of
    owners = np.array([owner_of(int(ns), world) for ns in recs["ns_id"]])
    order = np.argsort(owners, kind="stable")
    lim, _, _, _ = o.batch_records(0, recs[order])
    got = verdict.cpu().numpy()[pos.cpu().numpy().astype(np.int64)]
    want = np.zeros(n, dtype=np.uint8)
    want[order] = lim
    assert np.array_equal(got, want)
    assert_tables_equal(e, o, descs)
    # the oracle ignores the lane byte too (it checks the exchanged stream in the gloo test)
    o2 = H.oracle_with_limits(descs)
    laned = send.cpu().numpy().view(RECORD_DTYPE).reshape(-1)
    lim2, _, _, _ = o2.batch_records(0, laned)
    assert np.array_equal(lim2, verdict.cpu().numpy())
    # a set bit between the digest and the lane byte is still a key-range error
    bad = recs[recs["ns_id"] % 4 != 3][:8].copy()  # namespaces with qualified limits (single_row_limits)
    bad["key_hi"] |= np.uint64(1 << 40)
    with pytest.raises(EngineError):
        e.check_and_update_records(bad, False, stride=3)


def test_pipelined_device_calls_match_oracle():
    """RL_FLAG_PIPELINE: back-to-back device-memory calls overlap (partition of call s+1 with the
    replay of call s); after rl_fence/rl_sync the verdicts and the table equal the sequential ones."""
    import torch
    w = streams.WORKLOADS["C2"](batch=16384, n_rows=20000, n_ns=32)
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch, flags=2)
    e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, 1 << 16)
    nb = 12
    recs = [w.batch_records(b) for b in range(nb)]
    d_recs = [torch.from_numpy(r.view(np.int64).reshape(-1, 4).copy()).cuda() for r in recs]
    d_lim = [torch.zeros(w.batch, dtype=torch.uint8, device="cuda") for _ in range(nb)]
    d_first = [torch.zeros(w.batch, dtype=torch.int32, device="cuda") for _ in range(nb)]
    torch.cuda.synchronize()
    for b in range(nb):
        e.check_and_update_records_ptr(w.batch, d_recs[b].data_ptr(), d_lim[b].data_ptr(), 1,
                                       out_first_ptr=d_first[b].data_ptr(), stride=w.cells_per_row)
    e.fence()
    e.sync()
    for b in range(nb):
        want = o.batch_records(0, recs[b])
        assert np.array_equal(d_lim[b].cpu().numpy(), want[0]), f"batch {b}"
        assert np.array_equal(d_first[b].cpu().numpy().astype(np.uint32), want[1])
    assert_tables_equal(e, o, w.limits)
    # a host-memory call after pipelined ones is ordered behind them
    r = w.batch_records(nb)
    got = e.check_and_update_records(r, False, stride=w.cells_per_row)
    want = o.batch_records(0, r)
    assert np.array_equal(got[0], want[0])
    assert_tables_equal(e, o, w.limits)


def test_async_host_calls_match_oracle():
    """RL_MEM_HOST_ASYNC: pinned host buffers, calls only enqueue H2D + kernels + D2H; after
    rl_sync the verdicts in host memory equal the sequential ones (more calls than ring slots)."""
    import torch
    w = streams.WORKLOADS["C2"](batch=8192, n_rows=20000, n_ns=32)
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch, flags=2)
    e.limits_set(w.limits)
    o = H.oracle_with_limits(w.limits, 1 << 16)
    nb = 11
    recs = [w.batch_records(b) for b in range(nb)]
    h_recs = torch.stack([torch.from_numpy(r.view(np.int64).reshape(-1, 4).copy()) for r in recs]).pin_memory()
    h_lim = torch.zeros((nb, w.batch), dtype=torch.uint8).pin_memory()
    h_first = torch.zeros((nb, w.batch), dtype=torch.int32).pin_memory()
    for b in range(nb):
        e.check_and_update_records_ptr(w.batch, h_recs[b].data_ptr(), h_lim[b].data_ptr(), 2,
                                       out_first_ptr=h_first[b].data_ptr(), stride=w.cells_per_row)
    e.sync()
    for b in range(nb):
        want = o.batch_records(0, recs[b])
        assert np.array_equal(h_lim[b].numpy(), want[0]), f"batch {b}"
        assert np.array_equal(h_first[b].numpy().astype(np.uint32), want[1])
    assert_tables_equal(e, o, w.limits)


def test_batching_front_concurrent_callers_linearise():
    """rl_front: 8 threads issue single requests concurrently; the front coalesces them into
    batches.  Replaying the requests through the oracle in the front's drain order (out_seq)
    must reproduce every verdict, remaining and ttl — a valid linearisation, like concurrent
    callers of InMemoryStorage."""
    import threading
    from limitador_b200 import Front
    descs = H.mixed_limits(n_ns=12, seed=8)
    e = engine_with_limits(descs, 3, max_batch=4096)
    o = H.oracle_with_limits(descs)
    front = Front(e, max_batch=256, max_delay_us=200)
    n_threads, per_thread = 8, 300
    results = [[] for _ in range(n_threads)]

    def worker(t):
        off, ctrs, delta, now = H.random_csr_stream(descs, per_thread, 4000 + t, n_keys=5)
        for i in range(per_thread):
            c = ctrs[off[i]:off[i + 1]]
            # one clock for all threads would be the wall clock; use a fixed stamp per request so the
            # oracle replay is deterministic whatever the interleaving
            lim, first, seq, rem, ttl = front.check_and_update(c, int(delta[i]), now_us=H.T0 + 1, load_counters=True)
            results[t].append((seq, c.copy(), int(delta[i]), lim, first, rem.copy(), ttl.copy()))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    st = front.stats()
    front.close()
    allr = sorted([r for rs in results for r in rs], key=lambda r: r[0])
    assert [r[0] for r in allr if len(r[1])] == sorted(r[0] for r in allr if len(r[1]))
    assert st["requests"] == sum(1 for r in allr if len(r[1]))
    assert st["batches"] < st["requests"], "requests were never coalesced"
    for seq, c, d, lim, first, rem, ttl in allr:
        if len(c) == 0:
            assert lim is False
            continue
        wl, widx, wrem, wttl = o.check_and_update(c, d, True, H.T0 + 1)
        assert lim == wl, seq
        assert first == (None if widx is None else int(c[widx]["limit_id"]))
        assert rem.tolist() == wrem.tolist() and ttl.tolist() == wttl.tolist()
    assert_tables_equal(e, o, descs)


@pytest.mark.parametrize("load_counters", [False, True])
def test_hot_rows_get_partitions_of_their_own(load_counters, monkeypatch):
    """DESIGN §3.4: a row that dominates its k_main chunks is admitted to the hot-row table and from the next batch on
    its whole request list is replayed by one CTA of k_hot (no chained chunks); rows that cool down are dropped.
    Verdicts, named limits, remaining/ttl and the table equal the oracle's throughout — with windows rolling over
    (a 1-s limit), values accumulating (max 2^40), saturated rows (max 3) and mixed deltas on the hot rows."""
    monkeypatch.setenv("RL_HOT", "1")
    descs = np.array([(0, 0, 1, 1, 3, 1 * S), (1, 0, 1, 1, 1 << 40, 3600 * S), (2, 1, 1, 1, 50, 2 * S),
                      (3, 2, 0, 0, 1 << 40, 60 * S), (4, 3, 1, 1, 5, 60 * S)], dtype=LIMIT_DESC_DTYPE)
    e = engine_with_limits(descs, 3, capacity=1 << 15, regions=4)
    o = H.oracle_with_limits(descs)
    rng = np.random.default_rng(9)
    n = 20000
    t = H.T0
    for b in range(9):
        recs = np.zeros(n, dtype=RECORD_DTYPE)
        hot = rng.random(n) < (0.0 if b == 6 else 0.8)  # batch 6: the hot keys vanish, the table drains
        recs["ns_id"] = np.where(hot, rng.integers(0, 3, n), rng.integers(0, 4, n))
        recs["key_lo"] = np.where(hot, 1 + rng.integers(0, 2, n), 10 + rng.integers(0, 3000, n))
        recs["hits_addend"] = np.where(rng.random(n) < 0.9, 1, rng.integers(1, 4, n))
        recs["now_us"] = t + np.sort(rng.integers(0, 1_500_000, n)).astype(np.uint64)
        t += 1_600_000
        got = e.check_and_update_records(recs, load_counters, stride=3)
        want = o.batch_records(0, recs, load_counters, 3)
        assert got[0].tolist() == want[0].tolist(), f"batch {b}"
        assert got[1].tolist() == want[1].tolist()
        if load_counters:
            assert got[2].tolist() == want[2].tolist() and got[3].tolist() == want[3].tolist()
        assert_tables_equal(e, o, descs)
        hot_now = e.stats()["hot_rows"]
        if b in (2, 3, 4, 5):
            assert hot_now >= 4, f"batch {b}: {hot_now} hot rows"  # (ns 0..2) x (key 1..2), unqualified ns 2 -> one row
        if b == 8:
            assert hot_now >= 4
    # update_counters through the hot path as well
    for b in range(3):
        recs = np.zeros(n, dtype=RECORD_DTYPE)
        recs["ns_id"] = rng.integers(0, 3, n)
        recs["key_lo"] = 1 + rng.integers(0, 2, n)
        recs["hits_addend"] = 1
        recs["now_us"] = t + np.sort(rng.integers(0, 1_500_000, n)).astype(np.uint64)
        t += 1_600_000
        e.update_records(recs)
        o.batch_records(2, recs)
        assert_tables_equal(e, o, descs)


@pytest.mark.parametrize("hot", [0, 1])
@pytest.mark.parametrize("chunk,mult", [(128, 1), (256, 1), (128, 2)])
def test_chained_commit_stress(monkeypatch, chunk, mult, hot):
    """Optimistic-commit protocol under stress: RL_HEAVY_MULT=1 chains every partition above the
    average, and a tiny key space makes the chunks of a partition share written rows in every
    direction (earlier writer -> later reader AND later writer -> earlier reader, the case a
    round-1 bug missed).  Records and CSR forms, both load_counters values."""
    monkeypatch.setenv("RL_CHUNK", str(chunk))
    monkeypatch.setenv("RL_HEAVY_MULT", str(mult))
    monkeypatch.setenv("RL_HOT", str(hot))  # 0: every heavy partition stays on the chained path
    for cells in (1, 3):
        descs = single_row_limits(cells, seed=20 + cells)
        e = engine_with_limits(descs, cells, regions=4, flags=4)  # RL_FLAG_KERNEL_STATS: chunk accounting on
        o = H.oracle_with_limits(descs)
        for b in range(4):
            recs = H.random_records(descs, 6000, 300 + 10 * cells + b, n_keys=25, monotone=(b % 2 == 0))
            lc = bool(b & 1)
            got = e.check_and_update_records(recs, lc, stride=cells)
            want = o.batch_records(0, recs, lc, cells)
            assert got[0].tolist() == want[0].tolist(), (cells, b)
            assert got[1].tolist() == want[1].tolist()
            if lc:
                assert got[2].tolist() == want[2].tolist() and got[3].tolist() == want[3].tolist()
            assert_tables_equal(e, o, descs)
        if mult == 1 and not hot:  # every partition above the average is chained
            assert e.stats()["chained_chunks"] > 0 and e.stats()["ordered_chunks"] > 0
    # update_counters through the same chained path
    descs = single_row_limits(3, seed=31)
    e = engine_with_limits(descs, 3, regions=4)
    o = H.oracle_with_limits(descs)
    for b in range(3):
        recs = H.random_records(descs, 5000, 700 + b, n_keys=25)
        e.update_records(recs)
        o.batch_records(2, recs)
        assert_tables_equal(e, o, descs)
