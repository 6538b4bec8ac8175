"""Requests of 17..64 counters on the GPU (rl_config.max_counters_per_request, the wide position encoding), every output
compared with the CPU oracle: verdicts, first-limited ids, remaining / ttl and the full table.  The encoding itself is
run on the host in tests/test_wide_emu.py.  Sorted last on purpose: these entry points are new."""
import ctypes as C

import numpy as np
import pytest

from limitador_b200 import Engine, EngineError, streams
from limitador_b200 import engine as E
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests.test_rls import T0, CpuHarness, _req

pytestmark = pytest.mark.gpu
SCENARIOS = [(10, 50, 10, 0), (1, 1, 1, 1), (10, 10, 10, 10), (10, 50, 10, 10)]  # limitador/benches/bench.rs:65-90


def _wide_engine(descs, cells=7, wide=64, max_batch=4096, **kw):
    e = Engine(capacity_rows=1 << 16, cells_per_row=cells, max_batch=max_batch, max_counters=max_batch * 64,
               max_counters_per_request=wide, **kw)
    e.limits_set(descs)
    return e


def _same(got, want, n):
    for k in range(n):
        assert got[k].tolist() == want[k].tolist(), f"output {k} differs"


def _tables(e, o, descs):
    assert H.normalise_dump(e.dump(), descs) == H.normalise_dump(o.dump(), descs), "table differs"


def _csr_device(e, off, ctrs, delta, now, lc):
    """rl_check_and_update_batch with every array in device memory (torch tensors)."""
    import torch
    d = torch.device("cuda")
    t = {k: torch.from_numpy(v.view(np.uint8).copy()).to(d) for k, v in
         dict(off=off, ctrs=ctrs, delta=delta, now=now).items()}
    n, m = len(delta), len(ctrs)
    lim = torch.zeros(n, dtype=torch.uint8, device=d)
    fl = torch.zeros(n, dtype=torch.int32, device=d)
    rem = torch.zeros(max(m, 1), dtype=torch.int64, device=d)
    ttl = torch.zeros(max(m, 1), dtype=torch.int64, device=d)
    p = lambda x: C.c_void_p(x.data_ptr())
    e._check(e._lib.rl_check_and_update_batch(e._h, n, p(t["off"]), p(t["ctrs"]), p(t["delta"]), p(t["now"]), int(lc),
                                              E.MEM_DEVICE, p(lim), p(fl), p(rem) if lc else None,
                                              p(ttl) if lc else None))
    e.sync()
    return (lim.cpu().numpy(), fl.cpu().numpy().view(np.uint32), rem.cpu().numpy().view(np.uint64)[:m],
            ttl.cpu().numpy().view(np.uint64)[:m])


def _scenario(scn, small):
    n_ns, n_lim, n_cond, n_var = scn
    m = MT.Matcher()
    m.set_counter_cap(max(16, n_lim))
    conds = [f"cond_{i} == '1'" for i in range(n_cond)]
    vars_ = [f"var_{j}" for j in range(n_var)]
    descs = [m.add_limit(str(ns), (3 + (l * 7 + ns) % 11) if small else 2 ** 64 - 1, l * 60 + 10, conds, vars_)
             for ns in range(n_ns) for l in range(n_lim)]
    return m, np.array(descs, dtype=E.LIMIT_DESC_DTYPE)


def _scenario_batch(m, scn, n, rng):
    """CSR counters of n requests through the matcher; var_0 takes one of three values and the other variables are "1",
    so that keys repeat and small maxima bite."""
    n_ns, n_lim, n_cond, n_var = scn
    off, ctrs = [0], []
    ns_ids = [m.namespace_id(str(ns)) for ns in range(n_ns)]
    for i in range(n):
        ns = ns_ids[int(rng.integers(0, n_ns))]
        root = {f"cond_{c}": "1" for c in range(n_cond)}
        root.update({f"var_{v}": str(int(rng.integers(0, 3))) if v == 0 else "1" for v in range(n_var)})
        c = m.counters(ns, root=root)
        assert len(c) == n_lim
        ctrs.append(c)
        off.append(off[-1] + len(c))
    return np.array(off, dtype=np.uint32), np.concatenate(ctrs).astype(E.COUNTER_DTYPE)


@pytest.mark.parametrize("small", [False, True], ids=["as-written", "small-maxima"])
@pytest.mark.parametrize("scn", SCENARIOS, ids=["10x50x10x0", "1x1x1x1", "10x10x10x10", "10x50x10x10"])
def test_reference_scenarios_three_calls_match_oracle(scn, small):
    m, descs = _scenario(scn, small)
    rng = np.random.default_rng(hash(scn) & 0xFFFF)
    for mode in (1, 2, 0):  # is_rate_limited, update_counters, check_rate_limited_and_update
        e = _wide_engine(descs)
        o = H.oracle_with_limits(descs)
        for b in range(3):
            off, ctrs = _scenario_batch(m, scn, 600, rng)
            n = len(off) - 1
            delta = np.ones(n, dtype=np.uint64)
            now = np.full(n, T0 + b * 5_000_000, dtype=np.uint64) + np.arange(n, dtype=np.uint64)
            want = o.batch_csr(mode, off, ctrs, delta, now, mode == 0)
            if mode == 1:
                _same(e.is_within_limits_batch(off, ctrs, delta, now), want, 2)
            elif mode == 2:
                e.update_batch(off, ctrs, delta, now)
            else:
                _same(e.check_and_update_batch(off, ctrs, delta, now, True), want, 4)
                if small and b == 2 and scn[1] > 16:
                    assert len(set(want[1].tolist())) > 2  # the first-limited limit varies: several rows are involved
            _tables(e, o, descs)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("cells", [1, 3, 7])
def test_random_wide_csr_streams_match_oracle(device, cells):
    descs = H.wide_limits(cells)
    e = _wide_engine(descs, cells)
    o = H.oracle_with_limits(descs)
    for b in range(4):
        lc = b % 2 == 1
        off, ctrs, delta, now = H.wide_stream(descs, 500, 50 + b, n_keys=4, monotone=(b != 2), min_ctrs=1 if b == 3 else 17)
        want = o.batch_csr(0, off, ctrs, delta, now, lc)
        got = _csr_device(e, off, ctrs, delta, now, lc) if device else e.check_and_update_batch(off, ctrs, delta, now, lc)
        _same(got, want, 4 if lc else 2)
        _tables(e, o, descs)
    off, ctrs, delta, now = H.wide_stream(descs, 300, 99)
    e.update_batch(off, ctrs, delta, now)
    o.batch_csr(2, off, ctrs, delta, now)
    _tables(e, o, descs)


def test_mixed_narrow_and_wide_batch_matches_oracle():
    descs = H.wide_limits(5)
    e = _wide_engine(descs, 3)
    o = H.oracle_with_limits(descs)
    off, ctrs, delta, now = H.wide_stream(descs, 2000, 77, min_ctrs=1)
    sizes = np.diff(off)
    assert sizes.max() > 16 and sizes.min() <= 16
    _same(e.check_and_update_batch(off, ctrs, delta, now, True), o.batch_csr(0, off, ctrs, delta, now, True), 4)
    _tables(e, o, descs)


@pytest.mark.parametrize("cells", [3, 7])
def test_records_of_wide_namespaces_with_load_counters(cells):
    descs = H.wide_limits(cells + 20, sizes=(20, 64, 33, 2, 5))
    e = _wide_engine(descs, cells)
    o = H.oracle_with_limits(descs)
    for b in range(4):
        recs = H.random_records(descs, 1500, 300 + b, n_keys=4, monotone=(b != 1))
        lc = b != 2
        got = e.check_and_update_records(recs, lc, stride=64)
        want = o.batch_records(0, recs, lc, 64)
        _same(got, want, 4 if lc else 2)
        _tables(e, o, descs)
    recs = H.random_records(descs, 800, 999)
    e.update_records(recs)
    o.batch_records(2, recs)
    _tables(e, o, descs)
    # is_within_limits over namespaces of up to 64 limits
    recs = H.random_records(descs, 800, 1000)
    _same(e.is_within_limits_records(recs), o.batch_records(1, recs), 2)


def test_c2_through_a_wide_engine_is_byte_identical_to_a_default_engine():
    w = streams.WORKLOADS["C2"](batch=8192, n_rows=5000, n_ns=8)
    a = Engine(capacity_rows=1 << 14, cells_per_row=7, max_batch=8192)
    b = Engine(capacity_rows=1 << 14, cells_per_row=7, max_batch=8192, max_counters_per_request=64)
    for e in (a, b):
        e.limits_set(w.limits)
    for s in range(4):
        recs = w.batch_records(s)
        ga, gb = a.check_and_update_records(recs, s % 2 == 1, stride=4), b.check_and_update_records(recs, s % 2 == 1, stride=4)
        for x, y in zip(ga, gb):
            assert (x is None and y is None) or x.tobytes() == y.tobytes()
    assert sorted(a.dump()) == sorted(b.dump())


def test_a_request_over_the_engines_maximum_is_refused_with_the_table_untouched():
    descs = np.array([(k, 0, 1 + k % 3, 1, 5, 60_000_000) for k in range(40)], dtype=E.LIMIT_DESC_DTYPE)
    e = _wide_engine(descs, 3, wide=32)
    ok = np.array([(k, 0, 1, 0) for k in range(32)], dtype=E.COUNTER_DTYPE)
    e.check_and_update_batch(np.array([0, 32], dtype=np.uint32), ok, [1], [T0])
    before = sorted(e.dump())
    assert len(before) == 32
    many = np.array([(k, 0, 2, 0) for k in range(33)], dtype=E.COUNTER_DTYPE)
    off = np.array([0, 32, 65], dtype=np.uint32)
    with pytest.raises(EngineError, match="more than 32 counters.*before the table was touched"):
        e.check_and_update_batch(off, np.concatenate([ok, many]), [1, 1], [T0 + 1, T0 + 1])
    with pytest.raises(EngineError, match="more than 32 counters"):
        e.update_batch(off, np.concatenate([ok, many]), [1, 1], [T0 + 1, T0 + 1])
    assert sorted(e.dump()) == before
    # the record path: a namespace with more limits than the engine takes
    with pytest.raises(EngineError, match="more than 32 limits"):
        e.check_and_update_records(H.random_records(descs, 10, 1), False)


@pytest.mark.parametrize("bad", [1, 15, 65, 1000])
def test_engine_creation_refuses_a_maximum_out_of_range(bad):
    with pytest.raises(EngineError, match="max_counters_per_request"):
        Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=bad)
    for good in (0, 16, 17, 64):
        Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=good).close()


def test_is_within_limits_takes_any_number_of_counters_on_a_default_engine():
    descs = H.wide_limits(3, sizes=(50,))
    e = Engine(capacity_rows=1 << 12, cells_per_row=7, max_batch=4096, max_counters=4096 * 50)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    off, ctrs, delta, now = H.wide_stream(descs, 400, 5, min_ctrs=50)
    assert int(np.diff(off).min()) == 50
    _same(e.is_within_limits_batch(off, ctrs, delta, now), o.batch_csr(1, off, ctrs, delta, now), 2)


def _wide_rls_limits():
    limits = []
    for l in range(50):
        vars_ = ["descriptors[0].user"] if l % 3 else []
        limits.append(("wide", 2 + l % 5, 60 + l, ["descriptors[0].k == '1'"], vars_, f"l{l}" if l % 2 else None))
    limits.append(("api", 4, 60, [], ["descriptors[0].user"], "per-user"))
    return limits


def test_rls_should_rate_limit_over_a_50_limit_namespace_equals_the_cpu_mirror():
    limits = _wide_rls_limits()
    rng = np.random.default_rng(4)
    msgs = []
    for _ in range(1500):
        ns = "wide" if rng.random() < 0.8 else "api"
        d0 = [("k", str(rng.choice(["1", "1", "2"]))), ("user", f"u{int(rng.integers(0, 6))}")]
        msgs.append(_req(ns, [d0], int(rng.choice([0, 1, 1, 2]))))
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits, headers=R.HEADERS_DRAFT_VERSION_03, threads=2)
    h.m.set_counter_cap(64)
    # the mirror plans with a wide engine's maximum (the engine decides nothing: the oracle does)
    planning = Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=64)
    h.svc = R.RlsService(h.m, planning, R.HEADERS_DRAFT_VERSION_03, 2)
    m = MT.Matcher()
    m.set_counter_cap(64)
    e = Engine(capacity_rows=1 << 12, cells_per_row=7, max_batch=4096, max_counters=4096 * 50, max_counters_per_request=64)
    e.limits_set(np.array([m.add_limit(*l) for l in limits]))
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)
    for step in range(3):
        now = T0 + step * 20_000_000
        want = h.call(R.SHOULD_RATE_LIMIT, msgs, now)
        assert int(np.diff(h.last_plan["ctr_off"]).max()) == 50
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        got = [(g, R.decode_response(b) if g == 0 else None) for g, b in svc.responses()]
        assert got == want
    assert svc.metrics() == h.svc.metrics()
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


def test_front_check_and_update_with_50_counters():
    descs = H.wide_limits(9, sizes=(50,))
    e = _wide_engine(descs, 7)
    o = H.oracle_with_limits(descs)
    f = E.Front(e, max_batch=64, max_delay_us=0)
    off, ctrs, delta, now = H.wide_stream(descs, 60, 8, min_ctrs=50)
    for i in range(len(delta)):
        c = ctrs[off[i]:off[i + 1]]
        lim, first, _, rem, ttl = f.check_and_update(c, int(delta[i]), int(now[i]), load_counters=True)
        wl, wi, wr, wt = o.check_and_update(c, int(delta[i]), True, int(now[i]))
        assert lim == wl and rem.tolist() == list(wr) and ttl.tolist() == list(wt)
        assert first == (int(c[wi]["limit_id"]) if wl else None)
    f.close()
    _tables(e, o, descs)
