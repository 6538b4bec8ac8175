"""Limits in the matcher's boolean dialect served on the GPU (rl_rls_serve, rl_http_serve): responses, metrics and the
counter table against the CPU plan wrapped around the oracle, in both header modes, with 1 and 4 workers, across image
refreshes (limits added and deleted, the dialect changed), on a 65 536-request batch and on the 50-counter wide engine;
GET /counters lists the counters of boolean limits with their variables; and an ==-only limit set serves byte for byte
the same under both dialects."""
import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import boolean_corpora as BC
from tests import helpers as H
from tests.test_match_boolean_emu import boolean_harness
from tests.test_rls import T0, CpuHarness

METHODS = [R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT]


def _engine(limits, m, **kw):
    from limitador_b200 import Engine
    args = dict(capacity_rows=1 << 14, cells_per_row=3, max_batch=4096)
    args.update(kw)
    e = Engine(**args)
    if limits:
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
    return e


def _cpu(limits, headers=R.HEADERS_DRAFT_VERSION_03, threads=1, cap=None, planning_engine=None):
    """tests/test_rls.CpuHarness over a matcher in the boolean dialect."""
    h = CpuHarness([], headers, threads)
    h.svc.close()
    h.m = BC.matcher([], cap)
    for (ns, mx, secs, conds, vars_, name) in limits:
        d = h.m.add_limit(ns, mx, secs, conds, vars_, name)
        h.descs.append(d)
        h.o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    h.svc = R.RlsService(h.m, planning_engine, headers, threads)
    return h


def _responses(svc):
    return [(g, R.decode_response(b) if g == 0 else None) for g, b in svc.responses()]


def _dump_equal(e, h):
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("headers", [R.HEADERS_NONE, R.HEADERS_DRAFT_VERSION_03])
def test_rls_serve_equals_the_cpu_plan_around_the_oracle(headers, threads):
    msgs = BC.rls_messages(3, 3000)
    buf, off = R.pack_requests(msgs)
    h = _cpu(BC.LIMITS, headers, threads)
    m = BC.matcher([])
    e = _engine(BC.LIMITS, m)
    svc = R.RlsService(m, e, headers, threads)
    for step, method in enumerate(METHODS + METHODS[:2]):
        now = T0 + step * 4_000_000
        want = h.call(method, msgs, now)
        p = svc.plan_device(method, buf, off, now)
        assert p["n_store"] == h.last_plan["n_store"] and p["ctrs"].tobytes() == h.last_plan["ctrs"].tobytes()
        svc.serve(method, buf, off, now)
        assert _responses(svc) == want, (step, method)
    assert svc.metrics() == h.svc.metrics()
    _dump_equal(e, h)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4])
def test_http_serve_equals_the_cpu_plan_around_the_oracle(threads):
    bodies = BC.http_bodies(4, 3000)
    buf, off = HA.pack_bodies(bodies)
    h = boolean_harness(BC.LIMITS, threads)
    m = BC.matcher([])
    e = _engine(BC.LIMITS, m)
    api = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, threads))
    for step, ep in enumerate([HA.CHECK_AND_REPORT, HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT]):
        now = T0 + step * 4_000_000
        want = h.call(ep, bodies, now)
        api.serve(ep, buf, off, now)
        assert api.responses() == want, (step, ep)
    assert api.metrics() == h.api.metrics()
    _dump_equal(e, h)


@pytest.mark.gpu
def test_the_image_refreshes_after_limit_changes_and_a_dialect_change():
    """The matcher starts in the table dialect with its ==-only limit; boolean limits come after a dialect change, then a
    delete and a re-add: every change shows in the next served batch."""
    msgs = BC.rls_messages(5, 2000)
    buf, off = R.pack_requests(msgs)
    eq_only = BC.LIMITS[6]
    h = _cpu([], threads=2)
    m = MT.Matcher()
    e = _engine([eq_only], m)
    h.descs.append(h.m.add_limit(*eq_only))
    d = h.descs[0]
    h.o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)

    def both_add(l):
        dd = m.add_limit(*l)
        e.limits_set(np.array([dd]))
        dh = h.m.add_limit(*l)
        h.descs.append(dh)
        h.o.limit_set(int(dh["limit_id"]), int(dh["ns_id"]), int(dh["max_value"]), int(dh["window_us"]), bool(dh["qualified"]))
        assert int(dd["limit_id"]) == int(dh["limit_id"])

    def both_delete(lid):
        m.delete_limit(lid)
        e.limits_delete([lid])
        h.m.delete_limit(lid)
        h.o.limit_delete(lid)

    def dialect():
        m.set_dialect("boolean")
        with pytest.raises(MT.MatcherError):
            MT.Matcher().add_limit(*BC.LIMITS[0])

    changes = [lambda: None, dialect, lambda: both_add(BC.LIMITS[0]), lambda: both_add(BC.LIMITS[5]), lambda: both_delete(1),
               lambda: both_add(BC.LIMITS[0]), lambda: both_add(BC.LIMITS[3])]
    for step, change in enumerate(changes):
        change()
        now = T0 + step * 61_000_000
        want = h.call(R.SHOULD_RATE_LIMIT, msgs, now)
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        assert _responses(svc) == want, step
    assert svc.metrics() == h.svc.metrics()
    _dump_equal(e, h)


@pytest.mark.gpu
def test_a_65536_request_batch():
    msgs = BC.rls_messages(7, 65536)
    buf, off = R.pack_requests(msgs)
    h = _cpu(BC.LIMITS, threads=8)
    m = BC.matcher([])
    e = _engine(BC.LIMITS, m, max_batch=65536, max_counters=8 * 65536)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 8)
    want = h.call(R.SHOULD_RATE_LIMIT, msgs, T0)
    svc.serve(R.SHOULD_RATE_LIMIT, buf, off, T0)
    assert _responses(svc) == want
    bodies = BC.http_bodies(8, 65536)
    hh = boolean_harness(BC.LIMITS, 8)
    api = HA.HttpApi(svc)
    hb, ob = HA.pack_bodies(bodies)
    hh.o = h.o  # one store: the HTTP batch continues the RLS batch's counters
    hh.descs = h.descs
    api.serve(HA.CHECK_AND_REPORT, hb, ob, T0 + 1_000_000)
    assert api.responses() == hh.call(HA.CHECK_AND_REPORT, bodies, T0 + 1_000_000)
    _dump_equal(e, h)


@pytest.mark.gpu
def test_a_50_counter_namespace_on_a_wide_engine():
    from limitador_b200 import Engine
    limits = BC.wide_limits()
    msgs = BC.wide_messages(11, 1500)
    buf, off = R.pack_requests(msgs)
    planning = Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=64)  # the CPU plan takes the engine's maximum
    h = _cpu(limits, threads=2, cap=64, planning_engine=planning)
    m = BC.matcher([], cap=64)
    e = _engine(limits, m, cells_per_row=7, max_counters=4096 * 50, max_counters_per_request=64)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)
    for step in range(3):
        now = T0 + step * 20_000_000
        want = h.call(R.SHOULD_RATE_LIMIT, msgs, now)
        assert int(np.diff(h.last_plan["ctr_off"]).max()) == 50
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        assert _responses(svc) == want
    assert svc.metrics() == h.svc.metrics()
    _dump_equal(e, h)


@pytest.mark.gpu
def test_get_counters_lists_the_counters_of_boolean_limits_with_their_variables():
    from tests import test_zz9_counter_vars_gpu as CV

    class BoolService(CV.Service):
        def __init__(self, limits):
            from limitador_b200 import Engine
            self.m = BC.matcher([])
            self.e = Engine(capacity_rows=1 << 14, cells_per_row=3, max_batch=1 << 17)
            self.limits = list(limits)
            self.descs = [self.m.add_limit(*l) for l in limits]
            self.e.limits_set(np.array(self.descs))
            self.rls = R.RlsService(self.m, self.e, R.HEADERS_NONE, 2)
            self.api = HA.HttpApi(self.rls)
            self.rls.keep_counter_vars(1 << 16, 1 << 22)
            self.values = {}

    s = BoolService(BC.LIMITS)
    rng = np.random.default_rng(9)
    for step in range(3):
        now = T0 + step * 3_000_000
        infos = [(str(rng.choice(["api", "admin"])), dict(BC.descriptors(rng)[0]), 1, None) for _ in range(1500)]
        s.http(HA.CHECK_AND_REPORT, infos, now)
        reqs = [(str(rng.choice(["api", "admin"])), BC.descriptors(rng)[0]) for _ in range(1500)]
        s.rls_serve(R.SHOULD_RATE_LIMIT, reqs, now)
    for ns in ("api", "admin"):
        got = s.api.get_counters(ns, now + 1)
        assert got == s.expected(ns, now + 1), ns
        assert b'"set_variables":{"descriptors[0].user":' in got[1]
    assert s.rls.counter_vars_stats()["dropped"] == 0


@pytest.mark.gpu
def test_an_equality_only_limit_set_serves_the_same_under_both_dialects():
    limits = []
    for ns in range(8):
        limits.append((f"ns{ns}", 100, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"))
        limits.append((f"ns{ns}", 1000, 3600, [], ["descriptors[0].user"], "hourly-per-user"))
        limits.append((f"ns{ns}", 1 << 40, 60, ["descriptors[0].method != 'OPTIONS'"], [], None))
    rng = np.random.default_rng(2)
    msgs = [R.encode_request(f"ns{int(rng.integers(0, 9))}", [[("method", str(rng.choice(["GET", "POST", "OPTIONS"]))),
                                                                ("user", f"u{int(rng.integers(0, 40))}")]], 1) for _ in range(8192)]
    buf, off = R.pack_requests(msgs)
    sides = []
    for dialect in ("table", "boolean"):
        m = MT.Matcher(dialect=dialect)
        e = _engine(limits, m, max_batch=8192)
        sides.append((e, R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)))
    for step in range(4):
        out = []
        for e, svc in sides:
            svc.serve(R.SHOULD_RATE_LIMIT, buf, off, T0 + step * 10_000_000)
            out.append(svc.responses())
        assert out[0] == out[1]
    assert sides[0][0].dump() == sides[1][0].dump()
    assert sides[0][1].metrics() == sides[1][1].metrics()
