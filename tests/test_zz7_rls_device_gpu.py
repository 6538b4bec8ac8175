"""The RLS plan stage on the GPU (rl_rls_plan_device, and rl_rls_serve, which now plans on the device): the device plan
against the CPU plan array for array, and the served responses, metrics and counter table against the CPU stages
wrapped around the oracle (CpuHarness: plan -> oracle -> finish)."""
import numpy as np
import pytest

from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import rls_corpora as RC
from tests.test_rls import T0, CpuHarness, _gateway, _req

METHODS = [R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT]
PLAN_KEYS = ("ctr_off", "delta", "now_us", "store_index")


def _engine(limits, m, **kw):
    from limitador_b200 import Engine
    args = dict(capacity_rows=1 << 12, cells_per_row=3, max_batch=4096)
    args.update(kw)
    e = Engine(**args)
    if limits:
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
    return e


def _same_plan(got, want):
    assert got["n_store"] == want["n_store"] and got["load_counters"] == want["load_counters"]
    for k in PLAN_KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert got["ctrs"].tobytes() == want["ctrs"].tobytes()


def _responses(svc):
    return [(g, R.decode_response(b) if g == 0 else None) for g, b in svc.responses()]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(RC.corpora()))
def test_plan_device_equals_plan(name):
    limits, msgs = RC.corpora()[name]
    m = MT.Matcher()
    e = _engine(limits, m)
    buf, off = R.pack_requests(msgs)
    for headers in (R.HEADERS_NONE, R.HEADERS_DRAFT_VERSION_03):
        dev = R.RlsService(m, e, headers, 2)
        cpu = R.RlsService(m, e, headers, 3)
        for method in METHODS:
            want = cpu.plan(method, buf, off, T0)
            _same_plan(dev.plan_device(method, buf, off, T0), want)
            # finish after a device plan: the same responses as after the CPU plan
            k = want["n_store"]
            nc = int(want["ctr_off"][-1]) if k else 0
            rng = np.random.default_rng(k)
            outs = (rng.integers(0, 2, k).astype(np.uint8), np.full(k, 0xFFFFFFFF, np.uint32),
                    rng.integers(0, 9, nc).astype(np.uint64), rng.integers(0, 60_000_000, nc).astype(np.uint64))
            assert dev.finish(*outs) == cpu.finish(*outs)
        dev.close()
        cpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("headers", [R.HEADERS_NONE, R.HEADERS_DRAFT_VERSION_03])
def test_serve_equals_the_cpu_stages_around_the_oracle(headers, threads):
    limits, reqs = _gateway(17, 2500)
    msgs = [_req(ns, descs, hits) for ns, descs, hits in reqs] + RC.mutations(5, 300)[1] + RC.nul_bytes()[1]
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits, headers=headers, threads=threads, use_limit_name_label=True)
    m = MT.Matcher()
    e = _engine(limits, m)
    svc = R.RlsService(m, e, headers, threads, True)
    for step, method in enumerate([R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT, R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT]):
        now = T0 + step * 5_000_000
        want = h.call(method, msgs, now)
        svc.serve(method, buf, off, now)
        assert _responses(svc) == want, (step, method)
    assert svc.metrics() == h.svc.metrics()
    t = svc.timings()
    assert t["plan_us"] > 0 and t["store_us"] > 0 and t["finish_us"] > 0
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


@pytest.mark.gpu
def test_limits_added_updated_and_deleted_between_serve_calls():
    """The service re-uploads the matcher image when its generation moved: every change shows in the next batch."""
    limits, reqs = _gateway(23, 1500)
    msgs = [_req(ns, descs, hits) for ns, descs, hits in reqs]
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits[:3], threads=2)
    m = MT.Matcher()
    e = _engine(limits[:3], m)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)

    def both_add(l):
        d = m.add_limit(*l)
        e.limits_set(np.array([d]))
        dh = h.m.add_limit(*l)
        h.o.limit_set(int(dh["limit_id"]), int(dh["ns_id"]), int(dh["max_value"]), int(dh["window_us"]), bool(dh["qualified"]))
        return int(d["limit_id"])

    def both_delete(lid):
        m.delete_limit(lid)
        e.limits_delete([lid])
        h.m.delete_limit(lid)
        h.o.limit_delete(lid)

    changes = [lambda: both_add(limits[3]), lambda: both_add(limits[4]),
               lambda: both_add(limits[0][:1] + (1,) + limits[0][2:]),  # max_value 5 -> 1
               lambda: both_delete(1), lambda: both_add(limits[1]),     # back, now the newest limit of "api"
               lambda: None]
    for step, change in enumerate(changes):
        change()
        now = T0 + step * 61_000_000
        want = h.call(R.SHOULD_RATE_LIMIT, msgs, now)
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        assert _responses(svc) == want, step
    assert svc.metrics() == h.svc.metrics()


@pytest.mark.gpu
def test_a_65536_request_batch():
    limits, reqs = _gateway(29, 65536)
    msgs = [_req(ns, descs, hits) for ns, descs, hits in reqs]
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits, threads=8)
    m = MT.Matcher()
    e = _engine(limits, m, capacity_rows=1 << 14, max_batch=65536, max_counters=4 * 65536)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 8)
    want = h.call(R.SHOULD_RATE_LIMIT, msgs, T0)
    _same_plan(svc.plan_device(R.SHOULD_RATE_LIMIT, buf, off, T0), h.last_plan)
    svc.serve(R.SHOULD_RATE_LIMIT, buf, off, T0)
    assert _responses(svc) == want
    assert svc.metrics() == h.svc.metrics()


@pytest.mark.gpu
def test_a_50_counter_namespace_on_a_wide_engine():
    from limitador_b200 import Engine
    limits = RC.wide_limits()
    msgs = RC.wide_messages(11, 1500)
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits, threads=2)
    h.m.set_counter_cap(64)
    planning = Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=64)  # the CPU plan takes the engine's maximum
    h.svc = R.RlsService(h.m, planning, R.HEADERS_DRAFT_VERSION_03, 2)
    m = MT.Matcher()
    m.set_counter_cap(64)
    e = _engine(limits, m, cells_per_row=7, max_counters=4096 * 50, max_counters_per_request=64)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)
    for step in range(3):
        now = T0 + step * 20_000_000
        want = h.call(R.SHOULD_RATE_LIMIT, msgs, now)
        assert int(np.diff(h.last_plan["ctr_off"]).max()) == 50
        svc.serve(R.SHOULD_RATE_LIMIT, buf, off, now)
        assert _responses(svc) == want
    _same_plan(svc.plan_device(R.CHECK_RATE_LIMIT, buf, off, T0), h.svc.plan(R.CHECK_RATE_LIMIT, buf, off, T0))
    assert svc.metrics() == h.svc.metrics()
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


@pytest.mark.gpu
def test_cap_above_the_engine_refuses_only_the_oversize_requests():
    """The matcher's cap (40) raised past a default engine's 16: only the requests of more than 16 counters get gRPC 14;
    the rest is served as a service whose cap is the engine's own serves it."""
    limits = RC.over_cap_limits(30)
    msgs = RC.over_cap_messages()
    buf, off = R.pack_requests(msgs)
    h = CpuHarness(limits, threads=2)
    h.m.set_counter_cap(16)
    m = MT.Matcher()
    m.set_counter_cap(40)
    e = _engine(limits, m)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 2)
    want = h.call(R.SHOULD_RATE_LIMIT, msgs, T0)
    svc.serve(R.SHOULD_RATE_LIMIT, buf, off, T0)
    got = _responses(svc)
    assert got == want
    assert [g for g, _ in got] == [R.GRPC_UNAVAILABLE, 0, 0, 0] * 8
