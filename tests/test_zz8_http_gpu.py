"""The HTTP API on the GPU (rl_http_plan_device, rl_http_serve): the device plan against the CPU plan array for array,
and the served responses, metrics and counter table against the CPU stages wrapped around the oracle (HttpHarness:
plan -> oracle, one call per run -> finish)."""
import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import http_corpora as HC
from tests import rls_corpora as RC
from tests.http_corpora import T0, HttpHarness

ENDPOINTS = [HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT]
PLAN_KEYS = ("ctr_off", "delta", "now_us", "load_counters", "store_index")


def _engine(limits, m, **kw):
    from limitador_b200 import Engine
    args = dict(capacity_rows=1 << 12, cells_per_row=3, max_batch=4096)
    args.update(kw)
    e = Engine(**args)
    if limits:
        e.limits_set(np.array([m.add_limit(*l) for l in limits]))
    return e


def _same_plan(got, want):
    assert got["n_store"] == want["n_store"]
    for k in PLAN_KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert got["ctrs"].tobytes() == want["ctrs"].tobytes()


def _bodies(rng, n, headers=(None, None, "DraftVersion03", "other")):
    infos = HC.random_infos(rng, n)
    return [HA.encode_info(ns, v, d, headers[int(rng.integers(0, len(headers)))]) for ns, v, d, _ in infos]


@pytest.mark.gpu
def test_plan_device_equals_plan():
    rng = np.random.default_rng(1)
    bodies = _bodies(rng, 1500) + HC.corpus_bodies(rng, 600) + \
        [HA.encode_info("api", {"method": "GET", "user": "a\x00b"}, 1), b'{"namespace":"a\\u0070i","values":{"user":"u1"},"delta":1}']
    buf, off = HA.pack_bodies(bodies)
    m = MT.Matcher()
    e = _engine(HC.GATEWAY_LIMITS, m)
    dev = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, 2))
    cpu = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, 3))
    for ep in ENDPOINTS:
        want = cpu.plan(ep, buf, off, T0)
        _same_plan(dev.plan_device(ep, buf, off, T0), want)
        k = want["n_store"]
        nc = int(want["ctr_off"][-1]) if k else 0
        outs = (rng.integers(0, 2, k).astype(np.uint8), np.full(k, 0xFFFFFFFF, np.uint32),
                rng.integers(0, 9, nc).astype(np.uint64), rng.integers(0, 60_000_000, nc).astype(np.uint64))
        assert dev.finish(*outs) == cpu.finish(*outs)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("headers", ["off", "on", "mixed"])
def test_serve_equals_the_cpu_stages_around_the_oracle(headers, threads):
    rng = np.random.default_rng(7 + threads)
    hs = {"off": (None,), "on": ("DraftVersion03",), "mixed": (None, "DraftVersion03", "other")}[headers]
    bodies = _bodies(rng, 2500, hs) + HC.corpus_bodies(rng, 300)
    buf, off = HA.pack_bodies(bodies)
    h = HttpHarness(HC.GATEWAY_LIMITS, threads=threads, use_limit_name_label=True)
    m = MT.Matcher()
    e = _engine(HC.GATEWAY_LIMITS, m)
    api = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, threads, True))
    for step, ep in enumerate([HA.CHECK_AND_REPORT, HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT, HA.CHECK]):
        now = T0 + step * 5_000_000
        want = h.call(ep, bodies, now)
        api.serve(ep, buf, off, now)
        assert api.responses() == want, (step, ep)
        t = api.timings()
        assert t["store_calls"] == len(h.runs)
        if ep == HA.CHECK_AND_REPORT:
            assert (t["store_calls"] > 100) == (headers == "mixed")
    assert api.metrics() == h.api.metrics()
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


@pytest.mark.gpu
def test_limits_added_updated_and_deleted_between_serve_calls():
    limits = HC.GATEWAY_LIMITS
    rng = np.random.default_rng(23)
    bodies = _bodies(rng, 1500)
    buf, off = HA.pack_bodies(bodies)
    h = HttpHarness(limits[:3], threads=2)
    m = MT.Matcher()
    e = _engine(limits[:3], m)
    api = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, 2))

    def both_add(l):
        d = m.add_limit(*l)
        e.limits_set(np.array([d]))
        dh = h.m.add_limit(*l)
        h.o.limit_set(int(dh["limit_id"]), int(dh["ns_id"]), int(dh["max_value"]), int(dh["window_us"]), bool(dh["qualified"]))

    def both_delete(lid):
        m.delete_limit(lid)
        e.limits_delete([lid])
        h.m.delete_limit(lid)
        h.o.limit_delete(lid)

    changes = [lambda: both_add(limits[3]), lambda: both_add(limits[4]), lambda: both_add(limits[0][:1] + (1,) + limits[0][2:]),
               lambda: both_delete(1), lambda: both_add(limits[1]), lambda: None]
    for step, change in enumerate(changes):
        change()
        now = T0 + step * 61_000_000
        want = h.call(HA.CHECK_AND_REPORT, bodies, now)
        api.serve(HA.CHECK_AND_REPORT, buf, off, now)
        assert api.responses() == want, step
    assert api.metrics() == h.api.metrics()


@pytest.mark.gpu
def test_a_65536_body_batch():
    rng = np.random.default_rng(29)
    bodies = _bodies(rng, 65536, (None, "DraftVersion03"))
    buf, off = HA.pack_bodies(bodies)
    h = HttpHarness(HC.GATEWAY_LIMITS, threads=8)
    m = MT.Matcher()
    e = _engine(HC.GATEWAY_LIMITS, m, capacity_rows=1 << 14, max_batch=65536, max_counters=4 * 65536)
    api = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, 8))
    want = h.call(HA.CHECK_AND_REPORT, bodies, T0)
    _same_plan(api.plan_device(HA.CHECK_AND_REPORT, buf, off, T0), h.last_plan)
    api.serve(HA.CHECK_AND_REPORT, buf, off, T0)
    assert api.responses() == want
    assert api.timings()["store_calls"] == len(h.runs) > 1024  # more store calls than the first read brings back
    assert api.metrics() == h.api.metrics()


@pytest.mark.gpu
def test_a_50_counter_namespace_on_a_wide_engine():
    from limitador_b200 import Engine
    limits = RC.wide_limits()
    rng = np.random.default_rng(11)
    bodies = []
    for msg in RC.wide_messages(11, 1500):
        ns, descs, _ = R.decode_request(msg)
        bodies.append(HA.encode_info(ns, dict(descs[0]) if descs else {}, int(rng.integers(0, 3)),
                                     [None, "DraftVersion03"][int(rng.integers(0, 2))]))
    buf, off = HA.pack_bodies(bodies)
    h = HttpHarness(limits, threads=2)
    h.m.set_counter_cap(64)
    planning = Engine(capacity_rows=1 << 10, max_batch=64, max_counters_per_request=64)  # the CPU plan takes the engine's maximum
    h.rls = R.RlsService(h.m, planning, R.HEADERS_NONE, 2)
    h.api = HA.HttpApi(h.rls)
    m = MT.Matcher()
    m.set_counter_cap(64)
    e = _engine(limits, m, cells_per_row=7, max_counters=4096 * 50, max_counters_per_request=64)
    api = HA.HttpApi(R.RlsService(m, e, R.HEADERS_NONE, 2))
    for step in range(3):
        now = T0 + step * 20_000_000
        want = h.call(HA.CHECK_AND_REPORT, bodies, now)
        assert int(np.diff(h.last_plan["ctr_off"]).max()) > 16  # (values binds descriptors[0] only: up to 42 of the 50 apply)
        api.serve(HA.CHECK_AND_REPORT, buf, off, now)
        assert api.responses() == want
    assert api.metrics() == h.api.metrics()
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))


@pytest.mark.gpu
def test_rls_and_http_batches_interleaved_on_one_service():
    """One service, one engine, one metrics text: RLS and HTTP batches alternate against the same counters."""
    from tests.test_rls import CpuHarness
    limits = HC.GATEWAY_LIMITS
    rng = np.random.default_rng(31)
    h = HttpHarness(limits, threads=3, use_limit_name_label=True)
    hr = CpuHarness(limits, headers=R.HEADERS_DRAFT_VERSION_03, threads=3, use_limit_name_label=True)
    hr.m, hr.o, hr.descs = h.m, h.o, h.descs  # one matcher and one oracle behind both CPU surfaces
    hr.svc = h.rls
    h.rls.close()
    h.rls = R.RlsService(h.m, None, R.HEADERS_DRAFT_VERSION_03, 3, True)
    h.api = HA.HttpApi(h.rls)
    hr.svc = h.rls
    m = MT.Matcher()
    e = _engine(limits, m)
    svc = R.RlsService(m, e, R.HEADERS_DRAFT_VERSION_03, 3, True)
    api = HA.HttpApi(svc)
    for step in range(6):
        now = T0 + step * 3_000_000
        if step % 2:
            msgs = [R.encode_request(ns, [list(v.items())], d) for ns, v, d, _ in HC.random_infos(rng, 800)]
            want = hr.call(R.SHOULD_RATE_LIMIT, msgs, now)
            svc.serve(R.SHOULD_RATE_LIMIT, *R.pack_requests(msgs), now)
            assert [(g, R.decode_response(b) if g == 0 else None) for g, b in svc.responses()] == want
        else:
            bodies = _bodies(rng, 800)
            want = h.call(HA.CHECK_AND_REPORT, bodies, now)
            api.serve(HA.CHECK_AND_REPORT, *HA.pack_bodies(bodies), now)
            assert api.responses() == want
    assert svc.metrics() == api.metrics() == h.rls.metrics()
    assert H.normalise_dump(e.dump(), np.array(h.descs)) == H.normalise_dump(h.o.dump(), np.array(h.descs))
