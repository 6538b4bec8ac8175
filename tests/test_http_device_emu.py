"""The HTTP device plan (limitador_b200/csrc/rl_http_dev.cuh) without a GPU: the kernels run under tests/emu/cuda_shim.h
(tests/emu/emu_http.cpp) over the matcher's device image, and every array of the plan view, the store index, the outcome
class of every body and the store calls must equal the CPU plan's (rl_http_plan) on the same bodies.  The driver runs
once more under ASan + UBSan."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

from limitador_b200 import engine as E
from limitador_b200 import http_api as HA
from limitador_b200 import rls as R
from tests import helpers as H
from tests import http_corpora as HC
from tests import rls_corpora as RC
from tests.http_corpora import HttpHarness
from tests.test_rls_device_emu import _matcher, matcher_image

T0 = 1_700_000_000_000_000
REQ_DTYPE = np.dtype([("kind", "<u4"), ("store", "<u4"), ("dom_off", "<u4"), ("dom_len", "<u4"), ("headers", "<u4"), ("_pad", "<u4"),
                      ("delta", "<u8")])
ENDPOINTS = [HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT]


@functools.cache
def _emu():
    L = H.host_lib("emu_http.cpp", "librl_emu_http.so")
    vp, u64 = C.c_void_p, C.c_uint64
    L.emu_http_plan.restype = u64
    L.emu_http_plan.argtypes = [vp, C.c_int, u64, vp, vp, u64, C.c_uint32, vp, vp, vp, u64, vp, vp, vp, vp, vp, C.POINTER(u64),
                                C.POINTER(C.c_uint32)]
    L.emu_http_seed.argtypes = [u64]
    return L


def emu_plan(m, endpoint, bodies, now_us=T0, engine_max=16):
    buf, off = HA.pack_bodies(bodies)
    if len(buf) == 0:
        buf = np.zeros(1, np.uint8)
    img, _ = matcher_image(m)
    n = len(bodies)
    req = np.zeros(max(n, 1), REQ_DTYPE)
    ctr_off = np.zeros(n + 1, np.uint32)
    ctrs = np.zeros(64 * n + 1, E.COUNTER_DTYPE)
    delta, now, load = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint8)
    runs, ctr_run = np.zeros(3 * n + 3, np.uint32), np.zeros(2 * n + 2, np.uint32)
    n_ctr, n_runs = C.c_uint64(), C.c_uint32()
    k = _emu().emu_http_plan(img.ctypes.data, endpoint, n, buf.ctypes.data, off.ctypes.data, now_us, engine_max, req.ctypes.data,
                             ctr_off.ctypes.data, ctrs.ctypes.data, len(ctrs), delta.ctypes.data, now.ctypes.data, load.ctypes.data,
                             runs.ctypes.data, ctr_run.ctypes.data, C.byref(n_ctr), C.byref(n_runs))
    req = req[:n]
    return {"n_store": k, "ctr_off": ctr_off[:k + 1], "ctrs": ctrs[:n_ctr.value], "delta": delta[:k], "now_us": now[:k],
            "load_counters": load[:k], "store_index": req["store"].copy(), "req": req,
            "runs": runs[:3 * n_runs.value].reshape(-1, 3), "ctr_run": ctr_run[:k + n_runs.value]}


def _class(status):
    return np.where(status == 400, 1, np.where(status == 500, 5, 0))


def assert_same(m, h, endpoint, bodies, engine_max=16):
    got = emu_plan(m, endpoint, bodies, engine_max=engine_max)
    want = h.api.plan(endpoint, *HA.pack_bodies(bodies), T0)
    assert got["n_store"] == want["n_store"]
    for key in ("ctr_off", "delta", "now_us", "load_counters", "store_index"):
        assert np.array_equal(got[key], want[key]), key
    assert got["ctrs"].tobytes() == want["ctrs"].tobytes()
    # the outcome class of every body: 400 refused, 500 unshippable, else decided
    k = want["n_store"]
    nc = int(want["ctr_off"][-1]) if k else 0
    out = h.api.finish(np.zeros(k, np.uint8), np.full(k, 0xFFFFFFFF, np.uint32), np.zeros(nc, np.uint64), np.zeros(nc, np.uint64))
    kinds = got["req"]["kind"]
    assert np.array_equal(np.where(kinds == 1, 1, np.where(kinds == 5, 5, 0)), _class(np.array([s for s, _, _ in out])))
    # the store calls: maximal runs of equal flags, each with its own CSR from 0
    spans = HA.store_runs(want["load_counters"])
    assert [tuple(r[:1]) for r in got["runs"]] == [(j0,) for j0, _ in spans]
    for r, (j0, j1) in enumerate(spans):
        c0 = int(want["ctr_off"][j0])
        assert got["runs"][r][1] == c0 and got["runs"][r][2] == want["load_counters"][j0]
        assert np.array_equal(got["ctr_run"][j0 + r:j1 + r + 1], want["ctr_off"][j0:j1 + 1] - c0)
    return got


def _bodies(rng):
    infos = HC.random_infos(rng, 500)
    good = [HA.encode_info(*x) for x in infos]
    esc = [b'{"namespace":"a\\u0070i","values":{"\\u006dethod":"GET","user":"u\\u0031"},"delta":2,"response_headers":"Draft\\u0056ersion03"}',
           b'["api",{"method":"POST","user":"u2","user":"u3"},1,"x"]',
           HA.encode_info("api", {"method": "GET", "user": "a\x00b"}, 1, None), HA.encode_info("ad\x00min", {"user": "u1"}, 1, None)]
    return good + esc + HC.corpus_bodies(rng, 400)


@pytest.mark.parametrize("endpoint", ENDPOINTS)
@pytest.mark.parametrize("threads", [1, 3])
def test_device_plan_kernels_equal_the_cpu_plan(endpoint, threads):
    rng = np.random.default_rng(10 + threads)
    h = HttpHarness(HC.GATEWAY_LIMITS, threads=threads)
    bodies = _bodies(rng)
    _emu().emu_http_seed(threads)
    got = assert_same(h.m, h, endpoint, bodies)
    assert set(got["req"]["kind"].tolist()) == {1, 3, 4, 5}
    if endpoint == HA.CHECK_AND_REPORT:
        assert len(got["runs"]) > 100
    else:
        assert len(got["runs"]) == 1


def test_reference_scenarios_and_corpora():
    h = HttpHarness([HC.REF_LIMIT])
    for hd in (None, "DraftVersion03", "x"):
        body = HA.encode_info("test_namespace", {"req.method": "GET", "app.id": "1"}, 1, hd)
        for ep in ENDPOINTS:
            assert_same(h.m, h, ep, [body] * 3)
    assert_same(h.m, h, HA.CHECK, [])


def test_a_50_limit_namespace_with_requests_over_the_cap():
    """Cap 16 (a default engine's): requests that more than 16 of the 50 limits apply to are refused (500) in both plans."""
    limits = RC.wide_limits()
    m = _matcher(limits, cap=16)
    h = HttpHarness([])
    h.m = m
    h.rls = R.RlsService(m, None, R.HEADERS_NONE, 2)
    h.api = HA.HttpApi(h.rls)
    rng = np.random.default_rng(3)
    bodies = []
    for msg in RC.wide_messages(5, 300):
        ns, descs, _ = R.decode_request(msg)
        bodies.append(HA.encode_info(ns, dict(descs[0]) if descs else {}, int(rng.integers(0, 3)),
                                     [None, "DraftVersion03"][int(rng.integers(0, 2))]))
    got = assert_same(m, h, HA.CHECK_AND_REPORT, bodies, engine_max=16)
    assert (got["req"]["kind"] == 5).any() and (got["req"]["kind"] == 4).any()


def test_device_plan_driver_is_clean_under_asan_and_ubsan(tmp_path):
    """The kernels under the shim with ASan + UBSan over random and mutated bodies, each batch compared with the CPU plan
    (tests/san/san_http_dev.cpp)."""
    from tests.test_sanitizers import build_and_run
    root = H.ROOT
    csrc = os.path.join(root, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(root, "tests", "san", "san_http_dev.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(root, "include")], extra=("-std=c++17",))
    assert out.startswith("ok compared=")
