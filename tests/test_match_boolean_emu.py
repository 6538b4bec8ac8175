"""The device plans with limits in the matcher's boolean dialect, without a GPU: k_rls_plan and k_http_plan run under
tests/emu/cuda_shim.h over the matcher's image (tests and atoms sections), and every array of the store call, the store
index and the status of every request must equal the CPU plans' (rl_rls_plan, rl_http_plan), for all three RLS methods
and all three HTTP endpoints.  The corpora hold an `in` list, a startsWith + != group, presence tests, a group of six
atoms and a 50-limit namespace on a wide matcher.  The driver and a parser fuzz run once more under ASan + UBSan."""
import os

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import rls as R
from tests import boolean_corpora as BC
from tests import helpers as H
from tests.http_corpora import HttpHarness
from tests.test_http_device_emu import ENDPOINTS, assert_same
from tests.test_http_device_emu import _emu as _http_emu
from tests.test_rls_device_emu import METHODS, _emu, assert_same_plan, cpu_plan, emu_plan


def boolean_harness(limits, threads=1, cap=None):
    """tests/http_corpora.HttpHarness over a matcher in the boolean dialect."""
    h = HttpHarness([], threads)
    h.rls.close()
    h.m = BC.matcher([], cap)
    for (ns, mx, secs, conds, vars_, name) in limits:
        d = h.m.add_limit(ns, mx, secs, conds, vars_, name)
        h.descs.append(d)
        h.o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    h.rls = R.RlsService(h.m, None, R.HEADERS_NONE, threads)
    h.api = HA.HttpApi(h.rls)
    return h


@pytest.mark.parametrize("method", METHODS)
def test_rls_device_plan_equals_the_cpu_plan(method):
    m = BC.matcher(BC.LIMITS)
    msgs = BC.rls_messages(1, 1500)
    for threads in (1, 3):
        svc = R.RlsService(m, None, R.HEADERS_DRAFT_VERSION_03, threads)
        _emu().emu_rls_seed(threads)
        got = emu_plan(m, method, msgs)
        assert_same_plan(got, cpu_plan(svc, method, msgs))
        svc.close()
    # every boolean limit applies somewhere, and not everywhere
    ids = got["ctrs"]["limit_id"]
    assert set(np.unique(ids).tolist()) == set(range(len(BC.LIMITS)))
    assert (got["store_index"] == R.NO_STORE).sum() > 50


def test_rls_device_plan_on_the_wide_matcher():
    """Up to 50 counters per request (cap 64, a wide engine's), against rl_matcher_counters_batch_ns: the CPU plan of a
    service without an engine refuses requests past the default engine's 16 counters."""
    m = BC.matcher(BC.wide_limits(), cap=64)
    msgs = BC.wide_messages(5, 800)
    got = emu_plan(m, R.SHOULD_RATE_LIMIT, msgs, engine_max=64)
    ctx = [R.decode_request(b) for b in msgs]
    ctr_off, ctrs, status = m.counters_batch_ns([d for d, _, _ in ctx], [(None, [dict(x) for x in ds]) for _, ds, _ in ctx])
    assert (status == 0).all()
    j = 0
    for i in range(len(msgs)):
        if ctr_off[i + 1] == ctr_off[i]:
            assert got["store_index"][i] == R.NO_STORE
            continue
        assert got["store_index"][i] == j
        a, b = int(got["ctr_off"][j]), int(got["ctr_off"][j + 1])
        assert got["ctrs"][a:b].tobytes() == ctrs[ctr_off[i]:ctr_off[i + 1]].tobytes()
        j += 1
    assert j == got["n_store"] and int(np.diff(got["ctr_off"]).max()) == 50


@pytest.mark.parametrize("endpoint", ENDPOINTS)
@pytest.mark.parametrize("threads", [1, 3])
def test_http_device_plan_equals_the_cpu_plan(endpoint, threads):
    h = boolean_harness(BC.LIMITS, threads)
    _http_emu().emu_http_seed(threads)
    got = assert_same(h.m, h, endpoint, BC.http_bodies(2, 1500))
    assert set(got["req"]["kind"].tolist()) >= {3, 4}


def test_http_device_plan_on_the_wide_matcher_with_requests_over_the_cap():
    h = boolean_harness(BC.wide_limits(), 2, cap=16)
    rng = np.random.default_rng(3)
    bodies = []
    for msg in BC.wide_messages(6, 400):
        ns, descs, _ = R.decode_request(msg)
        bodies.append(HA.encode_info(ns, dict(descs[0]) if descs else {}, int(rng.integers(0, 3)), None))
    got = assert_same(h.m, h, HA.CHECK_AND_REPORT, bodies, engine_max=16)
    assert (got["req"]["kind"] == 5).any() and (got["req"]["kind"] == 4).any()


def test_boolean_driver_and_parser_fuzz_are_clean_under_asan_and_ubsan(tmp_path):
    """tests/san/san_bool.cpp: the RLS device plan under the shim over boolean limits, every batch compared with the CPU
    plan, then random and mutated expressions through the boolean parser."""
    from tests.test_sanitizers import build_and_run
    root = H.ROOT
    csrc = os.path.join(root, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(root, "tests", "san", "san_bool.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(root, "include")], extra=("-std=c++17",))
    assert out.startswith("ok compared=")


def test_get_limits_renders_a_boolean_condition_verbatim():
    """GET /limits/{namespace}: every condition's source as given, serde-escaped (tests/serde_render.py)."""
    from tests import serde_render as SR
    h = boolean_harness(BC.LIMITS)
    status, body = h.api.get_limits("api")
    assert status == 200
    assert body == SR.limits_body([l for l in BC.LIMITS if l[0] == "api"])
    assert SR.ser_str(BC.SIX).encode() in body and "contains('é')".encode() in body
