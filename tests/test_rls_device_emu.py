"""The RLS device plan (limitador_b200/csrc/rl_rls_dev.cuh) without a GPU: the kernels run under tests/emu/cuda_shim.h
(tests/emu/emu_rls.cpp) over the matcher's device image (rl_matcher_image), and every array the store call takes, the
store index and the gRPC status of every request must equal the CPU plan's (rl_rls_plan) on the same wire bytes.  The
shared BLAKE2b is checked against hashlib and rl_counter_key, and the driver runs once more under ASan + UBSan."""
import ctypes as C
import functools
import hashlib
import os

import numpy as np
import pytest

from limitador_b200 import engine as E
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import rls_corpora as RC

T0 = 1_700_000_000_000_000
REQ_DTYPE = np.dtype([("kind", "<u4"), ("hits", "<u4"), ("store", "<u4"), ("dom_off", "<u4"), ("dom_len", "<u4")])
REQ_BAD_WIRE, REQ_UNSUPPORTED = 1, 5
METHODS = [R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT]


@functools.cache
def _emu():
    L = H.host_lib("emu_rls.cpp", "librl_emu_rls.so")
    vp, u64 = C.c_void_p, C.c_uint64
    L.emu_rls_plan.restype = u64
    L.emu_rls_plan.argtypes = [vp, C.c_int, u64, vp, vp, u64, C.c_uint32, vp, vp, vp, u64, vp, vp, C.POINTER(u64)]
    L.emu_key_digest.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_uint32, C.POINTER(u64), C.POINTER(u64)]
    L.emu_blake2b.argtypes = [vp, u64, C.c_uint32, vp]
    L.emu_rls_seed.argtypes = [u64]
    return L


def matcher_image(m):
    """rl_matcher_image: the matcher as the device plan reads it (uint32 words) and its generation."""
    L = MT._lib()
    L.rl_matcher_image.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    need, gen = C.c_uint64(), C.c_uint64()
    L.rl_matcher_image(m._h, None, 0, C.byref(need), C.byref(gen))
    words = np.zeros(need.value, dtype=np.uint32)
    assert L.rl_matcher_image(m._h, words.ctypes.data, len(words), C.byref(need), C.byref(gen)) == 0
    return words, gen.value


def emu_plan(m, method, msgs, now_us=T0, engine_max=16):
    """The device plan under the shim -> the dict RlsService.plan returns, plus `grpc` and the raw per-request `req`."""
    buf, off = R.pack_requests(msgs)
    if len(buf) == 0:
        buf = np.zeros(1, np.uint8)
    img, _ = matcher_image(m)
    n = len(msgs)
    req = np.zeros(max(n, 1), REQ_DTYPE)
    ctr_off = np.zeros(n + 1, np.uint32)
    ctrs = np.zeros(64 * n + 1, E.COUNTER_DTYPE)
    delta, now = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
    n_ctr = C.c_uint64()
    m_store = _emu().emu_rls_plan(img.ctypes.data, method, n, buf.ctypes.data, off.ctypes.data, now_us, engine_max, req.ctypes.data,
                                  ctr_off.ctypes.data, ctrs.ctypes.data, len(ctrs), delta.ctypes.data, now.ctypes.data, C.byref(n_ctr))
    req = req[:n]
    grpc = np.where(req["kind"] == REQ_BAD_WIRE, R.GRPC_INTERNAL, np.where(req["kind"] == REQ_UNSUPPORTED, R.GRPC_UNAVAILABLE, R.GRPC_OK))
    return {"n_store": m_store, "ctr_off": ctr_off[:m_store + 1], "ctrs": ctrs[:n_ctr.value], "delta": delta[:m_store],
            "now_us": now[:m_store], "store_index": req["store"].copy(), "grpc": grpc.astype(np.uint8), "req": req}


def cpu_plan(svc, method, msgs, now_us=T0):
    """rl_rls_plan, then a finish with every store request allowed: the gRPC status of every request."""
    p = svc.plan(method, *R.pack_requests(msgs), now_us)
    k = p["n_store"]
    nc = int(p["ctr_off"][-1]) if k else 0
    svc.finish(np.zeros(k, np.uint8), np.full(k, 0xFFFFFFFF, np.uint32), np.zeros(nc, np.uint64), np.zeros(nc, np.uint64))
    p["grpc"] = svc.grpc_status()
    return p


def assert_same_plan(got, want):
    assert got["n_store"] == want["n_store"]
    for key in ("ctr_off", "delta", "now_us", "store_index", "grpc"):
        assert np.array_equal(got[key], want[key]), key
    assert got["ctrs"].tobytes() == want["ctrs"].tobytes()


def _matcher(limits, cap=None):
    m = MT.Matcher()
    if cap:
        m.set_counter_cap(cap)
    for l in limits:
        m.add_limit(*l)
    return m


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", sorted(RC.corpora()))
def test_device_plan_kernels_equal_the_cpu_plan(name, method):
    limits, msgs = RC.corpora()[name]
    m = _matcher(limits)
    for threads in (1, 3):
        svc = R.RlsService(m, None, R.HEADERS_DRAFT_VERSION_03, threads)
        _emu().emu_rls_seed(threads)
        assert_same_plan(emu_plan(m, method, msgs), cpu_plan(svc, method, msgs))
        svc.close()


def test_corpora_reach_every_request_kind():
    kinds = set()
    for limits, msgs in RC.corpora().values():
        kinds |= set(emu_plan(_matcher(limits), R.SHOULD_RATE_LIMIT, msgs)["req"]["kind"].tolist())
    assert kinds == {1, 2, 3, 4, 5}


def test_limits_deleted_and_added_again_between_batches():
    """A deleted limit leaves the image; added again it is the namespace's newest limit, so its counter comes last."""
    limits, reqs = RC._gateway(4, 400)
    msgs = [R.encode_request(ns, d, h) for ns, d, h in reqs]
    m = _matcher(limits)
    svc = R.RlsService(m, None, R.HEADERS_NONE, 2)
    gens = []
    for step in range(4):
        if step == 1:
            m.delete_limit(0)
        elif step == 2:
            m.add_limit(*limits[0])
            m.delete_limit(3)
        elif step == 3:
            m.add_limit(*limits[3][:1], 99, *limits[3][2:])  # back with a new max_value
        gens.append(matcher_image(m)[1])
        got, want = emu_plan(m, R.SHOULD_RATE_LIMIT, msgs), cpu_plan(svc, R.SHOULD_RATE_LIMIT, msgs)
        assert_same_plan(got, want)
        if step == 2:  # limit 0 is now the last limit of "api": where it applies, its counter comes last
            ids = got["ctrs"]["limit_id"].tolist()
            per_req = [ids[got["ctr_off"][j]:got["ctr_off"][j + 1]] for j in range(got["n_store"])]
            with_0 = [c for c in per_req if 0 in c]
            assert with_0 and all(c[-1] == 0 for c in with_0)
    assert gens == sorted(set(gens))  # every change moved the generation


def _contexts(msgs):
    out = []
    for b in msgs:
        dom, descs, _ = R.decode_request(b)
        out.append((dom, (None, [dict(d) for d in descs])))
    return out


def test_a_50_limit_namespace_with_cap_64():
    """The wide engine's case: up to 50 counters per request, against rl_matcher_counters_batch_ns."""
    m = _matcher(RC.wide_limits(), cap=64)
    msgs = RC.wide_messages(5, 600)
    got = emu_plan(m, R.SHOULD_RATE_LIMIT, msgs, engine_max=64)
    ctx = _contexts(msgs)
    ctr_off, ctrs, status = m.counters_batch_ns([d for d, _ in ctx], [c for _, c in ctx])
    assert (status == 0).all()
    j = 0
    widest = 0
    for i in range(len(msgs)):
        k = int(ctr_off[i + 1] - ctr_off[i])
        if k == 0:
            assert got["store_index"][i] == R.NO_STORE
            continue
        assert got["store_index"][i] == j
        a, b = int(got["ctr_off"][j]), int(got["ctr_off"][j + 1])
        assert got["ctrs"][a:b].tobytes() == ctrs[ctr_off[i]:ctr_off[i + 1]].tobytes()
        widest = max(widest, k)
        j += 1
    assert j == got["n_store"] and widest == 50


def test_requests_one_counter_over_the_cap():
    """Cap 4, five limits apply: the request gets gRPC 14 and no counter, in both plans."""
    m = _matcher(RC.over_cap_limits(5), cap=4)
    svc = R.RlsService(m, None, R.HEADERS_NONE, 2)
    msgs = RC.over_cap_messages()
    for method in METHODS:
        got = emu_plan(m, method, msgs)
        assert_same_plan(got, cpu_plan(svc, method, msgs))
        assert (got["grpc"][0::4] == R.GRPC_UNAVAILABLE).all() and (got["grpc"][2::4] == R.GRPC_OK).all()


def test_cap_above_the_engine_refuses_only_the_oversize_requests():
    """The matcher's cap raised past the engine's maximum (16): the device plan refuses exactly the requests of more than
    16 counters; every other request is planned as rl_matcher_counters_batch_ns matches it."""
    m = _matcher(RC.over_cap_limits(30), cap=40)
    msgs = RC.over_cap_messages()
    got = emu_plan(m, R.SHOULD_RATE_LIMIT, msgs, engine_max=16)
    assert (got["grpc"][0::4] == R.GRPC_UNAVAILABLE).all()  # 30 counters
    assert (got["grpc"][1::2] == R.GRPC_OK).all() and (got["grpc"][2::4] == R.GRPC_OK).all()
    ctx = _contexts(msgs[2:3])  # no `u`: only the 15 unqualified limits apply
    _, ctrs, _ = m.counters_batch_ns([d for d, _ in ctx], [c for _, c in ctx])
    assert len(ctrs) == 15
    assert got["n_store"] == 8 and (np.diff(got["ctr_off"]) == 15).all()
    for j in range(8):
        assert got["ctrs"][15 * j:15 * (j + 1)].tobytes() == ctrs.tobytes()


def test_blake2b_matches_hashlib_and_rl_counter_key():
    rng = np.random.default_rng(9)
    out = np.zeros(64, np.uint8)
    for ln in [0, 1, 111, 127, 128, 129, 255, 256, 257, 1000] + [int(x) for x in rng.integers(0, 600, 40)]:
        msg = rng.integers(0, 256, ln, dtype=np.uint8).tobytes()
        for size in (12, 32, 64):
            _emu().emu_blake2b(msg, ln, size, out.ctypes.data)
            assert out[:size].tobytes() == hashlib.blake2b(msg, digest_size=size).digest()
    for _ in range(50):
        k = int(rng.integers(1, 5))
        pairs = sorted({f"descriptors[0].v{int(rng.integers(0, 99))}": "ü" * int(rng.integers(0, 80)) + str(i) for i in range(k)}.items())
        lo, hi = C.c_uint64(), C.c_uint64()
        _emu().emu_key_digest(MT._strs([s for s, _ in pairs]), MT._strs([v for _, v in pairs]), len(pairs), C.byref(lo), C.byref(hi))
        assert (lo.value, hi.value) == MT.counter_key(dict(pairs))
        blob = b"".join(len(x.encode()).to_bytes(4, "little") + x.encode() for p in pairs for x in p)
        d = hashlib.blake2b(blob, digest_size=12).digest()
        assert lo.value == int.from_bytes(d[:8], "little") and hi.value == int.from_bytes(d[8:], "little")


def test_device_plan_driver_is_clean_under_asan_and_ubsan(tmp_path):
    """The kernels under the shim with ASan + UBSan, over random and mutated messages, each batch compared with the CPU
    plan (tests/san/san_rls_dev.cpp)."""
    from tests.test_sanitizers import build_and_run
    root = H.ROOT
    csrc = os.path.join(root, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(root, "tests", "san", "san_rls_dev.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(root, "include")], extra=("-std=c++17",))
    assert out.startswith("ok compared=")
