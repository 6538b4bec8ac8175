"""The counter variable dictionary (limitador_b200/csrc/rl_cvars_dev.cuh) without a GPU: the RLS and HTTP plan kernels and
k_counter_vars_record run under tests/emu/cuda_shim.h (tests/emu/emu_cvars.cpp), and the dictionary they leave must be
the map built in Python from the same requests: the CPU plan's counters, the decoded context (last duplicate key wins),
the limit's sorted variables.  Lookup and GC run under the shim as well.  The driver runs once more under ASan + UBSan."""
import ctypes as C
import functools
import os
import re
import struct

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import http_corpora as HC
from tests import rls_corpora as RC
from tests.test_http_device_emu import _bodies
from tests.test_rls_device_emu import _matcher, emu_plan, matcher_image

T0 = 1_700_000_000_000_000


@functools.cache
def _emu(simt=False):
    """tests/emu/emu_cvars.cpp under the host shim, or with simt=True under the fiber emulator (tests/emu/cuda_simt.h)."""
    L = H.host_lib("emu_cvars.cpp", "librl_emu_cvars_simt.so" if simt else "librl_emu_cvars.so", ["EMU_SIMT"] if simt else [])
    vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
    if simt:
        L.emu_cv_interleave.argtypes = [C.c_int, u64, C.c_double]
        L.emu_cv_interleave.restype = None
    L.emu_cv_seed.argtypes = [u64]
    L.emu_cv_create.restype = vp
    L.emu_cv_create.argtypes = [u64, u64]
    L.emu_cv_destroy.argtypes = [vp]
    L.emu_cv_stats.argtypes = [vp] + [C.POINTER(u64)] * 4
    L.emu_cv_plan_record.restype = u64
    L.emu_cv_plan_record.argtypes = [vp, C.c_int, vp, C.c_int, u64, vp, vp, u32]
    L.emu_cv_dump.restype = u64
    L.emu_cv_dump.argtypes = [vp, vp, vp, vp, vp, vp, u64]
    L.emu_cv_arena.restype = vp
    L.emu_cv_arena.argtypes = [vp]
    L.emu_cv_lookup.restype = u64
    L.emu_cv_lookup.argtypes = [vp, vp, u64, vp, vp, vp, vp, vp, vp, u64]
    L.emu_cv_gc.argtypes = [vp, vp, u64, vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
    return L


class Dict:
    """One dictionary under the shim; with interleave=(seed, p), under the fiber emulator with its interleaving mode on
    for every record call."""

    def __init__(self, max_keys=1 << 14, arena_bytes=1 << 20, interleave=None):
        self.L = _emu(interleave is not None)
        self.h = self.L.emu_cv_create(max_keys, arena_bytes)
        self.interleave = interleave

    def __del__(self):
        self.L.emu_cv_destroy(self.h)

    def record(self, m, http, endpoint, msgs, engine_max=16):
        buf, off = R.pack_requests(msgs)
        if len(buf) == 0:
            buf = np.zeros(1, np.uint8)
        img, _ = matcher_image(m)
        if self.interleave:
            self.L.emu_cv_interleave(1, *self.interleave)
        try:
            return self.L.emu_cv_plan_record(self.h, int(http), img.ctypes.data, endpoint, len(msgs), buf.ctypes.data,
                                             off.ctypes.data, engine_max)
        finally:
            if self.interleave:
                self.L.emu_cv_interleave(0, 0, 1.0)

    def stats(self):
        v = [C.c_uint64() for _ in range(4)]
        self.L.emu_cv_stats(self.h, *[C.byref(x) for x in v])
        return dict(zip(("slots", "keys", "arena_used", "dropped"), [x.value for x in v]))

    def entries(self):
        """-> {(varset, key_lo, key_hi): blob bytes}, and the blobs' (offset, length) in slot order."""
        cap = self.stats()["slots"]
        vs, lo, hi, bo = np.zeros(cap, np.uint32), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
        bl = np.zeros(cap, np.uint32)
        k = self.L.emu_cv_dump(self.h, vs.ctypes.data, lo.ctypes.data, hi.ctypes.data, bo.ctypes.data, bl.ctypes.data, cap)
        used = self.stats()["arena_used"]
        arena = C.string_at(self.L.emu_cv_arena(self.h), used) if used else b""
        out = {(int(vs[i]), int(lo[i]), int(hi[i])): arena[int(bo[i]):int(bo[i]) + int(bl[i])] for i in range(k)}
        return out, [(int(bo[i]), int(bl[i])) for i in range(k)]

    def lookup(self, m, ctrs):
        img, _ = matcher_image(m)
        n = len(ctrs)
        lid = np.ascontiguousarray([c[0] for c in ctrs] or [0], np.uint32)
        lo = np.ascontiguousarray([c[1] for c in ctrs] or [0], np.uint64)
        hi = np.ascontiguousarray([c[2] for c in ctrs] or [0], np.uint64)
        pos, un = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint8)
        out = np.zeros(1 << 20, np.uint8)
        self.L.emu_cv_lookup(self.h, img.ctypes.data, n, lid.ctypes.data, lo.ctypes.data, hi.ctypes.data, pos.ctypes.data,
                             un.ctypes.data, out.ctypes.data, len(out))
        return [None if un[i] else out[int(pos[i]):int(pos[i + 1])].tobytes() for i in range(n)]

    def gc(self, m, ctrs):
        img, _ = matcher_image(m)
        lid = np.ascontiguousarray([c[0] for c in ctrs] or [0], np.uint32)
        lo = np.ascontiguousarray([c[1] for c in ctrs] or [0], np.uint64)
        hi = np.ascontiguousarray([c[2] for c in ctrs] or [0], np.uint64)
        kept, freed = C.c_uint64(), C.c_uint64()
        self.L.emu_cv_gc(self.h, img.ctypes.data, len(ctrs), lid.ctypes.data, lo.ctypes.data, hi.ctypes.data, C.byref(kept), C.byref(freed))
        return kept.value, freed.value


_OPERAND = re.compile(r"""^descriptors\[(\d+)\](?:\.(\w+)|\[(['"])(.*)\3\])$""")


def var_value(source, descs):
    """limiter.py's variable resolution over descriptor maps (last duplicate key wins)."""
    mo = _OPERAND.match(source.strip())
    d, key = int(mo.group(1)), mo.group(2) if mo.group(2) is not None else mo.group(4)
    return descs[d][key]


def blob(values):
    return b"".join(struct.pack("<I", len(v.encode())) + v.encode() for v in values)


def unblob(b):
    out, at = [], 0
    while at < len(b):
        n = struct.unpack_from("<I", b, at)[0]
        out.append(b[at + 4:at + 4 + n].decode())
        at += 4 + n
    return out


class Limits:
    """limit id -> (varset_id, sorted variable sources) of the matcher's limits."""

    def __init__(self, m, limits):
        self.by_id = {}
        for l in limits:
            d = m.add_limit(*l)  # an equal limit: the same id (update_limit)
            self.by_id[int(d["limit_id"])] = (int(d["varset_id"]), sorted(set(l[4])))


def expected(lims, plan, contexts):
    """{(varset, key_lo, key_hi): blob} from the CPU plan's counters and the requests' decoded contexts."""
    out = {}
    for i, j in enumerate(plan["store_index"]):
        if j == R.NO_STORE:
            continue
        co = plan["ctr_off"]
        for c in plan["ctrs"][int(co[j]):int(co[j + 1])]:
            vs, srcs = lims.by_id[int(c["limit_id"])]
            if vs == 0:
                continue
            vals = [var_value(s, contexts[i]) for s in srcs]
            key = (vs, int(c["key_lo"]), int(c["key_hi"]))
            assert out.setdefault(key, blob(vals)) == blob(vals)
            assert MT.counter_key(dict(zip(srcs, vals))) == key[1:]
    return out


def rls_contexts(msgs):
    out = []
    for b in msgs:
        try:
            _, descs, _ = R.decode_request(b)
        except R.RlsError:
            descs = []
        out.append([dict(d) for d in descs])
    return out


def http_contexts(bodies):
    out = []
    for b in bodies:
        try:
            _, pairs, _, _ = HA.decode_body(b)
        except HA.HttpError:
            pairs = []
        out.append([dict(pairs)])
    return out


def check_entries(d, want, lims):
    got, _ = d.entries()
    assert got == want
    srcs = {vs: s for vs, s in lims.by_id.values()}
    for (vs, lo, hi), b in got.items():  # rl_counter_key(sources, recorded values) == key
        assert MT.counter_key(dict(zip(srcs[vs], unblob(b)))) == (lo, hi)


@pytest.mark.parametrize("name", sorted(RC.corpora()))
def test_rls_batches_record_the_values_behind_every_key(name):
    limits, msgs = RC.corpora()[name]
    m = MT.Matcher()
    lims = Limits(m, limits)
    svc = R.RlsService(m, None, R.HEADERS_NONE, 2)
    d = Dict()
    _emu().emu_cv_seed(5)
    want = {}
    for method in (R.SHOULD_RATE_LIMIT, R.CHECK_RATE_LIMIT, R.REPORT):
        n_store = d.record(m, False, method, msgs)
        p = svc.plan(method, *R.pack_requests(msgs), T0)
        assert n_store == p["n_store"]
        want.update(expected(lims, p, rls_contexts(msgs)))
    check_entries(d, want, lims)
    st = d.stats()
    # every key once: no waste in the arena when no two threads race for a key
    assert st["keys"] == len(want) and st["dropped"] == 0 and st["arena_used"] == sum(len(b) for b in want.values())


@pytest.mark.parametrize("endpoint", [HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT])
def test_http_batches_record_the_values_behind_every_key(endpoint):
    rng = np.random.default_rng(20 + endpoint)
    h = HC.HttpHarness([])
    lims = Limits(h.m, HC.GATEWAY_LIMITS + [("esc", 9, 60, [], ["descriptors[0]['a\"b']", "descriptors[0].z"], "q\"n")])
    bodies = _bodies(rng) + [HA.encode_info("esc", {"a\"b": "\x01\x7f\"\\é", "z": ""}, 1),
                             HA.encode_info("esc", {"a\"b": "x", "z": "1", "a\"b": "y"}, 1),
                             b'{"namespace":"esc","values":{"a\\"b":"dup1","z":"","a\\"b":"dup2"},"delta":1}']
    d = Dict()
    n_store = d.record(h.m, True, endpoint, bodies)
    p = h.api.plan(endpoint, *HA.pack_bodies(bodies), T0)
    assert n_store == p["n_store"]
    want = expected(lims, p, http_contexts(bodies))
    assert len(want) > 10 and any(k[0] == lims.by_id[5][0] for k in want)
    check_entries(d, want, lims)
    assert d.stats()["keys"] == len(want)


def test_rls_and_http_fill_one_dictionary_and_a_key_is_recorded_once():
    """The same keys from both surfaces and repeated within and across batches: one entry each."""
    h = HC.HttpHarness([])
    lims = Limits(h.m, HC.GATEWAY_LIMITS)
    users = [f"u{k}" for k in range(7)]
    bodies = [HA.encode_info("api", {"method": "GET", "user": u}, 1) for u in users * 5]
    msgs = [R.encode_request("api", [[("method", "GET"), ("user", u)]]) for u in users * 5]
    d = Dict()
    d.record(h.m, True, HA.CHECK_AND_REPORT, bodies)
    first = d.stats()
    d.record(h.m, False, R.SHOULD_RATE_LIMIT, msgs)
    assert d.stats() == first
    want = expected(lims, h.api.plan(HA.CHECK, *HA.pack_bodies(bodies), T0), http_contexts(bodies))
    assert first["keys"] == len(want) == 7  # one variable set (descriptors[0].user) for the three per-user limits
    check_entries(d, want, lims)


def test_the_50_limit_namespace_and_requests_over_the_cap():
    m = _matcher([], cap=64)
    lims = Limits(m, RC.wide_limits())
    msgs = RC.wide_messages(5, 300)
    d = Dict()
    d.record(m, False, R.SHOULD_RATE_LIMIT, msgs, engine_max=64)
    # (a service without an engine plans for 16 counters: the wide engine's plan is the device plan's, checked against
    # the matcher in test_rls_device_emu)
    want = expected(lims, emu_plan(m, R.SHOULD_RATE_LIMIT, msgs, engine_max=64), rls_contexts(msgs))
    assert len(want) > 10
    check_entries(d, want, lims)
    # over the engine's maximum: refused requests record nothing
    m2 = _matcher([], cap=40)
    lims2 = Limits(m2, RC.over_cap_limits(30))
    msgs2 = RC.over_cap_messages()
    d2 = Dict()
    d2.record(m2, False, R.SHOULD_RATE_LIMIT, msgs2, engine_max=16)
    p2 = emu_plan(m2, R.SHOULD_RATE_LIMIT, msgs2, engine_max=16)
    assert (p2["grpc"] == R.GRPC_UNAVAILABLE).any() and (p2["store_index"] != R.NO_STORE).any()
    check_entries(d2, expected(lims2, p2, rls_contexts(msgs2)), lims2)


def test_limits_deleted_and_added_again():
    h = HC.HttpHarness([])
    lims = Limits(h.m, HC.GATEWAY_LIMITS)
    rng = np.random.default_rng(4)
    d = Dict()
    want = {}
    for step in range(4):
        if step == 1:
            h.m.delete_limit(0)
            h.m.delete_limit(2)
        if step == 3:
            Limits(h.m, [HC.GATEWAY_LIMITS[2]])
        bodies = [HA.encode_info(*x) for x in HC.random_infos(rng, 300, users=40)]
        d.record(h.m, True, HA.CHECK_AND_REPORT, bodies)
        want.update(expected(lims, h.api.plan(HA.CHECK_AND_REPORT, *HA.pack_bodies(bodies), T0), http_contexts(bodies)))
    check_entries(d, want, lims)


def _users(n, ns="n"):
    return [HA.encode_info(ns, {"user": f"u{k:03d}"}, 1) for k in range(n)]


def test_a_full_table_drops_exactly_the_keys_over_it():
    h = HC.HttpHarness([])
    lims = Limits(h.m, [("n", 5, 60, [], ["descriptors[0].user"], None)])
    bodies = _users(40)
    d = Dict(max_keys=16)
    d.record(h.m, True, HA.CHECK, bodies + bodies)
    st = d.stats()
    assert st["slots"] == 16 and st["keys"] == 16 and st["dropped"] == 24 * 2
    want = expected(lims, h.api.plan(HA.CHECK, *HA.pack_bodies(bodies), T0), http_contexts(bodies))
    got, spans = d.entries()
    assert all(want[k] == b for k, b in got.items())  # no partial entry: every claimed slot has its blob
    assert all(ln == 8 for _, ln in spans)


def test_a_full_arena_drops_exactly_the_keys_over_it():
    h = HC.HttpHarness([])
    lims = Limits(h.m, [("n", 5, 60, [], ["descriptors[0].user"], None)])
    bodies = _users(30)
    d = Dict(max_keys=64, arena_bytes=8 * 10 + 3)  # a blob is 4 + 4 bytes
    d.record(h.m, True, HA.CHECK, bodies)
    st = d.stats()
    assert st["keys"] == 10 and st["dropped"] == 20 and st["arena_used"] == 8 * 10 + 3
    want = expected(lims, h.api.plan(HA.CHECK, *HA.pack_bodies(bodies), T0), http_contexts(bodies))
    got, _ = d.entries()
    assert len(got) == 10 and all(want[k] == b for k, b in got.items())


def test_lookup_and_gc():
    h = HC.HttpHarness([])
    lims = Limits(h.m, HC.GATEWAY_LIMITS)
    rng = np.random.default_rng(8)
    bodies = [HA.encode_info(*x) for x in HC.random_infos(rng, 800, users=60)]
    d = Dict()
    d.record(h.m, True, HA.CHECK_AND_REPORT, bodies)
    p = h.api.plan(HA.CHECK_AND_REPORT, *HA.pack_bodies(bodies), T0)
    want = expected(lims, p, http_contexts(bodies))
    ctrs = sorted({(int(c["limit_id"]), int(c["key_lo"]), int(c["key_hi"])) for c in p["ctrs"]})
    got = d.lookup(h.m, ctrs + [(0, 1, 2)])
    for (lid, lo, hi), b in zip(ctrs, got):
        vs = lims.by_id[lid][0]
        assert b == (want[(vs, lo, hi)] if vs else b"")
    assert got[-1] is None  # a qualified counter without an entry is unnamed
    # GC: keep what a third of the counters reference
    live = ctrs[::3]
    keep = {(lims.by_id[l][0], lo, hi) for l, lo, hi in live if lims.by_id[l][0]}
    before = d.stats()
    kept, freed = d.gc(h.m, live)
    st = d.stats()
    assert kept == st["keys"] == len(keep) and freed == before["keys"] - len(keep)
    assert st["arena_used"] == sum(len(want[k]) for k in keep)  # compacted
    got2, spans = d.entries()
    assert got2 == {k: want[k] for k in keep}
    assert sorted(spans) == sorted(spans) and sum(ln for _, ln in spans) == st["arena_used"]
    after = d.lookup(h.m, ctrs)
    for c, b0, b1 in zip(ctrs, got, after):
        vs = lims.by_id[c[0]][0]
        assert b1 == (b0 if (not vs or (vs, c[1], c[2]) in keep) else None)
    # new traffic after a GC records again
    d.record(h.m, True, HA.CHECK_AND_REPORT, bodies)
    assert d.entries()[0] == want


def test_driver_is_clean_under_asan_and_ubsan(tmp_path):
    """The recording, lookup and GC kernels under the shim with ASan + UBSan (tests/san/san_cvars.cpp)."""
    from tests.test_sanitizers import build_and_run
    root = H.ROOT
    csrc = os.path.join(root, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(root, "tests", "san", "san_cvars.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(root, "include")], extra=("-std=c++17",))
    assert out.startswith("ok entries=")
