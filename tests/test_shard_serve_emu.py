"""The general (CSR) form of the sharded exchange on the host (tests/emu/emu_shard_csr.cpp: k_ccount .. k_cgather and the
record exchange's waits under tests/emu/cuda_simt.h, over emulated engines), against ONE global oracle fed every source
batch in canonical order: (source rank, index at the source), one request at a time with its own op, load flag and
clock.  Namespaces never share a counter, so that order gives every owner's result."""
import ctypes as C
import functools

import numpy as np
import pytest

from limitador_b200.engine import COUNTER_DTYPE, LIMIT_DESC_DTYPE, NONE, owner_of
from oracle import binding as ob
from tests import helpers as H

T0 = 1_700_000_000_000_000
CHECK, WITHIN, UPDATE = 0, 1, 2
DIGEST = 0x5EED5EED5EED5EED


@functools.cache
def lib():
    L = H.host_lib("emu_shard_csr.cpp", "librl_emu_shard_csr.so")
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.emu_engine_create.restype = vp
    L.emu_engine_create.argtypes = [u32, u32, u32]
    L.emu_engine_destroy.argtypes = [vp]
    L.emu_engine_limits_set.argtypes = [vp, vp, u32]
    L.emu_engine_interleave.argtypes = [vp, C.c_int, u64, C.c_double]
    L.emu_engine_interleave.restype = None
    L.emu_cshard_create.restype = vp
    L.emu_cshard_create.argtypes = [vp, u32, u32, u32]
    L.emu_cshard_destroy.argtypes = [vp]
    L.emu_cshard_send.argtypes = [vp, u32, u32, u32, vp, vp, vp, vp, u32, vp, u32, C.c_ulonglong]
    L.emu_cshard_decide.argtypes = [vp, u32, C.c_ulonglong, vp]
    L.emu_cshard_collect.argtypes = [vp, u32, vp, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data if a is not None and len(a) else None


def make_limits(n_ns, per_ns, first_ns=0):
    """per_ns limits per namespace: alternately qualified (own variable set) and unqualified, small maxima."""
    d = np.zeros(n_ns * per_ns, dtype=LIMIT_DESC_DTYPE)
    for k in range(n_ns):
        for j in range(per_ns):
            i = k * per_ns + j
            q = j % 2 == 0
            d[i] = (i, first_ns + k, (j // 2 + 1) if q else 0, int(q), 2 + (i % 5), 10_000_000 * (1 + j % 3))
    return d


class Rig:
    """world emulated engines joined by the CSR exchange, and the global oracle."""

    def __init__(self, world, limits, cap_req=64, cap_ctr=1024, cells=3, log2P=2, log2R=6, small_owner=None, interleave=0):
        L = lib()
        self.world, self.limits = world, limits
        self.engines = []
        for r in range(world):
            lp, lr = (0, 1) if r == small_owner else (log2P, log2R)
            e = L.emu_engine_create(cells, lp, lr)
            assert L.emu_engine_limits_set(e, _p(limits), len(limits)) == 0
            if interleave:
                L.emu_engine_interleave(e, 1, interleave + r, 0.5)
            self.engines.append(e)
        arr = (C.c_void_p * world)(*self.engines)
        self.S = L.emu_cshard_create(arr, world, cap_req, cap_ctr)
        assert self.S
        self.orc = ob.Oracle(1 << 12)
        for d in limits:
            self.orc.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
        self.ns_limits = {}
        for d in limits:
            self.ns_limits.setdefault(int(d["ns_id"]), []).append(d)

    def close(self):
        L = lib()
        L.emu_cshard_destroy(self.S)
        for e in self.engines:
            L.emu_engine_destroy(e)

    def owner(self, ns):
        return owner_of(ns, self.world)

    def batch(self, rng, n, nss, max_ctrs=None, load_p=0.5):
        """n requests over namespaces nss: (off, ctrs, delta, now, load, ns of each request)."""
        off, ctrs, ns_of = [0], [], []
        for _ in range(n):
            ns = int(rng.choice(nss))
            lims = self.ns_limits[ns]
            k = len(lims) if max_ctrs is None else min(len(lims), max_ctrs)
            pick = sorted(rng.choice(len(lims), size=int(rng.integers(1, k + 1)), replace=False))
            for j in pick:
                d = lims[j]
                key = int(rng.integers(0, 6)) if d["qualified"] else 0
                ctrs.append((int(d["limit_id"]), 0, key * 0x9E3779B97F4A7C15 % (1 << 64), key))
            off.append(len(ctrs))
            ns_of.append(ns)
        return (np.array(off, np.uint32), np.array(ctrs, dtype=COUNTER_DTYPE), rng.integers(1, 3, n).astype(np.uint64),
                None, (rng.random(n) < load_p).astype(np.uint8), np.array(ns_of, np.int64))

    def step(self, batches, ops, nows, digests=None):
        """One step: every send, every decide, every collect.  batches[r] = Rig.batch output; nows[r] the rank's clock."""
        L = lib()
        W = self.world
        digests = digests or [DIGEST] * W
        keep, outs = [], []
        for r in range(W):
            off, ctrs, delta, _, load, _ = batches[r]
            n = len(delta)
            now = np.full(n, nows[r], np.uint64)
            keep.append((off, ctrs, delta, now, load))
            assert L.emu_cshard_send(self.S, r, n, int(off[-1]), _p(off), _p(ctrs), _p(delta), _p(now), ops[r], _p(load), 0,
                                     digests[r]) == 0
        status = []
        for r in range(W):
            head = np.zeros(4, np.uint32)
            status.append(L.emu_cshard_decide(self.S, r, digests[r], _p(head)))
        for r in range(W):
            off, ctrs, delta, now, load = keep[r]
            n, nc = len(delta), int(off[-1])
            o = (np.full(max(n, 1), 0x77, np.uint8), np.full(max(n, 1), 0x77777777, np.uint32), np.zeros(max(nc, 1), np.uint64),
                 np.zeros(max(nc, 1), np.uint64))
            c = L.emu_cshard_collect(self.S, r, *[_p(a) for a in o])
            outs.append((c, o[0][:n], o[1][:n], o[2][:nc], o[3][:nc]))
        return status, outs

    def oracle(self, batch, op, now, take=None):
        """The oracle's outputs for the requests of one source batch (take: a mask of the requests it decides)."""
        off, ctrs, delta, _, load, _ = batch
        n = len(delta)
        lim, first = np.zeros(n, np.uint8), np.full(n, NONE, np.uint32)
        rem, ttl = np.zeros(int(off[-1]), np.uint64), np.zeros(int(off[-1]), np.uint64)
        for i in range(n):
            if take is not None and not take[i]:
                continue
            a, b = int(off[i]), int(off[i + 1])
            lc = op == CHECK and bool(load[i])
            l1, f1, r1, t1 = self.orc.batch_csr(op, np.array([0, b - a], np.uint32), ctrs[a:b], delta[i:i + 1],
                                                np.array([now], np.uint64), lc)
            if op != UPDATE:
                lim[i], first[i] = l1[0], f1[0]
            if lc:
                rem[a:b], ttl[a:b] = r1, t1
        return lim, first, rem, ttl


def _check(got, want, mask=None, ctr_mask=None):
    c, lim, first, rem, ttl = got
    wl, wf, wr, wt = want
    m = np.ones(len(lim), bool) if mask is None else mask
    assert np.array_equal(lim[m], wl[m]) and np.array_equal(first[m], wf[m])
    cm = np.ones(len(rem), bool) if ctr_mask is None else ctr_mask
    assert np.array_equal(rem[cm], wr[cm]) and np.array_equal(ttl[cm], wt[cm])


def _run_steps(rig, rng, steps, sizes_fn, nss, ops_fn=None, max_ctrs=None):
    W = rig.world
    for s in range(steps):
        sizes = sizes_fn(s)
        batches = [rig.batch(rng, sizes[r], nss, max_ctrs) for r in range(W)]
        ops = ops_fn(s) if ops_fn else [int(rng.integers(0, 3)) for _ in range(W)]
        # per-rank clocks, not monotone in rank order
        nows = [T0 + s * 4_000_000 + (3_000_000 if r % 2 == 0 else 0) - 1000 * r for r in range(W)]
        status, outs = rig.step(batches, ops, nows)
        assert status == [0] * W and [o[0] for o in outs] == [0] * W
        for r in range(W):  # canonical order: rank by rank, each batch in its own order
            _check(outs[r], rig.oracle(batches[r], ops[r], nows[r]))


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_steps_against_one_oracle(world):
    rng = np.random.default_rng(world)
    limits = make_limits(12, 4)
    rig = Rig(world, limits)
    try:
        # ragged and empty blocks: sizes vary per rank and step, some ranks send nothing
        _run_steps(rig, rng, 4, lambda s: [0 if (s + r) % 3 == 0 else int(rng.integers(1, 64)) for r in range(world)],
                   list(range(12)))
    finally:
        rig.close()


def test_one_owner_takes_everything_under_interleaving():
    world = 3
    rng = np.random.default_rng(11)
    limits = make_limits(20, 4)
    rig = Rig(world, limits, interleave=77)
    try:
        mine = [ns for ns in range(20) if rig.owner(ns) == 1]
        assert mine
        _run_steps(rig, rng, 3, lambda s: [64, 37, 64], mine)
    finally:
        rig.close()


def test_requests_of_64_counters_on_a_wide_namespace():
    world = 2
    rng = np.random.default_rng(3)
    limits = np.concatenate([make_limits(1, 64), make_limits(3, 2, first_ns=1)])
    limits["limit_id"] = np.arange(len(limits))
    rig = Rig(world, limits, cells=7, log2R=10)
    try:
        _run_steps(rig, rng, 2, lambda s: [40, 40], [0, 1, 2, 3], ops_fn=lambda s: [CHECK, CHECK])
    finally:
        rig.close()


def test_source_over_its_caps_is_answered_with_error_verdicts():
    world = 3
    rng = np.random.default_rng(5)
    limits = make_limits(12, 4)
    rig = Rig(world, limits)
    try:
        batches = [rig.batch(rng, n, list(range(12))) for n in (30, 64 + 16, 20)]
        nows = [T0, T0, T0]
        status, outs = rig.step(batches, [CHECK] * 3, nows)
        assert outs[1][0] == 2 and np.all(outs[1][1] == 0xFF)  # never allowed
        for r in (0, 2):
            assert outs[r][0] == 0
            _check(outs[r], rig.oracle(batches[r], CHECK, nows[r]))
    finally:
        rig.close()


def test_registry_digest_mismatch_is_never_decided_across():
    world = 3
    rng = np.random.default_rng(6)
    limits = make_limits(12, 4)
    rig = Rig(world, limits)
    try:
        batches = [rig.batch(rng, 50, list(range(12))) for _ in range(world)]
        digests = [DIGEST, DIGEST ^ 1, DIGEST]
        status, outs = rig.step(batches, [CHECK] * 3, [T0] * 3, digests=digests)
        assert all(s & 2 for s in status)  # every owner saw a source with another digest
        for r in range(world):
            own = np.array([rig.owner(int(ns)) for ns in batches[r][5]])
            crossed = (own != r) & ((own == 1) | (r == 1))
            assert crossed.any() and np.all(outs[r][1][crossed] == 0xFF)
            want = rig.oracle(batches[r], CHECK, T0, take=~crossed)
            off = batches[r][0]
            cm = np.repeat(~crossed, np.diff(off))
            _check(outs[r], want, ~crossed, cm)
    finally:
        rig.close()


def test_full_region_on_one_owner_gives_error_verdicts_at_the_sources():
    world = 3
    rng = np.random.default_rng(7)
    limits = make_limits(12, 4)
    rig = Rig(world, limits, small_owner=2)
    try:
        # many distinct keys: owner 2's two-row table fills, its one run fails
        for s in range(2):
            batches = []
            for r in range(world):
                b = rig.batch(rng, 60, list(range(12)), load_p=0.0)
                b[1]["key_lo"] = rng.integers(0, 1 << 62, len(b[1])).astype(np.uint64)
                batches.append(b)
            status, outs = rig.step(batches, [CHECK] * 3, [T0 + s] * 3)
            assert status[2] & 4 and not status[0] & 4 and not status[1] & 4
            for r in range(world):
                own = np.array([rig.owner(int(ns)) for ns in batches[r][5]])
                failed = own == 2
                assert np.all(outs[r][1][failed] == 0xFF)  # error verdicts, never allow
                _check(outs[r], rig.oracle(batches[r], CHECK, T0 + s, take=~failed), ~failed, np.repeat(~failed, np.diff(batches[r][0])))
    finally:
        rig.close()
