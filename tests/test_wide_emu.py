"""The wide position encoding (requests of 17..64 counters, rl_core.h) run through the host emulator
(tests/emu/emu_wide.cpp) and compared bit for bit with the oracle: verdicts, first-limited ids, remaining / ttl in the
caller's order, and the table."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import helpers as H

ACCESS_DTYPE = np.dtype([("key_lo", "<u8"), ("hdr_hi", "<u8"), ("req", "<u4"), ("cells", "<u4"), ("posorig", "<u8")])
assert ACCESS_DTYPE.itemsize == 32


_wide = None


def wide_lib():
    """tests/emu/emu_wide.cpp compiled for the host (rebuilt when it or rl_core.h changes)."""
    global _wide
    if _wide is None:
        src = os.path.join(H.HERE, "emu", "emu_wide.cpp")
        so = os.path.join(H.HERE, "emu", "librl_emu_wide.so")
        core = os.path.join(os.path.dirname(H.HERE), "limitador_b200", "csrc", "rl_core.h")
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core)):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.emu_wide_create.restype = vp
        L.emu_wide_create.argtypes = [C.c_int]
        L.emu_wide_destroy.argtypes = [vp]
        L.emu_wide_set_tables.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32]
        L.emu_wide_batch_csr.argtypes = [vp, C.c_int, C.c_uint32, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
        L.emu_wide_resolve.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, vp, C.c_uint32, vp, vp]
        L.emu_wide_resolve.restype = C.c_int
        L.emu_wide_dump.restype = C.c_uint64
        L.emu_wide_dump.argtypes = [vp, C.c_uint64, vp, vp, vp, vp, vp]
        _wide = L
    return _wide


class WideEmu:
    """Sequential host run of the kernels' algorithm in the wide encoding (tests/emu/emu_wide.cpp)."""

    def __init__(self, descs, cells):
        self.L = wide_lib()
        self.h = self.L.emu_wide_create(cells)
        limits, desc, ngroups = H.assign_tables(descs, cells)
        self.L.emu_wide_set_tables(self.h, H._p(limits), len(limits), H._p(desc), ngroups)
        self.rounds = 0

    def __del__(self):
        if getattr(self, "h", None):
            self.L.emu_wide_destroy(self.h)

    def batch_csr(self, mode, off, ctrs, delta, now_us, load_counters=False):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=H.COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        n = len(delta)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, H.NONE, dtype=np.uint32)
        rem = np.zeros(len(ctrs), dtype=np.uint64)
        ttl = np.zeros(len(ctrs), dtype=np.uint64)
        rounds = C.c_int(0)
        r = self.L.emu_wide_batch_csr(self.h, mode, n, H._p(off), H._p(ctrs), H._p(delta), H._p(now_us),
                                      int(load_counters), H._p(lim), H._p(fl), H._p(rem), H._p(ttl), C.byref(rounds))
        assert r == 0, f"emu error {r}"
        self.rounds = rounds.value
        return lim, fl, rem, ttl

    def resolve(self, ctrs, wide=True, req=0, max_ctrs=64):
        ctrs = np.ascontiguousarray(ctrs, dtype=H.COUNTER_DTYPE)
        m = len(ctrs)
        acc = np.zeros(max(m, 1), dtype=ACCESS_DTYPE)
        perm = np.full(max(m, 1), 0xFF, dtype=np.uint8)
        r = self.L.emu_wide_resolve(self.h, int(wide), req, m, H._p(ctrs), max_ctrs, H._p(acc), H._p(perm))
        return r, acc, perm

    def dump(self):
        cap = 1 << 20
        lid = np.zeros(cap, dtype=np.uint32)
        lo, hi, val, exp = (np.zeros(cap, dtype=np.uint64) for _ in range(4))
        c = self.L.emu_wide_dump(self.h, cap, H._p(lid), H._p(lo), H._p(hi), H._p(val), H._p(exp))
        return sorted(zip(lid[:c].tolist(), lo[:c].tolist(), hi[:c].tolist(), val[:c].tolist(), exp[:c].tolist()))


def wide_limits(seed, sizes=(20, 33, 64, 3), small=True):
    """Namespaces of `sizes` limits, qualified (three variable sets) and unqualified interleaved in registration order,
    with small maxima so that the limits bite."""
    rng = np.random.default_rng(seed)
    descs, lid = [], 0
    for ns, size in enumerate(sizes):
        for _ in range(size):
            q = 1 if rng.random() < 0.7 else 0
            varset = int(rng.integers(1, 4)) if q else 0
            mx = int(rng.choice([0, 1, 2, 3, 5, 8, 20, 1 << 40])) if small else (1 << 62)
            win = int(rng.choice([1, 2, 10, 60, 3600])) * 1_000_000
            descs.append((lid, ns, varset, q, mx, win))
            lid += 1
    return np.array(descs, dtype=H.LIMIT_DESC_DTYPE)


def wide_stream(descs, n, seed, n_keys=3, monotone=True, min_ctrs=17):
    """Requests naming at least min_ctrs of their namespace's limits where it has that many (all of a smaller one),
    in shuffled order half of the time; per-variable-set keys from a tiny key space."""
    rng = np.random.default_rng(seed)
    by_ns = {}
    for d in descs:
        by_ns.setdefault(int(d["ns_id"]), []).append(d)
    nss = sorted(by_ns)
    off, ctrs = [0], []
    delta = np.zeros(n, dtype=np.uint64)
    now = np.zeros(n, dtype=np.uint64)
    t = H.T0
    for i in range(n):
        lims = by_ns[int(rng.choice(nss))]
        lo_k = min(min_ctrs, len(lims))
        k = int(rng.integers(lo_k, len(lims) + 1))
        pick = sorted(rng.choice(len(lims), size=k, replace=False).tolist())
        if rng.random() < 0.5:
            rng.shuffle(pick)
        vkeys = {}
        for j in pick:
            d = lims[j]
            vs = int(d["varset_id"]) if d["qualified"] else 0
            if vs not in vkeys:
                vkeys[vs] = (int(rng.integers(1, n_keys + 1)), int(rng.integers(0, 2)))
            lo, hi = vkeys[vs] if d["qualified"] else (0, 0)
            ctrs.append((int(d["limit_id"]), 0, lo, hi))
        off.append(len(ctrs))
        delta[i] = int(rng.choice([1, 1, 1, 2, 3, 7]))
        t += int(rng.choice([0, 0, 1, 1000, 400_000, 1_500_000]))
        now[i] = t if monotone else max(1, t - int(rng.choice([0, 0, 2_000_000])))
    return np.array(off, dtype=np.uint32), np.array(ctrs, dtype=H.COUNTER_DTYPE), delta, now


def run_both(descs, cells, batches, load_counters, mode=0):
    emu = WideEmu(descs, cells)
    orc = H.oracle_with_limits(descs)
    rounds = []
    for off, ctrs, delta, now in batches:
        e = emu.batch_csr(mode, off, ctrs, delta, now, load_counters)
        o = orc.batch_csr(mode, off, ctrs, delta, now, load_counters)
        rounds.append(emu.rounds)
        if mode == 0:
            assert e[0].tolist() == o[0].tolist(), "verdicts differ"
            assert e[1].tolist() == o[1].tolist(), "first-limited limit differs"
            if load_counters:
                assert e[2].tolist() == o[2].tolist(), "remaining differs"
                assert e[3].tolist() == o[3].tolist(), "ttl differs"
        assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs), "table differs"
    return rounds


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
@pytest.mark.parametrize("seed", [0, 1])
def test_wide_random_streams_match_oracle(cells, load_counters, seed):
    descs = wide_limits(seed)
    batches = [wide_stream(descs, 120, seed * 100 + b, monotone=(b % 2 == 0)) for b in range(4)]
    rounds = run_both(descs, cells, batches, load_counters)
    assert max(rounds) >= 1  # every wide request spans several rows


@pytest.mark.parametrize("load_counters", [False, True])
def test_wide_mixed_with_narrow_requests_matches_oracle(load_counters):
    descs = wide_limits(7)
    batches = [wide_stream(descs, 150, 700 + b, min_ctrs=1) for b in range(3)]
    assert any(int(np.diff(b[0]).max()) > 16 for b in batches) and any(int(np.diff(b[0]).min()) <= 16 for b in batches)
    run_both(descs, 3, batches, load_counters)


def test_wide_encoding_on_narrow_batches_matches_narrow_emulator():
    descs = H.mixed_limits(n_ns=12, seed=3)
    narrow, wide = H.Emu(descs, 3), WideEmu(descs, 3)
    for b in range(4):
        batch = H.random_csr_stream(descs, 250, 40 + b, n_keys=3)
        a, w = narrow.batch_csr(0, *batch, True), wide.batch_csr(0, *batch, True)
        for x, y in zip(a, w):
            assert x.tolist() == y.tolist()
    assert narrow.dump() == wide.dump()


def test_wide_update_mode_matches_oracle():
    descs = wide_limits(11)
    run_both(descs, 7, [wide_stream(descs, 100, 1100 + b) for b in range(3)], False, mode=2)


def test_wide_fixed_point_chain_at_64_counters():
    """The adversarial coupling of test_emu_algorithm (request i allowed iff i-1 denied, rows of max 1 shared
    pairwise), each request padded to 64 counters with limits that never bite, one row each."""
    descs = [(0, 0, 1, 1, 1, 3600_000_000), (1, 0, 2, 1, 1, 3600_000_000)]
    descs += [(2 + k, 0, 3 + k, 1, 1 << 40, 3600_000_000) for k in range(62)]
    descs = np.array(descs, dtype=H.LIMIT_DESC_DTYPE)
    n = 30
    off = np.arange(0, 64 * n + 1, 64, dtype=np.uint32)
    ctrs = np.zeros(64 * n, dtype=H.COUNTER_DTYPE)
    for i in range(n):
        row = [(2 + k, 0, 1000 + i, 0) for k in range(62)]
        row.insert(i % 62, (0, 0, 1 + i // 2, 0))        # row A_k shared by requests 2k, 2k+1
        row.insert(63 - i % 13, (1, 0, 1 + (i + 1) // 2, 0))  # row B_k shared by requests 2k-1, 2k
        ctrs[64 * i:64 * (i + 1)] = row
    delta = np.ones(n, dtype=np.uint64)
    now = np.full(n, H.T0, dtype=np.uint64)
    for lc in (False, True):
        rounds = run_both(descs, 1, [(off, ctrs, delta, now)], lc)
        assert rounds[0] >= n // 2


def test_wide_resolve_positions_permutation_and_high_bits():
    """64 counters of one namespace, unqualified ones last in the given order: they are processed first, so the
    positions and the permutation differ from the given order, and counters beyond bit 31 of `used` are grouped."""
    descs = [(k, 0, 0 if k >= 40 else 1 + k % 5, 0 if k >= 40 else 1, 1 << 40, 60_000_000) for k in range(64)]
    descs = np.array(descs, dtype=H.LIMIT_DESC_DTYPE)
    emu = WideEmu(descs, 7)
    ctrs = np.array([(k, 0, 9, 0) for k in range(64)], dtype=H.COUNTER_DTYPE)
    nacc, acc, perm = emu.resolve(ctrs, req=5)
    assert nacc > 1
    order = list(range(40, 64)) + list(range(40))  # unqualified first, then qualified, each in the given order
    assert perm.tolist() == order
    seen_pos, seen_orig = [], []
    for a in acc[:nacc]:
        assert a["req"] == 5 and a["hdr_hi"] != 0
        cells = int(a["cells"])
        cnt = (cells >> 28) & 7
        assert cells >> 31 == 1  # several accesses: coupled
        for k in range(cnt):
            pos = (int(a["posorig"]) >> (6 * k)) & 63
            seen_pos.append(pos)
            seen_orig.append(perm[pos])
        assert int(a["posorig"]) >> (6 * cnt) == 0
    assert sorted(seen_pos) == list(range(64)) and max(seen_pos) == 63
    assert sorted(seen_orig) == list(range(64))
    # one access per (row group, key): the 24 unqualified counters share groups of 7 cells
    assert all(a["hdr_hi"] == 0 for a in acc[nacc:])
    # the given order is kept inside each class
    assert [p for p in perm.tolist() if p >= 40] == list(range(40, 64))


def test_wide_resolve_limits():
    descs = np.array([(k, 0, 1, 1, 5, 60_000_000) for k in range(65)], dtype=H.LIMIT_DESC_DTYPE)
    emu = WideEmu(descs, 1)
    ctrs = np.array([(k, 0, 1, 0) for k in range(65)], dtype=H.COUNTER_DTYPE)
    too_many = 4  # RL_DEV_TOO_MANY_COUNTERS
    assert emu.resolve(ctrs)[0] == -too_many
    assert emu.resolve(ctrs[:33], max_ctrs=32)[0] == -too_many
    assert emu.resolve(ctrs[:32], max_ctrs=32)[0] == 32
    assert emu.resolve(ctrs[:64])[0] == 64
    assert emu.resolve(ctrs[:17], wide=False)[0] == -too_many
    assert emu.resolve(ctrs[:16], wide=False)[0] == 16
