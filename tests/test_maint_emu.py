"""The maintenance kernels (limitador_b200/csrc/rl_maint.cuh) run on the host under tests/emu/cuda_shim.h — the same
source the GPU compiles, one CUDA thread after the other in a shuffled order:
  * k_ns_metrics against a plain numpy reduction (prometheus_metrics.rs:93-125 semantics);
  * k_region_census / k_compact_move / k_compact_reinsert: a region rebuilt in place keeps every counter findable by the
    hot path's probing rule, frees its tombstones and leaves the other regions byte-identical.
The GPU runs of rl_compact / rl_ns_metrics_* through the C-ABI are in tests/test_zz3_maint_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from limitador_b200.engine import RECORD16_DTYPE, RECORD_DTYPE, pack_records16
from tests import helpers as H

TOMB = 0xFFFFFFFFFFFFFFFF


def metrics_by_numpy(ns, hits, limited, first, ns_cap, limits_cap):
    ok = (limited != 0xFF) & (ns < ns_cap)
    allowed, lim = ok & (limited == 0), ok & (limited != 0) & (limited != 0xFF)
    ac = np.bincount(ns[allowed], minlength=ns_cap).astype(np.uint64)
    ah = np.zeros(ns_cap, dtype=np.uint64)
    np.add.at(ah, ns[allowed], hits[allowed].astype(np.uint64))
    lc = np.bincount(ns[lim], minlength=ns_cap).astype(np.uint64)
    named = lim & (first < limits_cap)
    bl = np.bincount(first[named], minlength=limits_cap).astype(np.uint64)
    return ac, ah, lc, bl, int((~ok).sum())


@pytest.mark.parametrize("simt", [False, True], ids=["plain-path", "warp-aggregated-path"])
@pytest.mark.parametrize("n,ns_space,compact", [(1, 3, False), (31, 3, False), (5000, 40, False), (5000, 40, True), (3000, 1, True)])
def test_ns_metrics_kernel_equals_a_numpy_reduction(n, ns_space, compact, simt):
    """simt=False: the kernel's plain path, one thread after the other (cuda_shim.h).  simt=True: its DEVICE branch —
    __match_any_sync groups, __reduce_add_sync of the split hits, the leader's atomics — under the fiber emulator
    (cuda_simt.h), which also checks that every lane named in a mask reaches the rendezvous."""
    L = H.emu_maint_lib(simt)
    rng = np.random.default_rng(n + ns_space)
    ns_cap, limits_cap = 64, 16
    recs = np.zeros(n, dtype=RECORD_DTYPE)
    recs["ns_id"] = rng.integers(0, ns_space, size=n)
    recs["hits_addend"] = rng.choice([1, 1, 2, 255] if compact else [1, 1, 2, 70000, 2 ** 32 - 1], size=n)
    recs["key_lo"] = rng.integers(1, 2 ** 62, size=n)
    recs["key_hi"] = rng.integers(0, 2 ** 32, size=n)
    if not compact and n > 100:
        recs["ns_id"][::97] = 1000  # a namespace id beyond the tables: dropped, not counted
    limited = rng.choice([0, 0, 1, 0xFF], p=[0.5, 0.2, 0.28, 0.02], size=n).astype(np.uint8)
    first = rng.integers(0, 20, size=n).astype(np.uint32)
    first[limited == 0] = 0xFFFFFFFF
    wire = pack_records16(recs) if compact else recs
    out = np.zeros(3 * ns_cap + limits_cap + 1, dtype=np.uint64)
    L.emu_ns_metrics(H._p(wire), 2 if compact else 4, n, H._p(limited), H._p(first), ns_cap, limits_cap, H._p(out))
    ac, ah, lc, bl, dropped = metrics_by_numpy(recs["ns_id"].astype(np.int64), recs["hits_addend"], limited, first.astype(np.int64), ns_cap, limits_cap)
    assert out[:ns_cap].tolist() == ac.tolist()
    assert out[ns_cap:2 * ns_cap].tolist() == ah.tolist()
    assert out[2 * ns_cap:3 * ns_cap].tolist() == lc.tolist()
    assert out[3 * ns_cap:3 * ns_cap + limits_cap].tolist() == bl.tolist()
    assert int(out[-1]) == dropped
    # a second batch accumulates on top
    L.emu_ns_metrics(H._p(wire), 2 if compact else 4, n, H._p(limited), None, ns_cap, limits_cap, H._p(out))
    assert out[:ns_cap].tolist() == (2 * ac).tolist() and out[3 * ns_cap:3 * ns_cap + limits_cap].tolist() == bl.tolist()


class Table:
    def __init__(self, cells, log2P, log2R, simt=False):
        self.L = H.emu_maint_lib(simt)
        self.cells, self.log2P, self.log2R = cells, log2P, log2R
        self.h = self.L.emu_table_create(cells, log2P, log2R)

    def __del__(self):
        self.L.emu_table_destroy(self.h)

    def put(self, key, cells):
        a = np.ascontiguousarray(cells, dtype=np.uint64)
        assert len(a) == 2 * self.cells
        return self.L.emu_table_put(self.h, key[0], key[1], H._p(a))

    def get(self, key):
        a = np.zeros(2 * self.cells, dtype=np.uint64)
        r = self.L.emu_table_get(self.h, key[0], key[1], H._p(a))
        return (r, a.tolist()) if r >= 0 else (r, None)

    def tombstone(self, key):
        return self.L.emu_table_tombstone(self.h, key[0], key[1])

    def raw(self):
        n = self.L.emu_table_bytes(self.h)
        return np.ctypeslib.as_array(C.cast(self.L.emu_table_raw(self.h), C.POINTER(C.c_uint8)), shape=(n,)).copy()

    def compact(self, pct):
        st = np.zeros(7, dtype=np.uint64)
        sel = np.zeros(1 << self.log2P, dtype=np.uint8)
        self.L.emu_table_compact(self.h, pct, H._p(st), H._p(sel))
        return dict(zip(("regions", "regions_rebuilt", "rows_live", "rows_tombstoned", "rows_moved", "rows_reclaimed", "failures"),
                        [int(x) for x in st])), sel


@pytest.mark.parametrize("simt", [False, True], ids=["plain-path", "warp-aggregated-path"])
@pytest.mark.parametrize("cells,log2P,log2R,seed", [(1, 3, 6, 1), (3, 2, 7, 2), (7, 4, 5, 3), (1, 0, 8, 4), (3, 5, 3, 5)])
def test_a_rebuilt_region_keeps_every_counter_and_frees_its_tombstones(cells, log2P, log2R, seed, simt):
    """(3, 5, 3): regions of 8 rows — one warp of the census covers four regions (the __match_any_sync groups)."""
    H.emu_maint_lib(simt).emu_seed(seed)
    rng = np.random.default_rng(seed)
    t = Table(cells, log2P, log2R, simt)
    R, P = 1 << log2R, 1 << log2P
    live = {}
    keys = [(int(rng.integers(1, 2 ** 62)), (int(rng.integers(1, 9)) << 32) | int(rng.integers(0, 2 ** 32))) for _ in range(int(0.6 * R * P))]
    for k in keys:  # fill to ~60 %, long probe chains included
        c = rng.integers(1, 2 ** 40, size=2 * cells).tolist()
        if rng.random() < 0.1:
            c = [0] * (2 * cells)  # a row whose counters were all deleted: header only
        if t.put(k, c) >= 0:
            live[k] = c
    dead = [k for k in list(live) if rng.random() < 0.45]
    for k in dead:  # what rl_sweep leaves behind
        assert t.tombstone(k) >= 0
        del live[k]
    for k in keys[:len(keys) // 6]:  # and some rows claimed again through tombstones (rl_probe reuses the first one it passed)
        if k not in live:
            c = rng.integers(1, 2 ** 40, size=2 * cells).tolist()
            if t.put(k, c) >= 0:
                live[k] = c
    before = t.raw()
    stats, sel = t.compact(10)
    after = t.raw()
    assert stats["failures"] == 0 and stats["regions"] == P
    assert 0 < stats["regions_rebuilt"] == int(sel.sum())
    rb = 16 * (1 + cells)
    hdr_hi = after.view(np.uint64).reshape(-1, rb // 8)[:, 1].reshape(P, R)
    for g in range(P):
        region = slice(g * R * rb, (g + 1) * R * rb)
        if sel[g]:
            assert not (hdr_hi[g] == TOMB).any(), "a rebuilt region still holds tombstones"
        else:
            assert (before[region] == after[region]).all(), "a region that was not selected changed"
    n_empty = sum(1 for c in live.values() if not any(c))
    for k, c in live.items():  # the hot path's lookup rule finds every counter, with its cells
        r, got = t.get(k)
        if any(c):
            assert r >= 0 and got == c, k
    for k in dead[:300]:
        if k not in live:
            assert t.get(k)[0] < 0
    assert stats["rows_moved"] + stats["rows_reclaimed"] > 0
    assert stats["rows_reclaimed"] >= int((before.view(np.uint64).reshape(-1, rb // 8)[:, 1].reshape(P, R)[sel.astype(bool)] == TOMB).sum())
    # a second pass finds nothing left to do in the rebuilt regions; rebuilding every region with a tombstone (pct 0)
    # leaves a table without tombstones in which every counter is still found
    stats2, sel2 = t.compact(10)
    assert stats2["failures"] == 0 and not (sel2 & sel).any()
    stats3, _ = t.compact(0)
    assert stats3["failures"] == 0
    final = t.raw().view(np.uint64).reshape(-1, rb // 8)
    assert not (final[:, 1] == TOMB).any()
    # header-only rows survive only in regions that never held a tombstone (those are never rebuilt)
    assert len(live) - n_empty <= int((final[:, 1] != 0).sum()) <= len(live)
    for k, c in live.items():
        if any(c):
            assert t.get(k) == (t.get(k)[0], c) and t.get(k)[0] >= 0


def test_threshold_selects_regions_by_their_tombstone_share():
    t = Table(1, 2, 6)  # 4 regions of 64 rows
    rng = np.random.default_rng(9)
    placed = {g: [] for g in range(4)}
    while min(len(v) for v in placed.values()) < 40:
        k = (int(rng.integers(1, 2 ** 62)), (1 << 32) | int(rng.integers(0, 2 ** 32)))
        r = t.put(k, [5, 6])
        if r >= 0 and len(placed[r >> 6]) < 40:
            placed[r >> 6].append(k)
        elif r >= 0:
            t.tombstone(k)
            t.compact(0)
    t.compact(0)
    for g, want in ((0, 0), (1, 10), (2, 16), (3, 33)):  # tombstones per region: 0 %, 15.6 %, 25 %, 51.6 % of 64 rows
        for k in placed[g][:want]:
            t.tombstone(k)
    _, sel = Table.compact(t, 25)
    assert sel.tolist() == [0, 0, 1, 1]
    stats, sel = t.compact(1)
    assert sel.tolist() == [0, 1, 0, 0] and stats["rows_tombstoned"] == 10
    stats, sel = t.compact(0)
    assert sel.tolist() == [0, 0, 0, 0] and stats["rows_tombstoned"] == 0 and stats["rows_live"] == 4 * 40 - 59


def test_the_fiber_emulator_computes_the_intrinsics_and_refuses_what_would_hang_a_gpu(tmp_path):
    """tests/emu/cuda_simt.h on its own (tests/emu/simt_selftest.cpp): __match_any_sync groups reducing over their own
    masks, ballots, shuffles, __shfl_up_sync scans, the reducing barriers, poisoned per-block dynamic shared memory and a flag
    wait across two resident blocks against closed forms; then the mistakes it must abort on, the same flag wait with one
    resident block among them."""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    exe = str(tmp_path / "simt_selftest")
    subprocess.check_call(["g++", "-O1", "-std=c++17", os.path.join(here, "emu", "simt_selftest.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.startswith("ok simt"), r.stdout + r.stderr
    for case, message in (("exited", "names a thread that has exited"), ("mask", "cuda_simt: "),
                          ("barrier", "no thread of the block can make progress"),
                          ("spin", "waits in a __nanosleep loop")):
        r = subprocess.run([exe, case], capture_output=True, text=True, timeout=120)
        assert r.returncode != 0 and message in r.stderr and "not refused" not in r.stdout, (case, r.stdout, r.stderr)
