"""The decision kernels on the GPU at the batch geometries only a large batch reaches (the same geometries run on the
host under the fiber emulator in tests/test_decision_kernels_emu.py, at the sizes a CPU affords): 256-access chunks
over more than 256 tiles, the coupled and wide paths past one tile-merge pass, k_hot over more than 512 tiles with a
hot list longer than one sweep, and a chained partition whose chunk indices pass 2048.  Every batch is compared with
the CPU oracle, the table included, and every case asserts its geometry through Engine.stats().  These are ordinary
workloads: liveness of the chained commit is checked on the host, by the emulator's wait-loop detector."""
import numpy as np
import pytest

from limitador_b200 import Engine
from limitador_b200.engine import LIMIT_DESC_DTYPE, RECORD_DTYPE
from tests import helpers as H

pytestmark = pytest.mark.gpu
KERNEL_STATS, HOT_ROWS = 4, 16
M = (1 << 64) - 1


def _mix64(x):
    x = x ^ (x >> np.uint64(33))
    x = x * np.uint64(0xFF51AFD7ED558CCD)
    x = x ^ (x >> np.uint64(33))
    x = x * np.uint64(0xC4CEB9FE1A85EC53)
    return x ^ (x >> np.uint64(33))


def region_of(key_lo, key_hi, group, log2P):
    """rl_row_hash's region (rl_core.h) of a qualified row of row group `group`."""
    with np.errstate(over="ignore"):
        hdr = (np.uint64(group) << np.uint64(32)) | np.asarray(key_hi, dtype=np.uint64)
        h = _mix64(np.asarray(key_lo, dtype=np.uint64) ^ _mix64(hdr ^ np.uint64(0x9E3779B97F4A7C15)))
    return (h >> np.uint64(64 - log2P)).astype(np.int64)


def limits(n_ns, per_ns, mx=(40, 1 << 40, 7), win=(10, 60, 2)):
    descs, lid = [], 0
    for ns in range(n_ns):
        for k in range(per_ns):
            descs.append((lid, ns, 1, 1, mx[(ns + k) % len(mx)], win[(ns + k) % len(win)] * 1_000_000))
            lid += 1
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


def records(descs, n, seed, n_keys=2000, rowless=0.0, t0=H.T0):
    rng = np.random.default_rng(seed)
    r = np.zeros(n, dtype=RECORD_DTYPE)
    r["ns_id"] = rng.choice(sorted({int(d["ns_id"]) for d in descs}), size=n)
    r["ns_id"][rng.random(n) < rowless] = int(descs["ns_id"].max()) + 5
    r["hits_addend"] = rng.choice([1, 1, 2, 3], size=n)
    r["key_lo"] = rng.integers(1, n_keys + 1, size=n)
    r["key_hi"] = rng.integers(0, 2, size=n)
    r["now_us"] = t0 + np.cumsum(rng.choice([0, 1, 1000, 100_000], size=n))
    return r


def check(e, o, descs, recs, lc=False, stride=None):
    before = e.stats()
    lim, fl, rem, ttl = e.check_and_update_records(recs, load_counters=lc, stride=stride)
    after = e.stats()
    ol, of, orem, ottl = o.batch_records(0, recs, lc, stride=stride or e.cells_per_row)
    assert lim.tolist() == ol.tolist(), f"verdicts differ at {np.nonzero(lim != ol)[0][:10].tolist()}"
    assert fl.tolist() == of.tolist(), "first-limited ids differ"
    if lc:
        assert rem.tolist() == orem.tolist() and ttl.tolist() == ottl.tolist(), "remaining / ttl differ"
    assert H.normalise_dump(e.dump(), descs) == H.normalise_dump(o.dump(), descs), "table differs"
    return {k: after[k] - before[k] for k in ("chunks", "chained_chunks", "ordered_chunks")} | {
        "hot_rows": after["hot_rows"], "fixed_point_rounds": after["fixed_point_rounds"]}


def test_256_access_chunks_over_more_than_256_tiles(monkeypatch):
    monkeypatch.setenv("RL_CHUNK", "256")
    descs = limits(4, 3)
    n = 300 * 1024  # tiles of 512 accesses: 600 of them
    e = Engine(capacity_rows=1 << 16, cells_per_row=3, max_batch=n, regions=16, flags=KERNEL_STATS)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    for b in range(2):
        g = check(e, o, descs, records(descs, n, seed=b, rowless=0.7), lc=(b == 1))
        assert g["chunks"] > 0, g


def test_coupled_and_wide_paths_past_one_merge_pass():
    """Records of namespaces spanning several rows (the coupled fixed point, undo log of num_tiles * tile positions) and
    of a namespace of 20 limits (the wide encoding), each batch more than 128 tiles of accesses."""
    descs = H.mixed_limits(6, seed=3)
    n = 160 * 512 // 5
    e = Engine(capacity_rows=1 << 16, cells_per_row=7, max_batch=n, max_counters=n * 5, regions=8, flags=KERNEL_STATS)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    g = check(e, o, descs, records(descs, n, seed=7, n_keys=6, rowless=0.85), lc=True, stride=5)
    assert g["fixed_point_rounds"] >= 1, g
    wdescs = H.wide_limits(5, sizes=(20, 3))
    n = 160 * 512 // 20
    e = Engine(capacity_rows=1 << 16, cells_per_row=7, max_batch=n, max_counters=n * 20, regions=8,
               max_counters_per_request=64, flags=KERNEL_STATS)
    e.limits_set(wdescs)
    o = H.oracle_with_limits(wdescs)
    check(e, o, wdescs, records(wdescs, n, seed=8, n_keys=3, rowless=0.8), lc=True, stride=20)


def test_hot_rows_over_more_than_512_tiles_and_lists_longer_than_a_sweep():
    """A 2^20 batch with hot rows on: 1024 tiles, so k_hot merges in two passes, and one hot row with 40 000 requests,
    more than one k_hot sweep (32 768) looks at."""
    descs = limits(2, 2, mx=(30_000, 1 << 40), win=(3600, 60))
    n = 1 << 20
    e = Engine(capacity_rows=1 << 20, cells_per_row=3, max_batch=n, regions=64, flags=KERNEL_STATS | HOT_ROWS)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    t = H.T0
    for b in range(2):  # rows 5 and 6 of namespace 0 dominate their chunks: candidates, admitted by the next front
        r = np.zeros(256, dtype=RECORD_DTYPE)
        r["key_lo"] = np.repeat([5, 6], 128)
        r["hits_addend"] = 1
        r["now_us"] = t + np.arange(256)
        t += 1_000_000
        check(e, o, descs, r)
    assert e.stats()["hot_rows"] >= 2
    recs = records(descs, n, seed=3, n_keys=200_000, t0=t)
    rng = np.random.default_rng(4)
    hot5 = rng.choice(n, size=40_000, replace=False)
    recs["ns_id"][hot5] = 0
    recs["key_lo"][hot5] = 5
    recs["key_hi"][hot5] = 0
    g = check(e, o, descs, recs)
    assert g["hot_rows"] >= 2, g


def test_chained_partition_with_chunk_indices_past_2048():
    """2^20 records, 16 regions, hot rows off, a third of the keys in region 0: that partition is longer than two
    average ones and is chained in more than 2048 chunks of 128 — the chunks past 2048 wait for every earlier chunk."""
    descs = limits(1, 3, mx=(5000, 1 << 40, 90), win=(60, 3600, 10))
    n, log2P = 1 << 20, 4
    e = Engine(capacity_rows=1 << 20, cells_per_row=3, max_batch=n, regions=1 << log2P, flags=KERNEL_STATS)
    e.limits_set(descs)
    o = H.oracle_with_limits(descs)
    group = H.Emu(descs, 3).group_of(0)  # the row group the engine's registry gives limit 0
    rng = np.random.default_rng(5)
    keys = np.arange(1, 400_001, dtype=np.uint64)
    reg = region_of(keys, np.zeros_like(keys), group, log2P)
    home, other = keys[reg == 0][:3000], keys[reg != 0][:30_000]
    recs = np.zeros(n, dtype=RECORD_DTYPE)
    at_home = rng.random(n) < 0.33
    recs["key_lo"] = np.where(at_home, rng.choice(home, size=n), rng.choice(other, size=n))
    recs["hits_addend"] = rng.choice([1, 1, 2], size=n)
    recs["now_us"] = H.T0 + np.cumsum(rng.choice([0, 1, 100], size=n))
    g = check(e, o, descs, recs)
    assert g["chained_chunks"] > 2048 and g["ordered_chunks"] > 0, g
