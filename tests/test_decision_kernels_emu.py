"""The decision kernels themselves (k_front, k_hot, k_main and the general path's resolve, restore and fixed-point
kernels) run on the host under the fiber emulator (tests/emu/emu_engine.cpp over tests/emu/cuda_simt.h), at the
batch geometries whose code paths only large or unusual batches reach, against the C oracle: verdicts, first-limited
ids, remaining / ttl with load_counters, and the whole table (read back through k_scan's export) after every batch.
Every case asserts, from the call's geometry report, that it reached the geometry it is named for."""
from __future__ import annotations

import numpy as np
import pytest

from limitador_b200.engine import LIMIT_DESC_DTYPE, RECORD_DTYPE
from tests import helpers as H

RL_VERDICT_ERROR = 0xFF
RL_DEV_TABLE_FULL = 1


@pytest.fixture(scope="module", autouse=True)
def _built():
    H.emu_engine_lib()  # one build for the whole file


def single_row_limits(n_ns=4, per_ns=(1, 3, 2, 2), unqualified_ns=True, mx=(5, 40, 1 << 40, 3), win=(1, 10, 60, 2)):
    """Namespaces whose limits all sit in one row (one variable set): the record form replays them straight from the
    records; plus an unqualified namespace."""
    descs, lid = [], 0
    for ns in range(n_ns):
        for k in range(per_ns[ns % len(per_ns)]):
            descs.append((lid, ns, 1, 1, mx[(ns + k) % len(mx)], win[(ns + k) % len(win)] * 1_000_000))
            lid += 1
    if unqualified_ns:
        descs.append((lid, n_ns, 0, 0, 7, 1_000_000))
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


def records(descs, n, seed, n_keys=40, rowless=0.0, ns=None, t0=H.T0, step=(0, 1, 1000, 300_000)):
    """Records over the namespaces of `descs` (or `ns`), a share `rowless` of them naming a namespace without limits."""
    rng = np.random.default_rng(seed)
    nss = sorted({int(d["ns_id"]) for d in descs}) if ns is None else list(ns)
    r = np.zeros(n, dtype=RECORD_DTYPE)
    r["ns_id"] = rng.choice(nss, size=n)
    r["ns_id"][rng.random(n) < rowless] = int(descs["ns_id"].max()) + 5
    r["hits_addend"] = rng.choice([1, 1, 1, 2, 3], size=n)
    r["key_lo"] = rng.integers(1, n_keys + 1, size=n)
    r["key_hi"] = rng.integers(0, 2, size=n)
    r["now_us"] = t0 + np.cumsum(rng.choice(step, size=n))
    return r


def check_records(emu, orc, descs, recs, mode=0, lc=False):
    """One record batch through the emulated kernels and the oracle: everything must agree."""
    lim, fl, rem, ttl, err = emu.records(mode, recs, lc)
    assert err == 0, f"device error {err}"
    stride = len(rem) // max(len(recs), 1)
    ol, of, orem, ottl = orc.batch_records(mode, recs, lc, stride=stride)
    if mode == 0:
        bad = np.nonzero(lim != ol)[0]
        assert not len(bad), f"verdicts differ at {bad[:10].tolist()} ({len(bad)} of {len(recs)})"
        assert fl.tolist() == of.tolist(), "first-limited ids differ"
        if lc:
            assert rem.tolist() == orem.tolist(), "remaining differs"
            assert ttl.tolist() == ottl.tolist(), "ttl differs"
    assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs), "table differs"
    assert emu.geometry["rearmed"] == 1, "the front's and the replay's counters are not re-armed for the next batch"
    return emu.geometry


def check_csr(emu, orc, descs, batch, mode=0, lc=False):
    off, ctrs, delta, now = batch
    lim, fl, rem, ttl, err = emu.csr(mode, off, ctrs, delta, now, lc)
    assert err == 0, f"device error {err}"
    ol, of, orem, ottl = orc.batch_csr(mode, off, ctrs, delta, now, lc)
    if mode == 0:
        assert lim.tolist() == ol.tolist(), "verdicts differ"
        assert fl.tolist() == of.tolist(), "first-limited ids differ"
        if lc:
            assert rem.tolist() == orem.tolist(), "remaining differs"
            assert ttl.tolist() == ottl.tolist(), "ttl differs"
    assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs), "table differs"
    return emu.geometry


# ---- more tiles than one merge pass takes --------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [128, 256])
def test_record_path_merges_more_tiles_than_a_chunk_has_threads(chunk):
    """k_main merges a partition's per-tile runs CH tiles per pass: past CH tiles it takes a second pass (carry), and
    list_at searches prefixes over many tiles, most of whose runs for a given partition are empty.  262 tiles: three
    passes at CH = 128 (the carry of two earlier passes in the third), two at CH = 256."""
    descs = single_row_limits()
    n = 2 * 128 * 512 + 3000  # tiles of 512 accesses
    emu = H.EmuEngine(descs, 3, 4, 10, chunk=chunk)
    orc = H.oracle_with_limits(descs)
    for b in range(2):
        g = check_records(emu, orc, descs, records(descs, n, seed=b, rowless=0.9), lc=(b == 1))
        assert g["tiles"] > chunk and g["merge_passes_main"] == -(-262 // chunk) and g["ch"] == chunk, g


def test_coupled_records_merge_more_tiles_than_a_chunk_has_threads():
    """Records of namespaces spanning several rows: resolved into accesses (rows of slots, the unused ones rowless), then
    SNAPSHOT, SPEC rounds with k_restore over an undo log of num_tiles * tile positions, and COMMIT, past 128 tiles."""
    descs = H.mixed_limits(6, seed=3)
    emu = H.EmuEngine(descs, 7, 3, 10)
    orc = H.oracle_with_limits(descs)
    stride = 5  # mixed_limits' widest namespace
    n = 129 * 512 // stride + 400
    g = check_records(emu, orc, descs, records(descs, n, seed=7, n_keys=6, rowless=0.85), lc=True)
    assert g["tiles"] > 128 and g["merge_passes_main"] == 2 and g["fixed_point_rounds"] >= 1, g


def test_wide_records_merge_more_tiles_than_a_chunk_has_threads():
    """The wide path (a namespace of more than 16 limits): k_resolve_records_wide, AccSrcWide's k_main, k_wide_scatter."""
    descs = H.wide_limits(5, sizes=(20, 3))
    emu = H.EmuEngine(descs, 7, 3, 10)
    orc = H.oracle_with_limits(descs)
    n = 129 * 512 // 20 + 200
    g = check_records(emu, orc, descs, records(descs, n, seed=8, n_keys=3, rowless=0.8), lc=True)
    assert g["tiles"] > 128 and g["merge_passes_main"] == 2, g


def test_sharded_geometry_derives_256_access_tiles_on_the_device():
    """n_dev set: the tile is derived from the device-side count (rl_tile_of), 256 accesses over up to 256 tiles."""
    descs = single_row_limits()
    emu = H.EmuEngine(descs, 3, 4, 10, sharded=True)
    orc = H.oracle_with_limits(descs)
    for b, n in enumerate((33_500, 700, 257)):
        g = check_records(emu, orc, descs, records(descs, n, seed=20 + b, rowless=0.6))
        assert g["tile"] == 256 and g["tiles"] == min(256, -(-n // 256)), g
        if b == 0:
            assert g["tiles"] > 128 and g["merge_passes_main"] == 2, g


# ---- chained partitions -------------------------------------------------------------------------------------------
def region_heavy_records(emu, descs, n, seed, region=0, share=0.9, n_keys=60):
    """Records most of whose keys live in one table region: that partition is chained (longer than heavy_len)."""
    rng = np.random.default_rng(seed)
    pool = records(descs, 40 * n_keys, seed=seed + 1000, n_keys=n_keys * 20)
    home = [r for r in pool if emu.region_of(r) == region][:n_keys]
    other = [r for r in pool if emu.region_of(r) not in (region, -1)][:n_keys]
    assert len(home) == n_keys and other
    r = np.zeros(n, dtype=RECORD_DTYPE)
    pick_home = rng.random(n) < share
    for i in range(n):
        src = home if pick_home[i] else other
        r[i] = src[int(rng.integers(0, len(src)))]
    r["hits_addend"] = rng.choice([1, 1, 2], size=n)
    r["now_us"] = H.T0 + np.cumsum(rng.choice([0, 1, 50_000], size=n))
    return r


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_chained_partition_longer_than_a_chunk_scan_block_under_resident_blocks(seed):
    """A partition of more than CH chunks: the dependency scan runs in several blocks of CH chunks, and chunk indices
    reach past 64.  Two to four k_main blocks are resident and interleaved, so a chunk's first read races the commit of
    the chunk before it: the re-read of declared rows and the wait for exactly the chunks it depends on both matter."""
    descs = single_row_limits(n_ns=2, per_ns=(1, 3), unqualified_ns=False, mx=(60, 400), win=(10, 60))
    emu = H.EmuEngine(descs, 3, 2, 12, resident=1 + seed, interleave=(seed, 0.5))
    orc = H.oracle_with_limits(descs)
    g = check_records(emu, orc, descs, region_heavy_records(emu, descs, 150 * 128, seed, n_keys=40))
    assert g["max_w"] > 128 and g["chained_chunks"] > 128 and g["ordered_chunks"] > 0, g


# ---- hot rows -----------------------------------------------------------------------------------------------------
def hot_records(keys, reps, seed, t0, ns=0):
    """`reps` consecutive requests per key: each key dominates the chunk it falls in (a hot-row candidate)."""
    rng = np.random.default_rng(seed)
    r = np.zeros(len(keys) * reps, dtype=RECORD_DTYPE)
    r["ns_id"] = ns
    r["key_lo"] = np.repeat(np.asarray(keys, dtype=np.uint64), reps)
    r["hits_addend"] = rng.choice([1, 1, 2], size=len(r))
    r["now_us"] = t0 + np.cumsum(rng.choice([0, 1, 10_000], size=len(r)))
    return r


def test_hot_table_fills_drops_and_readmits_rows():
    """More than RL_HOT_CAND candidates in a batch, all RL_HOT_SLOTS slots taken, rows that cool down dropped and
    admitted again: k_front's tail under pressure, and k_hot replaying many hot rows beside k_main."""
    descs = single_row_limits(n_ns=1, per_ns=(2,), unqualified_ns=False, mx=(500, 3000), win=(60, 3600))
    emu = H.EmuEngine(descs, 3, 3, 12, hot=True)
    orc = H.oracle_with_limits(descs)
    t = H.T0
    seen = []
    plan = [range(1, 201), range(201, 401), range(1, 201), range(401, 601), range(1, 201)]
    for b, keys in enumerate(plan):
        recs = hot_records(list(keys), 40, seed=b, t0=t)
        t = int(recs["now_us"][-1]) + 1
        g = check_records(emu, orc, descs, recs, lc=(b % 2 == 1))
        seen.append(g)
    assert max(g["hot_candidates"] for g in seen) > 128, seen
    assert max(g["hot_after"] for g in seen) == 256, [g["hot_after"] for g in seen]
    assert any(g["hot_after"] < g["hot_in_use"] for g in seen), "no hot row was ever dropped"
    assert any(g["hot_in_use"] > 0 and g["hot_max_list"] > 0 for g in seen), "k_hot never replayed a list"


def test_hot_row_list_longer_than_one_sweep():
    """A hot row with more requests in one batch than one k_hot sweep looks at (RL_HOT_SWEEP = 32768)."""
    descs = single_row_limits(n_ns=1, per_ns=(1,), unqualified_ns=False, mx=(20_000,), win=(3600,))
    emu = H.EmuEngine(descs, 1, 2, 10, hot=True)
    orc = H.oracle_with_limits(descs)
    g = check_records(emu, orc, descs, hot_records([7, 8], 64, seed=1, t0=H.T0))
    assert g["hot_candidates"] >= 1, g
    check_records(emu, orc, descs, hot_records([9], 64, seed=3, t0=H.T0 + 5_000_000))  # its front admits them
    recs = hot_records([7], 33_000, seed=2, t0=H.T0 + 10_000_000)
    g = check_records(emu, orc, descs, recs)
    assert g["hot_in_use"] >= 1 and g["hot_max_list"] > 32_768 and g["hot_sweeps"] >= 2, g


# ---- the 7/4 -> 7/7 instantiation change with live counters ---------------------------------------------------------
def test_fifth_limit_joins_a_row_group_with_live_counters():
    """128-byte rows with at most 4 cells in use run k_main<7, 4>; a fifth limit joining a row group that already has
    counters switches to k_main<7, 7> (and k_restore to 7 active cells) without losing or misreading a counter."""
    base = [(0, 0, 1, 1, 30, 10_000_000), (1, 0, 1, 1, 200, 60_000_000), (2, 0, 1, 1, 9, 2_000_000),
            (3, 0, 1, 1, 1 << 40, 3600_000_000), (4, 1, 1, 1, 5, 1_000_000), (5, 1, 2, 1, 8, 1_000_000)]
    descs = np.array(base, dtype=LIMIT_DESC_DTYPE)
    emu = H.EmuEngine(descs, 7, 3, 10)
    orc = H.oracle_with_limits(descs)
    assert emu.max_cells_used == 4
    recs = records(descs, 3000, seed=1, n_keys=20, ns=[0])
    check_records(emu, orc, descs, recs, lc=True)
    csr = H.random_csr_stream(descs, 1500, seed=2, n_keys=20)
    check_csr(emu, orc, descs, csr, lc=True)
    more = np.array(base + [(6, 0, 1, 1, 12, 5_000_000)], dtype=LIMIT_DESC_DTYPE)
    emu.set_limits(more[6:])
    orc.limit_set(6, 0, 12, 5_000_000, True)
    assert emu.max_cells_used == 5
    recs = records(more, 3000, seed=3, n_keys=20, ns=[0], t0=int(recs["now_us"][-1]))
    check_records(emu, orc, more, recs, lc=True)
    check_csr(emu, orc, more, H.random_csr_stream(more, 1500, seed=4, n_keys=20), lc=True)


# ---- small and ragged batches ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 31, 33, 511, 513, 2049])
def test_small_and_ragged_batches(n):
    """Fewer accesses than a warp, one tile, a batch that is not a multiple of the tile, in both chunk sizes."""
    descs = single_row_limits()
    for chunk in (128, 256):
        emu = H.EmuEngine(descs, 3, 4, 8, chunk=chunk)
        orc = H.oracle_with_limits(descs)
        for b in range(2):
            g = check_records(emu, orc, descs, records(descs, n, seed=n + b, n_keys=4), lc=(b == 1))
            assert g["tiles"] == -(-n // 512), g


def test_partitions_only_in_the_first_or_the_last_tile_and_rowless_batches():
    descs = single_row_limits()
    emu = H.EmuEngine(descs, 3, 4, 8)
    orc = H.oracle_with_limits(descs)
    n = 5 * 512 + 17
    for where in ("first", "last", "none"):
        recs = records(descs, n, seed=len(where), rowless=1.0)
        live = records(descs, 300, seed=9, n_keys=5)
        if where == "first":
            recs[:300] = live
        elif where == "last":
            recs[-300:] = live
        g = check_records(emu, orc, descs, recs, lc=True)
        assert g["tiles"] == 6 and (g["items"] == 0) == (where == "none"), g


def test_a_full_region_inside_a_large_batch():
    """Regions of 16 rows and many keys: the probe finds regions full, those requests say RL_VERDICT_ERROR and touch
    nothing, and every other request is decided as if they were not there."""
    descs = single_row_limits(n_ns=1, per_ns=(2,), unqualified_ns=False)
    emu = H.EmuEngine(descs, 3, 4, 4)
    recs = records(descs, 6000, seed=4, n_keys=400)
    lim, fl, rem, ttl, err = emu.records(0, recs, True)
    assert err == RL_DEV_TABLE_FULL
    bad = lim == RL_VERDICT_ERROR
    assert 0 < bad.sum() < len(recs)
    orc = H.oracle_with_limits(descs)
    ol, of, orem, ottl = orc.batch_records(0, recs[~bad], True, stride=3)
    assert lim[~bad].tolist() == ol.tolist() and fl[~bad].tolist() == of.tolist()
    assert rem.reshape(-1, 3)[~bad].ravel().tolist() == orem.tolist()
    assert ttl.reshape(-1, 3)[~bad].ravel().tolist() == ottl.tolist()
    assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs)


# ---- the edge-arithmetic streams through every instantiation ------------------------------------------------------
@pytest.mark.parametrize("cells,per_ns,chunk", [(1, 1, 128), (3, 3, 256), (7, 4, 128), (7, 7, 256)])
def test_edge_streams_through_every_instantiation(cells, per_ns, chunk):
    """tests/helpers.py's edge-arithmetic record streams (u64 wrap, exact window boundaries, counters above their
    maximum, clocks going back) through k_main<1,1>, <3,3>, <7,4> and <7,7>, with update_counters and is_rate_limited
    batches between the check_and_update ones."""
    descs = H.edge_limits(cells * 10 + per_ns, shape="single", n_ns=6, cells=per_ns)
    emu = H.EmuEngine(descs, cells, 3, 9, chunk=chunk, weak=(cells == 7))
    orc = H.oracle_with_limits(descs)
    assert emu.max_cells_used <= (4 if per_ns <= 4 else 7)
    for b, (mode, recs) in enumerate(H.edge_batches(descs, cells + per_ns, 4, 700, form="records")):
        if mode == 1:
            lim, fl, err = emu.query_records(recs)
            ol, of, _, _ = orc.batch_records(1, recs)
            assert err == 0 and lim.tolist() == ol.tolist() and fl.tolist() == of.tolist()
            continue
        check_records(emu, orc, descs, recs, mode=mode, lc=(b % 2 == 0))


def test_hot_rows_over_more_tiles_than_k_hot_has_threads():
    """k_hot merges a hot row's per-tile runs 512 tiles per pass: a batch of more than 512 tiles (262 144 accesses)
    takes two, with the hot row's requests spread over all of them."""
    descs = single_row_limits(n_ns=1, per_ns=(2,), unqualified_ns=False, mx=(3000, 100_000), win=(60, 3600))
    emu = H.EmuEngine(descs, 3, 3, 10, hot=True)
    orc = H.oracle_with_limits(descs)
    check_records(emu, orc, descs, hot_records([5, 6], 64, seed=1, t0=H.T0))
    check_records(emu, orc, descs, hot_records([7], 64, seed=2, t0=H.T0 + 1_000_000))  # its front admits 5 and 6
    n = 513 * 512 + 100
    recs = records(descs, n, seed=3, rowless=1.0, t0=H.T0 + 2_000_000)
    hot_at = np.random.default_rng(4).random(n) < 0.01
    recs["ns_id"][hot_at] = 0
    recs["key_lo"][hot_at] = 5
    recs["key_hi"][hot_at] = 0
    g = check_records(emu, orc, descs, recs)
    assert g["tiles"] > 512 and g["merge_passes_hot"] == 2 and g["hot_in_use"] >= 1 and g["hot_max_list"] > 2000, g
