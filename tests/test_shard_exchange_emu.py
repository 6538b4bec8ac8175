"""The namespace-sharded peer exchange (limitador_b200/csrc/rl_shard.cuh, DESIGN.md §8) without a GPU: k_xcount,
k_xscatter, k_xwait, the record path over the segmented inbox with its verdict mirror, k_xreturn, k_xwaitv and k_xgather
run on the host under the fiber emulator (tests/emu/emu_engine.cpp's emu_shard_* over tests/emu/cuda_simt.h), `world`
emulated engines over host slabs laid out as rl_shard_create lays out the device ones.

Whole steps are checked against ONE global oracle that applies them in (step, source rank, source index) order — the
canonical stream order of the sharded store: the verdict of every request at its source, the union of the rank tables,
and every counter on its owner.  The send half alone is checked against a numpy stable bucketing by owner.  Every case
asserts, from the decide call's geometry report, that it reached what it is named for."""
from __future__ import annotations

import numpy as np
import pytest

from limitador_b200.engine import LIMIT_DESC_DTYPE, RECORD_DTYPE, pack_records16
from tests import helpers as H

RL_VERDICT_ERROR = 0xFF
RL_DEV_TABLE_FULL, RL_DEV_KEY_RANGE, RL_DEV_EXCHANGE = 1, 3, 6
POISON32 = 0xA5A5A5A5


@pytest.fixture(scope="module", autouse=True)
def _built():
    H.emu_engine_lib()  # one build for the whole file


def owner_of(ns_id, world):
    """rl_owner_dev: rl_mix64(ns_id + 0x51ed270b0a1f) % world, over a numpy array."""
    with np.errstate(over="ignore"):
        x = np.asarray(ns_id, dtype=np.uint64) + np.uint64(0x51ED270B0A1F)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xFF51AFD7ED558CCD)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xC4CEB9FE1A85EC53)
        x ^= x >> np.uint64(33)
    return (x % np.uint64(world)).astype(np.int64)


def namespaces_of_owner(owner, world, count, start=0):
    ns = np.arange(start, start + 64 * world * count + 64, dtype=np.uint64)
    got = ns[owner_of(ns, world) == owner][:count]
    assert len(got) == count
    return got.astype(np.uint32)


def limits(n_ns, per_ns, windows=(1, 60, 3600, 10, 2, 5, 30), maxes=(5, 100, 2000, 20, 8, 50, 300), ns_ids=None):
    """`per_ns` limits on one variable set per namespace: every namespace is one row (the record path)."""
    nss = range(n_ns) if ns_ids is None else ns_ids
    d, lid = [], 0
    for ns in nss:
        for k in range(per_ns):
            d.append((lid, int(ns), 1, 1, maxes[k], windows[k] * 1_000_000))
            lid += 1
    return np.array(d, dtype=LIMIT_DESC_DTYPE)


def recs_of(n, nss, seed, t0, n_keys=200, span_us=1_000_000, zipf=None, hits=(1, 1, 1, 2, 3)):
    """n records over the namespaces `nss`, clocks rising across [t0, t0 + span_us); zipf=(share, n_head_keys) puts a
    share of them on a few head keys of the first namespace."""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, dtype=RECORD_DTYPE)
    r["ns_id"] = rng.choice(np.asarray(nss, dtype=np.uint32), size=n)
    r["hits_addend"] = rng.choice(hits, size=n)
    r["key_lo"] = rng.integers(1, n_keys + 1, size=n)
    r["key_hi"] = rng.integers(0, 2, size=n)
    if zipf is not None:
        head = rng.random(n) < zipf[0]
        r["ns_id"][head] = nss[0]
        r["key_lo"][head] = rng.integers(1, zipf[1] + 1, size=int(head.sum()))
        r["key_hi"][head] = 0
    r["now_us"] = t0 + np.sort(rng.integers(0, span_us, size=n))
    return r


def make_shard(descs, cells, world, cap, lag, log2P=3, log2R=9, max_batch=None, **knobs):
    engines = [H.EmuEngine(descs, cells, log2P, log2R, **knobs) for _ in range(world)]
    return H.EmuShard(engines, cap, lag, max_batch), engines


def run_steps(sh, engines, steps, expect_err=None):
    """steps[st][r] = rank r's records of step st, issued phase by phase: every rank sends, every rank decides, every
    rank collects (what lag allows), then a flush.  Returns (verdicts [st][r], geometry reports, error words)."""
    world = sh.world
    outs, geos, errs = [], [], []
    for st, row in enumerate(steps):
        outs.append([sh.send(r, row[r]) for r in range(world)])
        buf = st % sh.depth
        for r in range(world):
            ctl = sh.ctl(r)
            assert ctl[buf, :, 1].tolist() == [st + 1] * world, f"step {st}: rflag of rank {r}'s blocks"
            fills = [int((owner_of(row[s]["ns_id"], world) == r).sum()) for s in range(world)]
            assert ctl[buf, :, 0].tolist() == fills, f"step {st}: fills of rank {r}'s inbox"
        for r in range(world):
            err = sh.decide(r)
            e = sh.err(r)
            errs.append((st, r, int(e[0]), int(e[7])))
            if expect_err is None:
                assert err == 0 and e[7] == 0, f"step {st} rank {r}: device error {err}, detail {e[7]:#x}"
            g = dict(engines[r].geometry, step=st, rank=r, fill=sum(
                int((owner_of(row[s]["ns_id"], world) == r).sum()) for s in range(world)))
            assert g["rearmed"] == 1, g
            geos.append(g)
        for r in range(world):
            assert sh.ctl(r)[buf, :, 2].tolist() == [st + 1] * world, f"step {st}: vflag of rank {r}'s verdicts"
            assert sh.ctrs(r)[:3].tolist() == [0, 0, 0], "blocks-done counters not re-armed"
        for r in range(world):
            sh.collect(r)
    for r in range(world):
        sh.collect(r, flush=True)
    return outs, geos, errs


def check_against_oracle(descs, world, engines, steps, outs, skip=None):
    """One oracle over (step, source rank, source index): verdicts at their sources, the union of the tables, every
    counter on its owner.  skip[(st, r)] = a boolean mask of requests the oracle does not see (their verdict is checked by
    the caller)."""
    o = H.oracle_with_limits(descs, 1 << 16)
    for st, row in enumerate(steps):
        for r in range(world):
            recs, got = row[r], outs[st][r]
            keep = np.ones(len(recs), dtype=bool) if skip is None or (st, r) not in skip else ~skip[(st, r)]
            if not keep.any():
                continue
            want = o.batch_records(0, recs[keep])[0]
            bad = np.nonzero(got[keep] != want)[0]
            assert not len(bad), f"step {st} rank {r}: {len(bad)} of {int(keep.sum())} verdicts differ, first at {bad[:8].tolist()}"
    union = [row for e in engines for row in e.dump()]
    assert H.normalise_dump(union, descs) == H.normalise_dump(o.dump(), descs), "the union of the rank tables differs"
    ns_of = {int(d["limit_id"]): int(d["ns_id"]) for d in descs}
    for r, e in enumerate(engines):
        for row in e.dump():
            assert owner_of(ns_of[row[0]], world) == r, f"a counter of namespace {ns_of[row[0]]} sits on rank {r}"


# ---- the send half: k_xcount and k_xscatter against a stable bucketing by owner -------------------------------------
def send_records(n, world, pattern, seed):
    rng = np.random.default_rng(seed)
    r = np.zeros(n, dtype=RECORD_DTYPE)
    if pattern == "one_owner":
        r["ns_id"] = rng.choice(namespaces_of_owner(world - 1, world, 3), size=n)
    elif pattern == "alternating":
        per = [namespaces_of_owner(o, world, 1)[0] for o in range(world)]
        r["ns_id"] = np.asarray(per, dtype=np.uint32)[np.arange(n) % world]
    else:
        r["ns_id"] = rng.integers(0, 4 * world + 7, size=n)
    r["hits_addend"] = np.arange(n) % 7 + 1
    r["key_lo"] = np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed)
    r["key_hi"] = np.arange(n) % 3
    r["now_us"] = H.T0 + np.arange(n)
    return r


@pytest.mark.parametrize("n,world,pattern", [
    (0, 1, "random"), (0, 32, "random"), (1, 2, "random"), (1, 32, "one_owner"), (255, 3, "alternating"),
    (256, 5, "random"), (257, 32, "alternating"), (257, 8, "one_owner"), (4097, 8, "random"), (4097, 5, "alternating"),
    (65_536, 3, "random"), (65_536, 2, "alternating"), (262_145, 2, "random"), (262_145, 2, "one_owner")])
def test_send_half_buckets_stably_by_owner(n, world, pattern):
    """Every inbox block holds its source's records of that owner in source order; dest[a] = owner << 27 | position;
    the fills and the step flags of every (buffer, peer) are published; the blocks-done counters are re-armed.  65 536
    records are 256 tiles (32 per warp in k_xcount's last-block scan), 262 145 are tiles of 512."""
    cap = max(16, -(-n // 16) * 16)
    sh, _ = make_shard(limits(1, 1), 1, world, cap, lag=1, log2P=0, log2R=4)
    small = min(n, 40)  # the other ranks send a little, so that every (owner, source) block is written
    for st in range(2):
        sent = [send_records(n if r == st % world else small, world, pattern, seed=10 * st + r) for r in range(world)]
        for r in range(world):
            sh.send(r, sent[r])
        for r in range(world):
            recs = sent[r]
            own = owner_of(recs["ns_id"], world)
            pos = np.zeros(len(recs), dtype=np.int64)
            for o in range(world):
                at = np.nonzero(own == o)[0]
                pos[at] = np.arange(len(at))
                block = sh.inbox(o, st, r)
                assert np.array_equal(block[:len(at)], recs[at]), f"step {st}: block {r} of owner {o}"
                c = sh.ctl(o)[st, r]
                assert (int(c[0]), int(c[1])) == (len(at), st + 1), f"step {st}: cnt / rflag of ({o}, {r})"
            dest = sh.dest(r, st)
            assert dest[:len(recs)].tolist() == ((own << 27) | pos).tolist(), f"step {st}: dest of rank {r}"
            assert (dest[len(recs):] == POISON32).all()
            assert sh.ctrs(r)[:2].tolist() == [0, 0], "k_xcount / k_xscatter blocks-done counters not re-armed"


# ---- k_xwait: fills into the inbox prefix, and the two refusals -----------------------------------------------------
def _xwait(world, cap, fills, step, n_max):
    sh, _ = make_shard(limits(1, 1), 1, world, cap, lag=2, log2P=0, log2R=4)
    buf = step % sh.depth
    ctl = np.zeros((sh.depth, world, 4), dtype=np.uint32)
    ctl[buf, :, 0] = fills
    ctl[buf, :, 1] = step + 1  # every block is complete: nothing waits
    sh.set_ctl(0, ctl)
    return sh.xwait(0, buf, step, n_max)


@pytest.mark.parametrize("world,fills", [
    (5, [0, 7, 0, 64, 0]), (3, [0, 0, 0]), (1, [48]), (32, [(r * 37) % 65 if r % 5 else 0 for r in range(32)]),
    (8, [0] * 7 + [1])])
def test_xwait_prefix_over_empty_and_ragged_blocks(world, fills):
    seg, n_dev, err = _xwait(world, 64, fills, step=4, n_max=world * 64)
    assert seg.tolist() == [0] + np.cumsum(fills).tolist() and n_dev == sum(fills)
    assert err.tolist() == [0] * 8


def test_xwait_refuses_a_fill_above_cap():
    seg, n_dev, err = _xwait(3, 64, [5, 65, 9], step=7, n_max=3 * 64)
    assert err[0] == RL_DEV_EXCHANGE and err[7] == (1 << 28) | (1 << 20) | 7
    assert seg.tolist() == [0, 5, 5, 14] and n_dev == 14  # the refused block counts as empty


def test_xwait_refuses_an_inbox_above_max_batch():
    seg, n_dev, err = _xwait(4, 64, [40, 0, 30, 1], step=0x12345, n_max=64)
    assert err[0] == RL_DEV_EXCHANGE and err[7] == (3 << 28) | 0x12345  # the step's low 20 bits
    assert seg.tolist() == [0] * 5 and n_dev == 0


# ---- whole steps ----------------------------------------------------------------------------------------------------
def ragged_steps(world, n_steps, cap, nss, seed, t0=H.T0, **kw):
    """Fills that are not multiples of 16 (block boundaries inside a front tile), one rank with nothing at all, and in
    step 1 every record on one owner (the other owners decide empty inboxes)."""
    rng = np.random.default_rng(seed)
    one = [x for x in nss if owner_of(x, world) == owner_of(nss[0], world)]
    steps = []
    for st in range(n_steps):
        row = []
        for r in range(world):
            n = 0 if r == st % world else int(rng.integers(1, cap + 1))
            if n % 16 == 0 and n:
                n -= 1
            row.append(recs_of(n, one if st == 1 else nss, seed=1000 * seed + 10 * st + r, t0=t0 + st * 700_000, **kw))
        steps.append(row)
    return steps


@pytest.mark.parametrize("world,lag,cells,per_ns", [(2, 0, 1, 1), (3, 1, 3, 3), (8, 2, 7, 4), (2, 3, 7, 7), (3, 4, 3, 2)])
def test_steps_reuse_every_buffer(world, lag, cells, per_ns):
    """2 x depth steps of ragged fills: every buffer, its flags and the verdict blocks are reused, through k_main<1,1>,
    <3,3>, <7,4> and <7,7>; the inbox fill is far below n_acc = world x cap, and the tile is derived from it."""
    cap = 304
    descs = limits(6, per_ns)
    sh, engines = make_shard(descs, cells, world, cap, lag)
    assert engines[0].max_cells_used == per_ns
    steps = ragged_steps(world, 2 * (lag + 2), cap, list(range(6)) + [9], seed=world * 10 + lag, n_keys=60)
    outs, geos, _ = run_steps(sh, engines, steps)
    check_against_oracle(descs, world, engines, steps, outs)
    for g in geos:
        assert g["tiles"] == min(256, -(-world * cap // 256)) and g["tile"] == 256, g
    assert any(g["fill"] == 0 for g in geos) and any(0 < g["fill"] < world * cap // 4 for g in geos)
    assert any(g["items"] > 0 and g["chunks"] > 0 for g in geos)


def test_one_owner_takes_every_record_and_its_partitions_chain():
    """Every namespace on one owner: its inbox takes world x cap records a step, far more than the partitions are sized
    for (one source batch), so its partitions are chained; the other owners decide empty inboxes."""
    world, cap = 3, 1024
    nss = namespaces_of_owner(1, world, 3)
    descs = limits(0, 2, ns_ids=nss)
    sh, engines = make_shard(descs, 3, world, cap, lag=1, log2P=2, log2R=10)
    steps = [[recs_of(cap - 3 * r, nss, seed=10 * st + r, t0=H.T0 + st * 300_000, n_keys=400) for r in range(world)]
             for st in range(4)]
    outs, geos, _ = run_steps(sh, engines, steps)
    check_against_oracle(descs, world, engines, steps, outs)
    own = [g for g in geos if g["rank"] == 1]
    assert all(g["fill"] == sum(cap - 3 * r for r in range(world)) for g in own)
    assert all(g["chained_chunks"] > 0 and g["heavy_items"] > 0 for g in own), own
    assert all(g["items"] == 0 for g in geos if g["rank"] != 1)


@pytest.mark.parametrize("cells,per_ns", [(1, 1), (3, 3)])
def test_hot_rows_replay_from_the_segmented_inbox(cells, per_ns):
    """Hot rows on, a Zipf head: k_main reports the head rows as candidates, the next front admits them, and k_hot
    replays them from the segmented inbox (RecordSrc::at) beside k_main."""
    world, cap = 2, 1024
    nss = namespaces_of_owner(0, world, 2)
    descs = limits(0, per_ns, ns_ids=nss, maxes=(400, 3000, 20000))
    sh, engines = make_shard(descs, cells, world, cap, lag=1, log2P=2, log2R=9, hot=True)
    steps = [[recs_of(cap - 5 - 7 * r, nss, seed=20 * st + r, t0=H.T0 + st * 200_000, zipf=(0.6, 3), n_keys=300)
              for r in range(world)] for st in range(6)]
    outs, geos, _ = run_steps(sh, engines, steps)
    check_against_oracle(descs, world, engines, steps, outs)
    own = [g for g in geos if g["rank"] == 0]
    assert any(g["hot_candidates"] > 0 for g in own), own
    assert any(g["hot_in_use"] > 0 and g["hot_max_list"] > 0 for g in own), own


@pytest.mark.parametrize("seed", [1, 2])
def test_resident_replay_blocks_interleaved(seed):
    """Two and four k_main blocks resident and interleaved (switch points at every global access with p = 0.5) while
    they replay a segmented inbox: a chained chunk's first read races the commit of the chunk before it."""
    world, cap = 3, 512
    nss = namespaces_of_owner(seed, world, 2)
    descs = limits(0, 3, ns_ids=nss, maxes=(60, 400, 3000))
    sh, engines = make_shard(descs, 3, world, cap, lag=1, log2P=1, log2R=10, resident=2 * seed, interleave=(seed, 0.5))
    steps = [[recs_of(cap - r, nss, seed=30 * st + r + seed, t0=H.T0 + st * 100_000, n_keys=50) for r in range(world)]
             for st in range(3)]
    outs, geos, _ = run_steps(sh, engines, steps)
    check_against_oracle(descs, world, engines, steps, outs)
    assert any(g["chained_chunks"] > 0 and g["ordered_chunks"] > 0 for g in geos), geos


def test_per_rank_clocks_are_not_monotone_in_the_canonical_order():
    """Rank r's clock runs r x 700 ms behind rank 0's, each step across a 1 s window: in (source rank, source index)
    order the clocks of one owner's inbox jump back and forth across 1 s windows."""
    world, cap = 3, 512
    descs = limits(5, 3, windows=(1, 2, 60), maxes=(3, 10, 200))
    sh, engines = make_shard(descs, 3, world, cap, lag=2)
    steps = []
    for st in range(6):
        steps.append([recs_of(cap - 11 * r, list(range(5)), seed=40 * st + r, n_keys=30, hits=(1, 2),
                              t0=H.T0 + st * 1_000_000 - r * 700_000) for r in range(world)])
    for row in steps:
        merged = np.concatenate([x["now_us"] for x in row])
        assert (np.diff(merged.astype(np.int64)) < 0).any()
    outs, geos, _ = run_steps(sh, engines, steps)
    check_against_oracle(descs, world, engines, steps, outs)
    assert sum(int((o == 1).sum()) for row in outs for o in row) > 0, "nothing was limited: the windows never mattered"


# ---- errors go back to their source position -------------------------------------------------------------------------
def test_key_out_of_range_is_an_error_verdict_at_its_source_position():
    """A record with key_hi >= 2^32: RL_VERDICT_ERROR at exactly its source's position, RL_DEV_KEY_RANGE on its owner,
    and every other request decided as if it were not there."""
    world, cap = 3, 256
    descs = limits(6, 2)
    sh, engines = make_shard(descs, 3, world, cap, lag=1)
    steps = [[recs_of(200 - 13 * r, list(range(6)), seed=50 * st + r, t0=H.T0 + st * 500_000, n_keys=20)
              for r in range(world)] for st in range(3)]
    bad_at = {(1, 2): 77, (2, 0): 0}
    skip = {}
    for (st, r), i in bad_at.items():
        steps[st][r]["key_hi"][i] = 1 << 32
        m = np.zeros(len(steps[st][r]), dtype=bool)
        m[i] = True
        skip[(st, r)] = m
    outs, _, errs = run_steps(sh, engines, steps, expect_err=True)
    for (st, r), i in bad_at.items():
        assert outs[st][r][i] == RL_VERDICT_ERROR
        assert np.nonzero(outs[st][r] == RL_VERDICT_ERROR)[0].tolist() == [i]
        owner = int(owner_of(steps[st][r]["ns_id"][i], world))
        assert (st, owner, RL_DEV_KEY_RANGE, 0) in errs, errs
    assert all(e[2] == 0 for e in errs if (e[0], e[1]) not in
               {(st, int(owner_of(steps[st][r]["ns_id"][i], world))) for (st, r), i in bad_at.items()}), errs
    check_against_oracle(descs, world, engines, steps, outs, skip=skip)


def test_a_full_region_in_one_owner_is_an_error_verdict_never_an_allow():
    """An owner whose table regions fill up: the requests of keys that found no row say RL_VERDICT_ERROR at their
    sources' positions, never an allow, and the rest are decided as if they were not there."""
    world, cap = 2, 512
    nss = namespaces_of_owner(1, world, 1)
    descs = limits(0, 2, ns_ids=nss, maxes=(50, 500))
    sh, engines = make_shard(descs, 3, world, cap, lag=0, log2P=2, log2R=4)  # 4 regions of 16 rows
    steps = [[recs_of(cap - 1 - r, nss, seed=60 * st + r, t0=H.T0 + st * 100_000, n_keys=120) for r in range(world)]
             for st in range(2)]
    outs, _, errs = run_steps(sh, engines, steps, expect_err=True)
    assert any(e[1] == 1 and e[2] == RL_DEV_TABLE_FULL for e in errs), errs
    skip, failed = {}, set()
    for st, row in enumerate(steps):
        for r in range(world):
            bad = outs[st][r] == RL_VERDICT_ERROR
            skip[(st, r)] = bad
            failed |= {(int(x["key_lo"]), int(x["key_hi"])) for x in row[r][bad]}
    assert failed, "no region filled up"
    for st, row in enumerate(steps):
        for r in range(world):
            keys = list(zip(row[r]["key_lo"].tolist(), row[r]["key_hi"].tolist()))
            for k, v in zip(keys, outs[st][r].tolist()):
                assert (k in failed) == (v == RL_VERDICT_ERROR), f"key {k}: verdict {v}"
    check_against_oracle(descs, world, engines, steps, outs, skip=skip)


# ---- the 16-byte record form ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cells,per_ns,n,hot", [(1, 1, 3000, False), (3, 3, 2500, True), (7, 7, 2000, False),
                                                (3, 2, 129 * 512 + 77, False)])
def test_sixteen_byte_records(cells, per_ns, n, hot):
    """rl_record16 batches stamped with one clock (RecordSrc's compact form): hits of 255, namespaces past the
    namespace table, hot rows, more than 128 tiles; verdicts, first-limited ids and the table equal the oracle's."""
    descs = limits(5, per_ns, maxes=(300, 600, 900, 1200, 1500, 1800, 2100))
    emu = H.EmuEngine(descs, cells, 3, 10, hot=hot)
    orc = H.oracle_with_limits(descs)
    seen = []
    for b in range(4 if hot else 2):
        recs = recs_of(n, [0, 1, 2, 3, 4, 700, 0xFFFFFF], seed=70 + b, t0=H.T0, n_keys=80, hits=(1, 1, 2, 255),
                       zipf=(0.5, 2) if hot else None)
        now = H.T0 + b * 3_000_000 + 17
        recs["now_us"] = now
        lim, fl, err = emu.records16(pack_records16(recs), now)
        assert err == 0
        ol, of, _, _ = orc.batch_records(0, recs)
        bad = np.nonzero(lim != ol)[0]
        assert not len(bad), f"batch {b}: verdicts differ at {bad[:8].tolist()}"
        assert fl.tolist() == of.tolist(), "first-limited ids differ"
        assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs), "table differs"
        assert (ol == 1).any() and (recs["hits_addend"] == 255).any()
        seen.append(dict(emu.geometry))
    if n > 128 * 512:
        assert seen[0]["tiles"] > 128 and seen[0]["merge_passes_main"] == 2, seen
    if hot:
        assert any(g["hot_in_use"] > 0 and g["hot_max_list"] > 0 for g in seen), seen
