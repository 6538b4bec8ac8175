"""The counter-import kernels (limitador_b200/csrc/rl_maint.cuh: k_import_resolve / k_import_claim / k_import_write) run
on the host under tests/emu/cuda_shim.h — the same source the GPU compiles, one CUDA thread after the other in a
shuffled order — and their warp-aggregated probe under tests/emu/cuda_simt.h:
  * an import into an empty table, or one partly filled with live rows and tombstones, leaves every counter where the
    hot path's probing rule (rl_kernels.cuh rl_probe, restated here) finds it, and every other row byte-identical;
  * every refusal (duplicate, unknown limit, key_hi >= 2^32, qualified expiry 0, full region) leaves the table
    byte-identical.
oracle_restore applies the same import to the CPU oracle through the oracle's own public calls (the GPU tests continue
a stream on it after an import); it is pinned here by a small known-answer test.
The GPU runs of rl_counters_export / rl_counters_import are in tests/test_zz4_snapshot_gpu.py."""
import numpy as np
import pytest

from limitador_b200.engine import LIMIT_DESC_DTYPE
from oracle import binding as ob
from tests import helpers as H

TOMB = 0xFFFFFFFFFFFFFFFF
M64 = (1 << 64) - 1
LIMIT_DEV = np.dtype([("group", "<u4"), ("cell", "<u4"), ("ns_id", "<u4"), ("qualified", "<u4")])
UNKNOWN_LIMIT, KEY_RANGE, NO_EXPIRY, DUPLICATE, TABLE_FULL = 1, 2, 3, 4, 5

def mix64(x):
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def row_hash(klo, hhi):  # rl_core.h rl_row_hash
    return mix64(klo ^ mix64(hhi ^ 0x9e3779b97f4a7c15))


class Table:
    """The hot path's counter table on the host: rows of a 16-byte header (key_lo, group << 32 | key_hi) and `cells`
    16-byte cells (value, expiry)."""

    def __init__(self, cells, log2P, log2R):
        self.cells, self.log2P, self.log2R = cells, log2P, log2R
        self.R = 1 << log2R
        self.w = np.zeros((1 << (log2P + log2R), 2 * (1 + cells)), dtype=np.uint64)  # row = 2 + 2 * cells words

    def probe(self, klo, hhi, create=False):
        """rl_probe (rl_kernels.cuh): home = low hash bits in the region the high bits pick, linear probing, an empty
        row ends the search, the first tombstone passed is reused on insert.  Row index or -1."""
        h = row_hash(klo, hhi)
        base = ((h >> (64 - self.log2P)) if self.log2P else 0) << self.log2R
        tomb = -1
        for i in range(self.R):
            r = base + ((h + i) & (self.R - 1))
            k0, k1 = int(self.w[r, 0]), int(self.w[r, 1])
            if (k0, k1) == (klo, hhi):
                return r
            if k0 == 0 and k1 == 0:
                if not create:
                    return -1
                t = tomb if tomb >= 0 else r
                self.w[t, 0], self.w[t, 1] = klo, hhi
                return t
            if k1 == TOMB and tomb < 0:
                tomb = r
        if create and tomb >= 0:
            self.w[tomb, 0], self.w[tomb, 1] = klo, hhi
            return tomb
        return -1

    def put(self, klo, hhi, cells):
        r = self.probe(klo, hhi, True)
        if r >= 0:
            self.w[r, 2:] = np.asarray(cells, dtype=np.uint64)
        return r

    def tombstone(self, klo, hhi):
        r = self.probe(klo, hhi)
        self.w[r] = 0
        self.w[r, 1] = TOMB

    def import_(self, simt, limits, lid, klo, khi, val, exp):
        cols = [np.ascontiguousarray(lid, dtype=np.uint32)] + [np.ascontiguousarray(c, dtype=np.uint64) for c in (klo, khi, val, exp)]
        unq = np.zeros(len(limits), dtype=np.uint8)
        L = H.emu_maint_lib(simt)
        err = L.emu_import(H._p(self.w), self.cells, self.log2P, self.log2R, H._p(limits), len(limits), len(cols[0]),
                           *[H._p(c) for c in cols], H._p(unq))
        return (None if err == M64 else (err >> 8, err & 0xFF)), unq


def make_limits(cells, n_groups, rng):
    """Limits on `n_groups` row groups (group 1.. ; the first is unqualified), `cells` limits each, plus an unregistered id."""
    rows = []
    for g in range(1, n_groups + 1):
        for c in range(cells):
            rows.append((g, c, g, 0 if g == 1 else 1))
    rows.append((0, 0, 0, 0))  # last id: not registered (group 0)
    return np.array(rows, dtype=LIMIT_DEV)


def key_of(limits, lid, klo, khi):
    d = limits[lid]
    if not d["qualified"]:
        return 0, int(d["group"]) << 32
    return klo, (int(d["group"]) << 32) | khi


def random_entries(limits, n_rows, rng):
    """Counters of n_rows distinct rows; several cells of one row are adjacent, as rl_counters_export writes them."""
    cells = int(limits["cell"].max()) + 1
    q_ids = [i for i in range(len(limits) - 1) if limits[i]["qualified"]]
    u_ids = [i for i in range(len(limits) - 1) if not limits[i]["qualified"]]
    out, seen_rows = [], set()
    for i in u_ids:  # the unqualified row
        if rng.random() < 0.7:
            out.append((i, 0, 0, int(rng.integers(0, 50)), int(rng.integers(0, 2 ** 40))))
    while len(seen_rows) < n_rows:
        g = int(rng.choice(sorted({int(limits[i]["group"]) for i in q_ids})))
        klo, khi = int(rng.integers(1, 2 ** 62)), int(rng.integers(0, 2 ** 32))
        if (g, klo, khi) in seen_rows:
            continue
        seen_rows.add((g, klo, khi))
        ids = [i for i in q_ids if limits[i]["group"] == g]
        for i in sorted(rng.choice(ids, size=int(rng.integers(1, cells + 1)), replace=False).tolist()):
            out.append((i, klo, khi, int(rng.integers(0, 2 ** 40)), int(rng.integers(1, 2 ** 50))))
    a = np.array(out, dtype=[("lid", "<u4"), ("klo", "<u8"), ("khi", "<u8"), ("val", "<u8"), ("exp", "<u8")])
    return a


def cols(a):
    return a["lid"], a["klo"], a["khi"], a["val"], a["exp"]


@pytest.mark.parametrize("simt", [False, True], ids=["plain-path", "warp-aggregated-path"])
@pytest.mark.parametrize("cells,log2P,log2R,prefill,seed", [(1, 2, 7, False, 1), (3, 3, 6, True, 2), (7, 0, 9, True, 3),
                                                            (4, 4, 5, True, 4)])
def test_imported_counters_sit_where_the_hot_path_probes(cells, log2P, log2R, prefill, simt, seed):
    H.emu_maint_lib(simt).emu_seed(seed)
    rng = np.random.default_rng(seed)
    limits = make_limits(cells, 4, rng)
    t = Table(cells, log2P, log2R)
    ents = random_entries(limits, int(0.35 * (1 << (log2P + log2R))), rng)
    live = {}
    if prefill:  # live rows (some of which the import names again) and tombstones on the probe chains
        for e in ents[: len(ents) // 3]:
            k = key_of(limits, int(e["lid"]), int(e["klo"]), int(e["khi"]))
            c = rng.integers(1, 2 ** 30, size=2 * cells).tolist()
            if t.put(*k, c) >= 0:
                live[k] = c
        for _ in range(len(ents) // 4):
            k = (int(rng.integers(1, 2 ** 62)), (2 << 32) | int(rng.integers(0, 2 ** 32)))
            if t.put(*k, rng.integers(1, 2 ** 30, size=2 * cells).tolist()) >= 0:
                live[k] = None
                if rng.random() < 0.6:
                    t.tombstone(*k)
                    del live[k]
    before = t.w.copy()
    err, unq = t.import_(simt, limits, *cols(ents))
    assert err is None
    touched = {}
    for e in ents:
        lid = int(e["lid"])
        k = key_of(limits, lid, int(e["klo"]), int(e["khi"]))
        r = t.probe(*k)
        assert r >= 0, "an imported counter is not where rl_probe looks"
        c = int(limits[lid]["cell"])
        assert (int(t.w[r, 2 + 2 * c]), int(t.w[r, 3 + 2 * c])) == (int(e["val"]), int(e["exp"]))
        touched.setdefault(r, set()).add(c)
    for k in live:  # rows that held a key before keep their index
        assert t.probe(*k) >= 0
    for r in range(len(t.w)):  # every row and cell the import did not name is byte-identical
        if r not in touched:
            assert (t.w[r] == before[r]).all(), f"row {r} changed"
        elif (t.w[r, :2] == before[r, :2]).all():
            for c in set(range(cells)) - touched[r]:
                assert (t.w[r, 2 + 2 * c:4 + 2 * c] == before[r, 2 + 2 * c:4 + 2 * c]).all(), f"row {r} cell {c} changed"
    named = {int(e["lid"]) for e in ents if not limits[int(e["lid"])]["qualified"]}
    assert sorted(np.flatnonzero(unq).tolist()) == sorted(named)


@pytest.mark.parametrize("simt", [False, True], ids=["plain-path", "warp-aggregated-path"])
def test_a_refused_import_changes_no_counter(simt):
    rng = np.random.default_rng(7)
    cells = 3
    limits = make_limits(cells, 4, rng)
    t = Table(cells, 2, 6)
    base = random_entries(limits, 60, rng)
    assert t.import_(simt, limits, *cols(base))[0] is None
    for k in [key_of(limits, int(e["lid"]), int(e["klo"]), int(e["khi"])) for e in base[::9]]:
        if k[0]:
            t.tombstone(*k)
    fresh = random_entries(limits, 50, np.random.default_rng(8))
    q = np.flatnonzero(limits["qualified"][fresh["lid"]] == 1)
    cases = []
    dup = fresh.copy()
    dup[-1] = dup[q[3]]
    dup[-1]["val"] += 1
    cases.append((dup, DUPLICATE))
    unk = fresh.copy()
    unk[q[5]]["lid"] = len(limits) - 1
    cases.append((unk, UNKNOWN_LIMIT))
    beyond = fresh.copy()
    beyond[q[6]]["lid"] = len(limits) + 10
    cases.append((beyond, UNKNOWN_LIMIT))
    wide = fresh.copy()
    wide[q[7]]["khi"] = 1 << 32
    cases.append((wide, KEY_RANGE))
    noexp = fresh.copy()
    noexp[q[8]]["exp"] = 0
    cases.append((noexp, NO_EXPIRY))
    for ents, why in cases:
        before = t.w.copy()
        err, _ = t.import_(simt, limits, *cols(ents))
        assert err is not None and err[1] == why, (err, why)
        # the claim pass gives back the rows it claimed: the table is byte-identical whichever pass refused
        assert (t.w == before).all(), "a refused import changed the table"
        if why == DUPLICATE:
            assert err[0] in (q[3], len(fresh) - 1)
        else:  # the resolve pass names the first bad entry
            assert err[0] == {KEY_RANGE: q[7], NO_EXPIRY: q[8]}.get(why, q[5] if ents is unk else q[6])
    # a full region: 16 rows, of which some hold rows and some are tombstones, 17 distinct rows named
    small = Table(cells, 0, 4)
    first = random_entries(limits, 10, np.random.default_rng(9))
    assert small.import_(simt, limits, *cols(first))[0] is None
    for e in first[-4:]:
        k = key_of(limits, int(e["lid"]), int(e["klo"]), int(e["khi"]))
        if k[0] and small.probe(*k) >= 0:
            small.tombstone(*k)
    before = small.w.copy()
    err, _ = small.import_(simt, limits, *cols(random_entries(limits, 17, np.random.default_rng(10))))
    assert err is not None and err[1] == TABLE_FULL
    assert (small.w == before).all(), "a refused import changed the table"


def oracle_restore(o, descs, limit_id, key_lo, key_hi, value, expiry_us):
    """What rl_counters_import does, applied to the CPU oracle through its own public calls: set each counter to exactly
    (value, expiry_us); a present counter is replaced, an unqualified one (key ignored) becomes present, other counters
    are untouched.  descs: the limits the oracle was given (limit_id, ns_id, max_value, window_us, qualified).

    The counters of every limit named are read back (dump), deleted (delete_counters) and created again with the
    imported ones merged in: update_counter(delta = value, now = expiry - window) creates exactly (value, expiry)
    (in_memory.rs:47-69), and limit_set again on an unqualified limit without a counter recreates the (0, EPOCH) default
    (add_counter, in_memory.rs:38-44).  A limit id the oracle does not know raises before anything changes."""
    by_id = {int(d["limit_id"]): d for d in descs}
    new = {}
    for l, lo, hi, v, x in zip(*[np.asarray(c).tolist() for c in (limit_id, key_lo, key_hi, value, expiry_us)]):
        if l not in by_id:
            raise ValueError(f"limit {l} is not registered")
        new[(l, lo, hi) if by_id[l]["qualified"] else (l, 0, 0)] = (v, x)
    touched = sorted({k[0] for k in new})
    state = {(l, lo, hi): (v, x) for l, lo, hi, v, x in o.dump() if l in touched}
    state.update(new)
    for (l, lo, hi), (v, x) in state.items():
        w = int(by_id[l]["window_us"])
        if x < w and (by_id[l]["qualified"] or (v, x) != (0, 0)):
            raise ValueError(f"counter {(l, lo, hi)}: expiry {x} is earlier than one window after the epoch")
    o.delete_counters(touched)
    for (l, lo, hi), (v, x) in sorted(state.items()):
        d = by_id[l]
        if not d["qualified"] and (v, x) == (0, 0):
            o.limit_set(l, int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), False)
        else:
            o.update_counters(ob.counters([(l, lo, hi)]), v, x - int(d["window_us"]))


def test_oracle_restore_sets_counters_exactly():
    W, T = 1_000_000, 5_000_000
    descs = np.array([(0, 0, 0, 0, 10, W), (1, 0, 1, 1, 10, W), (2, 1, 0, 0, 5, 2 * W)], dtype=LIMIT_DESC_DTYPE)
    o = ob.Oracle(64)
    for d in descs:
        o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    o.delete_counters([2])  # limit 2 now has no counter
    o.update_counters(ob.counters([(1, 7, 0)]), 3, T)  # (3, T + W)
    o.update_counters(ob.counters([(1, 8, 1)]), 2, T)
    assert o.dump() == [(0, 0, 0, 0, 0), (1, 7, 0, 3, T + W), (1, 8, 1, 2, T + W)]
    oracle_restore(o, descs, [1, 1, 0, 2], [7, 9, 55, 66], [0, 4, 0, 0], [6, 1, 4, 2], [T + 500, T + 900, T + 700, T + 2 * W])
    # a present counter replaced (even with an earlier expiry), a new one added, unqualified ones set with their key
    # ignored, limit 2 present again, counter (1, 8, 1) untouched
    assert o.dump() == [(0, 0, 0, 4, T + 700), (1, 7, 0, 6, T + 500), (1, 8, 1, 2, T + W), (1, 9, 4, 1, T + 900),
                        (2, 0, 0, 2, T + 2 * W)]
    assert o.check_and_update(ob.counters([(1, 7, 0)]), 5, False, T + 400)[0] is True  # 6 + 5 > 10 before expiry
    assert o.check_and_update(ob.counters([(1, 7, 0)]), 5, False, T + 500)[0] is False  # expired: a new window
    # the (0, EPOCH) default of an unqualified limit is restored as such
    o.delete_counters([0])
    oracle_restore(o, descs, [0], [0], [0], [0], [0])
    assert (0, 0, 0, 0, 0) in o.dump()
    before = o.dump()
    with pytest.raises(ValueError):
        oracle_restore(o, descs, [0, 3], [0, 0], [0, 0], [9, 9], [T, T])  # limit 3 is not registered
    assert o.dump() == before
