"""Persistent counters without a GPU: the change scan k_changes and the dictionary drain's mark k_counter_vars_since run
under tests/emu/cuda_shim.h (tests/emu/emu_journal.cpp) against a Python model of the shadow diff, and the journal
(limitador_b200/journal.py) is written, torn and corrupted on disk."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

from limitador_b200 import journal as J
from limitador_b200.engine import LIMIT_DESC_DTYPE, NONE, SNAPSHOT_VERSION
from tests import helpers as H

TOMB = 0xFFFFFFFFFFFFFFFF
CVSLOT_DTYPE = np.dtype([("fp", "<u8"), ("key_lo", "<u8"), ("key_hi", "<u4"), ("varset", "<u4"), ("off", "<u8"),
                         ("len", "<u4"), ("_pad", "<u4")])


@functools.cache
def lib():
    L = H.host_lib("emu_journal.cpp", "librl_emu_journal.so")
    vp = C.c_void_p
    L.emu_seed.argtypes = [C.c_uint64]
    L.emu_changes.restype = C.c_uint64
    L.emu_changes.argtypes = [vp, vp, C.c_uint32, C.c_uint64, vp, vp, C.c_uint64, vp, vp, vp, vp, vp]
    L.emu_cv_since.argtypes = [vp, C.c_uint64, C.c_uint64, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Table:
    """A counter table as the engine lays it out: row = (key_lo, group << 32 | key_hi) then `cells` (value, expiry)."""

    def __init__(self, cells, nrows, rng):
        self.cells, self.nrows, self.rng = cells, nrows, rng
        self.w = 2 * (1 + cells)
        self.rows = np.zeros((nrows, self.w), np.uint64)
        # row groups: 1..G, a qualified and an unqualified kind, some cells without a limit
        self.desc = np.zeros(8 * 9, dtype=H.CELLDESC_DTYPE)
        self.desc["limit_id"] = NONE
        lid = 0
        self.qualified_groups, self.unq_groups = [], []
        for g in range(1, 9):
            q = g % 3 != 0
            (self.qualified_groups if q else self.unq_groups).append(g)
            for c in range(cells):
                if rng.random() < 0.15:
                    continue  # a cell of no limit
                self.desc[g * 8 + c] = (100, 1000, lid, int(q))
                lid += 1
        self.n_limits = max(lid, 1)
        self.present = (rng.random(self.n_limits) < 0.8).astype(np.uint8)
        for g in self.qualified_groups:
            for c in range(cells):
                l = int(self.desc[g * 8 + c]["limit_id"])
                if l != NONE:
                    self.present[l] = 1  # qualified limits are always present
        self.unq_used = set()

    def cell(self, r, c):
        return self.rows[r, 2 + 2 * c], self.rows[r, 3 + 2 * c]

    def free_row(self, tomb_first):
        hdr = self.rows[:, 1]
        cand = np.flatnonzero(hdr == np.uint64(TOMB)) if tomb_first else np.array([], int)
        if not len(cand):
            cand = np.flatnonzero(hdr == 0)
        return int(self.rng.choice(cand)) if len(cand) else None

    def insert(self, tomb_first=False):
        r = self.free_row(tomb_first)
        if r is None:
            return
        if self.rng.random() < 0.2 and len(self.unq_used) < len(self.unq_groups):
            g = next(g for g in self.unq_groups if g not in self.unq_used)
            self.unq_used.add(g)
            lo, hi = 0, g << 32
        else:
            g = int(self.rng.choice(self.qualified_groups))
            lo, hi = int(self.rng.integers(1, 2**63)), (g << 32) | int(self.rng.integers(0, 2**32))
        self.rows[r, :] = 0
        self.rows[r, 0], self.rows[r, 1] = lo, hi
        for c in range(self.cells):
            if self.rng.random() < 0.7:
                self.rows[r, 2 + 2 * c] = self.rng.integers(0, 50)
                self.rows[r, 3 + 2 * c] = self.rng.integers(1, 2000)

    def live_rows(self):
        hdr = self.rows[:, 1]
        return np.flatnonzero((hdr != 0) & (hdr != np.uint64(TOMB)))

    def touch(self):
        live = self.live_rows()
        if not len(live):
            return
        r = int(self.rng.choice(live))
        c = int(self.rng.integers(0, self.cells))
        self.rows[r, 2 + 2 * c] += np.uint64(self.rng.integers(1, 5))
        if self.rng.random() < 0.3:
            self.rows[r, 3 + 2 * c] = self.rng.integers(1, 3000)

    def sweep(self, now):
        """k_reset mode 1: qualified cells with 0 < expiry <= now cleared, rows left without a counter -> tombstone."""
        for r in self.live_rows():
            g = int(self.rows[r, 1]) >> 32
            any_live = any_unq = False
            for c in range(self.cells):
                d = self.desc[g * 8 + c]
                v, e = self.cell(r, c)
                if d["limit_id"] != NONE and d["qualified"] and e != 0 and e <= now:
                    self.rows[r, 2 + 2 * c] = self.rows[r, 3 + 2 * c] = 0
                elif d["limit_id"] != NONE:
                    any_unq |= not d["qualified"]
                    any_live |= bool(d["qualified"]) and e != 0
            if not any_live and not any_unq:
                self.rows[r, :] = 0
                self.rows[r, 1] = np.uint64(TOMB)


def listed(rows, desc, present, cells):
    """rl_counters_export(now_us = 0) over the rows: {(limit, key_lo, key_hi): (value, expiry)}"""
    out = {}
    for r in range(len(rows)):
        lo, hi = int(rows[r, 0]), int(rows[r, 1])
        if hi == 0 or hi == TOMB:
            continue
        g = hi >> 32
        for c in range(cells):
            d = desc[g * 8 + c]
            l = int(d["limit_id"])
            if l == NONE or not present[l]:
                continue
            v, e = int(rows[r, 2 + 2 * c]), int(rows[r, 3 + 2 * c])
            if d["qualified"] and e == 0:
                continue
            out[(l, lo, hi & 0xFFFFFFFF)] = (v, e)
    return out


def model_delta(old, new, desc, present, cells):
    """The shadow diff k_changes computes, row by row, as a sorted list of entries."""
    out = []
    for r in range(len(new)):
        if np.array_equal(old[r], new[r]):
            continue
        a = listed(old[r:r + 1], desc, present, cells)
        b = listed(new[r:r + 1], desc, present, cells)
        same_key = a and b and old[r, 0] == new[r, 0] and old[r, 1] == new[r, 1]
        if same_key:
            out += [(k + v) for k, v in b.items() if a.get(k) != v]
            out += [(k + (0, 0)) for k in a if k not in b]
        else:
            out += [(k + (0, 0)) for k in a] + [(k + v) for k, v in b.items()]
    return sorted(out)


def drain(t, shadow, cap):
    out = [np.full(max(cap, 1), 0xAB, np.uint32)] + [np.full(max(cap, 1), 0xAB, np.uint64) for _ in range(4)]
    n = lib().emu_changes(_p(t.rows), _p(shadow), t.cells, t.nrows, _p(t.desc), _p(t.present), cap, *map(_p, out))
    return int(n), out


def apply_delta(state, entries, desc):
    """The journal's merge: absents first, the last value wins, then the absent qualified counters go (an unqualified
    counter at (0, 0) is present)."""
    qualified = {int(d["limit_id"]) for d in desc if d["limit_id"] != NONE and d["qualified"]}
    state = dict(state)
    for e in sorted(entries, key=lambda e: (e[3], e[4]) != (0, 0)):
        state[e[:3]] = e[3:]
    return {k: v for k, v in state.items() if not (k[0] in qualified and v == (0, 0))}


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_change_scan_matches_the_shadow_diff_model(cells, seed):
    rng = np.random.default_rng(seed * 10 + cells)
    lib().emu_seed(seed + 1)
    t = Table(cells, 512, rng)
    for _ in range(150):
        t.insert()
    shadow = t.rows.copy()
    state = listed(t.rows, t.desc, t.present, cells)
    kinds = {"insert": 0, "touch": 0, "sweep": 0, "reuse": 0}
    for step in range(12):
        old = shadow.copy()
        for _ in range(int(rng.integers(5, 40))):
            op = rng.choice(["insert", "touch", "touch", "sweep", "reuse"], p=[0.25, 0.3, 0.3, 0.05, 0.1])
            kinds[op] += 1
            if op == "insert":
                t.insert()
            elif op == "touch":
                t.touch()
            elif op == "sweep":
                t.sweep(int(rng.integers(200, 1500)))
            else:
                t.insert(tomb_first=True)  # a tombstone's position reused by another key
        want = model_delta(old, t.rows, t.desc, t.present, cells)
        n, out = drain(t, shadow, 1 << 14)
        got = sorted(zip(*(o[:n].tolist() for o in out)))
        assert got == want, f"step {step}"
        assert np.array_equal(shadow, t.rows)  # the drain brought the shadow up to date
        state = apply_delta(state, got, t.desc)
        assert state == listed(t.rows, t.desc, t.present, cells)  # replaying the deltas gives the export
    assert all(kinds.values())


def test_a_position_reused_by_another_key_emits_old_absent_and_new_present():
    rng = np.random.default_rng(7)
    t = Table(3, 64, rng)
    t.insert()
    r = int(t.live_rows()[0])
    shadow = t.rows.copy()
    old = listed(t.rows, t.desc, t.present, 3)
    t.sweep(10**9)  # every qualified counter expires: the row becomes a tombstone
    t.insert(tomb_first=True)
    assert t.rows[r, 1] != shadow[r, 1]
    n, out = drain(t, shadow, 64)
    got = sorted(zip(*(o[:n].tolist() for o in out)))
    assert [e for e in got if e[3:] == (0, 0)] == sorted(k + (0, 0) for k in old)
    assert apply_delta(old, got, t.desc) == listed(t.rows, t.desc, t.present, 3)


@pytest.mark.parametrize("cells", [1, 7])
def test_a_cap_too_small_leaves_the_shadow_and_the_outputs_untouched(cells):
    rng = np.random.default_rng(cells)
    t = Table(cells, 256, rng)
    for _ in range(60):
        t.insert()
    shadow = t.rows.copy()
    for _ in range(40):
        t.touch()
    t.sweep(900)
    before = shadow.copy()
    n, _ = drain(t, shadow, 1 << 12)  # count on a copy to know the size
    shadow[:] = before
    assert n > 1
    n2, out = drain(t, shadow, n - 1)
    assert n2 == n
    assert shadow.tobytes() == before.tobytes()
    assert all(np.all(o[:n - 1] == o.dtype.type(0xAB)) for o in out)
    n3, out = drain(t, shadow, n)  # the same drain, repeated with room
    assert n3 == n and np.array_equal(shadow, t.rows)


def test_an_unchanged_table_drains_nothing():
    t = Table(3, 128, np.random.default_rng(3))
    for _ in range(40):
        t.insert()
    shadow = t.rows.copy()
    assert drain(t, shadow, 0)[0] == 0


def test_cvars_drain_marks_exactly_the_slots_past_the_cursor():
    rng = np.random.default_rng(5)
    for nslots in (16, 1024):
        slots = np.zeros(nslots, CVSLOT_DTYPE)
        used = rng.random(nslots) < 0.6
        slots["fp"][used] = rng.integers(1, 2**63, used.sum())
        slots["off"] = rng.integers(0, 5000, nslots)
        for since in (0, 1, 2500, 4999, 5000):
            mark = np.full(nslots, 7, np.uint8)
            lib().emu_cv_since(_p(slots), nslots, since, _p(mark))
            assert np.array_equal(mark.astype(bool), used & (slots["off"] >= since))


# ---- the journal on disk -------------------------------------------------------------------------------------------
LIMITS = np.array([(0, 1, 1, 1, 10, 60_000_000), (1, 1, 1, 1, 20, 1_000_000), (2, 2, 0, 0, 5, 1_000_000)],
                  dtype=LIMIT_DESC_DTYPE)


def _cols(state):
    items = sorted(state.items())
    return (np.array([k[0] for k, _ in items], np.uint32), np.array([k[1] for k, _ in items], np.uint64),
            np.array([k[2] for k, _ in items], np.uint64), np.array([v[0] for _, v in items], np.uint64),
            np.array([v[1] for _, v in items], np.uint64))


def _vars(entries):
    blobs = [b for _, b in entries]
    off = np.zeros(len(blobs) + 1, np.uint64)
    np.cumsum([len(b) for b in blobs], out=off[1:])
    return (np.array([k[0] for k, _ in entries], np.uint32), np.array([k[1] for k, _ in entries], np.uint64),
            np.array([k[2] for k, _ in entries], np.uint64), off, np.frombuffer(b"".join(blobs), np.uint8).copy())


class FakeEngine:
    """Engine.drain_changes / save_counters over a Python dict: a full drain first and after a structural call."""

    def __init__(self):
        self.state, self.seen, self.full = {}, {}, True

    def track_changes(self, on=True):
        self.full = True

    def drain_changes(self):
        if self.full:
            self.full, self.seen = False, dict(self.state)
            return True, _cols(self.state)
        delta = {k: v for k, v in self.state.items() if self.seen.get(k) != v}
        delta.update({k: (0, 0) for k in self.seen if k not in self.state})
        self.seen = dict(self.state)
        return False, _cols(delta)

    def save_counters(self, path, now_us=0):
        lid, lo, hi, val, exp = _cols(self.state)
        with open(path, "wb") as f:
            np.savez(f, version=np.uint32(SNAPSHOT_VERSION), limits=LIMITS, limit_id=lid, key_lo=lo, key_hi=hi, value=val,
                     expiry_us=exp)


class FakeService:
    """RlsService.drain_counter_vars / counter_vars_gc / save_counters over a dict of entries."""

    def __init__(self):
        self._engine = FakeEngine()
        self.vars, self.new, self.full = {}, [], True

    def record(self, key, blob):
        if key not in self.vars:
            self.vars[key] = blob
            self.new.append(key)

    def drain_counter_vars(self):
        if self.full:
            self.full, self.new = False, []
            return True, _vars([])
        out, self.new = [(k, self.vars[k]) for k in self.new], []
        return False, _vars(out)

    def counter_vars_gc(self, now_us=0):
        used = {(1, k[1], k[2]) for k in self._engine.state if k[0] in (0, 1)}
        self.vars = {k: v for k, v in self.vars.items() if k in used}
        self.full = True

    def save_counters(self, path, now_us=0):
        self._engine.save_counters(path)
        ents = sorted(self.vars.items())
        vs, lo, hi, off, blobs = _vars(ents)
        with np.load(path) as z:
            arrays = dict(z)
        arrays.update(cv_varset=vs, cv_key_lo=lo, cv_key_hi=hi, cv_blob_off=off, cv_blobs=blobs)
        with open(path, "wb") as f:
            np.savez(f, **arrays)


def _step(svc, rng, t):
    e = svc._engine
    for _ in range(int(rng.integers(1, 8))):
        k = (int(rng.integers(0, 2)), int(rng.integers(1, 6)), int(rng.integers(0, 3)))
        v = e.state.get(k, (0, t + 1000))
        e.state[k] = (v[0] + int(rng.integers(1, 4)), v[1])
        svc.record((1, k[1], k[2]), f"user{k[1]}:{k[2]}".encode())
    if rng.random() < 0.3 and e.state:  # a sweep: some qualified counters become absent
        for k in list(e.state)[: int(rng.integers(1, 3))]:
            del e.state[k]
    e.state[(2, 0, 0)] = (t % 5, 0)  # an unqualified counter, (value, 0) is a present state


def _listed(svc):
    return {k: v for k, v in svc._engine.state.items()}


def _merged(directory):
    limits, cols, cvars, info = J.read_journal(directory, truncate=False)
    state = {(int(a), int(b), int(c)): (int(d), int(e)) for a, b, c, d, e in zip(*cols)}
    return {k: v for k, v in state.items() if not (k[0] != 2 and v[1] == 0)}, cvars, info


def _journal(tmp_path, steps, seed=0, structural_at=()):
    svc = FakeService()
    jr = J.CounterJournal(svc, str(tmp_path))
    rng = np.random.default_rng(seed)
    states = []
    for t in range(steps):
        _step(svc, rng, t)
        if t in structural_at:
            svc._engine.full = True
        r = jr.drain()
        states.append((_listed(svc), dict(svc.vars), r))
    jr.close()
    return svc, states


def test_the_journal_recovers_the_state_of_every_drain(tmp_path):
    for steps in range(1, 12):
        d = tmp_path / f"j{steps}"
        svc, states = _journal(d, steps, seed=steps, structural_at={4})
        state, cvars, info = _merged(str(d))
        assert state == states[-1][0]
        names = {(int(a), int(b), int(c)) for a, b, c in zip(*cvars[:3])}
        assert {(1, k[1], k[2]) for k in state if k[0] != 2} <= names
        assert sorted(os.listdir(d)) == [J._base_name(info["generation"]), J._log_name(info["generation"])]
    assert states[4][2]["full"] and not states[5][2]["full"]


def test_record_format_round_trips():
    rng = np.random.default_rng(1)
    counters = (rng.integers(0, 9, 17).astype(np.uint32),) + tuple(rng.integers(0, 2**63, 17).astype(np.uint64) for _ in range(4))
    cvars = _vars([((3, 5, 6), b"\x03\x00\x00\x00abc"), ((4, 7, 8), b"")])
    data = J.encode_record(1, counters, cvars) + J.encode_record(2, tuple(c[:0] for c in counters), cvars)
    recs, good = J.decode_records(data)
    assert good == len(data) and [r[0] for r in recs] == [1, 2]
    for a, b in zip(recs[0][1], counters):
        assert a.dtype == b.dtype and np.array_equal(a, b)
    for a, b in zip(recs[0][2], cvars):
        assert np.array_equal(a, b)


def test_a_log_truncated_anywhere_in_its_last_record_recovers_the_previous_drain(tmp_path):
    d = tmp_path / "j"
    svc, states = _journal(d, 8, seed=3)
    _, _, info = _merged(str(d))
    log = d / J._log_name(info["generation"])
    data = log.read_bytes()
    recs, good = J.decode_records(data)
    assert good == len(data) and len(recs) == 7
    last = len(data) - len(J.encode_record(7, recs[-1][1], recs[-1][2]))
    for cut in range(last, len(data)):
        log.write_bytes(data[:cut])
        state, _, info = _merged(str(d))
        assert info["records"] == 6 and state == states[-2][0], cut
    log.write_bytes(data[:last + 5])
    J.read_journal(str(d))  # truncate=True cuts the torn tail off
    assert log.read_bytes() == data[:last]


def test_a_flipped_byte_stops_the_replay_at_its_record(tmp_path):
    d = tmp_path / "j"
    svc, states = _journal(d, 6, seed=4)
    _, _, info = _merged(str(d))
    log = d / J._log_name(info["generation"])
    data = log.read_bytes()
    recs, _ = J.decode_records(data)
    starts = [0]
    for _, c, v in recs:
        starts.append(starts[-1] + len(J.encode_record(1, c, v)))
    rng = np.random.default_rng(0)
    for i in range(len(recs)):
        for at in sorted(set(rng.integers(starts[i], starts[i + 1], 25).tolist()) | {starts[i], starts[i + 1] - 1}):
            bad = bytearray(data)
            bad[at] ^= 0x5A
            log.write_bytes(bytes(bad))
            state, _, info = _merged(str(d))
            assert info["records"] == i and state == states[i][0], (i, at)
    log.write_bytes(data)
