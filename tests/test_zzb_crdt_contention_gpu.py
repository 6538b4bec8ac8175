"""The replicated counter value (include/rl_crdt.h) on the GPU where threads of one call collide, and at the edges of its
arithmetic, against oracle/crdt_oracle.c; then the counter variable dictionary with 65 536 requests sharing a few new
keys.  Each case runs once: the deterministic proof of the interleavings is tests/test_crdt_contention.py, under the
fiber emulator.  Sorted after the other GPU files on purpose."""
import ctypes as C

import numpy as np
import pytest

from limitador_b200 import crdt as CR
from oracle.crdt_binding import CrdtOracle
from tests.test_crdt import _keys

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000
SEC = 1_000_000
U64 = 2 ** 64
RL_MEM_DEVICE = 1
INCS = np.array([1, 2, 7, 1000, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)


def _status(f, *args):
    """0, or the status a call raised with."""
    try:
        f(*args)
        return 0
    except CR.CrdtError as e:
        return e.status


def _oracle_of(dump, actors, self_actor):
    """A replica holding exactly the rows of `dump`: a merge into an absent row at clock 0 takes the expiry and values."""
    o = CrdtOracle(actors, self_actor)
    for lo, hi, exp, vals in dump:
        o.merge_at((lo, hi), exp, {a: v for a, v in enumerate(vals)}, 0)
    assert o.dump() == dump
    return o


def _check(t, o, keys, now):
    val, exp = t.read(CR.keys_array(keys), now)
    assert val.tolist() == [o.read_at(k, now) % U64 for k in keys]
    assert exp.tolist() == [o.expiry(k) for k in keys]
    assert t.export(now) == o.export(now)
    assert t.dump() == o.dump()


# ---- contended increments ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("actors", [1, 4])
@pytest.mark.parametrize("n_keys", [1, 8, 256])
def test_65536_increments_of_a_few_keys(n_keys, actors):
    """Every call: 65 536 increments over n_keys keys, at clocks where the rows are absent, live, expired exactly at the
    clock and expired before it.  One actor: the value is the oracle's, whatever the order.  Four actors: on a row the
    call resets, each key's row is the oracle's for one choice of the actor whose request goes first."""
    rng = np.random.default_rng(n_keys * 10 + actors)
    self_actor = actors - 1
    t = CR.CrdtTable(1 << 12, actors, self_actor)
    keys = _keys(rng, n_keys, 50_000)
    n = 65536
    for now in (T0, T0 + SEC // 2, T0 + SEC, T0 + 3 * SEC):  # absent, live, expiry == now, expired
        before = t.dump()
        ki = rng.integers(0, n_keys, size=n)
        who = rng.integers(0, actors, size=n).astype(np.uint32)
        inc = rng.choice(INCS, size=n)
        t.inc(CR.keys_array([keys[int(j)] for j in ki]), who, inc, SEC, now)
        got = {(lo, hi): [exp, vals] for lo, hi, exp, vals in t.dump()}
        candidates = []
        for first in range(actors):
            o = _oracle_of(before, actors, self_actor)
            order = list(range(n))
            for k in range(n_keys):  # the key's first request of actor `first` goes first
                hits = np.flatnonzero((ki == k) & (who == first))
                assert len(hits), "every actor has requests for every key"
                order.insert(0, int(hits[0]))
            seen = set()
            for j in order:
                if j in seen:
                    continue
                seen.add(j)
                o.inc_actor_at(keys[int(ki[j])], int(who[j]), int(inc[j]), SEC, now)
            candidates.append({(lo, hi): [exp, vals] for lo, hi, exp, vals in o.dump()})
        assert set(got) == set(keys)
        for k in keys:
            assert any(got[k] == c[k] for c in candidates), (now, k, got[k], [c[k] for c in candidates])
        if actors == 1:
            sums = {k: 0 for k in keys}
            for j in range(n):
                sums[keys[int(ki[j])]] += int(inc[j])
            old = {(r[0], r[1]): r[3][0] for r in before}
            live = now == T0 + SEC // 2
            assert all(got[k][1][0] == ((old[k] if live else 0) + sums[k]) % U64 for k in keys)


# ---- edges of the arithmetic -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("actors", [1, 3, 5, 15])
def test_edges_against_the_oracle(actors):
    """Expiry at, one before and one after the clock for inc, merge, read and export; window 0; now + window wrapping past
    2^64; per-actor values and read sums wrapping; odd actor counts (a padding slot after the last actor); the extreme
    valid keys."""
    self_actor = actors // 2
    t, o = CR.CrdtTable(256, actors, self_actor), CrdtOracle(actors, self_actor)
    keys = [(0, 2 ** 64 - 2), (2 ** 64 - 1, 2 ** 64 - 2), (1, 0), (5, 6), (7, 8), (9, 10)]
    ka = CR.keys_array

    def inc(ks, a, v, w, now):
        t.inc(ka(ks), a, v, w, now)
        for k in ks:
            o.inc_actor_at(k, a, v, w, now)

    def merge(ups, now):
        t.merge(*CR.pack_updates(ups), now)
        for k, exp, vals in ups:
            o.merge_at(k, exp, vals, now)

    for a in range(actors):
        inc(keys, a, 2 ** 63 + a, SEC, T0)  # the read sums wrap
    exp0 = T0 + SEC
    for now in (exp0 - 1, exp0, exp0 + 1):
        _check(t, o, keys, now)
    inc(keys[:2], actors - 1, 2 ** 64 - 1, SEC, exp0 - 1)  # live: the actor's value wraps
    inc(keys[2:4], 0, 3, 2 * SEC, exp0)                     # expiry == now: a new window
    _check(t, o, keys, exp0)
    now = exp0
    merge([(keys[0], now, {0: 9}),                 # expiry == now: ignored
           (keys[1], now + 1, {actors - 1: 1}),    # one past: the earlier expiry wins
           (keys[4], now - 1, {0: 9}),             # already expired: ignored
           (keys[5], now + 1, {a: 2 ** 63 + 1 for a in range(actors)})], now)  # locally expired: reset to theirs
    for t_ in (now - 1, now, now + 1, now + 2):
        _check(t, o, keys, t_)
    # window 0: the new window is over as it starts; the next increment starts another
    now = T0 + 10 * SEC
    inc(keys[:3], 0, 5, 0, now)
    _check(t, o, keys, now)
    inc(keys[:3], 0, 6, 0, now)
    _check(t, o, keys, now)
    # now + window wrapping past 2^64: the expiry wraps as in the oracle (and is at once expired)
    now = 2 ** 64 - 5
    inc(keys[3:], actors - 1, 11, 10, now)
    _check(t, o, keys, now)
    merge([(keys[3], 2 ** 64 - 1, {0: 4})], now)
    _check(t, o, keys, now)
    _check(t, o, keys, 2 ** 64 - 1)


def test_invalid_keys_are_refused_and_change_nothing():
    t = CR.CrdtTable(64, 2, 0)
    t.inc(CR.keys_array([(0, 2 ** 64 - 2)]), 0, 1, SEC, T0)
    before = t.dump()
    for bad in [(0, 0), (1, 2 ** 64 - 1), (0, 2 ** 64 - 1)]:
        with pytest.raises(CR.CrdtError, match="key"):
            t.inc(CR.keys_array([bad]), 0, 1, SEC, T0)
        with pytest.raises(CR.CrdtError, match="key"):
            t.merge(*CR.pack_updates([(bad, T0 + SEC, {0: 1})]), T0)
        assert t.read(CR.keys_array([bad]), T0)[0].tolist() == [0]
    assert t.dump() == before


# ---- table geometry ----------------------------------------------------------------------------------------------------
def test_fill_to_capacity_in_one_call_refuse_the_next_clear_and_refill():
    rng = np.random.default_rng(31)
    t, o = CR.CrdtTable(4096, 3, 1), CrdtOracle(3, 1)
    keys = _keys(rng, 4096 + 600, 1_000_000)
    who = rng.integers(0, 3, size=4096).astype(np.uint32)
    t.inc(CR.keys_array(keys[:4096]), who, 4, SEC, T0)
    for k, a in zip(keys[:4096], who):
        o.inc_actor_at(k, int(a), 4, SEC, T0)
    before = t.dump(cap=8192)
    assert before == o.dump() and len(before) == 4096
    assert _status(t.inc, CR.keys_array([keys[4096]]), 0, 1, SEC, T0) == 1  # TRANSIENT: the table is full
    assert _status(t.merge, *CR.pack_updates([(keys[4097], T0 + SEC, {0: 1})]), T0) == 1
    assert t.dump(cap=8192) == before
    t.clear()
    assert t.dump() == []
    o = CrdtOracle(3, 1)
    t.inc(CR.keys_array(keys[600:]), 2, 5, SEC, T0 + 1)
    for k in keys[600:]:
        o.inc_actor_at(k, 2, 5, SEC, T0 + 1)
    assert t.dump(cap=8192) == o.dump()


@pytest.mark.parametrize("row", ["absent", "live", "expired"])
def test_65536_merges_onto_one_key(row):
    actors = 5
    rng = np.random.default_rng(41)
    t, o = CR.CrdtTable(64, actors, 0), CrdtOracle(actors, 0)
    key = (123, 456)
    now = T0 + SEC
    if row != "absent":
        for a in range(actors):
            t.inc(CR.keys_array([key]), a, 10 + a, SEC if row == "expired" else 5 * SEC, T0)
            o.inc_actor_at(key, a, 10 + a, SEC if row == "expired" else 5 * SEC, T0)
    ups = []
    for _ in range(65536):
        exp = now + int(rng.choice([-1, 0, 1, 2, SEC, 7 * SEC]))
        vals = {int(a): int(rng.choice(INCS)) for a in rng.choice(actors, size=int(rng.integers(0, 3)), replace=False)}
        ups.append((key, exp, vals))
    t.merge(*CR.pack_updates(ups), now)
    for k, exp, vals in ups:
        o.merge_at(k, exp, vals, now)
    _check(t, o, [key], now)


# ---- device memory and short outputs -----------------------------------------------------------------------------------
def test_device_memory_inputs_and_outputs():
    """RL_MEM_DEVICE for inc, merge and read: torch tensors through the C-ABI, against the same calls with host arrays."""
    import torch
    rng = np.random.default_rng(51)
    actors = 3
    t, h = CR.CrdtTable(1 << 12, actors, 0), CR.CrdtTable(1 << 12, actors, 0)
    L = t._lib

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()

    keys = _keys(rng, 3000, 100_000)
    for rnd in range(3):
        now = T0 + rnd * 700_000
        # distinct keys: with window 0 or several actors, repeats of a key may end in any of several orders' results
        ks = CR.keys_array([keys[int(j)] for j in rng.choice(len(keys), size=2500, replace=False)])
        who = rng.integers(0, actors, size=len(ks)).astype(np.uint32)
        inc = rng.choice(INCS, size=len(ks))
        win = rng.choice(np.array([0, SEC, 2 * SEC], dtype=np.uint64), size=len(ks))
        ups = [(keys[int(j)], now + int(rng.choice([-1, 0, 1, SEC])), {int(rng.integers(0, actors)): int(rng.integers(0, 99))})
               for j in rng.integers(0, len(keys), size=4000)]
        u, ua, uv = CR.pack_updates(ups)
        d = [dev(x) for x in (ks, who, inc, win, u, ua, uv)]
        torch.cuda.synchronize()
        assert L.rl_crdt_inc(t._h, len(ks), *[x.data_ptr() for x in d[:4]], now, RL_MEM_DEVICE) == 0
        assert L.rl_crdt_merge(t._h, len(u), d[4].data_ptr(), d[5].data_ptr(), d[6].data_ptr(), len(uv), now, RL_MEM_DEVICE) == 0
        h.inc(ks, who, inc, win, now)
        h.merge(u, ua, uv, now)
        probe = CR.keys_array(keys)
        pk = dev(probe)
        out_v = torch.zeros(len(probe), dtype=torch.int64, device="cuda")
        out_e = torch.zeros(len(probe), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        assert L.rl_crdt_read(t._h, len(probe), pk.data_ptr(), now, RL_MEM_DEVICE, out_v.data_ptr(), out_e.data_ptr()) == 0
        want_v, want_e = h.read(probe, now)
        assert out_v.cpu().numpy().view(np.uint64).tolist() == want_v.tolist()
        assert out_e.cpu().numpy().view(np.uint64).tolist() == want_e.tolist()
        assert t.dump(cap=8192) == h.dump(cap=8192)


def test_export_and_dump_with_more_rows_than_room():
    """cap below the count: cap rows, each one of the table's, and the true count."""
    rng = np.random.default_rng(61)
    actors = 2
    t, o = CR.CrdtTable(1024, actors, 1), CrdtOracle(actors, 1)
    keys = _keys(rng, 700, 100_000)
    t.inc(CR.keys_array(keys), 1, 3, SEC, T0)
    t.inc(CR.keys_array(keys[:100]), 0, 3, SEC, T0)
    for k in keys:
        o.inc_actor_at(k, 1, 3, SEC, T0)
    for k in keys[:100]:
        o.inc_actor_at(k, 0, 3, SEC, T0)
    L, cap = t._lib, 50
    k = np.zeros(cap, dtype=CR.KEY_DTYPE)
    val, exp = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    vals = np.zeros(cap * actors, np.uint64)
    n = C.c_uint64()
    assert L.rl_crdt_export(t._h, T0, cap, k.ctypes.data, val.ctypes.data, exp.ctypes.data, C.byref(n)) == 0
    assert n.value == 700
    got = set(zip(k["lo"].tolist(), k["hi"].tolist(), val.tolist(), exp.tolist()))
    assert len(got) == cap and got <= set(o.export(T0))
    n = C.c_uint64()
    assert L.rl_crdt_dump(t._h, cap, k.ctypes.data, exp.ctypes.data, vals.ctypes.data, C.byref(n)) == 0
    assert n.value == 700
    v = vals.reshape(cap, actors)
    got = {(int(k["lo"][i]), int(k["hi"][i]), int(exp[i]), tuple(v[i].tolist())) for i in range(cap)}
    assert len(got) == cap and got <= set(o.dump())


# ---- the counter variable dictionary -----------------------------------------------------------------------------------
@pytest.mark.parametrize("http", [False, True], ids=["rls", "http"])
@pytest.mark.parametrize("k", [1, 8])
def test_counter_vars_of_65536_requests_sharing_k_new_keys(k, http):
    """One batch of 65 536 requests naming k new keys: the dictionary lists exactly those keys with their values.  The
    arena bytes the racing reservations take are printed beside the sequential minimum, not asserted."""
    from limitador_b200 import http_api as HA
    from limitador_b200 import rls as R
    from tests.test_zz9_counter_vars_gpu import Service
    s = Service(capacity_rows=1 << 14)
    users = [f"shared-{j}-" + "y" * j for j in range(k)]
    if http:
        s.http(HA.CHECK_AND_REPORT, [("api", {"method": "GET", "user": users[i % k]}, 1, None) for i in range(65536)], T0)
    else:
        s.rls_serve(R.SHOULD_RATE_LIMIT, [("api", [("method", "GET"), ("user", users[i % k])]) for i in range(65536)], T0)
    st = s.rls.counter_vars_stats()
    assert st["keys"] == k and st["dropped"] == 0
    assert s.api.get_counters("api", T0 + 1) == s.expected("api", T0 + 1)
    minimum = sum(4 + len(u) for u in users)  # one variable: a u32 length and the bytes
    assert st["arena_used"] >= minimum
    print(f"counter vars {'http' if http else 'rls'} k={k}: arena {st['arena_used']} bytes, sequential minimum {minimum}")
