"""The CAS-claimed rows of the replicated counter value (csrc/rl_crdt.cuh) under real thread interleavings, without a GPU.

The kernels run under tests/emu/cuda_simt.h with its interleaving mode on: every global atomic and every load / 128-bit CAS
of rl_devmem.cuh may hand control to another thread of the block first, in a seeded order, so that the steps of threads
that claim a row or move its expiry and then write it interleave.  Blocks run one after the other, so every batch whose
requests must collide sits inside one 256-thread block.  Compared with oracle/crdt_oracle.c:

* one actor's repeats of a key in one inc call are exact: sum of the increments on an absent or expired row, old value
  plus that sum on a live one (wrapping), whatever the order;
* repeats across actors on an expired row equal the sequential order that starts with one of them (the request that
  resets the window): one outcome per request, the table must be one of them;
* merge batches are exact (merge_at commutes for one clock reading), also while other threads move the expiry;
* a table filled to its capacity in one call gives every key exactly one row.
The counter variable dictionary (csrc/rl_cvars_dev.cuh) claims its slots the same way: 256 recording threads of one
block racing for a few new keys must leave the dictionary the Python model builds.  The GPU runs of the same cases are
tests/test_zzb_crdt_contention_gpu.py."""
import numpy as np
import pytest

from limitador_b200 import crdt as CR
from limitador_b200 import http_api as HA
from limitador_b200 import rls as R
from oracle.crdt_binding import CrdtOracle
from tests import helpers as H
from tests import http_corpora as HC
from tests import test_counter_vars_emu as CV
from tests.test_snapshot_emu import row_hash

T0 = 1_700_000_000_000_000
SEC = 1_000_000
U64 = 2 ** 64
KEY = (0x1234_5678_9ABC, 7 << 32 | 3)
PRIOR = (5, 2 ** 63 + 11)  # what the row's two actors held before the call, in its earlier window

# every atomic switches (round robin in a random order), and about half of them do
MODES = [(101, 1.0), (202, 0.5)]


def _table(actors=2, self_actor=0, cap=1024, mode=MODES[0]):
    return H.EmuCrdt(cap, actors, self_actor, simt=True, interleave=mode)


def _prepare(t, o, row, actors):
    """Bring KEY's row to `row` ("fresh": absent, "expired": expiry == the call's clock, "live") and return the call's
    clock."""
    if row == "fresh":
        return T0
    for a in range(actors):
        v = PRIOR[a % 2]
        assert t.inc(CR.keys_array([KEY]), a, v, SEC, T0) == 0
        o.inc_actor_at(KEY, a, v, SEC, T0)
    return T0 + SEC if row == "expired" else T0 + SEC // 2


def _incs(rng, reps):
    return rng.choice(np.array([1, 2, 3, 1000, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64), size=reps)


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
@pytest.mark.parametrize("row", ["fresh", "expired", "live"])
@pytest.mark.parametrize("reps", [2, 3, 32, 100, 256])
def test_one_actors_repeats_of_a_key_all_count(reps, row, mode):
    rng = np.random.default_rng(reps)
    t, o = _table(mode=mode), CrdtOracle(2, 0)
    now = _prepare(t, o, row, 2)
    inc = _incs(rng, reps)
    assert t.inc(CR.keys_array([KEY] * reps), 1, inc, SEC, now) == 0
    for i in inc:
        o.inc_actor_at(KEY, 1, int(i), SEC, now)
    got, want = t.dump(), o.dump()
    lost = (want[0][3][1] - got[0][3][1]) % U64 if got and want else None
    assert got == want, f"lost increments: actor 1 holds {got[0][3][1]}, every order gives {want[0][3][1]} (lost {lost})"
    old = PRIOR[1] if row == "live" else 0
    assert want[0][3][1] == (old + int(sum(int(x) for x in inc))) % U64  # the oracle's order-free answer, restated
    assert t.read(CR.keys_array([KEY]), now)[0].tolist() == [o.read_at(KEY, now)]


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
@pytest.mark.parametrize("reps", [5, 64, 256])
def test_repeats_across_actors_equal_the_order_started_by_one_of_them(reps, mode):
    """On an expired row the request that resets the window decides the expiry (its window) and which actor takes its own
    increments as its value; the other actors add onto their stale values.  The table must equal the sequential run
    that starts with one of the requests."""
    actors = 4
    rng = np.random.default_rng(1000 + reps)
    t = _table(actors=actors, self_actor=2, mode=mode)
    now = _prepare(t, CrdtOracle(actors, 2), "expired", actors)
    who = rng.integers(0, actors, size=reps).astype(np.uint32)
    inc = _incs(rng, reps)
    win = rng.choice([SEC, 2 * SEC, 5 * SEC, 60 * SEC], size=reps).astype(np.uint64)
    assert t.inc(CR.keys_array([KEY] * reps), who, inc, win, now) == 0
    got = t.dump()

    outcomes = set()
    for first in range(reps):
        o = CrdtOracle(actors, 2)
        _prepare(H.EmuCrdt(8, actors, 2), o, "expired", actors)
        for j in [first] + [j for j in range(reps) if j != first]:
            o.inc_actor_at(KEY, int(who[j]), int(inc[j]), int(win[j]), now)
        outcomes.add(tuple(o.dump()))
    assert tuple(got) in outcomes, (got, sorted(outcomes)[:3])
    assert len(outcomes) > 1  # the batch can tell the orders apart


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
@pytest.mark.parametrize("actors,self_actor", [(2, 0), (3, 1), (5, 4)])
def test_merge_batches_with_repeats_are_exact(actors, self_actor, mode):
    """Updates of a few keys repeated inside one block: expiries at the clock (ignored), one past it, later, already
    expired; rows absent, live and expired at the start of the call (reset and zeroed by the thread whose CAS moves the
    expiry, while the others move it to the earliest one)."""
    rng = np.random.default_rng(actors * 10 + self_actor)
    t, o = _table(actors, self_actor, mode=mode), CrdtOracle(actors, self_actor)
    keys = [(k + 1, (k % 3) << 32 | 9) for k in range(6)]
    # keys 0-1 live, 2-3 expired at the call's clock, 4-5 absent
    for k in keys[:4]:
        for a in range(actors):
            assert t.inc(CR.keys_array([k]), a, 40 + a, SEC if k in keys[2:4] else 10 * SEC, T0) == 0
            o.inc_actor_at(k, a, 40 + a, SEC if k in keys[2:4] else 10 * SEC, T0)
    now = T0 + SEC
    for rnd in range(3):
        ups = []
        for j in rng.integers(0, len(keys), size=250):
            exp = now + int(rng.choice([-SEC, -1, 0, 1, 2, SEC // 2, 3 * SEC]))
            vals = {int(a): int(rng.choice(np.array([0, 1, 39, 50, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)))
                    for a in rng.choice(actors, size=int(rng.integers(0, actors + 1)), replace=False)}
            ups.append((keys[int(j)], exp, vals))
        assert t.merge(*CR.pack_updates(ups), now) == 0
        for k, exp, vals in ups:
            o.merge_at(k, exp, vals, now)
        assert t.dump() == o.dump()
        val, exp = t.read(CR.keys_array(keys), now)
        assert val.tolist() == [o.read_at(k, now) % U64 for k in keys]
        assert exp.tolist() == [o.expiry(k) for k in keys]
        now += SEC


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
def test_a_table_filled_to_capacity_in_one_call_gives_each_key_one_row(mode):
    """64 distinct keys into 64 rows from one block: every probe chain ends in a row of its own, some wrap past the
    table's end.  One more key is refused (status 1) and changes nothing already applied."""
    t, o = _table(actors=3, self_actor=0, cap=64, mode=mode), CrdtOracle(3, 0)
    rng = np.random.default_rng(64)
    keys = [(int(rng.integers(1, 2 ** 63)), int(rng.integers(0, 2 ** 63))) for _ in range(64)]
    who = rng.integers(0, 3, size=64).astype(np.uint32)
    inc = rng.integers(1, 100, size=64).astype(np.uint64)
    assert t.inc(CR.keys_array(keys), who, inc, SEC, T0) == 0
    for k, a, i in zip(keys, who, inc):
        o.inc_actor_at(k, int(a), int(i), SEC, T0)
    before = t.dump()
    assert before == o.dump() and len(before) == 64 and len({(lo, hi) for lo, hi, _, _ in before}) == 64
    homes = [row_hash(lo, hi) & 63 for lo, hi in keys]
    assert len(set(homes)) < 64  # collisions: chains that probe on (and, from the last rows, wrap to row 0)
    assert any(h >= 60 for h in homes)
    assert t.inc(CR.keys_array([(12345, 678)]), 0, 1, SEC, T0) == 1
    assert t.dump() == before
    # the same keys again, repeated: every increment lands on the key's one row
    assert t.inc(CR.keys_array(keys + keys[:32]), who.tolist() + who[:32].tolist(), 1, SEC, T0) == 0
    for k, a in zip(keys + keys[:32], who.tolist() + who[:32].tolist()):
        o.inc_actor_at(k, int(a), 1, SEC, T0)
    assert t.dump() == o.dump()


# ---- the counter variable dictionary (csrc/rl_cvars_dev.cuh): the second table whose rows are claimed by CAS ---------------
def _shared_key_batch(k, http):
    """256 requests (one recording block) of the gateway's `api` namespace naming k users in turn: k new keys of one
    variable set, each wanted by 256 / k threads at once."""
    users = [f"user-{j:02d}-" + "x" * (3 * j) for j in range(k)]  # blobs of different lengths
    if http:
        return [HA.encode_info("api", {"method": "GET", "user": users[i % k]}, 1) for i in range(256)]
    return [R.encode_request("api", [[("method", "GET"), ("user", users[i % k])]]) for i in range(256)]


def _record_shared(k, http, arena_bytes, mode):
    h = HC.HttpHarness([])
    lims = CV.Limits(h.m, HC.GATEWAY_LIMITS)
    msgs = _shared_key_batch(k, http)
    d = CV.Dict(max_keys=64, arena_bytes=arena_bytes, interleave=mode)
    if http:
        d.record(h.m, True, HA.CHECK_AND_REPORT, msgs)
        want = CV.expected(lims, h.api.plan(HA.CHECK_AND_REPORT, *HA.pack_bodies(msgs), T0), CV.http_contexts(msgs))
    else:
        d.record(h.m, False, R.SHOULD_RATE_LIMIT, msgs)
        svc = R.RlsService(h.m, None, R.HEADERS_NONE, 2)
        want = CV.expected(lims, svc.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests(msgs), T0), CV.rls_contexts(msgs))
    assert len(want) == k
    got, spans = d.entries()
    return d, lims, want, got, spans


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
@pytest.mark.parametrize("http", [False, True], ids=["rls", "http"])
@pytest.mark.parametrize("k", [1, 2, 8])
def test_counter_vars_recorded_by_racing_threads_equal_the_model(k, http, mode):
    """256 threads of one block record the same k new keys: every key once, with its values, however the threads'
    probes, reservations, blob writes and claims interleave; the losers' reservations are the only cost."""
    d, lims, want, got, spans = _record_shared(k, http, 1 << 16, mode)
    CV.check_entries(d, want, lims)
    st = d.stats()
    assert st["keys"] == len(got) == k and st["dropped"] == 0
    minimum = sum(len(b) for b in want.values())
    assert st["arena_used"] >= minimum
    assert all(ln == len(want[key]) for key, (_, ln) in zip(got, spans))


@pytest.mark.parametrize("mode", MODES, ids=["p1", "p05"])
@pytest.mark.parametrize("http", [False, True], ids=["rls", "http"])
@pytest.mark.parametrize("k", [2, 8])
def test_counter_vars_in_an_arena_that_fits_each_key_once(k, http, mode):
    """An arena of exactly the distinct keys' blobs: a sequential run keeps them all, racing duplicates may reserve the
    bytes a later key needs.  What holds either way (DESIGN §9i): no slot without its blob, and every key that is not
    recorded was counted in `dropped` (which counts refused reservations, so a key recorded by one thread and refused to
    another counts there too)."""
    minimum = sum(len(b) for b in _record_shared(k, http, 1 << 16, None)[2].values())
    seq, _, _, seq_got, _ = _record_shared(k, http, minimum, None)  # the host shim: one thread after the other
    assert len(seq_got) == k and seq.stats()["dropped"] == 0
    d, lims, want, got, spans = _record_shared(k, http, minimum, mode)
    assert all(want[key] == b for key, b in got.items())
    st = d.stats()
    assert st["keys"] == len(got) >= 1
    assert st["dropped"] >= len(want) - len(got)
    assert st["arena_used"] == minimum  # the cursor ran to the end (or past it)
