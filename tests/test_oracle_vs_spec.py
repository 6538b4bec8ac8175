"""The C oracle against the independent Python restatement (tests/spec_model.py) on random streams: all
three batch modes, both load_counters values, get_counters, delete_counters, re-registration, max_value
changes — starting from a tiny oracle table so that it rehashes under the stream."""
import numpy as np
import pytest

from tests import helpers as H
from tests.spec_model import SpecStore
from oracle import binding as ob


def both(descs, cap=16):
    o, s = ob.Oracle(cap), SpecStore()
    for d in descs:
        args = (int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
        o.limit_set(*args)
        s.limit_set(*args)
    return o, s


@pytest.mark.parametrize("seed", range(8))
def test_oracle_equals_the_python_spec_on_random_streams(seed):
    rng = np.random.default_rng(1000 + seed)
    descs = H.mixed_limits(n_ns=int(rng.choice([3, 6, 12])), seed=seed)
    o, s = both(descs)
    live = sorted(int(d["limit_id"]) for d in descs)
    t_last = H.T0
    for b in range(8):
        off, ctrs, delta, now = H.random_csr_stream(descs, int(rng.choice([50, 400, 1500])), seed * 100 + b,
                                                    n_keys=int(rng.choice([2, 30, 300])), monotone=bool(b & 1))
        mode = int(rng.choice([0, 0, 0, 1, 2]))
        lc = bool(rng.integers(0, 2)) and mode == 0
        got = o.batch_csr(mode, off, ctrs, delta, now, lc)
        want = H.spec_batch(s, mode, off, ctrs, delta, now, lc)
        assert np.array_equal(got[0], want[0]), f"verdicts, batch {b} mode {mode}"
        if mode != 2:
            assert np.array_equal(got[1], want[1]), f"first limited, batch {b} mode {mode}"
        if lc:
            assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3]), f"remaining/ttl, batch {b}"
        assert H.normalise_dump(o.dump(), descs) == H.normalise_dump(s.dump(), descs), f"state, batch {b}"
        t_last = max(t_last, int(now.max()))
        # maintenance between batches
        ev = rng.random()
        if ev < 0.25:
            ids = [int(x) for x in rng.choice(live, size=min(3, len(live)), replace=False)]
            assert sorted(o.get_counters(ids, t_last)) == s.get_counters(ids, t_last)
        elif ev < 0.45:
            ids = [int(x) for x in rng.choice(live, size=min(2, len(live)), replace=False)]
            o.delete_counters(ids)
            s.delete_counters(ids)
            for d in descs:  # the reference needs add_counter again before an unqualified limit is used (:107)
                if int(d["limit_id"]) in ids:
                    args = (int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
                    o.limit_set(*args)
                    s.limit_set(*args)
        elif ev < 0.6:
            d = descs[int(rng.integers(0, len(descs)))]
            mx = int(rng.choice([0, 1, 7, 1 << 33]))
            args = (int(d["limit_id"]), int(d["ns_id"]), mx, int(d["window_us"]), bool(d["qualified"]))
            o.limit_set(*args)
            s.limit_set(*args)
            d["max_value"] = mx
        assert H.normalise_dump(o.dump(), descs) == H.normalise_dump(s.dump(), descs), f"state after maintenance {b}"


def test_clear_drops_only_unqualified_counters_in_both():
    descs = H.mixed_limits(n_ns=6, seed=3)
    o, s = both(descs)
    off, ctrs, delta, now = H.random_csr_stream(descs, 600, 77, n_keys=20)
    o.batch_csr(0, off, ctrs, delta, now)
    H.spec_batch(s, 0, off, ctrs, delta, now, False)
    o.clear()
    s.clear()
    assert sorted(o.dump()) == s.dump()
    assert all(k[1:3] != (0, 0) or descs[descs["limit_id"] == k[0]]["qualified"][0] for k in s.dump())
