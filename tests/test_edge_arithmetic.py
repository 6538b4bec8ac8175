"""The edges of the counter arithmetic on the CPU layers: u64 wrap of value + delta, maxima up to 2^64-1, counters above
their maximum (update_counters, a lowered max_value), clocks exactly on a counter's expiry.
  * the edge streams of tests/helpers.py reach every one of those edges, counted (a generator change that loses one
    fails here);
  * the C oracle equals tests/spec_model.py on them: all three modes, both load_counters values, get_counters with the
    wrapping remaining, max_value lowered and raised between batches;
  * the host emulator (the kernels' rl_core.h replay, tests/emu) equals the oracle on them, narrow and wide;
  * the written-out known answers of helpers.EDGE_KATS hold on the oracle, spec_model and the emulator;
  * a run of allowed requests whose sum wraps is still decided in closed form (one replay step).
The same streams and known answers go through the GPU in tests/test_zz6_edges_gpu.py."""
import numpy as np
import pytest

from oracle import binding as ob
from tests import helpers as H
from tests.spec_model import SpecStore

M64 = H.M64
KEY = (0, 7, 0)  # the EDGE_KATS counter: limit 0, key_lo 7, key_hi 0


def _args(d):
    return int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"])


def _new_max(rng):
    """A max_value change on a live limit: far below (counters end up above it), to a u64 edge, or above."""
    return int(rng.choice([0, 1, 3])) if rng.random() < 0.5 else H._pick(rng, H.EDGE_MAXIMA)


# -- coverage -----------------------------------------------------------------------------------------------------------
CSR_FLOOR = dict(wrapped_sums=200, expiry_reads=200, stale_flips=40, above_max_reads=200, long_runs=3, wrapping_runs=3,
                 denied_runs=40)
RECORD_FLOOR = dict(expiry_reads=200, stale_flips=40, above_max_reads=100, long_runs=3, denied_runs=40)


@pytest.mark.parametrize("form,shape", [("csr", "mixed"), ("csr", "single"), ("records", "single")])
@pytest.mark.parametrize("seed", [1, 2])
def test_edge_streams_reach_every_edge(form, shape, seed):
    """Counted on spec_model, per stream of 6 batches of 2000 requests.  Records cannot wrap a value from zero (their
    delta is a u32): they reach 2^64 only from an imported state, which the GPU file seeds."""
    descs = H.edge_limits(seed, shape, cells=7)
    n = H.edge_coverage(descs, H.edge_batches(descs, seed, 6, 2000, form=form), form)
    floor = CSR_FLOOR if form == "csr" else RECORD_FLOOR
    for kind, least in floor.items():
        assert n[kind] >= least, f"{kind}: {n[kind]} < {least} ({n})"


# -- the oracle against spec_model ------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_the_python_spec_on_edge_streams(seed):
    rng = np.random.default_rng(500 + seed)
    descs = H.edge_limits(seed, "mixed" if seed % 2 else "single", n_ns=8)
    o = ob.Oracle(16)
    s = H.counting_spec(descs)
    for d in descs:
        o.limit_set(*_args(d))
    live = sorted(int(d["limit_id"]) for d in descs)
    wrapped_remaining = 0
    for b, (mode, (off, ctrs, delta, now)) in enumerate(H.edge_batches(descs, seed, 8, 1200)):
        lc = mode == 0 and bool(b & 2)
        got = o.batch_csr(mode, off, ctrs, delta, now, lc)
        want = H.spec_batch(s, mode, off, ctrs, delta, now, lc)
        assert np.array_equal(got[0], want[0]), f"verdicts, batch {b} mode {mode}"
        if mode != 2:
            assert np.array_equal(got[1], want[1]), f"first limited, batch {b} mode {mode}"
        if lc:
            assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3]), f"remaining/ttl, batch {b}"
        assert H.normalise_dump(o.dump(), descs) == H.normalise_dump(s.dump(), descs), f"state, batch {b}"
        # get_counters at the batch's last clock and one of its expiries: remaining wraps for counters above max
        for t in (int(now[-1]), int(now[len(now) // 2])):
            rows = o.get_counters(live, t)
            assert rows == s.get_counters(live, t), f"get_counters, batch {b}"
            mx = {int(d["limit_id"]): int(d["max_value"]) for d in descs}
            wrapped_remaining += sum(r[3] > mx[r[0]] for r in rows)
        # max_value lowered or raised under live counters
        for i in np.flatnonzero(rng.random(len(descs)) < 0.3):
            descs["max_value"][i] = _new_max(rng)
            o.limit_set(*_args(descs[i]))
            s.limit_set(*_args(descs[i]))
    assert wrapped_remaining > 0, "no get_counters row had a counter above its maximum"
    for kind in ("wrapped_sums", "expiry_reads", "above_max_reads", "denied_runs"):
        assert s.n[kind] > 0, f"the stream never reached {kind}: {s.n}"


# -- the emulator against the oracle ----------------------------------------------------------------------------------
def _emu_vs_oracle_with_max_changes(descs, cells, batches, lc, wide, seed):
    """helpers.emu_vs_oracle with max_value lowered / raised between batches; is_rate_limited batches (the emulator has
    no such call) run as check_and_update."""
    rng = np.random.default_rng(seed)
    emu, orc = H.Emu(descs, cells, wide), H.oracle_with_limits(descs)
    for b, (mode, (off, ctrs, delta, now)) in enumerate(batches):
        mode = 2 if mode == 2 else 0
        e = emu.batch_csr(mode, off, ctrs, delta, now, lc)
        o = orc.batch_csr(mode, off, ctrs, delta, now, lc)
        if mode == 0:
            assert e[0].tolist() == o[0].tolist(), f"verdicts differ, batch {b}"
            assert e[1].tolist() == o[1].tolist(), f"first-limited limit differs, batch {b}"
            if lc:
                assert e[2].tolist() == o[2].tolist(), f"remaining differs, batch {b}"
                assert e[3].tolist() == o[3].tolist(), f"ttl differs, batch {b}"
        assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs), f"table differs, batch {b}"
        for i in np.flatnonzero(rng.random(len(descs)) < 0.25):
            descs["max_value"][i] = _new_max(rng)
            orc.limit_set(*_args(descs[i]))
        emu.set_limits(descs)


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
def test_emulator_equals_oracle_on_edge_streams(cells, load_counters):
    for shape in ("mixed", "single"):
        descs = H.edge_limits(10 + cells, shape, n_ns=8, cells=cells)
        batches = H.edge_batches(descs, 20 + cells, 6, 1500)
        _emu_vs_oracle_with_max_changes(descs, cells, batches, load_counters, False, cells)


@pytest.mark.parametrize("load_counters", [False, True])
def test_wide_emulator_equals_oracle_on_edge_streams(load_counters):
    descs = H.edge_limits(4, "wide")
    batches = H.edge_batches(descs, 4, 5, 300, min_ctrs=17)
    _emu_vs_oracle_with_max_changes(descs, 7, batches, load_counters, True, 4)


# -- known answers ----------------------------------------------------------------------------------------------------
class _CsrLayer:
    """EDGE_KATS through a CSR batch interface (the oracle's or the emulator's)."""

    def __init__(self, kat):
        self.kat = kat

    def seed(self, value, now):
        self.batch(2, [value], [now], False)

    def check(self, deltas, nows, lc):
        lim, _, rem, ttl = self.batch(0, deltas, nows, lc)
        return lim.tolist(), rem.tolist(), ttl.tolist()

    def state(self):
        rows = [(v, x) for (l, lo, hi, v, x) in self.dump() if (l, lo, hi) == KEY]
        assert len(rows) == 1
        return rows[0]

    def _csr(self, n):
        return np.arange(n + 1, dtype=np.uint32), np.array([(KEY[0], 0, KEY[1], KEY[2])] * n, dtype=H.COUNTER_DTYPE)


class OracleLayer(_CsrLayer):
    def __init__(self, kat):
        super().__init__(kat)
        self.o = H.oracle_with_limits(H.edge_kat_limits(kat))

    def batch(self, mode, deltas, nows, lc):
        return self.o.batch_csr(mode, *self._csr(len(deltas)), deltas, nows, lc)

    def dump(self):
        return self.o.dump()

    def get(self, now):
        return [r[3:] for r in self.o.get_counters([0], now)]

    def set_max(self, mx):
        self.o.limit_set(*_args(H.edge_kat_limits(self.kat, mx)[0]))


class EmuLayer(_CsrLayer):
    def __init__(self, kat, cells=1, wide=False):
        super().__init__(kat)
        self.e = H.Emu(H.edge_kat_limits(kat), cells, wide)

    def batch(self, mode, deltas, nows, lc):
        return self.e.batch_csr(mode, *self._csr(len(deltas)), deltas, nows, lc)

    def dump(self):
        return self.e.dump()

    def get(self, now):
        return None  # the emulator has no get_counters

    def set_max(self, mx):
        self.e.set_limits(H.edge_kat_limits(self.kat, mx))


class SpecLayer:
    def __init__(self, kat):
        self.kat = kat
        self.s = SpecStore()
        self.s.limit_set(*_args(H.edge_kat_limits(kat)[0]))

    def seed(self, value, now):
        self.s.update_counters([KEY], value, now)

    def check(self, deltas, nows, lc):
        out = [self.s.check_and_update([KEY], d, lc, t) for d, t in zip(deltas, nows)]
        return [int(r[0]) for r in out], [r[2][0] for r in out], [r[3][0] for r in out]

    def state(self):
        return tuple(self.s.qualified[KEY])

    def get(self, now):
        return [r[3:] for r in self.s.get_counters([0], now)]

    def set_max(self, mx):
        self.s.limit_set(*_args(H.edge_kat_limits(self.kat, mx)[0]))


@pytest.mark.parametrize("name", sorted(H.EDGE_KATS))
@pytest.mark.parametrize("layer", ["oracle", "spec", "emu-1", "emu-7", "emu-wide"])
@pytest.mark.parametrize("batched", [False, True], ids=["one-call-each", "one-batch"])
@pytest.mark.parametrize("load_counters", [False, True])
def test_edge_known_answers(name, layer, batched, load_counters):
    kat = H.EDGE_KATS[name]
    mk = {"oracle": OracleLayer, "spec": SpecLayer, "emu-1": lambda k: EmuLayer(k, 1),
          "emu-7": lambda k: EmuLayer(k, 7), "emu-wide": lambda k: EmuLayer(k, 7, wide=True)}[layer]
    H.run_edge_kat(kat, mk(kat), batched, load_counters)


# -- closed form across a wrap ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cells", [1, 7])
def test_runs_across_the_wrap_stay_closed_form(cells):
    """Twelve allowed requests of delta 2^52 + 1 under max 2^64 - 2: from 2^64 - 1 - 2^54 the sum wraps past 2^64 at
    the fourth (no value is 2^64 - 1), from 5 it does not; the replay takes either as one run (one step).  Twelve
    delta-0 requests on a counter above its maximum are one denied run.  A B-test that saturated instead of wrapping
    would split the first run."""
    W, T, d = 60_000_000, H.T0, (1 << 52) + 1
    descs = np.array([(0, 0, 1, 1, M64 - 1, W)], dtype=H.LIMIT_DESC_DTYPE)
    off, ctrs = np.arange(13, dtype=np.uint32), np.array([(0, 0, 7, 0)] * 12, dtype=H.COUNTER_DTYPE)
    nows = [T + 1 + k for k in range(12)]
    for v0, wraps in ((M64 - (1 << 54), True), (5, False)):
        assert (v0 + 12 * d > M64) == wraps
        emu, orc = H.Emu(descs, cells), H.oracle_with_limits(descs)
        for x in (emu, orc):
            x.batch_csr(2, off[:2], ctrs[:1], [v0], [T])
        got = emu.batch_csr(0, off, ctrs, [d] * 12, nows, True)
        assert emu.steps == 1, f"from {v0}: {emu.steps} replay steps"
        want = orc.batch_csr(0, off, ctrs, [d] * 12, nows, True)
        assert got[0].tolist() == want[0].tolist() == [0] * 12
        assert got[2].tolist() == want[2].tolist()
        assert emu.dump() == orc.dump() == [(0, 7, 0, (v0 + 12 * d) & M64, T + W)]
    descs["max_value"] = 3
    emu, orc = H.Emu(descs, cells), H.oracle_with_limits(descs)
    for x in (emu, orc):
        x.batch_csr(2, off[:2], ctrs[:1], [10], [T])
    got = emu.batch_csr(0, off, ctrs, [0] * 12, nows, True)
    assert emu.steps == 1 and got[0].tolist() == [1] * 12
    assert got[2].tolist() == orc.batch_csr(0, off, ctrs, [0] * 12, nows, True)[2].tolist()
