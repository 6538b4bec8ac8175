"""The edges of the counter arithmetic through every decision path of the GPU engine, every batch compared with the CPU
oracle (verdicts, first-limited ids, remaining / ttl where the call returns them, the whole table): u64 deltas and
wrapping sums, maxima up to 2^64-1, counters above their maximum, clocks exactly on a counter's expiry
(tests/helpers.py edge_limits / edge_csr_stream / edge_records; their coverage is counted in
tests/test_edge_arithmetic.py).  The run-length replay decides whole runs in closed form (DESIGN.md §3.3); these are the
values at which a 32-bit product, a saturating add or an exclusive expiry bound would change its answers.  Sorted last
on purpose: it reruns the streams of the files before it at the edges."""
import numpy as np
import pytest

from limitador_b200 import Engine
from limitador_b200.engine import COUNTER_DTYPE, LIMIT_DESC_DTYPE, RECORD_DTYPE, pack_records16
from tests import helpers as H

pytestmark = pytest.mark.gpu
S = 1_000_000
M64 = H.M64


def _engine(descs, cells, capacity=1 << 14, max_batch=1 << 14, regions=4, flags=0, **kw):
    e = Engine(capacity_rows=capacity, cells_per_row=cells, max_batch=max_batch, regions=regions, flags=flags, **kw)
    e.limits_set(descs)
    return e


def _tables(e, o, descs, what=""):
    assert H.normalise_dump(e.dump(), descs) == H.normalise_dump(o.dump(), descs), f"table differs {what}"


def _same(got, want, n, what):
    for k in range(n):
        assert got[k].tolist() == want[k].tolist(), f"output {k} differs, {what}"


def _change_max(e, o, descs, rng, share=0.3):
    """max_value lowered (under live counters) or raised, on the engine and the oracle."""
    idx = np.flatnonzero(rng.random(len(descs)) < share)
    for i in idx:
        descs["max_value"][i] = int(rng.choice([0, 1, 3])) if rng.random() < 0.5 else H._pick(rng, H.EDGE_MAXIMA)
        d = descs[i]
        o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    if len(idx):
        e.limits_set(descs[idx])


def _get_counters(e, o, descs, t):
    ids = descs["limit_id"]
    got = e.get_counters(ids, t)
    assert got == o.get_counters(ids, t), "get_counters differs"
    mx = {int(d["limit_id"]): int(d["max_value"]) for d in descs}
    return sum(r[3] > mx[r[0]] for r in got)  # rows whose remaining wrapped (counter above its maximum)


# -- 32-byte records ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
def test_records_at_the_edges(cells, load_counters):
    """Host calls: check_and_update, update_counters and is_within_limits batches of one edge stream, max_value changed
    between batches, get_counters on counters above their maximum."""
    descs = H.edge_limits(30 + cells, "single", n_ns=9, cells=cells)
    e, o = _engine(descs, cells), H.oracle_with_limits(descs)
    rng = np.random.default_rng(cells)
    above = 0
    for b, (mode, recs) in enumerate(H.edge_batches(descs, 40 + cells, 6, 3000, form="records")):
        if mode == 0:
            got = e.check_and_update_records(recs, load_counters, stride=cells)
            _same(got, o.batch_records(0, recs, load_counters, cells), 4 if load_counters else 2, f"batch {b}")
        elif mode == 1:
            _same(e.is_within_limits_records(recs), o.batch_records(1, recs), 2, f"batch {b}")
        else:
            e.update_records(recs)
            o.batch_records(2, recs)
        _tables(e, o, descs, f"batch {b}")
        above += _get_counters(e, o, descs, int(recs["now_us"][-1]))
        _change_max(e, o, descs, rng)
    assert above > 0


@pytest.mark.parametrize("load_counters", [False, True])
def test_pipelined_device_records_at_the_edges(load_counters):
    """RL_FLAG_PIPELINE: back-to-back device-memory calls, outputs read after rl_fence / rl_sync."""
    import torch
    cells = 3
    descs = H.edge_limits(50, "single", n_ns=9, cells=cells)
    e, o = _engine(descs, cells, flags=2), H.oracle_with_limits(descs)
    shadow = H.spec_with_limits(descs)
    recs = [H.edge_records(descs, 3000, 60 + b, shadow=shadow, monotone=(b % 2 == 0)) for b in range(6)]
    n = len(recs[0])
    dev = [torch.from_numpy(r.view(np.int64).reshape(-1, 4).copy()).cuda() for r in recs]
    outs = [[torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
             torch.zeros(n * cells, dtype=torch.int64, device="cuda"),
             torch.zeros(n * cells, dtype=torch.int64, device="cuda")] for _ in recs]
    torch.cuda.synchronize()
    for d, (lim, fl, rem, ttl) in zip(dev, outs):
        e.check_and_update_records_ptr(n, d.data_ptr(), lim.data_ptr(), 1, load_counters, out_first_ptr=fl.data_ptr(),
                                       out_rem_ptr=rem.data_ptr() if load_counters else 0,
                                       out_ttl_ptr=ttl.data_ptr() if load_counters else 0, stride=cells)
    e.fence()
    e.sync()
    for b, r in enumerate(recs):
        want = o.batch_records(0, r, load_counters, cells)
        got = [outs[b][0].cpu().numpy(), outs[b][1].cpu().numpy().view(np.uint32),
               outs[b][2].cpu().numpy().view(np.uint64), outs[b][3].cpu().numpy().view(np.uint64)]
        _same(got, want, 4 if load_counters else 2, f"batch {b}")
    _tables(e, o, descs)


@pytest.mark.parametrize("cells", [1, 7])
def test_compact_records_at_the_edges(cells):
    """rl_record16, hits 1..255, one clock per batch aimed at a live counter's expiry (- 1, + 0, + 1)."""
    descs = H.edge_limits(70 + cells, "single", n_ns=9, cells=cells)
    e, o = _engine(descs, cells), H.oracle_with_limits(descs)
    rng = np.random.default_rng(cells)
    shadow = H.spec_with_limits(descs)
    t = H.T0
    for b in range(8):
        recs = H.edge_records(descs, 4000, 80 + b, shadow=shadow, hits=(1, 255))
        live = [x for (_, _, _, _, x) in o.dump() if x > t]
        t = (int(rng.choice(live)) + int(rng.integers(-1, 2))) if live and b % 2 else t + 1000
        recs["now_us"] = t
        lim, fl = e.check_and_update_compact(pack_records16(recs), t)
        want = o.batch_records(0, recs)
        assert lim.tolist() == want[0].tolist() and fl.tolist() == want[1].tolist(), f"batch {b}"
        _tables(e, o, descs, f"batch {b}")


# -- the general (CSR) form -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
def test_csr_u64_deltas_and_coupled_requests(cells, load_counters):
    """u64 deltas on every row shape, coupled (multi-row) requests decided by the fixed point, update_counters and
    is_within_limits batches, max_value changes, get_counters above the maximum."""
    descs = H.edge_limits(90 + cells, "mixed", n_ns=12)
    e, o = _engine(descs, cells), H.oracle_with_limits(descs)
    rng = np.random.default_rng(cells)
    above = 0
    for b, (mode, (off, ctrs, delta, now)) in enumerate(H.edge_batches(descs, 100 + cells, 6, 2500)):
        if mode == 0:
            got = e.check_and_update_batch(off, ctrs, delta, now, load_counters)
            _same(got, o.batch_csr(0, off, ctrs, delta, now, load_counters), 4 if load_counters else 2, f"batch {b}")
        elif mode == 1:
            _same(e.is_within_limits_batch(off, ctrs, delta, now), o.batch_csr(1, off, ctrs, delta, now), 2, f"batch {b}")
        else:
            e.update_batch(off, ctrs, delta, now)
            o.batch_csr(2, off, ctrs, delta, now)
        _tables(e, o, descs, f"batch {b}")
        above += _get_counters(e, o, descs, int(now[-1]))
        _change_max(e, o, descs, rng)
    assert above > 0
    assert e.stats()["fixed_point_rounds"] >= 1


@pytest.mark.parametrize("load_counters", [False, True])
def test_wide_requests_at_the_edges(load_counters):
    """max_counters_per_request=64: requests of 17..64 counters on wide_limits-shaped edge limits."""
    descs = H.edge_limits(110, "wide")
    e = _engine(descs, 7, capacity=1 << 15, max_batch=4096, max_counters=4096 * 64, max_counters_per_request=64)
    o = H.oracle_with_limits(descs)
    rng = np.random.default_rng(5)
    for b, (mode, (off, ctrs, delta, now)) in enumerate(H.edge_batches(descs, 111, 5, 600, min_ctrs=17)):
        if mode == 2:
            e.update_batch(off, ctrs, delta, now)
            o.batch_csr(2, off, ctrs, delta, now)
        else:
            got = e.check_and_update_batch(off, ctrs, delta, now, load_counters)
            _same(got, o.batch_csr(0, off, ctrs, delta, now, load_counters), 4 if load_counters else 2, f"batch {b}")
        _tables(e, o, descs, f"batch {b}")
        _change_max(e, o, descs, rng, 0.1)


# -- k_hot and the chained path -------------------------------------------------------------------------------------------
def _hot_limits():
    """ns 0: max 2^64 - 1 (values wrap, never denied); ns 1: max 2^36, 2-s window (each window's run crosses the maximum
    after ~16 large hits); ns 2: max 2^63 (crossed from an imported value); ns 3: unqualified, 1-µs window."""
    return np.array([(0, 0, 1, 1, M64, 1 << 40), (1, 1, 1, 1, 1 << 36, 2 * S), (2, 2, 1, 1, 1 << 63, 60 * S),
                     (3, 3, 0, 0, (1 << 32) - 1, 1)], dtype=LIMIT_DESC_DTYPE)


def _seed_near_the_top(e, o, descs, t):
    """Hot keys 1 and 2 of namespaces 0 and 2 imported just below 2^64 and 2^63: the batches' runs wrap and cross."""
    rows = [(0, k, 0, M64 - (1 << 44) * k, t + (1 << 40)) for k in (1, 2)] + \
           [(2, k, 0, (1 << 63) - (1 << 43) * k, t + 60 * S) for k in (1, 2)]
    cols = [np.array(c, dtype=np.uint32 if j == 0 else np.uint64) for j, c in enumerate(zip(*rows))]
    e.import_counters(*cols)
    H.oracle_restore(o, descs, *cols)
    _tables(e, o, descs, "after the import")


@pytest.mark.parametrize("load_counters", [False, True])
def test_hot_rows_replay_runs_across_the_wrap(load_counters, monkeypatch):
    """RL_HOT=1: one key per namespace dominates consecutive batches, so k_hot replays its whole request list; its runs
    of equal large hits (2^31 .. 2^32-1) add up past 2^32 per run, wrap past 2^64 (ns 0) and cross the maximum inside
    a run (ns 1, ns 2)."""
    monkeypatch.setenv("RL_HOT", "1")
    descs = _hot_limits()
    e, o = _engine(descs, 3, capacity=1 << 15, max_batch=1 << 15), H.oracle_with_limits(descs)
    rng = np.random.default_rng(11)
    t, n = H.T0, 20000
    _seed_near_the_top(e, o, descs, t)
    big = np.array(H.RECORD_BIG_DELTAS, dtype=np.uint32)
    for b in range(7):
        recs = np.zeros(n, dtype=RECORD_DTYPE)
        hot = rng.random(n) < 0.8
        recs["ns_id"] = np.where(hot, rng.integers(0, 3, n), rng.integers(0, 4, n))
        recs["key_lo"] = np.where(hot, 1 + rng.integers(0, 2, n), 10 + rng.integers(0, 3000, n))
        d = big[b % len(big)]  # one large delta per batch; one request in ten takes another
        recs["hits_addend"] = np.where(rng.random(n) < 0.9, d, big[rng.integers(0, len(big), n)])
        recs["now_us"] = t + np.sort(rng.integers(0, 1_500_000, n)).astype(np.uint64)
        t += 1_600_000
        got = e.check_and_update_records(recs, load_counters, stride=3)
        _same(got, o.batch_records(0, recs, load_counters, 3), 4 if load_counters else 2, f"batch {b}")
        _tables(e, o, descs, f"batch {b}")
        if b >= 2:
            assert e.stats()["hot_rows"] > 0, f"batch {b}: no hot row"
    values = {(l, lo): v for (l, lo, _, v, _) in o.dump()}
    assert all(values[(0, k)] < M64 - (1 << 44) * k for k in (1, 2)), "the ns-0 counters did not wrap"


@pytest.mark.parametrize("load_counters", [False, True])
def test_chained_chunks_at_the_edges(load_counters, monkeypatch):
    """RL_CHUNK=128, RL_HEAVY_MULT=1, RL_HOT=0: every partition above the average is chained, and a tiny key space makes
    its chunks share rows; edge records and update batches."""
    monkeypatch.setenv("RL_CHUNK", "128")
    monkeypatch.setenv("RL_HEAVY_MULT", "1")
    monkeypatch.setenv("RL_HOT", "0")
    for cells in (1, 3):
        descs = H.edge_limits(120 + cells, "single", n_ns=9, cells=cells)
        e, o = _engine(descs, cells, flags=4), H.oracle_with_limits(descs)  # RL_FLAG_KERNEL_STATS
        for b, (mode, recs) in enumerate(H.edge_batches(descs, 130 + cells, 5, 6000, form="records", n_keys=25)):
            if mode == 2:
                e.update_records(recs)
                o.batch_records(2, recs)
            else:
                got = e.check_and_update_records(recs, load_counters, stride=cells)
                _same(got, o.batch_records(0, recs, load_counters, cells), 4 if load_counters else 2, f"batch {b}")
            _tables(e, o, descs, f"cells {cells} batch {b}")
        st = e.stats()
        assert st["chained_chunks"] > 0 and st["ordered_chunks"] > 0


# -- imported edge states -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cells", [1, 7])
def test_imported_edge_states(cells):
    """import_counters seeds values near 2^64, counters above their maximum and expiries equal to the next request's
    clock (oracle_restore does the same on the oracle); an edge stream goes on from there in both forms."""
    descs = H.edge_limits(140 + cells, "mixed", n_ns=12)
    e, o = _engine(descs, cells), H.oracle_with_limits(descs)
    rng = np.random.default_rng(cells)
    shadow = H.spec_with_limits(descs)
    off, ctrs, delta, now = H.edge_csr_stream(descs, 2000, 150 + cells, shadow=shadow)
    # one row per counter the stream names; expiry = the clock of its first request, or one window later
    seen, rows, aimed = set(), [], 0
    for i in range(len(delta)):
        for c in ctrs[off[i]:off[i + 1]]:
            d = descs[descs["limit_id"] == c["limit_id"]][0]
            k = (int(c["limit_id"]),) + ((int(c["key_lo"]), int(c["key_hi"])) if d["qualified"] else (0, 0))
            if k in seen:
                continue
            seen.add(k)
            mx = int(d["max_value"])
            v = H._pick(rng, [M64, M64 - 1, M64 - int(delta[i]), (mx + 1) & M64, (mx + 5) & M64, 1 << 63, mx])
            x = int(now[i]) if rng.random() < 0.5 else int(now[i]) + int(d["window_us"])
            x = max(x, int(d["window_us"]))
            aimed += x == int(now[i])
            rows.append((*k, v, x))
    cols = [np.array(c, dtype=np.uint32 if j == 0 else np.uint64) for j, c in enumerate(zip(*rows))]
    e.import_counters(*cols)
    H.oracle_restore(o, descs, *cols)
    _tables(e, o, descs, "after the import")
    assert aimed > 0 and _get_counters(e, o, descs, int(now[0])) > 0
    _same(e.check_and_update_batch(off, ctrs, delta, now, True), o.batch_csr(0, off, ctrs, delta, now, True), 4, "csr")
    _tables(e, o, descs, "after the CSR batch")
    _get_counters(e, o, descs, int(now[-1]))
    recs = H.edge_records(descs, 2000, 160 + cells, shadow=shadow)
    _same(e.check_and_update_records(recs, True, stride=5), o.batch_records(0, recs, True, 5), 4, "records")
    _tables(e, o, descs, "after the records")


# -- known answers ----------------------------------------------------------------------------------------------------
class EngineLayer:
    """helpers.EDGE_KATS through the engine's CSR calls."""

    def __init__(self, kat, cells):
        self.kat = kat
        self.e = _engine(H.edge_kat_limits(kat), cells, capacity=1 << 10, max_batch=1 << 12, regions=1)

    def _csr(self, n):
        return np.arange(n + 1, dtype=np.uint32), np.array([(0, 0, 7, 0)] * n, dtype=COUNTER_DTYPE)

    def seed(self, value, now):
        self.e.update_batch(*self._csr(1), [value], [now])

    def check(self, deltas, nows, lc):
        lim, _, rem, ttl = self.e.check_and_update_batch(*self._csr(len(deltas)), deltas, nows, lc)
        return lim.tolist(), rem.tolist(), ttl.tolist()

    def state(self):
        rows = [(v, x) for (l, lo, hi, v, x) in self.e.dump() if (l, lo, hi) == (0, 7, 0)]
        assert len(rows) == 1
        return rows[0]

    def get(self, now):
        return [r[3:] for r in self.e.get_counters([0], now)]

    def set_max(self, mx):
        self.e.limits_set(H.edge_kat_limits(self.kat, mx))


@pytest.mark.parametrize("name", sorted(H.EDGE_KATS))
@pytest.mark.parametrize("cells", [1, 7])
@pytest.mark.parametrize("batched", [False, True], ids=["one-call-each", "one-batch"])
@pytest.mark.parametrize("load_counters", [False, True])
def test_edge_known_answers_on_the_engine(name, cells, batched, load_counters):
    H.run_edge_kat(H.EDGE_KATS[name], EngineLayer(H.EDGE_KATS[name], cells), batched, load_counters)


@pytest.mark.parametrize("cells", [1, 7])
def test_a_run_across_the_wrap_takes_the_rounds_of_any_run(cells):
    """200 allowed requests of delta 2^52 + 1 on one key under max 2^64 - 2: from 2^64 - 1 - 2^58 the sum wraps past
    2^64 on the way (no value is 2^64 - 1), from 5 it does not.  k_main decides both in the same number of replay rounds
    (closed form); a B-test that saturated instead of wrapping would apply the requests at the wrap one per round."""
    W, T, n, d = 60 * S, H.T0, 200, (1 << 52) + 1
    descs = np.array([(0, 0, 1, 1, M64 - 1, W)], dtype=LIMIT_DESC_DTYPE)
    off, ctrs = np.arange(n + 1, dtype=np.uint32), np.array([(0, 0, 7, 0)] * n, dtype=COUNTER_DTYPE)
    rounds = {}
    for v0 in (M64 - (1 << 58), 5):
        e, o = _engine(descs, cells, capacity=1 << 10, max_batch=1 << 12, regions=1, flags=4), H.oracle_with_limits(descs)
        e.update_batch(off[:2], ctrs[:1], [v0], [T])
        o.batch_csr(2, off[:2], ctrs[:1], [v0], [T])
        before = e.stats()["replay_rounds"]
        args = (off, ctrs, np.full(n, d, dtype=np.uint64), T + 1 + np.arange(n, dtype=np.uint64))
        _same(e.check_and_update_batch(*args, True), o.batch_csr(0, *args, True), 4, f"from {v0}")
        assert e.dump() == o.dump() == [(0, 7, 0, (v0 + n * d) & M64, T + W)]
        rounds[v0] = e.stats()["replay_rounds"] - before
    assert (M64 - (1 << 58) + n * d) > M64 >= 5 + n * d
    assert rounds[M64 - (1 << 58)] == rounds[5], rounds
