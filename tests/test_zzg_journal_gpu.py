"""Persistent counters on the GPU (limitador_b200/journal.py over rl_counters_drain and rl_rls_counter_vars_drain):
mixed RLS and HTTP traffic through a service that keeps counter variables, drained after every batch, on a default,
a 64-counter and a pipelined engine.  After every drain a fresh service recovered from a copy of the directory lists
the same counters and answers GET /counters and GET /limits as the live one; structural calls between drains give a
full drain, a sweep a delta, and recovery stays exact; the recovered service then serves the rest of the stream as
limiter.RateLimiter over the CPU oracle does.  A crash is only ever simulated by copying the journal's files."""
import shutil

import numpy as np
import pytest

from limitador_b200 import journal as J
from limitador_b200.engine import RECORD_DTYPE
from tests.http_corpora import T0
from tests.test_zzd_configure_gpu import AD, G, GL, HR, NAMESPACES, P, PA, Pair

PIPELINE = 2  # RL_FLAG_PIPELINE
CONFIGS = [[G, P, HR, GL, AD], [dict(G, max_value=8), P, HR, AD, PA]]  # the second deletes GL and adds PA


def _export(e):
    return sorted(zip(*(c.tolist() for c in e.export_counters())))


def _fresh(kw, n_configs):
    b = Pair(**kw)
    for c in CONFIGS[:n_configs]:
        b.configure(c)
    return b


def _gets(p, now):
    return [(p.api.get_counters(ns, now), p.api.get_limits(ns)) for ns in NAMESPACES]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [{}, {"max_counters_per_request": 64}, {"flags": PIPELINE}], ids=["default", "wide", "pipelined"])
def test_a_recovered_service_lists_answers_and_serves_as_the_live_one(tmp_path, kw):
    rng = np.random.default_rng(5)
    a = _fresh(kw, 1)
    jr = J.CounterJournal(a.rls, str(tmp_path / "live"))
    n_configs, now, fulls = 1, T0, []
    for step in range(9):
        now = T0 + step * 7_000_000
        if step == 3:
            a.configure(CONFIGS[1])  # a deletion: rows of GL are reset, cells re-mapped
            n_configs = 2
        if step == 5:
            a.e.sweep(now)  # the admin and path-a windows (10 s) of two steps ago end: tombstones to reclaim
            a.rl.storage.o.invalidate_expired(now)  # the oracle's sweep
            assert a.e.compact(0)["regions_rebuilt"] > 0
        if step == 7:
            assert a.e.sweep(now) > 0
            a.rl.storage.o.invalidate_expired(now)
        a.traffic(rng, step, now)
        r = jr.drain()
        fulls.append(r["full"])
        copy = tmp_path / f"copy{step}"
        shutil.copytree(tmp_path / "live", copy)
        b = _fresh(kw, n_configs)
        info = J.recover(str(copy), b.rls)
        assert info["truncated_bytes"] == 0
        assert _export(b.e) == _export(a.e), step
        assert _gets(b, now) == _gets(a, now), step
        if step == 8:
            # the recovered service takes over the stream; the oracle goes with it
            b.rl, b.clock = a.rl, a.clock
            for s2 in range(3):
                b.traffic(rng, step + 1 + s2, now + (s2 + 1) * 2_000_000)
            assert b.metrics() == {k: v for k, v in b.want_m.items() if v}  # a series at 0 is not written
        b.close()
    # the first drain, the configure_with and the compaction give bases; the sweep a delta
    assert fulls == [True, False, False, True, False, True, False, False, False]
    jr.close()
    a.close()


@pytest.mark.gpu
def test_a_delta_after_a_sweep_and_a_reinsert_into_the_same_row(tmp_path):
    from limitador_b200 import Engine
    e = Engine(capacity_rows=256, cells_per_row=3, max_batch=4096, regions=1)
    e.limits_set([(0, 0, 1, 1, 100, 1_000_000), (1, 0, 1, 1, 100, 5_000_000), (2, 1, 0, 0, 50, 1_000_000)])
    jr = J.CounterJournal(e, str(tmp_path / "j"))
    rng = np.random.default_rng(1)
    now = T0
    for step in range(10):
        now += 3_000_000
        recs = np.zeros(200, dtype=RECORD_DTYPE)
        recs["ns_id"] = rng.integers(0, 2, len(recs))
        recs["hits_addend"] = 1
        recs["key_lo"] = rng.integers(1, 60, len(recs))  # few keys: rows emptied by a sweep are claimed again
        recs["now_us"] = now
        e.check_and_update_records(recs)
        if step % 2:
            e.sweep(now + 1_500_000)
        r = jr.drain()
        assert r["full"] == (step == 0)
        copy = tmp_path / f"c{step}"
        shutil.copytree(tmp_path / "j", copy)
        f = Engine(capacity_rows=512, cells_per_row=1, max_batch=4096)
        f.limits_set(e.limits_get())
        J.recover(str(copy), f)
        assert _export(f) == _export(e), step
        f.close()
    assert e.compact(0)["rows_tombstoned"] > 0  # rows were tombstoned along the way
    jr.close()


@pytest.mark.gpu
def test_a_million_qualified_keys_round_trip_through_base_and_deltas(tmp_path):
    from limitador_b200 import Engine
    e = Engine(capacity_rows=1 << 21, cells_per_row=1, max_batch=1 << 16)
    e.limits_set([(0, 0, 1, 1, 10 ** 9, 3_600_000_000)])
    jr = J.CounterJournal(e, str(tmp_path / "j"))
    n, batch = 1 << 20, 1 << 16
    for s in range(0, n, batch):
        recs = np.zeros(batch, dtype=RECORD_DTYPE)
        recs["hits_addend"] = 1 + (s // batch) % 3
        recs["key_lo"] = np.arange(s, s + batch, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(1)
        recs["key_hi"] = np.arange(s, s + batch, dtype=np.uint64) & np.uint64(0xFFFF)
        recs["now_us"] = T0 + s
        e.update_records(recs)
        r = jr.drain()
        assert r["full"] == (s == 0) and (s == 0 or r["counters"] == batch)
    f = Engine(capacity_rows=1 << 21, cells_per_row=3, max_batch=1 << 16)
    f.limits_set(e.limits_get())
    info = J.recover(str(tmp_path / "j"), f)
    assert info["records"] == n // batch - 1 and info["counters"] == n
    ea, eb = e.export_counters(), f.export_counters()
    oa, ob = np.lexsort((ea[2], ea[1], ea[0])), np.lexsort((eb[2], eb[1], eb[0]))
    assert all(np.array_equal(x[oa], y[ob]) for x, y in zip(ea, eb))
    jr.close()
