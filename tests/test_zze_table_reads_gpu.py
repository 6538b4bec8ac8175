"""The table reads (rl_get_counters, rl_counters_export) when the output arrays are too small: at most cap rows written,
each a row of the full result, and *out_count the exact number found, on a table that holds expired qualified counters,
an unqualified limit whose cell sits in a row after delete_counters (present in the row, absent as a counter) and an
unqualified limit that was never touched.  The full results are the oracle's."""
import ctypes as C

import numpy as np
import pytest

from limitador_b200 import Engine
from limitador_b200.engine import COUNTER_DTYPE, LIMIT_DESC_DTYPE, MEM_DEVICE, MEM_HOST, _p
from tests import helpers as H

pytestmark = pytest.mark.gpu
S = 1_000_000
SENTINEL = 0x25A5A5A5  # fits an int32 tensor

# ns 0: two qualified limits on one variable set (one row per key; the 1 s one expires), two unqualified limits in one
# row; ns 1: an unqualified limit no request names
LIMITS = np.array([(0, 0, 1, 1, 1000, 1 * S), (1, 0, 1, 1, 1000, 60 * S), (2, 0, 0, 0, 1000, 60 * S),
                   (3, 0, 0, 0, 1000, 60 * S), (4, 1, 0, 0, 1000, 60 * S)], dtype=LIMIT_DESC_DTYPE)
IDS = np.arange(len(LIMITS), dtype=np.uint32)


def _table():
    e = Engine(capacity_rows=1 << 10, cells_per_row=3, max_batch=1024)
    e.limits_set(LIMITS)
    o = H.oracle_with_limits(LIMITS)
    n = 24
    off = np.arange(0, 4 * n + 1, 4, dtype=np.uint32)
    per_key = lambda k: [(0, 0, k, k & 1), (1, 0, k, k & 1), (2, 0, 0, 0), (3, 0, 0, 0)]  # noqa: E731
    ctrs = np.array([c for k in range(1, n + 1) for c in per_key(k)], dtype=COUNTER_DTYPE)
    delta = np.ones(n, dtype=np.uint64)
    now = H.T0 + np.arange(n, dtype=np.uint64) * 1000
    got, want = e.check_and_update_batch(off, ctrs, delta, now), o.batch_csr(0, off, ctrs, delta, now)
    assert got[0].tolist() == want[0].tolist()
    e.delete_counters([2])  # limit 2's cell stays in the row, (0, 0), and is no counter any more
    o.delete_counters([2])
    return e, o


def _rows(cols, n):
    return [tuple(int(c[i]) for c in cols) for i in range(n)]


def _host_call(fn, cap):
    """fn(cap, five pointers, count pointer) with host arrays one longer than cap -> (count, rows written, untouched)"""
    cols = [np.full(cap + 1, SENTINEL, dtype=np.uint32 if k == 0 else np.uint64) for k in range(5)]
    cnt = C.c_uint64(SENTINEL)
    ptrs = [_p(c) for c in cols] if cap else [None] * 5
    assert fn(cap, *ptrs, C.byref(cnt)) == 0
    n = min(cnt.value, cap)
    return cnt.value, _rows(cols, n), all(int(c[n]) == SENTINEL for c in cols)


def _device_call(fn, cap):
    import torch
    cols = [torch.full((cap + 1,), SENTINEL, dtype=torch.int32 if k == 0 else torch.int64, device="cuda")
            for k in range(5)]
    torch.cuda.synchronize()
    cnt = C.c_uint64(SENTINEL)
    ptrs = [C.c_void_p(c.data_ptr()) for c in cols] if cap else [None] * 5
    assert fn(cap, *ptrs, C.byref(cnt)) == 0
    n = min(cnt.value, cap)
    host = [c.cpu().numpy().view(np.uint32 if k == 0 else np.uint64) for k, c in enumerate(cols)]
    return cnt.value, _rows(host, n), all(int(c[n]) == SENTINEL for c in host)


def _check_caps(call, fn, full):
    for cap in (0, 1, len(full) - 1):
        cnt, rows, untouched = call(fn, cap)
        assert cnt == len(full), f"cap {cap}: *out_count {cnt}, {len(full)} found with room for all"
        assert len(rows) == min(cap, len(full)) and set(rows) <= set(full), f"cap {cap}: rows not of the full result"
        assert untouched, f"cap {cap}: written beyond cap"


def test_get_counters_with_a_short_cap_counts_exactly():
    e, o = _table()
    L = e._lib
    for t in (H.T0 + S // 2, H.T0 + 2 * S):  # limit 0's counters live, then expired
        fn = lambda cap, *out: L.rl_get_counters(e._h, _p(IDS), len(IDS), t, cap, *out)  # noqa: E731
        cnt, full, _ = _host_call(fn, 1 << 10)
        assert sorted(full) == o.get_counters(IDS, t) and len(full) == cnt
        assert {r[0] for r in full} == ({0, 1, 3} if t < H.T0 + S else {1, 3})
        _check_caps(_host_call, fn, full)
        assert e.get_counters(IDS, t, cap=1) == sorted(full)


@pytest.mark.parametrize("mem", [MEM_HOST, MEM_DEVICE], ids=["host", "device"])
def test_export_with_a_short_cap_counts_exactly(mem):
    e, o = _table()
    L = e._lib
    fn = lambda cap, *out: L.rl_counters_export(e._h, None, 0, 0, cap, mem, *out)  # noqa: E731
    call = _host_call if mem == MEM_HOST else _device_call
    cnt, full, _ = call(fn, 1 << 10)
    assert len(full) == cnt and len(set(full)) == cnt
    assert (4, 0, 0, 0, 0) in full and 2 not in {r[0] for r in full}  # never touched: present; deleted: absent
    assert H.normalise_dump(full, LIMITS) == H.normalise_dump(o.dump(), LIMITS)
    _check_caps(call, fn, full)
    assert sorted(zip(*[c.tolist() for c in e.dump_arrays(cap=1)])) == sorted(full)
