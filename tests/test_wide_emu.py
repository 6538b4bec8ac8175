"""The wide position encoding (requests of 17..64 counters, rl_core.h) run through the host emulator
(tests/emu/emu.cpp, wide=True) and compared bit for bit with the oracle: verdicts, first-limited ids, remaining / ttl in the
caller's order, and the table."""
import numpy as np
import pytest

from tests import helpers as H


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
@pytest.mark.parametrize("seed", [0, 1])
def test_wide_random_streams_match_oracle(cells, load_counters, seed):
    descs = H.wide_limits(seed)
    batches = [H.wide_stream(descs, 120, seed * 100 + b, monotone=(b % 2 == 0)) for b in range(4)]
    rounds = H.emu_vs_oracle(descs, cells, batches, load_counters, wide=True)
    assert max(rounds) >= 1  # every wide request spans several rows


@pytest.mark.parametrize("load_counters", [False, True])
def test_wide_mixed_with_narrow_requests_matches_oracle(load_counters):
    descs = H.wide_limits(7)
    batches = [H.wide_stream(descs, 150, 700 + b, min_ctrs=1) for b in range(3)]
    assert any(int(np.diff(b[0]).max()) > 16 for b in batches) and any(int(np.diff(b[0]).min()) <= 16 for b in batches)
    H.emu_vs_oracle(descs, 3, batches, load_counters, wide=True)


def test_wide_encoding_on_narrow_batches_matches_narrow_emulator():
    descs = H.mixed_limits(n_ns=12, seed=3)
    narrow, wide = H.Emu(descs, 3), H.Emu(descs, 3, wide=True)
    for b in range(4):
        batch = H.random_csr_stream(descs, 250, 40 + b, n_keys=3)
        a, w = narrow.batch_csr(0, *batch, True), wide.batch_csr(0, *batch, True)
        for x, y in zip(a, w):
            assert x.tolist() == y.tolist()
    assert narrow.dump() == wide.dump()


def test_wide_update_mode_matches_oracle():
    descs = H.wide_limits(11)
    H.emu_vs_oracle(descs, 7, [H.wide_stream(descs, 100, 1100 + b) for b in range(3)], False, mode=2, wide=True)


def test_wide_fixed_point_chain_at_64_counters():
    """The adversarial coupling of test_emu_algorithm (request i allowed iff i-1 denied, rows of max 1 shared
    pairwise), each request padded to 64 counters with limits that never bite, one row each."""
    descs = [(0, 0, 1, 1, 1, 3600_000_000), (1, 0, 2, 1, 1, 3600_000_000)]
    descs += [(2 + k, 0, 3 + k, 1, 1 << 40, 3600_000_000) for k in range(62)]
    descs = np.array(descs, dtype=H.LIMIT_DESC_DTYPE)
    n = 30
    off = np.arange(0, 64 * n + 1, 64, dtype=np.uint32)
    ctrs = np.zeros(64 * n, dtype=H.COUNTER_DTYPE)
    for i in range(n):
        row = [(2 + k, 0, 1000 + i, 0) for k in range(62)]
        row.insert(i % 62, (0, 0, 1 + i // 2, 0))        # row A_k shared by requests 2k, 2k+1
        row.insert(63 - i % 13, (1, 0, 1 + (i + 1) // 2, 0))  # row B_k shared by requests 2k-1, 2k
        ctrs[64 * i:64 * (i + 1)] = row
    delta = np.ones(n, dtype=np.uint64)
    now = np.full(n, H.T0, dtype=np.uint64)
    for lc in (False, True):
        rounds = H.emu_vs_oracle(descs, 1, [(off, ctrs, delta, now)], lc, wide=True)
        assert rounds[0] >= n // 2


def test_wide_resolve_positions_permutation_and_high_bits():
    """64 counters of one namespace, unqualified ones last in the given order: they are processed first, so the
    positions and the permutation differ from the given order, and counters beyond bit 31 of `used` are grouped."""
    descs = [(k, 0, 0 if k >= 40 else 1 + k % 5, 0 if k >= 40 else 1, 1 << 40, 60_000_000) for k in range(64)]
    descs = np.array(descs, dtype=H.LIMIT_DESC_DTYPE)
    emu = H.Emu(descs, 7, wide=True)
    ctrs = np.array([(k, 0, 9, 0) for k in range(64)], dtype=H.COUNTER_DTYPE)
    nacc, acc, perm = emu.resolve(ctrs, req=5)
    assert nacc > 1
    order = list(range(40, 64)) + list(range(40))  # unqualified first, then qualified, each in the given order
    assert perm.tolist() == order
    seen_pos, seen_orig = [], []
    for a in acc[:nacc]:
        assert a["req"] == 5 and a["hdr_hi"] != 0
        cells = int(a["cells"])
        cnt = (cells >> 28) & 7
        assert cells >> 31 == 1  # several accesses: coupled
        for k in range(cnt):
            pos = (int(a["posorig"]) >> (6 * k)) & 63
            seen_pos.append(pos)
            seen_orig.append(perm[pos])
        assert int(a["posorig"]) >> (6 * cnt) == 0
    assert sorted(seen_pos) == list(range(64)) and max(seen_pos) == 63
    assert sorted(seen_orig) == list(range(64))
    # one access per (row group, key): the 24 unqualified counters share groups of 7 cells
    assert all(a["hdr_hi"] == 0 for a in acc[nacc:])
    # the given order is kept inside each class
    assert [p for p in perm.tolist() if p >= 40] == list(range(40, 64))


def test_wide_resolve_limits():
    descs = np.array([(k, 0, 1, 1, 5, 60_000_000) for k in range(65)], dtype=H.LIMIT_DESC_DTYPE)
    emu = H.Emu(descs, 1, wide=True)
    ctrs = np.array([(k, 0, 1, 0) for k in range(65)], dtype=H.COUNTER_DTYPE)
    too_many = 4  # RL_DEV_TOO_MANY_COUNTERS
    assert emu.resolve(ctrs)[0] == -too_many
    assert emu.resolve(ctrs[:33], max_ctrs=32)[0] == -too_many
    assert emu.resolve(ctrs[:32], max_ctrs=32)[0] == 32
    assert emu.resolve(ctrs[:64])[0] == 64
    assert emu.resolve(ctrs[:17], wide=False)[0] == -too_many
    assert emu.resolve(ctrs[:16], wide=False)[0] == 16
