"""The batching ALGORITHM the kernels implement (rl_core.h: request -> row accesses,
stream-order replay per row, fixed-point rounds for requests spanning several rows) run
sequentially on the host (tests/emu) and compared bit-for-bit with the oracle."""
import numpy as np
import pytest

from tests import helpers as H


@pytest.mark.parametrize("cells", [1, 3, 7])
@pytest.mark.parametrize("load_counters", [False, True])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_streams_match_oracle(cells, load_counters, seed):
    descs = H.mixed_limits(n_ns=12, seed=seed)
    batches = [H.random_csr_stream(descs, 300, seed * 100 + b, n_keys=3, monotone=(b % 2 == 0)) for b in range(6)]
    rounds = H.emu_vs_oracle(descs, cells, batches, load_counters)
    assert max(rounds) >= 1  # the mixed table always has multi-row requests


def test_update_mode_matches_oracle():
    descs = H.mixed_limits(n_ns=12, seed=5)
    emu = H.Emu(descs, 3)
    orc = H.oracle_with_limits(descs)
    for b in range(4):
        off, ctrs, delta, now = H.random_csr_stream(descs, 200, 900 + b, n_keys=3)
        emu.batch_csr(2, off, ctrs, delta, now)
        orc.batch_csr(2, off, ctrs, delta, now)
        assert H.normalise_dump(emu.dump(), descs) == H.normalise_dump(orc.dump(), descs)


def test_long_dependency_chain_converges():
    """Adversarial coupling: request i is allowed iff request i-1 was denied (limits max 1 on
    two rows shared pairwise) — the fixed point needs many rounds but stays exact."""
    descs = np.array([(0, 0, 1, 1, 1, 3600_000_000), (1, 0, 2, 1, 1, 3600_000_000)], dtype=H.LIMIT_DESC_DTYPE)
    n = 40
    off = np.arange(0, 2 * n + 1, 2, dtype=np.uint32)
    ctrs = np.zeros(2 * n, dtype=H.COUNTER_DTYPE)
    for i in range(n):
        ctrs[2 * i] = (0, 0, 1 + i // 2, 0)          # row A_k shared by requests 2k, 2k+1
        ctrs[2 * i + 1] = (1, 0, 1 + (i + 1) // 2, 0)  # row B_k shared by requests 2k-1, 2k
    delta = np.ones(n, dtype=np.uint64)
    now = np.full(n, H.T0, dtype=np.uint64)
    rounds = H.emu_vs_oracle(descs, 1, [(off, ctrs, delta, now)], False)
    assert rounds[0] > 2


@pytest.mark.parametrize("cells,load_counters,seed", [(1, True, 11), (3, False, 12), (7, True, 13)])
def test_wide_key_space_streams_match_oracle(cells, load_counters, seed):
    """Many distinct keys with few requests each (state carried across batches, windows expiring
    between them, the oracle's table growing under it) — the shape the GPU fuzzing found the oracle's
    rehash bug with."""
    descs = H.mixed_limits(n_ns=12, seed=seed)
    batches = [H.random_csr_stream(descs, 2500, seed * 100 + b, n_keys=120, monotone=bool(b & 1)) for b in range(4)]
    H.emu_vs_oracle(descs, cells, batches, load_counters)
