"""The namespace-sharded peer exchange (rl_shard_*, SURVEY §8e) on ONE GPU: `world` engines in one
process, each with its own table and exchange slab, connected by plain device pointers
(rl_shard_connect_ptrs) — the same kernels, flags and buffer rotation as the one-process-per-GPU
deployment, where the slabs are CUDA-IPC mappings and the stores cross NVLink.

Checked against ONE global oracle that applies the steps in (step, source rank, source index) order —
the canonical stream order of the sharded store (SURVEY §8e) — verdicts of every request and the union
of the per-rank tables."""
import time

import numpy as np
import pytest

from limitador_b200 import Engine, EngineError, streams
from limitador_b200.engine import RECORD_DTYPE, Shard
from limitador_b200 import exchange
from tests import helpers as H

pytestmark = pytest.mark.gpu


def _run(world, lag, n_steps, batch, n_rows, n_ns, ragged=False, cells=7, seed=0, hot=False, per_rank_clock=False,
         monkeypatch=None):
    """C2 traffic through `world` shards.  cells: rows of 1, 3 or 7 cells (C2's first `cells` limits of every namespace
    when that is fewer than its 4, so that every namespace stays one row); hot: hot rows on (RL_HOT=1); per_rank_clock:
    each step spans 1 s of clock and rank r's clock runs r x 700 ms behind rank 0's, so that the canonical order of an
    inbox is not monotone in time.  Prints the wall time and the device memory the engines and shards took."""
    import torch
    t_start = time.perf_counter()
    if hot:
        monkeypatch.setenv("RL_HOT", "1")
    w = streams.WORKLOADS["C2"](batch=batch, n_rows=n_rows, n_ns=n_ns)
    descs = w.limits[w.limits["limit_id"] % 4 < min(cells, 4)]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    engines = [Engine(capacity_rows=w.capacity_rows, cells_per_row=cells, max_batch=world * batch, flags=2)
               for _ in range(world)]
    for e in engines:
        e.limits_set(descs)
    shards = [Shard(engines[r], r, world, batch, lag) for r in range(world)]
    slabs = [s.slab for s in shards]
    for s in shards:
        s.connect_ptrs(slabs)
    rng = np.random.default_rng(seed)
    recs = [[w.batch_records(1000 * r + st) for r in range(world)] for st in range(n_steps)]
    for st in range(n_steps):  # one clock for all ranks of a step, as in a global batch
        for r in range(world):
            recs[st][r]["now_us"] = recs[st][0]["now_us"]
            if per_rank_clock:
                recs[st][r]["now_us"] = (H.T0 + st * 1_000_000 - r * 700_000
                                         + np.arange(batch, dtype=np.uint64) * np.uint64(1_000_000) // np.uint64(batch))
        if ragged:
            for r in range(world):
                recs[st][r] = recs[st][r][: int(rng.integers(0, batch + 1))]
            recs[st][st % world] = recs[st][st % world][:0]  # and one rank with nothing at all
    d_recs = [[torch.from_numpy(x.view(np.int64).reshape(-1, 4).copy()).cuda() for x in row] for row in recs]
    d_out = [[torch.full((max(len(x), 1),), 7, dtype=torch.uint8, device="cuda") for x in row] for row in recs]
    torch.cuda.synchronize()
    for st in range(n_steps):
        # phase by phase over the ranks: every wait kernel is enqueued after the kernels it waits for
        for r in range(world):
            shards[r].send(len(recs[st][r]), d_recs[st][r].data_ptr(), d_out[st][r].data_ptr())
        for r in range(world):
            shards[r].decide()
        for r in range(world):
            shards[r].collect()
    for s in shards:
        s.flush()
    for e in engines:
        e.sync()
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    o = H.oracle_with_limits(descs, 1 << 16)
    limited = 0
    for st in range(n_steps):
        for r in range(world):
            if len(recs[st][r]) == 0:
                continue
            want = o.batch_records(0, recs[st][r])[0]
            got = d_out[st][r].cpu().numpy()[: len(want)]
            assert np.array_equal(got, want), f"step {st} rank {r}: {int((got != want).sum())} verdicts differ"
            limited += int(want.sum())
    assert limited > 0, "no request was limited: the limits never mattered"
    # the union of the rank tables is the oracle's table, and every counter sits on its owner
    union = []
    for r, e in enumerate(engines):
        d = e.dump()
        union.extend(d)
    assert H.normalise_dump(union, descs) == H.normalise_dump(o.dump(), descs)
    ns_of = {int(d["limit_id"]): int(d["ns_id"]) for d in descs}
    for r, e in enumerate(engines):
        for row in e.dump():
            assert exchange.owner_of(ns_of[int(row[0])], world) == r
    for s in shards:
        s.close()
    for e in engines:
        e.close()
    print(f"world {world} lag {lag} batch {batch} cells {cells} hot {int(hot)}: {time.perf_counter() - t_start:.1f} s, "
          f"engines and shards took {used / 2**30:.2f} GiB of device memory")


@pytest.mark.parametrize("world,lag", [(1, 0), (2, 1), (2, 2), (3, 2), (4, 0)])
def test_peer_exchange_matches_global_oracle(world, lag):
    _run(world, lag, n_steps=7, batch=4096, n_rows=5000, n_ns=16)


def test_peer_exchange_ragged_and_empty_steps():
    _run(3, 2, n_steps=8, batch=2048, n_rows=3000, n_ns=12, ragged=True, seed=5)


def test_peer_exchange_world_8_batch_65536():
    """Eight ranks of full-size C2 batches: 256 tiles per send (32 per warp in k_xcount's last-block scan)."""
    _run(8, 2, n_steps=4, batch=65536, n_rows=400_000, n_ns=64)


def test_peer_exchange_tiles_of_512():
    """A batch of 300 000 records per rank: k_xcount / k_xscatter tiles of 512 records, more than 16 tiles per warp in
    the last-block scan."""
    _run(2, 1, n_steps=3, batch=300_000, n_rows=500_000, n_ns=64)


@pytest.mark.parametrize("lag", [3, 4])
def test_peer_exchange_deep_lag(lag):
    """lag 3 and 4: 5 and 6 rotating buffers, 12 steps, so every buffer is reused at least twice."""
    _run(3, lag, n_steps=12, batch=2048, n_rows=5000, n_ns=16, ragged=True, seed=lag)


@pytest.mark.parametrize("cells", [1, 3])
def test_peer_exchange_hot_rows(cells, monkeypatch):
    """Rows of 1 and 3 cells (k_main<1,1> and <3,3>) with hot rows on: C2's Zipf head replayed by k_hot from the
    segmented inbox."""
    _run(2, 1, n_steps=6, batch=16384, n_rows=20_000, n_ns=4, cells=cells, hot=True, monkeypatch=monkeypatch)


def test_peer_exchange_per_rank_clocks():
    """Rank r's clock r x 700 ms behind rank 0's within every step: an inbox in canonical order jumps back and forth
    across C2's 1 s windows."""
    _run(3, 2, n_steps=6, batch=4096, n_rows=3000, n_ns=8, per_rank_clock=True)


def test_peer_exchange_hot_owner():
    """Every namespace on one owner: its inbox takes world x batch records in a step."""
    import torch
    world, batch = 3, 1024
    w = streams.WORKLOADS["C2"](batch=batch, n_rows=2000, n_ns=1)
    engines = [Engine(capacity_rows=w.capacity_rows, cells_per_row=7, max_batch=world * batch, flags=2) for _ in range(world)]
    for e in engines:
        e.limits_set(w.limits)
    shards = [Shard(engines[r], r, world, batch, 1) for r in range(world)]
    for s in shards:
        s.connect_ptrs([x.slab for x in shards])
    o = H.oracle_with_limits(w.limits, 1 << 16)
    for st in range(4):
        recs = [w.batch_records(10 * st + r) for r in range(world)]
        d = [torch.from_numpy(x.view(np.int64).reshape(-1, 4).copy()).cuda() for x in recs]
        out = [torch.zeros(batch, dtype=torch.uint8, device="cuda") for _ in range(world)]
        for r in range(world):
            shards[r].send(batch, d[r].data_ptr(), out[r].data_ptr())
        for r in range(world):
            shards[r].decide()
        for s in shards:
            s.flush()
        for e in engines:
            e.sync()
        for r in range(world):
            assert np.array_equal(out[r].cpu().numpy(), o.batch_records(0, recs[r])[0])


def test_peer_exchange_refuses_an_inbox_larger_than_the_engine():
    """rl_config.max_batch bounds an owner's inbox: a larger one fails the step loudly (RL_FATAL at rl_sync),
    never a silent allow."""
    import torch
    world, batch = 2, 1024
    w = streams.WORKLOADS["C2"](batch=batch, n_rows=2000, n_ns=1)
    engines = [Engine(capacity_rows=w.capacity_rows, cells_per_row=7, max_batch=batch, flags=2) for _ in range(world)]
    for e in engines:
        e.limits_set(w.limits)
    shards = [Shard(engines[r], r, world, batch, 0) for r in range(world)]
    for s in shards:
        s.connect_ptrs([x.slab for x in shards])
    recs = [w.batch_records(r) for r in range(world)]
    d = [torch.from_numpy(x.view(np.int64).reshape(-1, 4).copy()).cuda() for x in recs]
    out = [torch.zeros(batch, dtype=torch.uint8, device="cuda") for _ in range(world)]
    for r in range(world):
        shards[r].send(batch, d[r].data_ptr(), out[r].data_ptr())
    for r in range(world):
        shards[r].decide()
    for s in shards:
        s.flush()
    owner = exchange.owner_of(0, world)
    with pytest.raises(EngineError):
        engines[owner].sync()


def test_shard_refuses_a_slab_the_device_cannot_hold():
    """A slab larger than the device is refused with RL_TRANSIENT and its exact size in bytes (the shard is freed before
    the message is written), and the engine stays usable: the refused allocation does not fail its next launch."""
    from limitador_b200.engine import RL_TRANSIENT
    world, cap, lag = 32, 1 << 27, 4
    depth = lag + 2
    align = lambda x: (x + 255) & ~255
    slab_bytes = (align(depth * world * cap * RECORD_DTYPE.itemsize) + align(depth * world * cap)
                  + align(depth * world * 16))  # records | verdicts | one 16-byte control block per (buffer, peer)
    assert slab_bytes > 4 * (80 << 30)  # far beyond an 80 GB device
    w = streams.WORKLOADS["C2"](batch=1024, n_rows=2000, n_ns=1)
    e = Engine(capacity_rows=w.capacity_rows, cells_per_row=w.cells_per_row, max_batch=w.batch, flags=2)
    e.limits_set(w.limits)
    with pytest.raises(EngineError) as err:
        Shard(e, 0, world, cap, lag)
    assert err.value.status == RL_TRANSIENT
    assert f"cannot allocate the {slab_bytes}-byte exchange slab" in str(err.value)
    recs = w.batch_records(0)
    lim = e.check_and_update_records(recs, True, stride=w.cells_per_row)[0]
    assert np.array_equal(lim, H.oracle_with_limits(w.limits, 1 << 16).batch_records(0, recs, True, w.cells_per_row)[0])
    e.close()
