"""Namespace-sharded execution of one batch over `world` ranks (SURVEY.md §8e).

Every counter a request touches belongs to the request's namespace
(limitador/src/lib.rs:512), so a request has exactly one owner rank,
`rl_owner_of(ns_id, world)`, and counters are never replicated.  One step =
  bucket my slice of the global batch by owner (stable)  ->  all-to-all of the 32-B records
  ->  decide locally (stream order = source rank, source index)  ->  all-to-all of the verdict
  bytes back  ->  restore request order.
The only collective on the path is that personalised all-to-all (NCCL over NVLink on GPUs).
`sharded_step` is the plain two-collective form; `LanePipelinedExchange` is the pipelined form
bench.py runs (fixed-size blocks, one all-to-all per step, no host synchronisation).
The orchestration is backend-agnostic: bench.py plugs in the engine's kernels on GPU tensors,
tests/test_exchange_gloo.py plugs in numpy + the oracle on CPU tensors over gloo.
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np


def sharded_step(recs, world: int, dist, bucket: Callable, decide: Callable, unpermute: Callable, out_limited,
                 recv_buf=None, verdict_recv=None, verdict_back=None):
    """Run one sharded step.

    recs         : [n, 4] int64 tensor (bytes = rl_record[n]) — this rank's slice of the global batch
    bucket(recs) : -> (send [n,4] tensor grouped by owner, stably; src_idx [n] tensor; counts: list[int] per owner)
    decide(recv, m, verdict) : run check_and_update on the first m received records, writing verdict[:m] (uint8)
    unpermute(verdict_back, src_idx, out_limited): out_limited[src_idx[i]] = verdict_back[i]
    Returns the number of requests this rank decided.
    """
    import torch

    n = recs.shape[0]
    send, src_idx, send_counts = bucket(recs)
    sc = torch.tensor(send_counts, dtype=torch.int64, device=recs.device)
    rc = torch.empty_like(sc)
    dist.all_to_all_single(rc, sc)
    recv_counts = rc.cpu().tolist()
    m = int(sum(recv_counts))
    if recv_buf is None or recv_buf.shape[0] < m:
        recv_buf = torch.empty((max(m, 1), 4), dtype=torch.int64, device=recs.device)
    if verdict_recv is None or verdict_recv.shape[0] < m:
        verdict_recv = torch.empty(max(m, 1), dtype=torch.uint8, device=recs.device)
    if verdict_back is None or verdict_back.shape[0] < n:
        verdict_back = torch.empty(max(n, 1), dtype=torch.uint8, device=recs.device)
    dist.all_to_all_single(recv_buf[:m], send, recv_counts, list(send_counts))
    if m:
        decide(recv_buf, m, verdict_recv)
    dist.all_to_all_single(verdict_back[:n], verdict_recv[:m], list(send_counts), recv_counts)
    unpermute(verdict_back, src_idx, out_limited)
    return m


def stable_bucket_numpy(recs_np: np.ndarray, owners: np.ndarray, world: int):
    """Reference (CPU) bucketing: stable sort by owner.  Returns (permuted records, src index, counts)."""
    order = np.argsort(owners, kind="stable")
    counts = np.bincount(owners, minlength=world).astype(np.int64)
    return recs_np[order], order.astype(np.int32), counts.tolist()


class LanePipelinedExchange:
    """Sharded steps with ONE all-to-all each (include/rl_engine.h: rl_record_lane_put/_gather).

    Blocks are fixed-size (`slot_cap` record slots per peer, unused slots are no-op records), so no
    counts travel and nothing synchronises with the host.  A record that does not fit its owner's block is NOT
    decided: its verdict byte comes back as RL_VERDICT_ERROR (0xFF, include/rl_engine.h) — never as 0 = allowed —
    and the bucket kernel raises the overflow flag the caller passed (bench.py fails the run on it).  The peer
    exchange of the engine (`rl_shard_*`, engine.Shard) has no such limit and is what bench.py runs by default.  The verdict byte of the record that sat in
    slot (p, k) of step s-lag rides back in the lane byte of slot (p, k) of step s: the reverse
    all-to-all of the two-collective scheme disappears, and the decisions of the last lag-1 steps
    overlap the exchange of step s (a step's period is bounded by (decision latency + exchange) / lag,
    not by their sum).  A step's verdicts are therefore delivered `lag` steps later (`step` returns
    the output tensor that has just been completed); `flush` delivers what is still in flight with
    lane-only exchanges.

    `ops` supplies the device work (bench.py: the engine's kernels on CUDA tensors; the gloo test:
    numpy + the oracle):
      bucket(recs, send, pos)        send[world*slot_cap, 4] <- recs bucketed by owner (+ padding), pos[n] <- slot
      lane_put(send, lane)           lane byte of send[i] <- lane[i]
      decide(recv, verdict)          check_and_update over every slot of recv, verdict[i] <- limited (may be asynchronous)
      lane_gather(recv, pos, out)    out[i] <- lane byte of recv[pos[i]]
      fence(age)                     order the current stream after the decide call `age` calls back (0 = the last)
    """

    def __init__(self, world: int, batch: int, slot_cap: int, dist, ops, device, lag: int = 2):
        import torch
        assert lag >= 1
        self.world, self.batch, self.slot_cap, self.dist, self.ops, self.lag = world, batch, slot_cap, dist, ops, lag
        self.depth = depth = lag + 1  # buffer sets: a set is reused lag+1 steps later
        slots = world * slot_cap
        self.send = torch.empty((slots, 4), dtype=torch.int64, device=device)
        self.recv = [torch.empty((slots, 4), dtype=torch.int64, device=device) for _ in range(depth)]
        self.pos = [torch.zeros(batch, dtype=torch.int32, device=device) for _ in range(depth)]
        self.verdict = [torch.zeros(slots, dtype=torch.uint8, device=device) for _ in range(depth)]
        self.outs = [None] * depth  # output tensor of the step that used buffer set b, until delivered
        self.seq = 0

    def step(self, recs, out_limited):
        """Enqueue one step for `recs` ([batch, 4] int64 = rl_record[batch]); its verdicts land in
        `out_limited` `lag` steps (or a flush) later.  Returns the output tensor completed by this
        step's exchange, or None."""
        ops, s, lag = self.ops, self.seq, self.lag
        b, bl = s % self.depth, (s - lag) % self.depth
        ops.bucket(recs, self.send, self.pos[b])  # independent of any decision: runs while they finish
        ops.fence(lag - 1)  # the decisions of step s-lag are final (later steps may still be running)
        ops.lane_put(self.send, self.verdict[bl])
        self.dist.all_to_all_single(self.recv[b], self.send)
        ops.decide(self.recv[b], self.verdict[b])
        done = self.outs[bl] if s >= lag else None
        if done is not None:
            ops.lane_gather(self.recv[b], self.pos[bl], done)
            self.outs[bl] = None
        self.outs[b] = out_limited
        self.seq += 1
        return done

    def flush(self):
        """Deliver the verdicts of the (up to `lag`) steps still in flight; returns their outputs."""
        ops, done = self.ops, []
        ops.fence(0)  # every decide call so far
        for back in range(self.lag, 0, -1):
            b = (self.seq - back) % self.depth
            if self.seq < back or self.outs[b] is None:
                continue
            self.send.fill_(-1)  # no records, only lanes
            ops.lane_put(self.send, self.verdict[b])
            spare = self.recv[(self.seq + back) % self.depth]  # no decide call is reading any of them now
            self.dist.all_to_all_single(spare, self.send)
            ops.lane_gather(spare, self.pos[b], self.outs[b])
            done.append(self.outs[b])
            self.outs[b] = None
        return done


def owner_of(ns_id: int, world: int) -> int:
    """rl_owner_of (include/rl_engine.h): the rank that owns a namespace."""
    from . import engine as _eng
    return int(_eng.load_library().rl_owner_of(int(ns_id), int(world)))


def namespaces_owned(ns_ids, rank: int, world: int) -> np.ndarray:
    """The namespaces of `ns_ids` that `rank` owns in a store of `world` ranks (uint32, ascending).  Re-sharding a
    store to a new world size: every old rank exports, for each new rank r, its counters of namespaces_owned(all, r,
    new_world) (Engine.export_counters(ns_ids=...)), and new rank r imports what every old rank exported for it."""
    ids = sorted({int(n) for n in np.asarray(ns_ids).ravel().tolist()})
    return np.array([n for n in ids if owner_of(n, world) == rank], dtype=np.uint32)


def observed_block_max(recs, owner_lut, world: int) -> int:
    """Largest number of records one step of `recs` ([steps, batch, 4] int64 = rl_record) sends to one owner.
    `owner_lut[ns_id]` = owner rank (a tensor on the records' device)."""
    import torch
    worst = 0
    for s in range(recs.shape[0]):
        ns = recs[s, :, 0] & 0xFFFFFFFF  # rl_record word 0 = ns_id | hits_addend << 32
        worst = max(worst, int(torch.bincount(owner_lut[ns], minlength=world).max().item()))
    return worst


def slot_cap_for(largest_block: int, batch: int, headroom: float = 1.2) -> int:
    """Exchange block size (record slots per peer) for an observed largest block: headroom on top, a multiple
    of 256, never more than a whole batch."""
    return int(min(batch, (int(largest_block * headroom) + 255) // 256 * 256))


def balanced_namespace_ids(load, world: int):
    """A static namespace -> GPU placement (SURVEY §8e "Skew": "allow a static namespace→GPU override table") without
    touching the data path: the owner of a request is rl_owner_of(ns_id, world) and ns_id is an interned id the front
    chooses, so the front gives every namespace an id whose owner is the rank it wants the namespace on.

    load[j] = observed traffic of namespace j (any unit).  Namespaces are placed heaviest first on the least loaded
    rank (LPT), then given the smallest unused id that hashes to that rank.  Returns (ids int64[len(load)],
    owner_load float64[world]); ids[j] replaces j everywhere the front names the namespace (rl_limit_desc.ns_id,
    rl_record.ns_id).  Deterministic: equal inputs give equal ids on every rank."""
    import numpy as np
    load = np.asarray(load, dtype=np.float64)
    n = len(load)
    owner_load = np.zeros(world, dtype=np.float64)
    want = np.zeros(n, dtype=np.int64)
    for j in np.argsort(-load, kind="stable"):
        r = int(np.argmin(owner_load))  # ties: the lowest rank
        want[j] = r
        owner_load[r] += load[j]
    need = np.bincount(want, minlength=world)
    pools = [[] for _ in range(world)]
    cand = 0
    while any(len(pools[r]) < need[r] for r in range(world)):
        r = owner_of(cand, world)
        if len(pools[r]) < need[r]:
            pools[r].append(cand)
        cand += 1
        if cand > (1 << 24):
            raise RuntimeError("no namespace ids left below 2^24 (the 16-byte record form's id range)")
    ids = np.zeros(n, dtype=np.int64)
    taken = [0] * world
    for j in range(n):  # ids in namespace order inside a rank: stable and easy to read in a dump
        r = int(want[j])
        ids[j] = pools[r][taken[r]]
        taken[r] += 1
    return ids, owner_load


def remap_namespace_ids(recs, id_lut):
    """In place: rl_record word 0 (ns_id | hits_addend << 32) of `recs` ([..., 4] int64) gets ns_id = id_lut[ns_id].
    `id_lut` is an int64 tensor on the records' device."""
    flat = recs.view(-1, 4)
    step = 1 << 22
    for a in range(0, flat.shape[0], step):
        w0 = flat[a:a + step, 0]
        flat[a:a + step, 0] = id_lut[w0 & 0xFFFFFFFF] | ((w0 >> 32) << 32)
    return recs
