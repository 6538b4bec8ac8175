"""ctypes binding of librl_engine.so (include/rl_engine.h).

The engine is the product: hand-written sm_90a kernels behind a C-ABI.  There is no CPU
fallback — constructing an Engine without the built library or without a CUDA device
raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

RL_OK, RL_TRANSIENT, RL_FATAL = 0, 1, 2
MEM_HOST, MEM_DEVICE, MEM_HOST_ASYNC = 0, 1, 2
NONE = 0xFFFFFFFF

RECORD_DTYPE = np.dtype(
    [("ns_id", "<u4"), ("hits_addend", "<u4"), ("key_lo", "<u8"), ("key_hi", "<u8"), ("now_us", "<u8")]
)
RECORD16_DTYPE = np.dtype([("ns_hits_keyhi", "<u8"), ("key_lo", "<u8")])
COUNTER_DTYPE = np.dtype([("limit_id", "<u4"), ("_pad", "<u4"), ("key_lo", "<u8"), ("key_hi", "<u8")])


def pack_records16(recs: np.ndarray) -> np.ndarray:
    """rl_record[] -> rl_record16[] (include/rl_engine.h); the records' now_us is dropped: the batch is stamped
    with one clock reading at the call.  Raises if a record does not fit the 16-byte form."""
    recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
    if len(recs) and (int(recs["ns_id"].max()) >= 1 << 24 or int(recs["hits_addend"].max()) > 255
                      or int((recs["key_hi"] & np.uint64(0x00FFFFFFFFFFFFFF)).max()) >= 1 << 32):
        raise ValueError("record does not fit rl_record16: ns_id < 2^24, hits_addend <= 255, key_hi < 2^32")
    out = np.zeros(len(recs), dtype=RECORD16_DTYPE)
    out["ns_hits_keyhi"] = (recs["ns_id"].astype(np.uint64) | (recs["hits_addend"].astype(np.uint64) << np.uint64(24))
                            | ((recs["key_hi"] & np.uint64(0xFFFFFFFF)) << np.uint64(32)))
    out["key_lo"] = recs["key_lo"]
    return out
LIMIT_DESC_DTYPE = np.dtype(
    [("limit_id", "<u4"), ("ns_id", "<u4"), ("varset_id", "<u4"), ("qualified", "<u4"),
     ("max_value", "<u8"), ("window_us", "<u8")]
)

# every symbol include/rl_engine.h declares (tests check the library exports them all)
ABI_SYMBOLS = [
    "rl_shard_batch_create", "rl_shard_batch_destroy", "rl_shard_batch_slab", "rl_shard_batch_engine", "rl_shard_batch_ipc_handle",
    "rl_shard_batch_connect_ipc", "rl_shard_batch_connect_ptrs", "rl_shard_batch_send", "rl_shard_batch_decide",
    "rl_shard_batch_collect", "rl_shard_batch_step",
    "rl_engine_create", "rl_engine_destroy", "rl_last_error", "rl_engine_set_stream", "rl_engine_stream",
    "rl_engine_max_counters_per_request",
    "rl_sync", "rl_get_stats", "rl_limits_set", "rl_limits_delete", "rl_check_and_update_records",
    "rl_check_and_update_batch", "rl_is_within_limits_batch", "rl_is_within_limits_records",
    "rl_update_batch", "rl_update_records", "rl_get_counters", "rl_delete_counters", "rl_clear",
    "rl_sweep", "rl_bucket_by_owner", "rl_unpermute_u8", "rl_owner_of",
    "rl_profile_begin", "rl_profile_end", "rl_bucket_by_owner_padded", "rl_gather_u8", "rl_record_lane_put", "rl_record_lane_gather", "rl_fence", "rl_fence_call",
    "rl_front_create", "rl_front_destroy", "rl_front_check_and_update", "rl_front_stats",
    "rl_shard_create", "rl_shard_destroy", "rl_shard_ipc_handle", "rl_shard_connect_ipc", "rl_shard_connect_ptrs",
    "rl_shard_slab", "rl_shard_slab_bytes", "rl_shard_send", "rl_shard_decide", "rl_shard_collect", "rl_shard_step",
    "rl_shard_flush", "rl_shard_debug", "rl_trace_dump", "rl_check_and_update_compact", "rl_shard_fence",
    "rl_compact", "rl_ns_metrics_enable", "rl_ns_metrics_accumulate", "rl_ns_metrics_read",
    "rl_counters_export", "rl_counters_import", "rl_limits_get", "rl_counters_track", "rl_counters_drain",
]

SNAPSHOT_VERSION = 1  # format of Engine.save_counters files


class RlConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("capacity_rows", C.c_uint64),
        ("cells_per_row", C.c_uint32), ("max_batch", C.c_uint32), ("max_counters", C.c_uint32),
        ("regions", C.c_uint32), ("flags", C.c_uint32), ("max_counters_per_request", C.c_uint32),
    ]


class RlStats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64), ("batches", C.c_uint64), ("requests", C.c_uint64),
        ("capacity_rows", C.c_uint64), ("regions", C.c_uint32), ("row_bytes", C.c_uint32),
        ("fixed_point_rounds", C.c_uint32), ("_pad", C.c_uint32),
        ("chunks", C.c_uint64), ("replay_rounds", C.c_uint64), ("chained_chunks", C.c_uint64),
        ("ordered_chunks", C.c_uint64), ("phase_cycles", C.c_uint64 * 6),
        ("hot_rows", C.c_uint32), ("_pad2", C.c_uint32),
    ]


class EngineError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"[{'TRANSIENT' if status == RL_TRANSIENT else 'FATAL'}] {msg}")
        self.status = status
        self.transient = status == RL_TRANSIENT


_lib = None


def load_library(path: str | None = None):
    """Load librl_engine.so and declare the ABI.  Raises if it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or os.environ.get("RL_ENGINE_LIB") or _build.LIB_PATH
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -m limitador_b200.build` "
            "(limitador_b200 has no CPU fallback)")
    L = C.CDLL(path)
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
    L.rl_engine_create.argtypes = [C.POINTER(RlConfig), C.POINTER(vp)]
    L.rl_engine_destroy.argtypes = [vp]
    L.rl_engine_destroy.restype = None
    L.rl_last_error.argtypes = [vp]
    L.rl_last_error.restype = C.c_char_p
    L.rl_engine_max_counters_per_request.argtypes = [vp]
    L.rl_engine_max_counters_per_request.restype = u32
    L.rl_engine_set_stream.argtypes = [vp, vp]
    L.rl_engine_stream.argtypes = [vp]
    L.rl_engine_stream.restype = vp
    L.rl_sync.argtypes = [vp]
    L.rl_fence.argtypes = [vp]
    L.rl_fence_call.argtypes = [vp, u32]
    L.rl_get_stats.argtypes = [vp, C.POINTER(RlStats)]
    L.rl_limits_set.argtypes = [vp, vp, u32]
    L.rl_limits_delete.argtypes = [vp, vp, u32]
    L.rl_check_and_update_records.argtypes = [vp, u64, vp, i32, i32, vp, vp, vp, vp, u32]
    L.rl_check_and_update_batch.argtypes = [vp, u64, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp]
    L.rl_is_within_limits_batch.argtypes = [vp, u64, vp, vp, vp, vp, i32, vp, vp]
    L.rl_is_within_limits_records.argtypes = [vp, u64, vp, i32, vp, vp]
    L.rl_update_batch.argtypes = [vp, u64, vp, vp, vp, vp, i32]
    L.rl_update_records.argtypes = [vp, u64, vp, i32]
    L.rl_get_counters.argtypes = [vp, vp, u32, u64, u64, vp, vp, vp, vp, vp, vp]
    L.rl_delete_counters.argtypes = [vp, vp, u32]
    L.rl_clear.argtypes = [vp]
    L.rl_sweep.argtypes = [vp, u64, vp]
    L.rl_compact.argtypes = [vp, u32, vp]
    L.rl_ns_metrics_enable.argtypes = [vp, i32]
    L.rl_ns_metrics_accumulate.argtypes = [vp, u64, vp, u32, vp, vp, i32]
    L.rl_ns_metrics_read.argtypes = [vp, u32, vp, vp, vp, u32, vp, vp, i32]
    L.rl_counters_export.argtypes = [vp, vp, u32, u64, u64, i32, vp, vp, vp, vp, vp, vp]
    L.rl_counters_import.argtypes = [vp, u64, vp, vp, vp, vp, vp, i32]
    L.rl_limits_get.argtypes = [vp, u32, vp, vp]
    L.rl_counters_track.argtypes = [vp, i32]
    L.rl_counters_drain.argtypes = [vp, u64, i32, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int)]
    L.rl_bucket_by_owner.argtypes = [vp, u64, vp, u32, vp, vp, vp]
    L.rl_unpermute_u8.argtypes = [vp, u64, vp, vp, vp]
    L.rl_bucket_by_owner_padded.argtypes = [vp, u64, vp, u32, u32, vp, vp, vp]
    L.rl_gather_u8.argtypes = [vp, u64, vp, vp, vp]
    L.rl_record_lane_put.argtypes = [vp, u64, vp, vp]
    L.rl_record_lane_gather.argtypes = [vp, u64, vp, vp, vp]
    L.rl_profile_begin.argtypes = [vp]
    L.rl_profile_end.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
    L.rl_front_create.argtypes = [vp, u32, u32, C.POINTER(vp)]
    L.rl_front_destroy.argtypes = [vp]
    L.rl_front_destroy.restype = None
    L.rl_front_check_and_update.argtypes = [vp, vp, u32, u64, u64, i32, vp, vp, vp, vp, vp]
    L.rl_front_stats.argtypes = [vp, vp, vp]
    L.rl_owner_of.argtypes = [u32, u32]
    L.rl_owner_of.restype = u32
    L.rl_shard_create.argtypes = [vp, u32, u32, u32, u32, C.POINTER(vp)]
    L.rl_shard_destroy.argtypes = [vp]
    L.rl_shard_destroy.restype = None
    L.rl_shard_ipc_handle.argtypes = [vp, vp]
    L.rl_shard_connect_ipc.argtypes = [vp, vp]
    L.rl_shard_connect_ptrs.argtypes = [vp, vp]
    L.rl_shard_slab.argtypes = [vp]
    L.rl_shard_slab.restype = vp
    L.rl_shard_slab_bytes.argtypes = [vp]
    L.rl_shard_slab_bytes.restype = u64
    L.rl_shard_send.argtypes = [vp, u64, vp, vp]
    L.rl_shard_decide.argtypes = [vp]
    L.rl_shard_collect.argtypes = [vp, C.POINTER(vp)]
    L.rl_shard_step.argtypes = [vp, u64, vp, vp, C.POINTER(vp)]
    L.rl_shard_flush.argtypes = [vp]
    L.rl_shard_fence.argtypes = [vp]
    L.rl_shard_debug.argtypes = [vp, vp]
    L.rl_trace_dump.argtypes = [vp, u32, vp, vp, vp, vp]
    L.rl_shard_batch_create.argtypes = [vp, u32, u32, u32, u32, C.POINTER(vp)]
    L.rl_shard_batch_destroy.argtypes = [vp]
    L.rl_shard_batch_destroy.restype = None
    L.rl_shard_batch_slab.argtypes = [vp]
    L.rl_shard_batch_slab.restype = vp
    L.rl_shard_batch_engine.argtypes = [vp]
    L.rl_shard_batch_engine.restype = vp
    L.rl_shard_batch_ipc_handle.argtypes = [vp, vp]
    L.rl_shard_batch_connect_ipc.argtypes = [vp, vp]
    L.rl_shard_batch_connect_ptrs.argtypes = [vp, vp]
    L.rl_shard_batch_send.argtypes = [vp, u64, u64, vp, vp, vp, vp, i32, vp, i32]
    L.rl_shard_batch_decide.argtypes = [vp]
    L.rl_shard_batch_collect.argtypes = [vp, vp, vp, vp, vp]
    L.rl_shard_batch_step.argtypes = [vp, u64, u64, vp, vp, vp, vp, i32, vp, i32, vp, vp, vp, vp]
    L.rl_check_and_update_compact.argtypes = [vp, u64, vp, u64, i32, vp, vp]
    if path == _build.LIB_PATH:
        _lib = L
    return L


def _p(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    """One GPU-resident counter table (one per process / per GPU)."""

    def __init__(self, capacity_rows: int, cells_per_row: int = 1, max_batch: int = 65536,
                 max_counters: int = 0, regions: int = 0, device: int = 0, flags: int = 0,
                 max_counters_per_request: int = 0):
        """max_counters_per_request: counters one request may name (and limits one namespace may have on the
        record path); 0 = 16, up to 64.  Batches without a longer request run the same kernels either way."""
        self._lib = load_library()
        self._h = C.c_void_p()
        cfg = RlConfig(C.sizeof(RlConfig), device, capacity_rows, cells_per_row, max_batch, max_counters,
                       regions, flags, max_counters_per_request)
        st = self._lib.rl_engine_create(C.byref(cfg), C.byref(self._h))
        if st != RL_OK:
            msg = "rl_engine_create failed (no CUDA device? limitador_b200 has no CPU fallback)"
            if self._h:
                msg = self._lib.rl_last_error(self._h).decode() or msg
                self._lib.rl_engine_destroy(self._h)
                self._h = C.c_void_p()
            raise EngineError(st, msg)
        self.cells_per_row = cells_per_row
        self.max_batch = max_batch
        self.device = device
        self.max_counters_per_request = int(self._lib.rl_engine_max_counters_per_request(self._h))

    # -- lifecycle --
    def close(self):
        if getattr(self, "_h", None):
            self._lib.rl_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int):
        if st != RL_OK:
            raise EngineError(st, self._lib.rl_last_error(self._h).decode())

    def sync(self):
        self._check(self._lib.rl_sync(self._h))

    def fence(self):
        """Order every pipelined call issued so far before later work on the engine's stream."""
        self._check(self._lib.rl_fence(self._h))

    def set_stream(self, cuda_stream_ptr: int | None):
        self._check(self._lib.rl_engine_set_stream(self._h, C.c_void_p(cuda_stream_ptr or 0)))

    @property
    def stream(self) -> int:
        return int(self._lib.rl_engine_stream(self._h) or 0)

    def stats(self) -> dict:
        s = RlStats()
        self._check(self._lib.rl_get_stats(self._h, C.byref(s)))
        d = {f[0]: getattr(s, f[0]) for f in RlStats._fields_ if not f[0].startswith("_")}
        d["phase_cycles"] = list(d["phase_cycles"])
        return d

    def trace_dump(self, cap: int = 65536):
        """RL_FLAG_TRACE: list of (event name, is_end, seq, gpu_ns), in ring order; clears the ring."""
        names = {1: "front", 2: "main", 3: "xcount", 4: "xscatter", 5: "xwait", 6: "xreturn", 7: "xwaitv", 8: "xgather", 9: "hot"}
        ev = np.zeros(cap, dtype=np.uint32)
        seq = np.zeros(cap, dtype=np.uint32)
        ns = np.zeros(cap, dtype=np.uint64)
        cnt = C.c_uint32(0)
        self._check(self._lib.rl_trace_dump(self._h, cap, _p(ev), _p(seq), _p(ns), C.byref(cnt)))
        return [(names.get(int(ev[i]) & 0xFF, "?"), int(ev[i]) >> 8, int(seq[i]), int(ns[i])) for i in range(cnt.value)]

    def fence_call(self, age: int):
        """Order only the pipelined call issued `age` calls ago (0 = last, 1 = the one before)."""
        self._check(self._lib.rl_fence_call(self._h, age))

    def profile_begin(self):
        self._check(self._lib.rl_profile_begin(self._h))

    def profile_end(self):
        """(summed k_main device ms, k_main launches) since profile_begin."""
        ms, n = C.c_double(0), C.c_uint64(0)
        self._check(self._lib.rl_profile_end(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # -- limits --
    def limits_set(self, descs):
        """descs: iterable of (limit_id, ns_id, varset_id, qualified, max_value, window_us) or array."""
        if not isinstance(descs, np.ndarray):
            descs = np.array([tuple(d) for d in descs], dtype=LIMIT_DESC_DTYPE)
        descs = np.ascontiguousarray(descs, dtype=LIMIT_DESC_DTYPE)
        self._check(self._lib.rl_limits_set(self._h, _p(descs), len(descs)))

    def limits_delete(self, limit_ids):
        ids = np.ascontiguousarray(limit_ids, dtype=np.uint32)
        self._check(self._lib.rl_limits_delete(self._h, _p(ids), len(ids)))

    # -- host-memory (numpy) calls: synchronous --
    def check_and_update_records(self, recs, load_counters=False, stride=None, want_first=True):
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        n = len(recs)
        stride = stride or self.cells_per_row
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32) if want_first else None
        rem = np.zeros(n * stride, dtype=np.uint64) if load_counters else None
        ttl = np.zeros(n * stride, dtype=np.uint64) if load_counters else None
        self._check(self._lib.rl_check_and_update_records(
            self._h, n, _p(recs), int(load_counters), MEM_HOST, _p(lim), _p(fl), _p(rem), _p(ttl), stride))
        return lim, fl, rem, ttl

    def check_and_update_compact(self, recs16, now_us: int, want_first=True):
        """16-byte records, all stamped now_us (host memory, synchronous)."""
        recs16 = np.ascontiguousarray(recs16, dtype=RECORD16_DTYPE)
        n = len(recs16)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32) if want_first else None
        self._check(self._lib.rl_check_and_update_compact(self._h, n, _p(recs16), now_us, MEM_HOST, _p(lim), _p(fl)))
        return lim, fl

    def check_and_update_compact_ptr(self, n: int, recs_ptr: int, now_us: int, out_limited_ptr: int, mem: int,
                                     out_first_ptr: int = 0):
        self._check(self._lib.rl_check_and_update_compact(self._h, n, C.c_void_p(recs_ptr), now_us, mem,
                                                          C.c_void_p(out_limited_ptr), C.c_void_p(out_first_ptr or None)))

    def check_and_update_batch(self, off, ctrs, delta, now_us, load_counters=False):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        n = len(delta)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32)
        rem = np.zeros(len(ctrs), dtype=np.uint64)
        ttl = np.zeros(len(ctrs), dtype=np.uint64)
        self._check(self._lib.rl_check_and_update_batch(
            self._h, n, _p(off), _p(ctrs), _p(delta), _p(now_us), int(load_counters), MEM_HOST,
            _p(lim), _p(fl), _p(rem) if load_counters else None, _p(ttl) if load_counters else None))
        return lim, fl, rem, ttl

    def is_within_limits_batch(self, off, ctrs, delta, now_us):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        n = len(delta)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32)
        self._check(self._lib.rl_is_within_limits_batch(
            self._h, n, _p(off), _p(ctrs), _p(delta), _p(now_us), MEM_HOST, _p(lim), _p(fl)))
        return lim, fl

    def is_within_limits_records(self, recs):
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        n = len(recs)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32)
        self._check(self._lib.rl_is_within_limits_records(self._h, n, _p(recs), MEM_HOST, _p(lim), _p(fl)))
        return lim, fl

    def update_batch(self, off, ctrs, delta, now_us):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        self._check(self._lib.rl_update_batch(self._h, len(delta), _p(off), _p(ctrs), _p(delta), _p(now_us), MEM_HOST))

    def update_records(self, recs):
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        self._check(self._lib.rl_update_records(self._h, len(recs), _p(recs), MEM_HOST))

    # -- raw-pointer calls (device or pinned host memory; ints from tensor.data_ptr()) --
    def check_and_update_records_ptr(self, n, recs_ptr, out_limited_ptr, mem, load_counters=False,
                                     out_first_ptr=0, out_rem_ptr=0, out_ttl_ptr=0, stride=0):
        self._check(self._lib.rl_check_and_update_records(
            self._h, n, C.c_void_p(recs_ptr), int(load_counters), mem, C.c_void_p(out_limited_ptr),
            C.c_void_p(out_first_ptr or 0), C.c_void_p(out_rem_ptr or 0), C.c_void_p(out_ttl_ptr or 0),
            stride or self.cells_per_row))

    def bucket_by_owner_ptr(self, n, recs_ptr, world, out_recs_ptr, out_src_ptr):
        counts = np.zeros(world, dtype=np.uint64)
        self._check(self._lib.rl_bucket_by_owner(self._h, n, C.c_void_p(recs_ptr), world,
                                                 C.c_void_p(out_recs_ptr), C.c_void_p(out_src_ptr), _p(counts)))
        return counts

    def bucket_by_owner_padded_ptr(self, n, recs_ptr, world, slot_cap, out_recs_ptr, out_pos_ptr, overflow_ptr):
        self._check(self._lib.rl_bucket_by_owner_padded(self._h, n, C.c_void_p(recs_ptr), world, slot_cap,
                                                        C.c_void_p(out_recs_ptr), C.c_void_p(out_pos_ptr),
                                                        C.c_void_p(overflow_ptr)))

    def gather_u8_ptr(self, n, in_ptr, pos_ptr, out_ptr):
        self._check(self._lib.rl_gather_u8(self._h, n, C.c_void_p(in_ptr), C.c_void_p(pos_ptr), C.c_void_p(out_ptr)))

    def record_lane_put_ptr(self, n_slots, recs_ptr, lane_ptr):
        self._check(self._lib.rl_record_lane_put(self._h, n_slots, C.c_void_p(recs_ptr), C.c_void_p(lane_ptr)))

    def record_lane_gather_ptr(self, n, recs_ptr, pos_ptr, out_ptr):
        self._check(self._lib.rl_record_lane_gather(self._h, n, C.c_void_p(recs_ptr), C.c_void_p(pos_ptr),
                                                    C.c_void_p(out_ptr)))

    def unpermute_u8_ptr(self, n, in_ptr, src_ptr, out_ptr):
        self._check(self._lib.rl_unpermute_u8(self._h, n, C.c_void_p(in_ptr), C.c_void_p(src_ptr), C.c_void_p(out_ptr)))

    # -- maintenance --
    def _read_table(self, call, cap, device=False):
        """Count, then fetch (again if the table grew in between).  call(cap, five output pointers, count pointer) is
        rl_get_counters or rl_counters_export with every other argument bound; the first call fetches `cap` rows.
        Returns five numpy arrays (uint32, then uint64), or with device=True torch tensors on the engine's GPU
        (int32 / int64 holding the same bits)."""
        cnt = C.c_uint64(0)
        while True:
            if device:
                import torch
                dev = torch.device("cuda", self.device)
                arrs = [torch.empty(max(cap, 1), dtype=torch.int32, device=dev)] + [
                    torch.empty(max(cap, 1), dtype=torch.int64, device=dev) for _ in range(4)]
                ptrs = [C.c_void_p(a.data_ptr()) for a in arrs]
            else:
                arrs = [np.zeros(cap, dtype=np.uint32)] + [np.zeros(cap, dtype=np.uint64) for _ in range(4)]
                ptrs = [_p(a) for a in arrs]
            self._check(call(cap, *ptrs, C.byref(cnt)))
            if cnt.value <= cap:
                return tuple(a[:cnt.value] for a in arrs)
            cap = int(cnt.value)

    def get_counters(self, limit_ids, now_us, cap=1 << 20):
        """Sorted list of (limit_id, key_lo, key_hi, remaining, ttl_us) of every counter with ttl(now_us) > 0 in the
        namespaces of the given limits.  cap: rows of the first fetch."""
        ids = np.ascontiguousarray(limit_ids, dtype=np.uint32)
        cols = self._read_table(
            lambda cap, *out: self._lib.rl_get_counters(self._h, _p(ids), len(ids), now_us, cap, *out), cap)
        return sorted(zip(*(c.tolist() for c in cols)))

    def delete_counters(self, limit_ids):
        ids = np.ascontiguousarray(limit_ids, dtype=np.uint32)
        self._check(self._lib.rl_delete_counters(self._h, _p(ids), len(ids)))

    def clear(self):
        self._check(self._lib.rl_clear(self._h))

    def sweep(self, now_us) -> int:
        cnt = C.c_uint64(0)
        self._check(self._lib.rl_sweep(self._h, now_us, C.byref(cnt)))
        return cnt.value

    def compact(self, min_tombstone_pct: int = 25) -> dict:
        """rl_compact: rebuild the regions whose tombstones reach the given share of their rows -> rl_compact_stats."""
        st = (C.c_uint64 * 6)()
        self._check(self._lib.rl_compact(self._h, min_tombstone_pct, st))
        return dict(zip(("regions", "regions_rebuilt", "rows_live", "rows_tombstoned", "rows_moved", "rows_reclaimed"),
                        [int(x) for x in st]))

    def ns_metrics_enable(self, on: bool = True):
        """Per-namespace authorized_calls / authorized_hits / limited_calls reduced on the device behind every
        check_and_update_records / _compact call from now on."""
        self._check(self._lib.rl_ns_metrics_enable(self._h, int(on)))

    def ns_metrics_accumulate(self, recs, limited, first_limited=None):
        """Add an already decided batch (RECORD_DTYPE or RECORD16_DTYPE records + verdict bytes [+ limit ids named])."""
        recs = np.ascontiguousarray(recs)
        limited = np.ascontiguousarray(limited, dtype=np.uint8)
        fl = None if first_limited is None else np.ascontiguousarray(first_limited, dtype=np.uint32)
        self._check(self._lib.rl_ns_metrics_accumulate(self._h, len(recs), _p(recs), recs.dtype.itemsize, _p(limited),
                                                       None if fl is None else _p(fl), MEM_HOST))

    def ns_metrics_read(self, ns_cap: int, limits_cap: int = 0, reset: bool = False) -> dict:
        ac, ah, lc = (np.zeros(max(ns_cap, 1), dtype=np.uint64) for _ in range(3))
        bl = np.zeros(max(limits_cap, 1), dtype=np.uint64)
        dropped = C.c_uint64(0)
        self._check(self._lib.rl_ns_metrics_read(self._h, ns_cap, _p(ac), _p(ah), _p(lc), limits_cap, _p(bl), C.byref(dropped), int(reset)))
        return {"authorized_calls": ac[:ns_cap], "authorized_hits": ah[:ns_cap], "limited_calls": lc[:ns_cap],
                "limited_by_limit": bl[:limits_cap], "dropped": int(dropped.value)}

    def dump_arrays(self, cap=1 << 22):
        """export_counters() as numpy arrays, with a first fetch of `cap` rows."""
        return self._read_table(
            lambda cap, *out: self._lib.rl_counters_export(self._h, None, 0, 0, cap, MEM_HOST, *out), cap)

    def dump(self):
        """Sorted list of (limit_id, key_lo, key_hi, value, expiry_us) for every present counter."""
        lid, lo, hi, val, exp = self.dump_arrays()
        return sorted(zip(lid.tolist(), lo.tolist(), hi.tolist(), val.tolist(), exp.tolist()))

    # -- snapshots: restart, resize or re-shard without losing counters --
    def limits_get(self) -> np.ndarray:
        """Every registered limit (LIMIT_DESC_DTYPE), ascending id."""
        n = C.c_uint32(0)
        self._check(self._lib.rl_limits_get(self._h, 0, None, C.byref(n)))
        out = np.zeros(n.value, dtype=LIMIT_DESC_DTYPE)
        self._check(self._lib.rl_limits_get(self._h, len(out), _p(out), C.byref(n)))
        return out

    def export_counters(self, now_us: int = 0, ns_ids=None, device: bool = False):
        """rl_counters_export -> (limit_id, key_lo, key_hi, value, expiry_us).  numpy arrays (uint32, then uint64), or
        with device=True torch tensors on the engine's GPU (int32 / int64 holding the same bits), written there by the
        scan itself.  ns_ids=None: every namespace.  now_us > 0 leaves out the qualified counters rl_sweep(now_us)
        would drop."""
        ids = None if ns_ids is None else np.ascontiguousarray(ns_ids, dtype=np.uint32)
        n_ids = 0 if ids is None else len(ids)
        mem = MEM_DEVICE if device else MEM_HOST
        return self._read_table(
            lambda cap, *out: self._lib.rl_counters_export(self._h, _p(ids), n_ids, now_us, cap, mem, *out), 0, device)

    def import_counters(self, limit_id, key_lo, key_hi, value, expiry_us):
        """rl_counters_import: set each counter to exactly (value, expiry_us), all or nothing.  numpy arrays, or torch
        CUDA tensors on the engine's GPU (4- and 8-byte integers as export_counters(device=True) returns them)."""
        cols = (limit_id, key_lo, key_hi, value, expiry_us)
        n = len(limit_id)
        if any(len(c) != n for c in cols):
            raise ValueError("import_counters: the five arrays must have the same length")
        if all(hasattr(c, "is_cuda") and c.is_cuda for c in cols):
            import torch
            cols = [c.contiguous() for c in cols]
            if cols[0].element_size() != 4 or any(c.element_size() != 8 for c in cols[1:]):
                raise ValueError("import_counters: limit_id must be a 4-byte and the other columns 8-byte tensors")
            torch.cuda.current_stream(cols[0].device).synchronize()  # the engine's stream reads them next
            ptrs, mem = [C.c_void_p(c.data_ptr()) for c in cols], MEM_DEVICE
        elif any(hasattr(c, "is_cuda") and c.is_cuda for c in cols):
            raise ValueError("import_counters: either all five columns are CUDA tensors or none is")
        else:
            cols = [np.ascontiguousarray(cols[0], dtype=np.uint32)] + [np.ascontiguousarray(c, dtype=np.uint64) for c in cols[1:]]
            ptrs, mem = [_p(c) for c in cols], MEM_HOST
        self._check(self._lib.rl_counters_import(self._h, n, *ptrs, mem))

    def _snapshot_arrays(self, now_us: int = 0) -> dict:
        """The arrays of a save_counters file, in file order: the limits (rl_limits_get) and every counter
        (export_counters(now_us)) sorted by (limit_id, key) so that the same table always gives the same file."""
        limits = self.limits_get()
        lid, lo, hi, val, exp = self.export_counters(now_us)
        order = np.lexsort((hi, lo, lid))
        return dict(version=np.uint32(SNAPSHOT_VERSION), limits=limits, limit_id=lid[order], key_lo=lo[order],
                    key_hi=hi[order], value=val[order], expiry_us=exp[order])

    def save_counters(self, path: str, now_us: int = 0):
        """Write the limits and every counter (_snapshot_arrays(now_us)) to one .npz file at `path`."""
        with open(path, "wb") as f:
            np.savez(f, **self._snapshot_arrays(now_us))

    def load_counters(self, path: str):
        """Import a save_counters file.  Limit ids are interned by the caller: this engine must have registered the same
        limits under the same ids (the same configuration, registered in the same order) before the call.  Refused
        before any counter changes if a limit of the file is registered here with another namespace, window or
        qualified flag (a limit's identity, limit.rs:177-214; max_value may differ, as after update_limit)."""
        with np.load(path) as z:
            if int(z["version"]) != SNAPSHOT_VERSION:
                raise ValueError(f"{path}: snapshot format {int(z['version'])}, this build reads {SNAPSHOT_VERSION}")
            limits = z["limits"]
            cols = [z[k] for k in ("limit_id", "key_lo", "key_hi", "value", "expiry_us")]
        self.import_snapshot(limits, cols, path)

    def import_snapshot(self, limits, cols, source: str = "snapshot"):
        """load_counters on arrays: the limits the counters were saved under (LIMIT_DESC_DTYPE) and the five counter
        columns.  Refused before any counter changes if a limit the counters use is registered here with another
        namespace, window or qualified flag."""
        mine = {int(d["limit_id"]): d for d in self.limits_get()}
        used = set(np.unique(cols[0]).tolist())
        bad = sorted(int(d["limit_id"]) for d in limits if int(d["limit_id"]) in used and int(d["limit_id"]) in mine
                     and any(int(d[k]) != int(mine[int(d["limit_id"])][k]) for k in ("ns_id", "window_us", "qualified")))
        if bad:
            raise ValueError(f"{source}: limits {bad} are registered here with another namespace, window or qualified flag")
        self.import_counters(*cols)

    # -- change tracking: what a journal on disk drains (limitador_b200.journal) --
    def track_changes(self, on: bool = True):
        """rl_counters_track: keep a device shadow of the table (one more copy of it in HBM) so that drain_changes can
        list what changed; the next drain is full.  on=False frees the shadow."""
        self._check(self._lib.rl_counters_track(self._h, int(on)))

    def drain_changes(self, cap: int = 1 << 16):
        """rl_counters_drain -> (full, (limit_id, key_lo, key_hi, value, expiry_us)).  full: every counter, exactly
        export_counters().  Otherwise the counters changed since the last drain, an absent one as value = expiry = 0
        (apply those before the others).  cap: rows of the first fetch; a drain that does not fit is fetched again,
        whole.  Serialise with the decision calls."""
        full = C.c_int(0)
        cols = self._read_table(
            lambda cap, *out: self._lib.rl_counters_drain(self._h, cap, MEM_HOST, *out, C.byref(full)), cap)
        return bool(full.value), cols


def owner_of(ns_id: int, world: int) -> int:
    return int(load_library().rl_owner_of(ns_id, world))


class Front:
    """The batching front: blocking, thread-safe single-request calls over one Engine."""

    def __init__(self, engine: Engine, max_batch: int = 1024, max_delay_us: int = 50):
        self._lib = load_library()
        self._engine = engine  # keep alive
        self._h = C.c_void_p()
        st = self._lib.rl_front_create(engine._h, max_batch, max_delay_us, C.byref(self._h))
        if st != RL_OK:
            raise EngineError(st, "rl_front_create failed")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rl_front_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check_and_update(self, ctrs, delta: int, now_us: int = 0, load_counters: bool = False):
        """ctrs: COUNTER_DTYPE array.  Returns (limited, first_limited_id|None, seq, remaining, ttl)."""
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        m = len(ctrs)
        lim, first, seq = C.c_uint8(0), C.c_uint32(NONE), C.c_uint64(0)
        rem = np.zeros(max(m, 1), dtype=np.uint64)
        ttl = np.zeros(max(m, 1), dtype=np.uint64)
        st = self._lib.rl_front_check_and_update(self._h, _p(ctrs), m, delta, now_us, int(load_counters),
                                                 C.addressof(lim), C.addressof(first), _p(rem), _p(ttl),
                                                 C.addressof(seq))
        if st != RL_OK:
            raise EngineError(st, self._lib.rl_last_error(self._engine._h).decode())
        return bool(lim.value), (None if first.value == NONE else first.value), seq.value, rem[:m], ttl[:m]

    def stats(self):
        b, r = C.c_uint64(0), C.c_uint64(0)
        self._lib.rl_front_stats(self._h, C.addressof(b), C.addressof(r))
        return {"batches": b.value, "requests": r.value}


class Shard:
    """Namespace-sharded peer exchange of one rank (include/rl_engine.h: rl_shard_*): records travel to
    their owner GPU and verdicts back by direct NVLink stores into IPC-mapped slabs, no NCCL on the data
    path.  All pointers are device pointers (ints); every call only enqueues."""

    def __init__(self, engine: "Engine", rank: int, world: int, cap: int, lag: int = 2):
        self._lib = engine._lib
        self._eng = engine
        self._h = C.c_void_p()
        engine._check(self._lib.rl_shard_create(engine._h, rank, world, cap, lag, C.byref(self._h)))
        self.rank, self.world, self.cap, self.lag = rank, world, cap, lag

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rl_shard_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def slab(self) -> int:
        return int(self._lib.rl_shard_slab(self._h) or 0)

    @property
    def slab_bytes(self) -> int:
        return int(self._lib.rl_shard_slab_bytes(self._h))

    def ipc_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._eng._check(self._lib.rl_shard_ipc_handle(self._h, buf))
        return buf.raw

    def connect_ipc(self, handles: bytes):
        assert len(handles) == 64 * self.world
        self._eng._check(self._lib.rl_shard_connect_ipc(self._h, C.c_char_p(handles)))

    def connect_ptrs(self, slabs):
        arr = (C.c_void_p * self.world)(*[C.c_void_p(int(p)) for p in slabs])
        self._eng._check(self._lib.rl_shard_connect_ptrs(self._h, arr))

    def send(self, n: int, recs_ptr: int, out_ptr: int):
        self._eng._check(self._lib.rl_shard_send(self._h, n, C.c_void_p(recs_ptr), C.c_void_p(out_ptr)))

    def decide(self):
        self._eng._check(self._lib.rl_shard_decide(self._h))

    def collect(self):
        """Returns the device pointer of the out_limited buffer whose delivery was enqueued, or None."""
        done = C.c_void_p()
        self._eng._check(self._lib.rl_shard_collect(self._h, C.byref(done)))
        return done.value

    def step(self, n: int, recs_ptr: int, out_ptr: int):
        done = C.c_void_p()
        self._eng._check(self._lib.rl_shard_step(self._h, n, C.c_void_p(recs_ptr), C.c_void_p(out_ptr), C.byref(done)))
        return done.value

    def flush(self):
        self._eng._check(self._lib.rl_shard_flush(self._h))

    def fence(self):
        """Order the engine's stream after every verdict delivery enqueued so far (no host blocking)."""
        self._eng._check(self._lib.rl_shard_fence(self._h))

    def debug(self):
        """{'ctl': [buf][peer] -> (fill, record flag, verdict flag), 'sent', 'decided', 'collected'} of this rank."""
        depth = self.lag + 2
        out = np.zeros(depth * self.world * 4 + 3, dtype=np.uint32)
        self._lib.rl_shard_debug(self._h, _p(out))
        ctl = out[:-3].reshape(depth, self.world, 4)[:, :, :3].tolist()
        return {"ctl": ctl, "sent": int(out[-3]), "decided": int(out[-2]), "collected": int(out[-1])}


class ShardBatch:
    """The general (CSR) form of the namespace-sharded peer exchange of one rank (include/rl_engine.h: rl_shard_batch_*):
    served requests travel to the GPU that owns their namespace, outputs come back, one step at a time.  Attach it to an
    RlsService (RlsService.attach_shard) to serve RLS and HTTP batches on a sharded store; send / decide / collect take
    device pointers (ints) for drivers of their own."""

    CHECK_AND_UPDATE, IS_WITHIN, UPDATE = 0, 1, 2

    def __init__(self, engine: "Engine", rank: int, world: int, cap_requests: int, cap_counters: int):
        self._lib = engine._lib
        self._eng = engine
        self._h = C.c_void_p()
        engine._check(self._lib.rl_shard_batch_create(engine._h, rank, world, cap_requests, cap_counters, C.byref(self._h)))
        self.rank, self.world, self.cap_requests, self.cap_counters = rank, world, cap_requests, cap_counters

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rl_shard_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def slab(self) -> int:
        return int(self._lib.rl_shard_batch_slab(self._h) or 0)

    def ipc_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._eng._check(self._lib.rl_shard_batch_ipc_handle(self._h, buf))
        return buf.raw

    def connect_ipc(self, handles: bytes):
        assert len(handles) == 64 * self.world
        self._eng._check(self._lib.rl_shard_batch_connect_ipc(self._h, C.c_char_p(handles)))

    def connect_ptrs(self, slabs):
        arr = (C.c_void_p * self.world)(*[C.c_void_p(int(p)) for p in slabs])
        self._eng._check(self._lib.rl_shard_batch_connect_ptrs(self._h, arr))

    def send(self, n: int, n_ctr: int, off_ptr: int, ctrs_ptr: int, delta_ptr: int, now_ptr: int, op: int,
             load_ptr: int = 0, load_all: bool = False):
        v = C.c_void_p
        self._eng._check(self._lib.rl_shard_batch_send(self._h, n, n_ctr, v(off_ptr), v(ctrs_ptr), v(delta_ptr), v(now_ptr), op,
                                                       v(load_ptr or 0), int(load_all)))

    def decide(self):
        """Decide this rank's inbox.  Raises on a source with other limits (after the outputs went back) and on a failed
        engine call (its requests were answered with error verdicts)."""
        self._eng._check(self._lib.rl_shard_batch_decide(self._h))

    def step(self, n: int, n_ctr: int, off_ptr: int, ctrs_ptr: int, delta_ptr: int, now_ptr: int, op: int, limited_ptr: int,
             first_ptr: int = 0, remaining_ptr: int = 0, ttl_ptr: int = 0, load_ptr: int = 0, load_all: bool = False):
        """send + decide + collect: the one call of a one-process-per-GPU deployment."""
        v = C.c_void_p
        self._eng._check(self._lib.rl_shard_batch_step(self._h, n, n_ctr, v(off_ptr), v(ctrs_ptr), v(delta_ptr), v(now_ptr), op,
                                                       v(load_ptr or 0), int(load_all), v(limited_ptr), v(first_ptr or 0),
                                                       v(remaining_ptr or 0), v(ttl_ptr or 0)))

    def collect(self, limited_ptr: int, first_ptr: int = 0, remaining_ptr: int = 0, ttl_ptr: int = 0):
        v = C.c_void_p
        self._eng._check(self._lib.rl_shard_batch_collect(self._h, v(limited_ptr), v(first_ptr or 0), v(remaining_ptr or 0),
                                                          v(ttl_ptr or 0)))
