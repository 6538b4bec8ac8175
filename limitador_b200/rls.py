"""ctypes binding of the Envoy RLS v3 wire surface (include/rl_rls.h, csrc/rl_rls.cpp).

`RlsService` serves batches of `envoy.service.ratelimit.v3.RateLimitRequest` wire messages:
decode + counters_that_apply on the engine's GPU, ONE engine call for the whole batch, then
`RateLimitResponse` bytes on a pool of CPU workers (envoy_rls/server.rs:91-208, kuadrant_service.rs:27-186).
`plan`/`finish` are the CPU stages on their own (drivable without a GPU), `plan_device` is the GPU plan on its
own; `serve` runs plan_device -> engine -> finish.
`encode_request` / `decode_response` are small pure-Python helpers for callers and tests (the tests
cross-check them against the protobuf runtime).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import engine as _eng
from . import matcher as _m

CODE_UNKNOWN, CODE_OK, CODE_OVER_LIMIT = 0, 1, 2
HEADERS_NONE, HEADERS_DRAFT_VERSION_03 = 0, 1
SHOULD_RATE_LIMIT, CHECK_RATE_LIMIT, REPORT = 0, 1, 2
GRPC_OK, GRPC_INTERNAL, GRPC_UNAVAILABLE = 0, 13, 14
NO_STORE = 0xFFFFFFFF

RLS_SYMBOLS = (
    "rl_rls_attach_shard", "rl_rls_serve_sharded", "rl_rls_send", "rl_rls_decide", "rl_rls_collect",
    "rl_rls_decode_request", "rl_rls_encode_response", "rl_rls_create", "rl_rls_destroy", "rl_rls_last_error",
    "rl_rls_plan", "rl_rls_plan_view", "rl_rls_finish", "rl_rls_responses", "rl_rls_serve", "rl_rls_metrics_render",
    "rl_rls_last_timings", "rl_rls_plan_device", "rl_rls_keep_counter_vars", "rl_rls_counter_vars_stats",
    "rl_rls_counter_vars_gc", "rl_rls_counter_vars_export", "rl_rls_counter_vars_import", "rl_rls_configure",
    "rl_rls_config_status", "rl_rls_counter_vars_drain",
)

ENTRY_DTYPE = np.dtype([("descriptor", "<u4"), ("key_off", "<u4"), ("key_len", "<u4"), ("val_off", "<u4"), ("val_len", "<u4")])


class RlsRequest(C.Structure):
    _fields_ = [("domain_off", C.c_uint32), ("domain_len", C.c_uint32), ("hits_addend", C.c_uint32),
                ("n_descriptors", C.c_uint32), ("n_entries", C.c_uint32)]


class RlsError(RuntimeError):
    pass


class ConfigureError(RlsError):
    """A configuration refused by RlsService.configure_with; `index` is the refused entry (None when the engine's delete
    call failed).  Nothing changed."""

    def __init__(self, msg: str, index: Optional[int]):
        super().__init__(msg)
        self.index = index


class LimitSpec(C.Structure):
    _fields_ = [("ns", C.c_char_p), ("max_value", C.c_uint64), ("seconds", C.c_uint64),
                ("conditions", C.POINTER(C.c_char_p)), ("n_cond", C.c_uint32), ("_pad0", C.c_uint32),
                ("variables", C.POINTER(C.c_char_p)), ("n_var", C.c_uint32), ("_pad1", C.c_uint32),
                ("name", C.c_char_p), ("id", C.c_char_p)]


class ConfigureReport(C.Structure):
    _fields_ = [("kept", C.c_uint32), ("added", C.c_uint32), ("updated", C.c_uint32), ("deleted", C.c_uint32),
                ("first_refused", C.c_uint32), ("_pad", C.c_uint32)]


def _field(limit, key):
    return limit[key] if isinstance(limit, dict) else getattr(limit, key)


def _lib():
    L = _m._lib()
    if getattr(L, "_rl_rls_ready", False):
        return L
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.rl_rls_decode_request.argtypes = [vp, u64, C.POINTER(RlsRequest), vp, u32]
    L.rl_rls_encode_response.argtypes = [u32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), u32, vp, u64, C.POINTER(u64)]
    L.rl_rls_create.argtypes = [vp, vp, i32, u32, i32, C.POINTER(vp)]
    L.rl_rls_destroy.argtypes = [vp]
    L.rl_rls_destroy.restype = None
    L.rl_rls_last_error.argtypes = [vp]
    L.rl_rls_last_error.restype = C.c_char_p
    L.rl_rls_plan.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_rls_plan_device.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_rls_plan_view.argtypes = [vp, C.POINTER(u64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                   C.POINTER(i32), C.POINTER(vp)]
    L.rl_rls_finish.argtypes = [vp, i32, vp, vp, vp, vp]
    L.rl_rls_responses.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.rl_rls_serve.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_rls_metrics_render.argtypes = [vp, vp, u64, C.POINTER(u64)]
    L.rl_rls_last_timings.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.rl_rls_keep_counter_vars.argtypes = [vp, u64, u64]
    L.rl_rls_counter_vars_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.rl_rls_counter_vars_gc.argtypes = [vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.rl_rls_counter_vars_export.argtypes = [vp, vp, u32, u64, u64, u64, vp, vp, vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
    L.rl_rls_counter_vars_import.argtypes = [vp, u64, vp, vp, vp, vp, vp, C.POINTER(u64)]
    L.rl_rls_counter_vars_drain.argtypes = [vp, u64, u64, vp, vp, vp, vp, vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(i32)]
    L.rl_rls_configure.argtypes = [vp, C.POINTER(LimitSpec), u32, i32, C.POINTER(ConfigureReport)]
    L.rl_rls_config_status.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.rl_rls_attach_shard.argtypes = [vp, vp]
    L.rl_rls_serve_sharded.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_rls_send.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_rls_decide.argtypes = [vp]
    L.rl_rls_collect.argtypes = [vp]
    L._rl_rls_ready = True
    return L


# ---- pure-Python wire helpers ------------------------------------------------------------------------------------
def _varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _len_field(tag: int, payload: bytes) -> bytes:
    return _varint((tag << 3) | 2) + _varint(len(payload)) + payload


def encode_request(domain: str, descriptors: Sequence[Sequence[Tuple[str, str]]], hits_addend: int = 0) -> bytes:
    """RateLimitRequest{domain = 1, descriptors = 2 (entries = 1 {key = 1, value = 2}), hits_addend = 3}; proto3:
    empty strings and a zero hits_addend are not written."""
    out = bytearray()
    if domain:
        out += _len_field(1, domain.encode())
    for d in descriptors:
        body = bytearray()
        for k, v in d:
            e = (_len_field(1, k.encode()) if k else b"") + (_len_field(2, v.encode()) if v else b"")
            body += _len_field(1, e)
        out += _len_field(2, bytes(body))
    if hits_addend:
        out += _varint(3 << 3) + _varint(hits_addend)
    return bytes(out)


def pack_requests(msgs: Sequence[bytes]) -> Tuple[np.ndarray, np.ndarray]:
    """-> (buf uint8, off uint64[n+1]): the batch layout rl_rls_plan / rl_rls_serve take."""
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    if msgs:
        off[1:] = np.cumsum([len(m) for m in msgs], dtype=np.uint64)
    buf = np.frombuffer(b"".join(msgs), dtype=np.uint8) if msgs else np.zeros(0, dtype=np.uint8)
    return np.ascontiguousarray(buf), off


def _read_varint(b: bytes, p: int) -> Tuple[int, int]:
    v = s = 0
    while True:
        c = b[p]
        p += 1
        v |= (c & 0x7F) << s
        s += 7
        if not c & 0x80:
            return v, p


def decode_response(b: bytes) -> Tuple[int, List[Tuple[str, str]]]:
    """RateLimitResponse bytes -> (overall_code, response_headers_to_add as (key, value) pairs)."""
    code, headers, p = 0, [], 0
    while p < len(b):
        key, p = _read_varint(b, p)
        tag, wt = key >> 3, key & 7
        if wt == 0:
            v, p = _read_varint(b, p)
            if tag == 1:
                code = v
        elif wt == 2:
            n, p = _read_varint(b, p)
            body, p = b[p:p + n], p + n
            if tag == 3:
                k = v = ""
                q = 0
                while q < len(body):
                    kk, q = _read_varint(body, q)
                    ln, q = _read_varint(body, q)
                    s, q = body[q:q + ln].decode(), q + ln
                    if kk >> 3 == 1:
                        k = s
                    elif kk >> 3 == 2:
                        v = s
                headers.append((k, v))
        else:
            raise ValueError(f"unexpected wire type {wt}")
    return code, headers


def decode_request(msg: bytes, cap_entries: int = 64):
    """The native decoder on one message -> (domain, descriptors as lists of (key, value), hits_addend as on the wire);
    raises RlsError for a message prost would refuse."""
    L = _lib()
    arr = np.frombuffer(msg, dtype=np.uint8) if msg else np.zeros(1, dtype=np.uint8)
    q = RlsRequest()
    ent = np.zeros(max(cap_entries, 1), dtype=ENTRY_DTYPE)
    if L.rl_rls_decode_request(arr.ctypes.data, len(msg), C.byref(q), ent.ctypes.data, cap_entries) != 0:
        raise RlsError("malformed RateLimitRequest")
    if q.n_entries > cap_entries:
        return decode_request(msg, q.n_entries)
    descs: List[List[Tuple[str, str]]] = [[] for _ in range(q.n_descriptors)]
    for e in ent[:q.n_entries]:
        descs[int(e["descriptor"])].append((msg[int(e["key_off"]):int(e["key_off"]) + int(e["key_len"])].decode(),
                                            msg[int(e["val_off"]):int(e["val_off"]) + int(e["val_len"])].decode()))
    return msg[q.domain_off:q.domain_off + q.domain_len].decode(), descs, q.hits_addend


def encode_response(code: int, headers: Sequence[Tuple[str, str]] = ()) -> bytes:
    L = _lib()
    ks = _m._strs([k for k, _ in headers])
    vs = _m._strs([v for _, v in headers])
    need = C.c_uint64()
    buf = np.zeros(64 + sum(len(k) + len(v) + 16 for k, v in headers), dtype=np.uint8)
    if L.rl_rls_encode_response(code, ks, vs, len(headers), buf.ctypes.data, len(buf), C.byref(need)) != 0:
        raise RlsError("rl_rls_encode_response failed")
    return buf[:need.value].tobytes()


def _view(ptr, n, dtype):
    if not ptr or n == 0:
        return np.zeros(0, dtype=dtype)
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(n * np.dtype(dtype).itemsize,)).view(dtype)


def _batch_call(svc, fn, method: int, buf, off, now_us: int) -> int:
    """fn(handle, method, n, buf, off, now_us), a plan or serve call, on svc's service; svc keeps the batch's arrays
    alive -> n."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    svc._keep = (buf, off)
    svc._check(fn(svc._h, method, len(off) - 1, buf.ctypes.data if len(buf) else None, off.ctypes.data, now_us))
    return len(off) - 1


def _read_plan(view_fn, h, check, n: int, load_per_request: bool):
    """The planned batch of n requests through rl_rls_plan_view / rl_http_plan_view -> dict(n_store, ctr_off, ctrs, delta,
    now_us, load_counters, store_index), copies of its arrays.  load_counters is one bool for the batch, or with
    load_per_request one flag per store request."""
    ns = C.c_uint64()
    p_off, p_ctr, p_delta, p_now, p_idx = (C.c_void_p() for _ in range(5))
    lc = C.c_void_p() if load_per_request else C.c_int()
    check(view_fn(h, C.byref(ns), C.byref(p_off), C.byref(p_ctr), C.byref(p_delta), C.byref(p_now), C.byref(lc), C.byref(p_idx)))
    m = ns.value
    ctr_off = _view(p_off.value, m + 1, np.uint32).copy()
    return {
        "n_store": m, "ctr_off": ctr_off,
        "ctrs": _view(p_ctr.value, int(ctr_off[-1]) if m else 0, _eng.COUNTER_DTYPE).copy(),
        "delta": _view(p_delta.value, m, np.uint64).copy(), "now_us": _view(p_now.value, m, np.uint64).copy(),
        "load_counters": _view(lc.value, m, np.uint8).copy() if load_per_request else bool(lc.value),
        "store_index": _view(p_idx.value, n, np.uint32).copy(),
    }


def _ptr(a, dtype, keep: list):
    """a's address as a contiguous dtype array for a C call (None for None or an empty array); the array is appended to
    keep, which the caller holds until the call returns."""
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=dtype)
    keep.append(a)
    return a.ctypes.data if len(a) else None


class RlsService:
    """One RLS front over a Matcher and (optionally) an Engine.  Not thread-safe: one batch at a time."""

    def __init__(self, matcher: _m.Matcher, engine: Optional[_eng.Engine] = None, headers: int = HEADERS_NONE,
                 threads: int = 0, use_limit_name_label: bool = False):
        self._lib = _lib()
        self._matcher, self._engine = matcher, engine  # keep them alive
        h = C.c_void_p()
        eh = engine._h if engine is not None else None
        if self._lib.rl_rls_create(matcher._h, eh, headers, threads, int(use_limit_name_label), C.byref(h)) != 0:
            raise RlsError("rl_rls_create failed")
        self._h = h

    def close(self):
        if self._h:
            self._lib.rl_rls_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status):
        if status != 0:
            raise RlsError(self._lib.rl_rls_last_error(self._h).decode())

    def plan(self, method: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Stage 1 on the CPU workers -> dict(n_store, ctr_off, ctrs, delta, now_us, load_counters, store_index): copies of
        the store call."""
        return self._plan(self._lib.rl_rls_plan, method, buf, off, now_us)

    def plan_device(self, method: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Stage 1 on the engine's device (the service needs an engine); the same dict as `plan`, array for array."""
        return self._plan(self._lib.rl_rls_plan_device, method, buf, off, now_us)

    def _plan(self, fn, method, buf, off, now_us):
        n = _batch_call(self, fn, method, buf, off, now_us)
        return _read_plan(self._lib.rl_rls_plan_view, self._h, self._check, n, False)

    def finish(self, limited=None, first_limited=None, remaining=None, ttl_us=None, store_status: int = 0):
        keep = []
        self._check(self._lib.rl_rls_finish(self._h, store_status, _ptr(limited, np.uint8, keep),
                                            _ptr(first_limited, np.uint32, keep), _ptr(remaining, np.uint64, keep),
                                            _ptr(ttl_us, np.uint64, keep)))
        return self.responses()

    def attach_shard(self, shard: Optional[_eng.ShardBatch]):
        """Serve on a namespace-sharded store: from now on `serve` ships every store request to the rank that owns its
        namespace (every rank runs its own service with the same limits and issues the same serve calls).  None
        detaches."""
        self._check(self._lib.rl_rls_attach_shard(self._h, shard._h if shard is not None else None))
        self._shard = shard  # keep it alive

    def send(self, method: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Sharded step, phase 1: plan on the device and send the store requests to their owners.  A one-process driver of
        several ranks calls every rank's send, then every decide, then every collect."""
        _batch_call(self, self._lib.rl_rls_send, method, buf, off, now_us)

    def decide(self):
        """Sharded step, phase 2: decide this rank's inbox."""
        self._check(self._lib.rl_rls_decide(self._h))

    def collect(self):
        """Sharded step, phase 3: collect this rank's outputs and finish its responses -> responses()."""
        self._check(self._lib.rl_rls_collect(self._h))
        return self.responses()

    def responses(self) -> List[Tuple[int, bytes]]:
        """-> [(grpc_status, response bytes)] of the last finished batch."""
        pb, po, pg, pc = (C.c_void_p() for _ in range(4))
        self._check(self._lib.rl_rls_responses(self._h, C.byref(pb), C.byref(po), C.byref(pg), C.byref(pc)))
        n = len(self._keep[1]) - 1
        off = _view(po.value, n + 1, np.uint64)
        raw = _view(pb.value, int(off[-1]) if n else 0, np.uint8).tobytes()
        grpc = _view(pg.value, n, np.uint8)
        return [(int(grpc[i]), raw[int(off[i]):int(off[i + 1])]) for i in range(n)]

    def codes(self) -> np.ndarray:
        """overall_code of every response of the last finished batch (0 where the gRPC status is not OK)."""
        pc = C.c_void_p()
        self._check(self._lib.rl_rls_responses(self._h, None, None, None, C.byref(pc)))
        return _view(pc.value, len(self._keep[1]) - 1, np.uint8).copy()

    def grpc_status(self) -> np.ndarray:
        pg = C.c_void_p()
        self._check(self._lib.rl_rls_responses(self._h, None, None, C.byref(pg), None))
        return _view(pg.value, len(self._keep[1]) - 1, np.uint8).copy()

    def serve(self, method: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """plan -> ONE engine call -> finish.  Needs an engine (no CPU store exists in the product)."""
        _batch_call(self, self._lib.rl_rls_serve, method, buf, off, now_us)

    def timings(self) -> Dict[str, float]:
        a, b, c = C.c_double(), C.c_double(), C.c_double()
        self._lib.rl_rls_last_timings(self._h, C.byref(a), C.byref(b), C.byref(c))
        return {"plan_us": a.value, "store_us": b.value, "finish_us": c.value}

    def keep_counter_vars(self, max_keys: int, arena_bytes: int):
        """Record the variable values behind the counter keys of every device plan (GET /counters needs them) in a
        dictionary of max_keys slots and arena_bytes of values on the engine's device; (0, 0) turns it off."""
        self._check(self._lib.rl_rls_keep_counter_vars(self._h, max_keys, arena_bytes))

    def counter_vars_stats(self) -> Dict[str, int]:
        k, a, d = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._check(self._lib.rl_rls_counter_vars_stats(self._h, C.byref(k), C.byref(a), C.byref(d)))
        return {"keys": k.value, "arena_used": a.value, "dropped": d.value}

    def counter_vars_gc(self, now_us: int = 0) -> Dict[str, int]:
        """Keep the entries the engine's present counters reference (0 = wall clock) -> {kept, freed}."""
        k, f = C.c_uint64(), C.c_uint64()
        self._check(self._lib.rl_rls_counter_vars_gc(self._h, now_us, C.byref(k), C.byref(f)))
        return {"kept": k.value, "freed": f.value}

    # -- snapshots: the dictionary beside the counters --
    def export_counter_vars(self, now_us: int = 0, ns_ids=None):
        """The dictionary entries the counters Engine.export_counters(now_us, ns_ids) lists refer to -> numpy arrays
        (varset uint32, key_lo, key_hi, blob_off [n + 1], blobs uint8): entry i's values are blobs[blob_off[i] ..
        blob_off[i + 1]), a u32 little-endian length then the bytes per variable, in no particular order.  Empty while
        keeping is off."""
        ids = None if ns_ids is None else np.ascontiguousarray(ns_ids, dtype=np.uint32)
        n_ids = 0 if ids is None else len(ids)
        p_ids = None if ids is None else (ids.ctypes.data if n_ids else np.zeros(1, np.uint32).ctypes.data)
        cnt, nb, cap, bcap = C.c_uint64(0), C.c_uint64(0), 0, 0
        while True:  # count, then fetch (again if the dictionary grew in between)
            vs, lo, hi = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint64), np.zeros(max(cap, 1), np.uint64)
            off, blobs = np.zeros(cap + 1, np.uint64), np.zeros(max(bcap, 1), np.uint8)
            self._check(self._lib.rl_rls_counter_vars_export(self._h, p_ids, n_ids, now_us, cap, bcap, vs.ctypes.data,
                                                             lo.ctypes.data, hi.ctypes.data, off.ctypes.data,
                                                             blobs.ctypes.data, C.byref(cnt), C.byref(nb)))
            if cap and cnt.value <= cap and nb.value <= bcap:
                n = cnt.value
                return vs[:n], lo[:n], hi[:n], off[:n + 1], blobs[:int(off[n])]
            if cnt.value == 0:
                return vs[:0], lo[:0], hi[:0], np.zeros(1, np.uint64), blobs[:0]
            cap, bcap = int(cnt.value), int(nb.value)

    def import_counter_vars(self, varset, key_lo, key_hi, blob_off, blobs) -> int:
        """Add dictionary entries (the arrays export_counter_vars returns), all or nothing -> the keys added (keys the
        dictionary holds already are skipped).  Every entry must match a qualified limit of the matcher and digest to its
        key; a refused call raises RlsError naming the first refused entry and changes nothing."""
        vs = np.ascontiguousarray(varset, dtype=np.uint32)
        lo, hi = np.ascontiguousarray(key_lo, dtype=np.uint64), np.ascontiguousarray(key_hi, dtype=np.uint64)
        off, b = np.ascontiguousarray(blob_off, dtype=np.uint64), np.ascontiguousarray(blobs, dtype=np.uint8)
        n = len(vs)
        if len(lo) != n or len(hi) != n or len(off) != n + 1:
            raise ValueError("import_counter_vars: varset, key_lo and key_hi need n entries and blob_off n + 1")
        if n and int(off.max()) > len(b):
            raise ValueError("import_counter_vars: blob_off points past blobs")
        added = C.c_uint64(0)
        self._check(self._lib.rl_rls_counter_vars_import(self._h, n, vs.ctypes.data, lo.ctypes.data, hi.ctypes.data,
                                                         off.ctypes.data, b.ctypes.data if len(b) else None, C.byref(added)))
        return added.value

    def drain_counter_vars(self):
        """rl_rls_counter_vars_drain -> (full, (varset, key_lo, key_hi, blob_off, blobs)): the dictionary entries recorded
        since the last drain, in export_counter_vars' layout.  full = True (and no entries) after keep_counter_vars,
        counter_vars_gc or import_counter_vars: take export_counter_vars() then.  Serialise with serve."""
        cnt, nb, full, cap, bcap = C.c_uint64(0), C.c_uint64(0), C.c_int(0), 0, 0
        while True:  # count, then fetch: a drain that does not fit is not consumed
            vs, lo, hi = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint64), np.zeros(max(cap, 1), np.uint64)
            off, blobs = np.zeros(cap + 1, np.uint64), np.zeros(max(bcap, 1), np.uint8)
            self._check(self._lib.rl_rls_counter_vars_drain(self._h, cap, bcap, vs.ctypes.data, lo.ctypes.data, hi.ctypes.data,
                                                            off.ctypes.data, blobs.ctypes.data, C.byref(cnt), C.byref(nb),
                                                            C.byref(full)))
            if full.value or (cnt.value <= cap and nb.value <= bcap):
                n = 0 if full.value else cnt.value
                return bool(full.value), (vs[:n], lo[:n], hi[:n], off[:n + 1], blobs[:int(off[n])])
            cap, bcap = int(cnt.value), int(nb.value)

    def save_counters(self, path: str, now_us: int = 0):
        """Engine.save_counters(path, now_us) of the service's engine, plus the dictionary entries those counters refer
        to (cv_varset, cv_key_lo, cv_key_hi, cv_blob_off, cv_blobs), sorted by (varset, key) so that the same state
        always gives the same file.  Engine.load_counters reads the file as well (it ignores the cv_ arrays)."""
        vs, lo, hi, off, blobs = self.export_counter_vars(now_us)
        order = np.lexsort((hi, lo, vs))
        ln = np.diff(off)[order]
        new_off = np.zeros(len(order) + 1, np.uint64)
        np.cumsum(ln, out=new_off[1:])
        # byte t of sorted blob k comes from off[order[k]] + (t - new_off[k])
        src = np.repeat(off[:-1][order].astype(np.int64) - new_off[:-1].astype(np.int64), ln.astype(np.int64))
        src += np.arange(int(new_off[-1]), dtype=np.int64)
        arrays = self._engine._snapshot_arrays(now_us)
        arrays.update(cv_varset=vs[order], cv_key_lo=lo[order], cv_key_hi=hi[order], cv_blob_off=new_off, cv_blobs=blobs[src])
        with open(path, "wb") as f:
            np.savez(f, **arrays)

    def load_counters(self, path: str) -> int:
        """Import a save_counters file: the dictionary entries first (keeping must be on), then the counters through
        Engine.load_counters.  Returns the keys added to the dictionary.  A file without cv_ arrays (Engine.save_counters)
        loads exactly as Engine.load_counters loads it.  If the counter import is refused after the dictionary import,
        the added entries refer to no counter, and the next counter_vars_gc drops them."""
        with np.load(path) as z:
            cv = [z[k] for k in ("cv_varset", "cv_key_lo", "cv_key_hi", "cv_blob_off", "cv_blobs")] if "cv_varset" in z else None
        added = self.import_counter_vars(*cv) if cv is not None else 0
        self._engine.load_counters(path)
        return added

    # -- configuration --
    def configure_with(self, limits, dry_run: bool = False) -> Dict[str, int]:
        """RateLimiter::configure_with (lib.rs:475-505) over rl_rls_configure: the service then holds exactly `limits`
        (limiter.Limit objects, or dicts as limits_file.parse_limits returns them).  Kept limits keep their counters; the
        first of two entries with one identity wins; all or nothing.  dry_run checks and counts without changing anything.
        -> {kept, added, updated, deleted}; raises ConfigureError naming the refused entry."""
        limits = list(limits)
        keep = []  # the encoded strings live until the call returns

        def enc(v):
            return None if v is None else str(v).encode()

        specs = (LimitSpec * max(len(limits), 1))()
        for i, l in enumerate(limits):
            conds, vars_ = [str(c) for c in _field(l, "conditions")], [str(v) for v in _field(l, "variables")]
            ca, va = _m._strs(conds), _m._strs(vars_)
            keep += [ca, va]
            specs[i] = LimitSpec(enc(_field(l, "namespace")), int(_field(l, "max_value")), int(_field(l, "seconds")), ca, len(conds), 0,
                                 va, len(vars_), 0, enc(_field(l, "name")), enc(_field(l, "id")))
        rep = ConfigureReport()
        if self._lib.rl_rls_configure(self._h, specs, len(limits), int(dry_run), C.byref(rep)) != 0:
            raise ConfigureError(self._lib.rl_rls_last_error(self._h).decode(),
                                 None if rep.first_refused == NO_STORE else rep.first_refused)
        return {"kept": rep.kept, "added": rep.added, "updated": rep.updated, "deleted": rep.deleted}

    def load_limits_file(self, path: str, dry_run: bool = False) -> Dict[str, int]:
        """configure_with the limits of a limitador-server limits file (limits_file.load_limits_file)."""
        from . import limits_file
        return self.configure_with(limits_file.load_limits_file(path), dry_run)

    def config_status(self) -> Dict[str, int]:
        """Status::config_version / config_err_since (limitador-server main.rs:218-235) of the configure_with calls."""
        v, e = C.c_uint64(), C.c_uint64()
        self._check(self._lib.rl_rls_config_status(self._h, C.byref(v), C.byref(e)))
        return {"config_version": v.value, "config_err_since": e.value}

    def metrics(self) -> str:
        need = C.c_uint64()
        self._lib.rl_rls_metrics_render(self._h, None, 0, C.byref(need))
        buf = C.create_string_buffer(need.value)
        self._check(self._lib.rl_rls_metrics_render(self._h, buf, need.value, C.byref(need)))
        return buf.value.decode()
