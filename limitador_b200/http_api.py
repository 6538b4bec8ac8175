"""ctypes binding of Limitador's HTTP API surface (include/rl_http.h, csrc/rl_rls.cpp).

`HttpApi(rls_service)` serves batches of `CheckAndReportInfo` JSON bodies for one endpoint at a time — POST /check,
/report or /check_and_report (limitador-server/src/http_api/server.rs:129-260) — through the RLS service's matcher,
engine, workers and metrics: decode + counters_that_apply on the engine's GPU, one engine call per run of equal
load_counters flags, then status / body / X-RateLimit-* headers on the CPU workers.  `plan` / `finish` are the CPU stages
on their own (drivable without a GPU), `plan_device` is the GPU plan on its own; `serve` runs plan_device -> engine ->
finish.  `encode_info` writes a body as serde_json serialises the struct.  `get_counters` / `get_limits` answer
GET /counters/{namespace} and GET /limits/{namespace} (server.rs:88-125); `render_counters` is the rendering of the
former on its own.
"""
from __future__ import annotations

import ctypes as C
import json
from typing import Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import engine as _eng
from . import rls as _rls

CHECK, REPORT, CHECK_AND_REPORT = 0, 1, 2
HEADERS_NONE, HEADERS_DRAFT_VERSION_03, HEADERS_OTHER = 0, 1, 2
HEADER_NAMES = ("X-RateLimit-Limit", "X-RateLimit-Remaining", "X-RateLimit-Reset")

HTTP_SYMBOLS = (
    "rl_http_serve_sharded", "rl_http_send", "rl_http_decide", "rl_http_collect",
    "rl_http_decode_body", "rl_http_create", "rl_http_destroy", "rl_http_last_error", "rl_http_plan", "rl_http_plan_device",
    "rl_http_plan_view", "rl_http_finish", "rl_http_responses", "rl_http_serve", "rl_http_last_timings", "rl_http_get_limits",
    "rl_http_get_counters", "rl_http_render_counters", "rl_http_get_response",
)


class HttpInfo(C.Structure):
    _fields_ = [("ns_off", C.c_uint32), ("ns_len", C.c_uint32), ("delta", C.c_uint64), ("n_entries", C.c_uint32),
                ("response_headers", C.c_uint32)]


class HttpError(RuntimeError):
    pass


def _lib():
    L = _rls._lib()
    if getattr(L, "_rl_http_ready", False):
        return L
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.rl_http_decode_body.argtypes = [vp, u64, vp, C.POINTER(HttpInfo), vp, u32]
    L.rl_http_create.argtypes = [vp, C.POINTER(vp)]
    L.rl_http_destroy.argtypes = [vp]
    L.rl_http_destroy.restype = None
    L.rl_http_last_error.argtypes = [vp]
    L.rl_http_last_error.restype = C.c_char_p
    L.rl_http_plan.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_http_plan_device.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_http_plan_view.argtypes = [vp, C.POINTER(u64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                    C.POINTER(vp), C.POINTER(vp)]
    L.rl_http_finish.argtypes = [vp, vp, vp, vp, vp, vp]
    L.rl_http_responses.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.rl_http_serve.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_http_serve_sharded.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_http_send.argtypes = [vp, i32, u64, vp, vp, u64]
    L.rl_http_decide.argtypes = [vp]
    L.rl_http_collect.argtypes = [vp]
    L.rl_http_last_timings.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(u32)]
    L.rl_http_get_limits.argtypes = [vp, C.c_char_p, u32]
    L.rl_http_get_counters.argtypes = [vp, C.c_char_p, u32, u64]
    L.rl_http_render_counters.argtypes = [vp, C.c_char_p, u32, u64, vp, vp, vp, vp, vp, vp]
    L.rl_http_get_response.argtypes = [vp, C.POINTER(C.c_uint16), C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]
    L._rl_http_ready = True
    return L


def encode_info(namespace: str, values: Mapping[str, str], delta: int, response_headers: Optional[str] = None) -> bytes:
    """CheckAndReportInfo as serde_json::to_vec writes it: compact, fields in declaration order, `values` in the given
    order, the short escapes and lower-case \\u00XX for other control characters, everything else as UTF-8."""
    d = {"namespace": namespace, "values": dict(values), "delta": int(delta), "response_headers": response_headers}
    return json.dumps(d, ensure_ascii=False, separators=(",", ":")).encode()


pack_bodies = _rls.pack_requests  # -> (buf uint8, off uint64[n+1]): the batch layout rl_http_plan / rl_http_serve take


def decode_body(body: bytes, cap_entries: int = 64):
    """The native decoder on one body -> (namespace, values as (key, value) pairs in body order, delta, response_headers
    state); raises HttpError for a body the Json extractor refuses (HTTP 400)."""
    L = _lib()
    arr = np.frombuffer(body, dtype=np.uint8) if body else np.zeros(1, dtype=np.uint8)
    txt = np.zeros(max(len(body), 1), dtype=np.uint8)
    q = HttpInfo()
    ent = np.zeros(max(cap_entries, 1), dtype=_rls.ENTRY_DTYPE)
    if L.rl_http_decode_body(arr.ctypes.data, len(body), txt.ctypes.data, C.byref(q), ent.ctypes.data, cap_entries) != 0:
        raise HttpError("body refused")
    if q.n_entries > cap_entries:
        return decode_body(body, q.n_entries)
    t = txt.tobytes()
    s = lambda o, n: t[o:o + n].decode()  # noqa: E731
    pairs = [(s(int(e["key_off"]), int(e["key_len"])), s(int(e["val_off"]), int(e["val_len"]))) for e in ent[:q.n_entries]]
    return s(q.ns_off, q.ns_len), pairs, q.delta, q.response_headers


_view, _ptr = _rls._view, _rls._ptr


class HttpApi:
    """The HTTP API over an RlsService (its matcher, engine, workers and metrics).  Not thread-safe, and not to be used
    concurrently with the RlsService: one batch of either surface at a time."""

    def __init__(self, rls_service: _rls.RlsService):
        self._lib = _lib()
        self._rls = rls_service  # keep it alive
        h = C.c_void_p()
        if self._lib.rl_http_create(rls_service._h, C.byref(h)) != 0:
            raise HttpError("rl_http_create failed")
        self._h = h
        self._n = 0

    def close(self):
        if self._h:
            self._lib.rl_http_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status):
        if status != 0:
            raise HttpError(self._lib.rl_http_last_error(self._h).decode())

    def plan(self, endpoint: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Stage 1 on the CPU workers -> dict(n_store, ctr_off, ctrs, delta, now_us, load_counters, store_index): copies
        of the store requests (load_counters: one flag per store request)."""
        return self._plan(self._lib.rl_http_plan, endpoint, buf, off, now_us)

    def plan_device(self, endpoint: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Stage 1 on the engine's device; the same dict as `plan`, array for array."""
        return self._plan(self._lib.rl_http_plan_device, endpoint, buf, off, now_us)

    def _plan(self, fn, endpoint, buf, off, now_us):
        self._n = n = len(off) - 1
        _rls._batch_call(self, fn, endpoint, buf, off, now_us)
        return _rls._read_plan(self._lib.rl_http_plan_view, self._h, self._check, n, True)

    def finish(self, limited=None, first_limited=None, remaining=None, ttl_us=None, store_status=None):
        """Stage 3.  store_status: one status per store request (None = all OK)."""
        keep = []
        self._check(self._lib.rl_http_finish(self._h, _ptr(store_status, np.int32, keep), _ptr(limited, np.uint8, keep),
                                             _ptr(first_limited, np.uint32, keep), _ptr(remaining, np.uint64, keep),
                                             _ptr(ttl_us, np.uint64, keep)))
        return self.responses()

    def responses(self) -> List[Tuple[int, bytes, Dict[str, str]]]:
        """-> [(status, body, headers)] of the last finished batch; headers holds the X-RateLimit-* headers present."""
        ps, pb, pbo, ph, pho = (C.c_void_p() for _ in range(5))
        self._check(self._lib.rl_http_responses(self._h, C.byref(ps), C.byref(pb), C.byref(pbo), C.byref(ph), C.byref(pho)))
        n = self._n
        status = _view(ps.value, n, np.uint16)
        bo = _view(pbo.value, n + 1, np.uint64)
        ho = _view(pho.value, 3 * n + 1, np.uint64)
        body = _view(pb.value, int(bo[-1]) if n else 0, np.uint8).tobytes()
        hv = _view(ph.value, int(ho[-1]) if n else 0, np.uint8).tobytes()
        out = []
        for i in range(n):
            hdrs = {}
            for k, name in enumerate(HEADER_NAMES):
                v = hv[int(ho[3 * i + k]):int(ho[3 * i + k + 1])]
                if v:
                    hdrs[name] = v.decode()
            out.append((int(status[i]), body[int(bo[i]):int(bo[i + 1])], hdrs))
        return out

    def serve(self, endpoint: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """plan_device -> the engine (one call per run) -> finish.  Needs an engine."""
        self._n = len(off) - 1
        _rls._batch_call(self, self._lib.rl_http_serve, endpoint, buf, off, now_us)

    def send(self, endpoint: int, buf: np.ndarray, off: np.ndarray, now_us: int = 0):
        """Sharded step (the RLS service has a ShardBatch attached), phase 1: plan and send; then decide and collect, as
        RlsService.send / decide / collect."""
        self._n = len(off) - 1
        _rls._batch_call(self, self._lib.rl_http_send, endpoint, buf, off, now_us)

    def decide(self):
        self._check(self._lib.rl_http_decide(self._h))

    def collect(self):
        self._check(self._lib.rl_http_collect(self._h))
        return self.responses()

    def timings(self) -> Dict[str, float]:
        a, b, c, k = C.c_double(), C.c_double(), C.c_double(), C.c_uint32()
        self._lib.rl_http_last_timings(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(k))
        return {"plan_us": a.value, "store_us": b.value, "finish_us": c.value, "store_calls": k.value}

    def get_limits(self, namespace: str) -> Tuple[int, bytes]:
        """GET /limits/{namespace} -> (status, body)."""
        ns = namespace.encode()
        self._check(self._lib.rl_http_get_limits(self._h, ns, len(ns)))
        return self._get_response()[:2]

    def get_counters(self, namespace: str, now_us: int = 0) -> Tuple[int, bytes]:
        """GET /counters/{namespace} at now_us (0 = wall clock) -> (status, body).  Needs an engine, and the RLS service
        keeping counter variables (RlsService.keep_counter_vars) for any qualified counter to be listed."""
        ns = namespace.encode()
        self._check(self._lib.rl_http_get_counters(self._h, ns, len(ns), now_us))
        status, body, self.last_unnamed = self._get_response()
        return status, body

    def render_counters(self, namespace: str, ctrs, remaining, ttl_us, blobs: bytes, blob_off, unnamed=None) -> Tuple[int, bytes]:
        """The rendering stage of get_counters on its own: counters (COUNTER_DTYPE), remaining / ttl_us per counter, the
        blobs packed (counter i's at blobs[blob_off[i]:blob_off[i + 1]]) and the unnamed flags -> (status, body)."""
        ns = namespace.encode()
        ctrs = np.ascontiguousarray(ctrs, dtype=_eng.COUNTER_DTYPE)
        n = len(ctrs)
        rem = np.ascontiguousarray(remaining, dtype=np.uint64)
        ttl = np.ascontiguousarray(ttl_us, dtype=np.uint64)
        bl = np.frombuffer(bytes(blobs) or b"\0", dtype=np.uint8)
        bo = np.ascontiguousarray(blob_off, dtype=np.uint64)
        un = None if unnamed is None else np.ascontiguousarray(unnamed, dtype=np.uint8)
        p = lambda a: a.ctypes.data if a is not None and len(a) else None  # noqa: E731
        self._check(self._lib.rl_http_render_counters(self._h, ns, len(ns), n, p(ctrs), p(rem), p(ttl), p(bl), p(bo), p(un)))
        status, body, self.last_unnamed = self._get_response()
        return status, body

    def _get_response(self):
        st, pb, ln, un = C.c_uint16(), C.c_void_p(), C.c_uint64(), C.c_uint64()
        self._check(self._lib.rl_http_get_response(self._h, C.byref(st), C.byref(pb), C.byref(ln), C.byref(un)))
        return int(st.value), _view(pb.value, ln.value, np.uint8).tobytes(), un.value

    def metrics(self) -> str:
        """The shared metrics text (rl_rls_metrics_render): the same as the RLS service's."""
        return self._rls.metrics()


def store_runs(load_counters: np.ndarray) -> List[Tuple[int, int]]:
    """The store calls of a plan: maximal runs [j0, j1) of equal load_counters flags."""
    lc = np.asarray(load_counters)
    if len(lc) == 0:
        return []
    cuts = [0] + [int(j) for j in np.flatnonzero(lc[1:] != lc[:-1]) + 1] + [len(lc)]
    return list(zip(cuts[:-1], cuts[1:]))
