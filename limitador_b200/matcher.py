"""ctypes binding of the native CPU front (include/rl_match.h, csrc/rl_match.cpp): limits -> counters.

`Matcher` is the compiled counterpart of `limiter.RateLimiter.counters_that_apply` (lib.rs:507-522): it
interns limits, namespaces and variable sets the same way `limiter.RateLimiter` does, matches a request's
context against the namespace's limits and returns the CSR of `rl_counter` that
`Engine.check_and_update_batch` takes.  No decision is computed here.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import engine as _eng

BIND_ROOT = 0xFFFFFFFF

MATCH_SYMBOLS = (
    "rl_matcher_create", "rl_matcher_destroy", "rl_matcher_last_error", "rl_matcher_add_limit",
    "rl_matcher_delete_limit", "rl_matcher_namespace_id", "rl_matcher_limit_name", "rl_matcher_counters",
    "rl_matcher_counters_batch", "rl_counter_key", "rl_matcher_response_headers",
    "rl_matcher_add_limit_ex", "rl_matcher_limit_name_copy", "rl_matcher_last_error_copy",
    "rl_front_check_and_update_bindings", "rl_matcher_set_counter_cap", "rl_matcher_counters_batch_ns",
    "rl_matcher_response_headers_batch",
)


class RlBinding(C.Structure):
    _fields_ = [("descriptor", C.c_uint32), ("_pad", C.c_uint32), ("key", C.c_char_p), ("value", C.c_char_p)]


class MatcherError(RuntimeError):
    pass


def _lib():
    L = _eng.load_library()
    if getattr(L, "_rl_match_ready", False):
        return L
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.rl_matcher_create.argtypes = [C.POINTER(vp)]
    L.rl_matcher_destroy.argtypes = [vp]
    L.rl_matcher_destroy.restype = None
    L.rl_matcher_last_error.argtypes = [vp]
    L.rl_matcher_last_error.restype = C.c_char_p
    L.rl_matcher_add_limit.argtypes = [vp, C.c_char_p, u64, u64, C.POINTER(C.c_char_p), u32, C.POINTER(C.c_char_p), u32,
                                       C.c_char_p, vp]
    L.rl_matcher_add_limit_ex.argtypes = [vp, C.c_char_p, u64, u64, C.POINTER(C.c_char_p), u32, C.POINTER(C.c_char_p), u32,
                                          C.c_char_p, C.c_int, vp, C.POINTER(C.c_int)]
    L.rl_matcher_limit_name_copy.argtypes = [vp, u32, C.c_char_p, u32, C.POINTER(C.c_int)]
    L.rl_matcher_last_error_copy.argtypes = [vp, C.c_char_p, u32]
    L.rl_matcher_delete_limit.argtypes = [vp, u32]
    L.rl_matcher_set_counter_cap.argtypes = [vp, u32]
    L.rl_matcher_counters_batch_ns.argtypes = [vp, u64, C.POINTER(C.c_char_p), vp, C.POINTER(RlBinding), vp, vp, u64, vp]
    L.rl_matcher_response_headers_batch.argtypes = [vp, u64, vp, vp, vp, vp, vp, u64, vp, C.POINTER(u64)]
    L.rl_matcher_namespace_id.argtypes = [vp, C.c_char_p, C.POINTER(u32)]
    L.rl_matcher_limit_name.argtypes = [vp, u32]
    L.rl_matcher_limit_name.restype = C.c_char_p
    L.rl_matcher_counters.argtypes = [vp, u32, C.POINTER(RlBinding), u32, vp, u32, C.POINTER(u32)]
    L.rl_matcher_counters_batch.argtypes = [vp, u64, vp, vp, C.POINTER(RlBinding), vp, vp, u64]
    L.rl_matcher_response_headers.argtypes = [vp, vp, vp, vp, u32, C.c_char_p, u32, C.c_char_p, u32, C.c_char_p, u32]
    L.rl_counter_key.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), u32, C.POINTER(u64), C.POINTER(u64)]
    L.rl_counter_key.restype = None
    L.rl_front_check_and_update_bindings.argtypes = [vp, vp, C.c_char_p, C.POINTER(RlBinding), u32, u64, u64, C.c_int, vp, vp, vp,
                                                     vp, vp, vp, vp]
    L._rl_match_ready = True
    return L


def _strs(items: Sequence[str]):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode()
    return arr


def counter_key(set_variables: Dict[str, str]) -> Tuple[int, int]:
    """(key_lo, key_hi) of resolved variables: the digest `limiter.Counter.key` computes with hashlib."""
    ks = list(set_variables)
    lo, hi = C.c_uint64(), C.c_uint64()
    _lib().rl_counter_key(_strs(ks), _strs([set_variables[k] for k in ks]), len(ks), C.byref(lo), C.byref(hi))
    return lo.value, hi.value


def _bindings(root: Optional[Dict[str, str]], descriptors: Optional[List[Dict[str, str]]]):
    flat = [(BIND_ROOT, k, v) for k, v in (root or {}).items()]
    for i, d in enumerate(descriptors or []):
        flat += [(i, k, v) for k, v in d.items()]
    return flat


class Matcher:
    def __init__(self):
        self._lib = _lib()
        h = C.c_void_p()
        if self._lib.rl_matcher_create(C.byref(h)) != 0:
            raise MatcherError("rl_matcher_create failed")
        self._h = h

    def close(self):
        if self._h:
            self._lib.rl_matcher_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status):
        if status != 0:
            raise MatcherError(self._lib.rl_matcher_last_error(self._h).decode())

    def add_limit(self, namespace: str, max_value: int, seconds: int, conditions: Iterable[str] = (),
                  variables: Iterable[str] = (), name: Optional[str] = None) -> np.void:
        """-> one LIMIT_DESC_DTYPE row (limit_id, ns_id, varset_id, qualified, max_value, window_us)."""
        conds, vars_ = list(conditions), list(variables)
        desc = np.zeros(1, dtype=_eng.LIMIT_DESC_DTYPE)
        self._check(self._lib.rl_matcher_add_limit(self._h, namespace.encode(), max_value, seconds, _strs(conds), len(conds),
                                                   _strs(vars_), len(vars_), None if name is None else name.encode(),
                                                   desc.ctypes.data))
        return desc[0]

    def add_limit_keep(self, namespace: str, max_value: int, seconds: int, conditions: Iterable[str] = (),
                       variables: Iterable[str] = (), name: Optional[str] = None):
        """Storage::add_limit (storage/mod.rs:60-65): an equal live limit keeps its max_value and name.
        -> (LIMIT_DESC_DTYPE row as the limit now stands, existed)."""
        conds, vars_ = list(conditions), list(variables)
        desc = np.zeros(1, dtype=_eng.LIMIT_DESC_DTYPE)
        existed = C.c_int(0)
        self._check(self._lib.rl_matcher_add_limit_ex(self._h, namespace.encode(), max_value, seconds, _strs(conds), len(conds),
                                                      _strs(vars_), len(vars_), None if name is None else name.encode(), 1,
                                                      desc.ctypes.data, C.byref(existed)))
        return desc[0], bool(existed.value)

    def set_counter_cap(self, cap: int):
        """Counters one request may produce (default 16 = what a default engine takes); raise it to the engine's
        max_counters_per_request (up to 64) to ship wider requests, or past it to match without the engine."""
        self._check(self._lib.rl_matcher_set_counter_cap(self._h, cap))

    def delete_limit(self, limit_id: int):
        self._check(self._lib.rl_matcher_delete_limit(self._h, limit_id))

    def namespace_id(self, namespace: str) -> Optional[int]:
        out = C.c_uint32()
        return out.value if self._lib.rl_matcher_namespace_id(self._h, namespace.encode(), C.byref(out)) == 0 else None

    def limit_name(self, limit_id: int) -> Optional[str]:
        buf = C.create_string_buffer(1024)
        has = C.c_int(0)
        self._check(self._lib.rl_matcher_limit_name_copy(self._h, limit_id, buf, 1024, C.byref(has)))
        return buf.value.decode() if has.value else None

    def counters(self, ns_id: int, root: Optional[Dict[str, str]] = None,
                 descriptors: Optional[List[Dict[str, str]]] = None, cap: int = 64) -> np.ndarray:
        """counters_that_apply for one request -> COUNTER_DTYPE array (registration order)."""
        flat = _bindings(root, descriptors)
        binds = (RlBinding * max(len(flat), 1))()
        for i, (d, k, v) in enumerate(flat):
            binds[i] = RlBinding(d, 0, k.encode(), v.encode())
        out = np.zeros(cap, dtype=_eng.COUNTER_DTYPE)
        n = C.c_uint32()
        self._check(self._lib.rl_matcher_counters(self._h, ns_id, binds, len(flat), out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    def response_headers(self, ctrs: np.ndarray, remaining, ttl_us) -> Dict[str, str]:
        """CheckResult::response_header (lib.rs:235-275) of one request from its load_counters outputs."""
        ctrs = np.ascontiguousarray(ctrs, dtype=_eng.COUNTER_DTYPE)
        rem = np.ascontiguousarray(remaining, dtype=np.uint64)
        ttl = np.ascontiguousarray(ttl_us, dtype=np.uint64)
        bl, br, bs = C.create_string_buffer(64 + 96 * max(len(ctrs), 1) + 300 * len(ctrs)), C.create_string_buffer(32), C.create_string_buffer(32)
        self._check(self._lib.rl_matcher_response_headers(self._h, ctrs.ctypes.data, rem.ctypes.data, ttl.ctypes.data, len(ctrs),
                                                          bl, len(bl), br, len(br), bs, len(bs)))
        if len(ctrs) == 0:
            return {}
        return {"X-RateLimit-Limit": bl.value.decode(), "X-RateLimit-Remaining": br.value.decode(),
                "X-RateLimit-Reset": bs.value.decode()}

    def counters_batch_ns(self, namespaces: Sequence[str], contexts: Sequence[Tuple[Optional[dict], Optional[list]]]):
        """rl_matcher_counters_batch_ns: requests named by namespace string, one reader section for the whole batch.
        -> (ctr_off uint32[n+1], ctrs COUNTER_DTYPE, status uint8[n]: 0 matched, 1 namespace without limits, 2 too many counters)."""
        n = len(namespaces)
        flats = [_bindings(r, d) for r, d in contexts]
        off = np.zeros(n + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(f) for f in flats])
        binds = (RlBinding * max(int(off[-1]), 1))()
        j = 0
        for f in flats:
            for d, k, v in f:
                binds[j] = RlBinding(d, 0, k.encode(), v.encode())
                j += 1
        ctr_off = np.zeros(n + 1, dtype=np.uint32)
        ctrs = np.zeros(64 * (n + 1), dtype=_eng.COUNTER_DTYPE)
        status = np.zeros(max(n, 1), dtype=np.uint8)
        self._check(self._lib.rl_matcher_counters_batch_ns(self._h, n, _strs(list(namespaces)), off.ctypes.data, binds, ctr_off.ctypes.data,
                                                           ctrs.ctypes.data, len(ctrs), status.ctypes.data))
        return ctr_off, ctrs[:int(ctr_off[-1])], status[:n]

    def response_headers_batch(self, ctr_off, ctrs, remaining, ttl_us, cap: int = 0) -> List[Dict[str, str]]:
        """rl_matcher_response_headers_batch: the draft-03 header values of every request of a CSR in one call."""
        ctr_off = np.ascontiguousarray(ctr_off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=_eng.COUNTER_DTYPE)
        rem = np.ascontiguousarray(remaining, dtype=np.uint64)
        ttl = np.ascontiguousarray(ttl_us, dtype=np.uint64)
        n = len(ctr_off) - 1
        out_off = np.zeros(n + 1, dtype=np.uint64)
        need = C.c_uint64()
        buf = C.create_string_buffer(max(cap, 1))
        st = self._lib.rl_matcher_response_headers_batch(self._h, n, ctr_off.ctypes.data, ctrs.ctypes.data, rem.ctypes.data, ttl.ctypes.data,
                                                         buf, cap, out_off.ctypes.data, C.byref(need))
        if st != 0 and need.value > cap:  # too small: the call said how much it needs
            return self.response_headers_batch(ctr_off, ctrs, rem, ttl, int(need.value))
        self._check(st)
        raw = buf.raw
        out = []
        for i in range(n):
            lim, r, rst = raw[int(out_off[i]):int(out_off[i + 1])].split(b"\0")[:3]
            out.append({} if ctr_off[i + 1] == ctr_off[i] else
                       {"X-RateLimit-Limit": lim.decode(), "X-RateLimit-Remaining": r.decode(), "X-RateLimit-Reset": rst.decode()})
        return out

    def counters_batch(self, ns_ids: Sequence[int], contexts: Sequence[Tuple[Optional[dict], Optional[list]]],
                       cap: Optional[int] = None):
        """-> (ctr_off[n+1] uint32, ctrs COUNTER_DTYPE): the inputs of Engine.check_and_update_batch."""
        n = len(ns_ids)
        flats = [_bindings(r, d) for r, d in contexts]
        off = np.zeros(n + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(f) for f in flats])
        binds = (RlBinding * max(int(off[-1]), 1))()
        j = 0
        for f in flats:
            for d, k, v in f:
                binds[j] = RlBinding(d, 0, k.encode(), v.encode())
                j += 1
        cap = cap or 64 * max(n, 1)
        ctr_off = np.zeros(n + 1, dtype=np.uint32)
        ctrs = np.zeros(cap, dtype=_eng.COUNTER_DTYPE)
        ids = np.ascontiguousarray(ns_ids, dtype=np.uint32)
        self._check(self._lib.rl_matcher_counters_batch(self._h, n, ids.ctypes.data, off.ctypes.data, binds,
                                                        ctr_off.ctypes.data, ctrs.ctypes.data, cap))
        return ctr_off, ctrs[:int(ctr_off[-1])]


def front_check_and_update(front, matcher: "Matcher", namespace: str, root: Optional[Dict[str, str]] = None,
                           descriptors: Optional[List[Dict[str, str]]] = None, delta: int = 1, now_us: int = 0,
                           load_counters: bool = False):
    """rl_front_check_and_update_bindings: RateLimiter::check_rate_limited_and_update for one request — the native
    matcher on the calling thread, then the batching front.  -> (limited, first_limited limit id | None, seq, counters
    (COUNTER_DTYPE), remaining, ttl_us)."""
    L = _lib()
    flat = _bindings(root, descriptors)
    binds = (RlBinding * max(len(flat), 1))()
    for i, (d, k, v) in enumerate(flat):
        binds[i] = RlBinding(d, 0, k.encode(), v.encode())
    lim, first, seq, n = C.c_uint8(0), C.c_uint32(_eng.NONE), C.c_uint64(0), C.c_uint32(0)
    ctrs = np.zeros(16, dtype=_eng.COUNTER_DTYPE)
    rem = np.zeros(16, dtype=np.uint64)
    ttl = np.zeros(16, dtype=np.uint64)
    st = L.rl_front_check_and_update_bindings(front._h, matcher._h, namespace.encode(), binds, len(flat), delta, now_us,
                                              int(load_counters), C.addressof(lim), C.addressof(first), ctrs.ctypes.data,
                                              C.addressof(n), rem.ctypes.data, ttl.ctypes.data, C.addressof(seq))
    if st != 0:
        raise MatcherError(L.rl_matcher_last_error(matcher._h).decode() or "rl_front_check_and_update_bindings failed")
    k = n.value
    return bool(lim.value), (None if first.value == _eng.NONE else first.value), seq.value, ctrs[:k], rem[:k], ttl[:k]
