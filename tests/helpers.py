"""Shared test helpers: oracle-backed CounterStorage, the host emulator binding, random stream
builders, the edge-domain streams and known answers of the counter arithmetic, and oracle_restore
(an import applied to the CPU oracle)."""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

from oracle import binding as ob
from limitador_b200.engine import COUNTER_DTYPE, LIMIT_DESC_DTYPE, NONE, RECORD_DTYPE
from limitador_b200.limiter import Authorization

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
T0 = 1_700_000_000_000_000

CELLDESC_DTYPE = np.dtype([("max_value", "<u8"), ("window_us", "<u8"), ("limit_id", "<u4"), ("qualified", "<u4")])


def host_lib(src, name, defines=()):
    """tests/emu/<src> compiled for the host into tests/emu/<name> (with -D<defines>).  It is rebuilt when it is older than
    any source in tests/emu/, any .h / .cuh in limitador_b200/csrc/ or any header in include/: everything it can
    include."""
    so = os.path.join(HERE, "emu", name)
    dirs = {os.path.join(HERE, "emu"): (".cpp", ".h"), os.path.join(ROOT, "limitador_b200", "csrc"): (".h", ".cuh"),
            os.path.join(ROOT, "include"): (".h",)}
    deps = [os.path.join(d, f) for d, ext in dirs.items() for f in os.listdir(d) if f.endswith(ext)]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        tmp = f"{so}.{os.getpid()}.so"  # a process that has the old library loaded keeps its copy
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", *[f"-D{d}" for d in defines], "-o", tmp,
                               os.path.join(HERE, "emu", src)])
        os.replace(tmp, so)
    return C.CDLL(so)


@functools.cache
def emu_lib():
    L = host_lib("emu.cpp", "librl_emu.so")
    vp = C.c_void_p
    L.emu_create.restype = vp
    L.emu_create.argtypes = [C.c_int]
    L.emu_destroy.argtypes = [vp]
    L.emu_limits_set.argtypes = [vp, vp, C.c_uint32, C.c_char_p, C.c_uint32]
    L.emu_limits_set.restype = C.c_int
    L.emu_limit_group.argtypes = [vp, C.c_uint32]
    L.emu_limit_group.restype = C.c_uint32
    L.emu_batch_csr.argtypes = [vp, C.c_int, C.c_int, C.c_uint32, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.emu_resolve.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, vp, C.c_uint32, vp, vp]
    L.emu_resolve.restype = C.c_int
    L.emu_dump.restype = C.c_uint64
    L.emu_dump.argtypes = [vp, C.c_uint64, vp, vp, vp, vp, vp]
    L.emu_steps.restype = C.c_uint64
    L.emu_steps.argtypes = [vp]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


ACCESS_DTYPE = np.dtype([("key_lo", "<u8"), ("hdr_hi", "<u8"), ("req", "<u4"), ("cells", "<u4"), ("posorig", "<u8")])
assert ACCESS_DTYPE.itemsize == 32


class Emu:
    """Sequential host run of the kernels' algorithm (tests/emu/emu.cpp), in the narrow position encoding or, with
    wide=True, the wide one (requests of up to 64 counters)."""

    def __init__(self, descs: np.ndarray, cells: int, wide: bool = False):
        self.L = emu_lib()
        self.wide = wide
        self.h = self.L.emu_create(cells)
        self.cells = cells
        self.set_limits(descs)
        self.rounds = self.steps = 0

    def set_limits(self, descs):
        """rl_limits_set through the engine's registry (new ids, or live ids with another max_value; the counters
        stay).  Raises ValueError with the engine's message when the registry refuses a limit."""
        d = np.ascontiguousarray(descs, dtype=LIMIT_DESC_DTYPE)
        err = C.create_string_buffer(512)
        if self.L.emu_limits_set(self.h, _p(d), len(d), err, len(err)) != 0:
            raise ValueError(err.value.decode())

    def group_of(self, limit_id):
        """The row group the registry gave a limit (0: not defined)."""
        return int(self.L.emu_limit_group(self.h, limit_id))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.emu_destroy(self.h)

    def batch_csr(self, mode, off, ctrs, delta, now_us, load_counters=False):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        n = len(delta)
        lim = np.zeros(n, dtype=np.uint8)
        fl = np.full(n, NONE, dtype=np.uint32)
        rem = np.zeros(len(ctrs), dtype=np.uint64)
        ttl = np.zeros(len(ctrs), dtype=np.uint64)
        rounds = C.c_int(0)
        r = self.L.emu_batch_csr(self.h, int(self.wide), mode, n, _p(off), _p(ctrs), _p(delta), _p(now_us),
                                 int(load_counters), _p(lim), _p(fl), _p(rem), _p(ttl), C.byref(rounds))
        assert r == 0, f"emu error {r}"
        self.rounds = rounds.value
        self.steps = int(self.L.emu_steps(self.h))  # replay steps: a closed-form run counts one
        return lim, fl, rem, ttl

    def resolve(self, ctrs, req=0, max_ctrs=64, wide=None):
        """rl_resolve_request alone on one request (in the emulator's encoding unless `wide` says otherwise): the number
        of accesses or a negative RL_DEV_* code, the accesses and (wide) the permutation."""
        wide = self.wide if wide is None else wide
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        m = len(ctrs)
        acc = np.zeros(max(m, 1), dtype=ACCESS_DTYPE)
        perm = np.full(max(m, 1), 0xFF, dtype=np.uint8)
        r = self.L.emu_resolve(self.h, int(wide), req, m, _p(ctrs), max_ctrs, _p(acc), _p(perm))
        return r, acc, perm

    def dump(self):
        cap = 1 << 20
        lid = np.zeros(cap, dtype=np.uint32)
        lo = np.zeros(cap, dtype=np.uint64)
        hi = np.zeros(cap, dtype=np.uint64)
        val = np.zeros(cap, dtype=np.uint64)
        exp = np.zeros(cap, dtype=np.uint64)
        c = self.L.emu_dump(self.h, cap, _p(lid), _p(lo), _p(hi), _p(val), _p(exp))
        return sorted(zip(lid[:c].tolist(), lo[:c].tolist(), hi[:c].tolist(), val[:c].tolist(), exp[:c].tolist()))


def emu_vs_oracle(descs, cells, batches, load_counters, mode=0, wide=False):
    """Run `batches` (CSR tuples) through the emulator and the oracle and compare them bit for bit: verdicts,
    first-limited ids and (load_counters) remaining / ttl for check_and_update (mode 0), the table after every batch.
    Returns the emulator's fixed-point rounds per batch."""
    emu = Emu(descs, cells, wide)
    orc = oracle_with_limits(descs)
    rounds = []
    for off, ctrs, delta, now in batches:
        e = emu.batch_csr(mode, off, ctrs, delta, now, load_counters)
        o = orc.batch_csr(mode, off, ctrs, delta, now, load_counters)
        rounds.append(emu.rounds)
        if mode == 0:
            assert e[0].tolist() == o[0].tolist(), "verdicts differ"
            assert e[1].tolist() == o[1].tolist(), "first-limited limit differs"
            if load_counters:
                assert e[2].tolist() == o[2].tolist(), "remaining differs"
                assert e[3].tolist() == o[3].tolist(), "ttl differs"
        assert normalise_dump(emu.dump(), descs) == normalise_dump(orc.dump(), descs), "table differs"
    return rounds


def normalise_dump(dump, descs):
    """Unqualified counters: a never-touched row and a present (0, EPOCH) entry are the same
    state; drop the (0,0) ones so both sides compare equal."""
    unq = {int(d["limit_id"]) for d in descs if not d["qualified"]}
    return sorted(t for t in dump if not (t[0] in unq and t[3] == 0 and t[4] == 0))


def oracle_with_limits(descs, capacity_hint=1024) -> "ob.Oracle":
    o = ob.Oracle(capacity_hint)
    for d in descs:
        o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    return o


class OracleStorage:
    """The RateLimiter mirror's CounterStorage protocol over the CPU oracle (tests only)."""

    def __init__(self):
        self.o = ob.Oracle(1024)

    def set_limit(self, limit_id, ns_id, varset_id, qualified, max_value, window_us):
        self.o.limit_set(limit_id, ns_id, max_value, window_us, qualified)

    def forget_limit(self, limit_id):
        self.o.limit_delete(limit_id)

    @staticmethod
    def _ctrs(counters):
        return ob.counters([(c.limit_id, *c.key()) for c in counters])

    def is_within_limits(self, counter, delta, now_us):
        return self.o.is_within_limits(self._ctrs([counter]), delta, now_us)

    def first_limited(self, counters, delta, now_us):
        if not counters:
            return None
        limited, idx = self.o.is_rate_limited(self._ctrs(counters), delta, now_us)
        return counters[idx] if limited else None

    def update_counter(self, counter, delta, now_us):
        self.o.update_counters(self._ctrs([counter]), delta, now_us)

    def check_and_update(self, counters, delta, load_counters, now_us):
        limited, idx, rem, ttl = self.o.check_and_update(self._ctrs(counters), delta, load_counters, now_us)
        if load_counters:
            for j, c in enumerate(counters):
                c.remaining = int(rem[j])
                c.expires_in_us = int(ttl[j])
        return Authorization(limited, counters[idx].limit.name if limited else None)

    def check_and_update_many(self, counter_lists, deltas, nows, load_counters):
        return [self.check_and_update(cl, d, load_counters, t) if cl else Authorization(False)
                for cl, d, t in zip(counter_lists, deltas, nows)]

    def get_counters(self, limit_ids, now_us):
        return self.o.get_counters(limit_ids, now_us)

    def delete_counters(self, limit_ids):
        self.o.delete_counters(limit_ids)

    def clear(self):
        self.o.clear()


# ---------------------------------------------------------------------------------------
def _plain_limit(rng):
    """max 0 / tiny / huge, 1 s .. 1 h windows"""
    mx = int(rng.choice([0, 1, 2, 3, 5, 8, 20, 1 << 40]))
    win = int(rng.choice([1, 2, 10, 60, 3600])) * 1_000_000
    return mx, win


def mixed_limits(n_ns=6, seed=0, draw=_plain_limit):
    """A limits table exercising every row shape: single qualified limit, several limits on
    one variable set (one row), two variable sets (two rows), unqualified + qualified,
    unqualified only; (max_value, window_us) from `draw`."""
    rng = np.random.default_rng(seed)
    descs = []
    lid = 0
    shapes = ["q1", "q4", "q2v", "uq", "u", "q3u2"]
    for ns in range(n_ns):
        shape = shapes[ns % len(shapes)]
        plan = {
            "q1": [(1, 1)],
            "q4": [(1, 1)] * 4,
            "q2v": [(1, 1), (1, 1), (2, 1)],
            "uq": [(0, 0), (1, 1)],
            "u": [(0, 0), (0, 0)],
            "q3u2": [(1, 1), (0, 0), (1, 1), (2, 1), (0, 0)],
        }[shape]
        for varset, q in plan:
            mx, win = draw(rng)
            descs.append((lid, ns, varset, q, mx, win))
            lid += 1
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


def random_csr_stream(descs, n, seed, n_keys=5, monotone=True, subset=True):
    """Random requests over `descs`: request = a namespace, a random non-empty subset of its
    limits (or all), per-varset keys drawn from a tiny key space (heavy duplicates)."""
    rng = np.random.default_rng(seed)
    by_ns = {}
    for d in descs:
        by_ns.setdefault(int(d["ns_id"]), []).append(d)
    nss = sorted(by_ns)
    off = [0]
    ctrs = []
    delta = np.zeros(n, dtype=np.uint64)
    now = np.zeros(n, dtype=np.uint64)
    t = T0
    for i in range(n):
        ns = int(rng.choice(nss))
        lims = by_ns[ns]
        if subset and rng.random() < 0.4:
            k = int(rng.integers(0, len(lims) + 1))
            pick = sorted(rng.choice(len(lims), size=k, replace=False).tolist()) if k else []
        else:
            pick = list(range(len(lims)))
        if rng.random() < 0.3:
            rng.shuffle(pick)
        vkeys = {}
        for j in pick:
            d = lims[j]
            vs = int(d["varset_id"]) if d["qualified"] else 0
            if vs not in vkeys:
                vkeys[vs] = (int(rng.integers(1, n_keys + 1)), int(rng.integers(0, 2)))
            lo, hi = vkeys[vs] if d["qualified"] else (0, 0)
            ctrs.append((int(d["limit_id"]), 0, lo, hi))
        off.append(len(ctrs))
        delta[i] = int(rng.choice([1, 1, 1, 2, 3, 7]))
        step = int(rng.choice([0, 0, 1, 1000, 400_000, 1_500_000]))
        t += step
        now[i] = t if monotone else max(1, t - int(rng.choice([0, 0, 2_000_000])))
    return (np.array(off, dtype=np.uint32), np.array(ctrs, dtype=COUNTER_DTYPE) if ctrs else np.zeros(0, COUNTER_DTYPE),
            delta, now)


def wide_limits(seed, sizes=(20, 33, 64, 3), small=True, draw=_plain_limit):
    """Namespaces of `sizes` limits, qualified (three variable sets) and unqualified interleaved in registration order,
    with small maxima so that the limits bite (or all 2^62 with small=False); windows and maxima from `draw`."""
    rng = np.random.default_rng(seed)
    descs, lid = [], 0
    for ns, size in enumerate(sizes):
        for _ in range(size):
            q = 1 if rng.random() < 0.7 else 0
            varset = int(rng.integers(1, 4)) if q else 0
            mx, win = draw(rng) if small else (1 << 62, int(rng.choice([1, 2, 10, 60, 3600])) * 1_000_000)
            descs.append((lid, ns, varset, q, mx, win))
            lid += 1
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


def wide_stream(descs, n, seed, n_keys=3, monotone=True, min_ctrs=17):
    """Requests naming at least min_ctrs of their namespace's limits where it has that many (all of a smaller one),
    in shuffled order half of the time; per-variable-set keys from a tiny key space."""
    rng = np.random.default_rng(seed)
    by_ns = {}
    for d in descs:
        by_ns.setdefault(int(d["ns_id"]), []).append(d)
    nss = sorted(by_ns)
    off, ctrs = [0], []
    delta = np.zeros(n, dtype=np.uint64)
    now = np.zeros(n, dtype=np.uint64)
    t = T0
    for i in range(n):
        lims = by_ns[int(rng.choice(nss))]
        lo_k = min(min_ctrs, len(lims))
        k = int(rng.integers(lo_k, len(lims) + 1))
        pick = sorted(rng.choice(len(lims), size=k, replace=False).tolist())
        if rng.random() < 0.5:
            rng.shuffle(pick)
        vkeys = {}
        for j in pick:
            d = lims[j]
            vs = int(d["varset_id"]) if d["qualified"] else 0
            if vs not in vkeys:
                vkeys[vs] = (int(rng.integers(1, n_keys + 1)), int(rng.integers(0, 2)))
            lo, hi = vkeys[vs] if d["qualified"] else (0, 0)
            ctrs.append((int(d["limit_id"]), 0, lo, hi))
        off.append(len(ctrs))
        delta[i] = int(rng.choice([1, 1, 1, 2, 3, 7]))
        t += int(rng.choice([0, 0, 1, 1000, 400_000, 1_500_000]))
        now[i] = t if monotone else max(1, t - int(rng.choice([0, 0, 2_000_000])))
    return np.array(off, dtype=np.uint32), np.array(ctrs, dtype=COUNTER_DTYPE), delta, now


def random_records(descs, n, seed, n_keys=5, monotone=True):
    rng = np.random.default_rng(seed)
    nss = sorted({int(d["ns_id"]) for d in descs}) + [int(descs["ns_id"].max()) + 3]  # + a namespace without limits
    r = np.zeros(n, dtype=RECORD_DTYPE)
    r["ns_id"] = rng.choice(nss, size=n)
    r["hits_addend"] = rng.choice([1, 1, 1, 2, 3, 7], size=n)
    r["key_lo"] = rng.integers(1, n_keys + 1, size=n)
    r["key_hi"] = rng.integers(0, 2, size=n)
    steps = rng.choice([0, 0, 1, 1000, 400_000, 1_500_000], size=n)
    t = T0 + np.cumsum(steps)
    if not monotone:
        t = t - rng.choice([0, 0, 2_000_000], size=n)
    r["now_us"] = t
    return r


@functools.cache
def emu_maint_lib(simt: bool = False):
    """tests/emu/emu_maint.cpp: the maintenance, counter-import and CRDT kernels (rl_maint.cuh, rl_crdt.cuh) compiled for
    the host — under tests/emu/cuda_shim.h (one CUDA thread after the other; the kernels' warp-aggregated branches
    compiled out), or with simt=True under tests/emu/cuda_simt.h (fibers + warp rendezvous: the device branches
    themselves run)."""
    L = host_lib("emu_maint.cpp", "librl_emu_simt.so" if simt else "librl_emu_maint.so", ["EMU_SIMT"] if simt else [])
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.emu_seed.argtypes = [u64]
    L.emu_ns_metrics.argtypes = [vp, u32, u32, vp, vp, u32, u32, vp]
    L.emu_ns_metrics.restype = None
    L.emu_table_create.restype = vp
    L.emu_table_create.argtypes = [u32, u32, u32]
    L.emu_table_destroy.argtypes = [vp]
    L.emu_table_raw.restype = vp
    L.emu_table_raw.argtypes = [vp]
    L.emu_table_bytes.restype = u64
    L.emu_table_bytes.argtypes = [vp]
    for f in (L.emu_table_put, L.emu_table_get):
        f.restype = C.c_int64
        f.argtypes = [vp, u64, u64, vp]
    L.emu_table_tombstone.restype = C.c_int64
    L.emu_table_tombstone.argtypes = [vp, u64, u64]
    L.emu_table_compact.argtypes = [vp, u32, vp, vp]
    L.emu_table_compact.restype = None
    L.emu_crdt_create.restype = vp
    L.emu_crdt_create.argtypes = [u64, u32, u32]
    L.emu_crdt_destroy.argtypes = [vp]
    L.emu_crdt_inc.argtypes = [vp, u32, vp, vp, vp, vp, u64]
    L.emu_crdt_inc.restype = u32
    L.emu_crdt_merge.argtypes = [vp, u32, vp, vp, vp, u64, u64]
    L.emu_crdt_merge.restype = u32
    L.emu_crdt_read.argtypes = [vp, u32, vp, u64, vp, vp]
    L.emu_crdt_read.restype = u32
    L.emu_crdt_scan.argtypes = [vp, C.c_int, u64, u64, vp, vp, vp, vp]
    L.emu_crdt_scan.restype = u64
    L.emu_import.restype = u64
    L.emu_import.argtypes = [vp, u32, u32, u32, vp, u32, u64, vp, vp, vp, vp, vp, vp]
    if simt:
        L.emu_simt_interleave.argtypes = [C.c_int, u64, C.c_double]
        L.emu_simt_interleave.restype = None
    return L


class EmuCrdt:
    """The CRDT kernels on the host (same interface as limitador_b200.crdt.CrdtTable).  interleave=(seed, p) (simt=True
    only): every call runs under cuda_simt.h's interleaving mode, the n-th call of the table with seed + n."""

    def __init__(self, capacity_rows, actors, self_actor, simt=False, interleave=None):
        from limitador_b200 import crdt as CR
        assert interleave is None or simt
        self.CR = CR
        self.L = emu_maint_lib(simt)
        self.actors, self.self_actor = actors, self_actor
        self.h = self.L.emu_crdt_create(capacity_rows, actors, self_actor)
        self.capacity = capacity_rows
        self.interleave, self.calls = interleave, 0

    def _call(self, f, *args):
        if self.interleave is None:
            return f(*args)
        seed, p = self.interleave
        self.calls += 1
        self.L.emu_simt_interleave(1, seed + self.calls, p)
        try:
            return f(*args)
        finally:
            self.L.emu_simt_interleave(0, 0, 1.0)  # the library is shared: leave the mode off for everybody else

    def __del__(self):
        try:
            self.L.emu_crdt_destroy(self.h)
        except Exception:
            pass

    def inc(self, keys, actor, increment, window_us, now_us):
        keys = np.ascontiguousarray(keys, dtype=self.CR.KEY_DTYPE)
        n = len(keys)
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(actor, dtype=np.uint32), (n,)))
        inc = np.ascontiguousarray(np.broadcast_to(np.asarray(increment, dtype=np.uint64), (n,)))
        win = np.ascontiguousarray(np.broadcast_to(np.asarray(window_us, dtype=np.uint64), (n,)))
        return self._call(self.L.emu_crdt_inc, self.h, n, _p(keys), _p(a), _p(inc), _p(win), now_us)

    def merge(self, ups, actors, values, now_us):
        ups = np.ascontiguousarray(ups, dtype=self.CR.UPDATE_DTYPE)
        actors = np.ascontiguousarray(actors, dtype=np.uint32)
        values = np.ascontiguousarray(values, dtype=np.uint64)
        return self._call(self.L.emu_crdt_merge, self.h, len(ups), _p(ups), _p(actors), _p(values), len(values), now_us)

    def read(self, keys, now_us):
        keys = np.ascontiguousarray(keys, dtype=self.CR.KEY_DTYPE)
        val = np.zeros(len(keys), dtype=np.uint64)
        exp = np.zeros(len(keys), dtype=np.uint64)
        assert self._call(self.L.emu_crdt_read, self.h, len(keys), _p(keys), now_us, _p(val), _p(exp)) == 0
        return val, exp

    def export(self, now_us, cap=1 << 16):
        k = np.zeros(cap, dtype=self.CR.KEY_DTYPE)
        val = np.zeros(cap, dtype=np.uint64)
        exp = np.zeros(cap, dtype=np.uint64)
        n = self._call(self.L.emu_crdt_scan, self.h, 0, now_us, cap, _p(k), _p(val), _p(exp), None)
        return sorted(zip(k["lo"][:n].tolist(), k["hi"][:n].tolist(), val[:n].tolist(), exp[:n].tolist()))

    def dump(self, cap=1 << 16):
        k = np.zeros(cap, dtype=self.CR.KEY_DTYPE)
        exp = np.zeros(cap, dtype=np.uint64)
        vals = np.zeros(cap * self.actors, dtype=np.uint64)
        n = self._call(self.L.emu_crdt_scan, self.h, 1, 0, cap, _p(k), None, _p(exp), _p(vals))
        v = vals[:n * self.actors].reshape(n, self.actors)
        return sorted((int(k["lo"][i]), int(k["hi"][i]), int(exp[i]), tuple(v[i].tolist())) for i in range(n))


def oracle_restore(o, descs, limit_id, key_lo, key_hi, value, expiry_us):
    """What rl_counters_import does, applied to the CPU oracle through its own public calls: set each counter to exactly
    (value, expiry_us); a present counter is replaced, an unqualified one (key ignored) becomes present, other counters
    are untouched.  descs: the limits the oracle was given (limit_id, ns_id, max_value, window_us, qualified).

    The counters of every limit named are read back (dump), deleted (delete_counters) and created again with the
    imported ones merged in: update_counter(delta = value, now = expiry - window) creates exactly (value, expiry)
    (in_memory.rs:47-69), and limit_set again on an unqualified limit without a counter recreates the (0, EPOCH) default
    (add_counter, in_memory.rs:38-44).  A limit id the oracle does not know raises before anything changes."""
    by_id = {int(d["limit_id"]): d for d in descs}
    new = {}
    for l, lo, hi, v, x in zip(*[np.asarray(c).tolist() for c in (limit_id, key_lo, key_hi, value, expiry_us)]):
        if l not in by_id:
            raise ValueError(f"limit {l} is not registered")
        new[(l, lo, hi) if by_id[l]["qualified"] else (l, 0, 0)] = (v, x)
    touched = sorted({k[0] for k in new})
    state = {(l, lo, hi): (v, x) for l, lo, hi, v, x in o.dump() if l in touched}
    state.update(new)
    for (l, lo, hi), (v, x) in state.items():
        w = int(by_id[l]["window_us"])
        if x < w and (by_id[l]["qualified"] or (v, x) != (0, 0)):
            raise ValueError(f"counter {(l, lo, hi)}: expiry {x} is earlier than one window after the epoch")
    o.delete_counters(touched)
    for (l, lo, hi), (v, x) in sorted(state.items()):
        d = by_id[l]
        if not d["qualified"] and (v, x) == (0, 0):
            o.limit_set(l, int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), False)
        else:
            o.update_counters(ob.counters([(l, lo, hi)]), v, x - int(d["window_us"]))


# ---------------------------------------------------------------------------------------
# The edges of the counter arithmetic: u64 wrap of value + delta, maxima up to 2^64-1, counters above their maximum,
# clocks exactly on a counter's expiry.  The closed-form replay (DESIGN.md §3.3) is exact only if it wraps and bounds
# exactly like n sequential adds; the streams below reach those values on purpose, and CountingSpec proves they did.
M64 = (1 << 64) - 1
EDGE_MAXIMA = [0, 1, (1 << 32) - 1, 1 << 32, (1 << 63) - 1, 1 << 63, (1 << 64) - 2, M64]
EDGE_WINDOWS = [1, 2, 1_000_000, 60_000_000, 1 << 40]
SMALL_DELTAS = [0, 1, 1, 2, 3, 7]
CSR_BIG_DELTAS = [1 << 31, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, 1 << 62, 3 << 62, 1 << 63, M64]
RECORD_BIG_DELTAS = [1 << 31, (1 << 31) + 1, 3 << 30, (1 << 32) - 1]  # hits_addend is a u32


def _pick(rng, pool):
    return pool[int(rng.integers(len(pool)))]


def _edge_limit(rng):
    """Maxima at the u32 / i64 / u64 boundaries or small enough to bite; windows of 1 µs .. 2^40 µs."""
    mx = _pick(rng, EDGE_MAXIMA) if rng.random() < 0.6 else _pick(rng, [1, 2, 3, 5, 8, 20])
    return mx, _pick(rng, EDGE_WINDOWS)


def edge_limits(seed, shape="mixed", n_ns=6, cells=7, sizes=(20, 33, 64, 3)):
    """Limits with edge maxima and windows in the row shapes of mixed_limits ("mixed"), of one row per namespace
    ("single": 1..cells limits on one variable set, every fourth namespace unqualified, maxima >= 2^63-1 in the
    second of every four) or of wide_limits ("wide")."""
    if shape == "mixed":
        return mixed_limits(n_ns, seed, draw=_edge_limit)
    if shape == "wide":
        return wide_limits(seed, sizes, draw=_edge_limit)
    rng = np.random.default_rng(seed)
    descs, lid = [], 0
    for ns in range(n_ns):
        q = 0 if ns % 4 == 3 else 1
        for _ in range(int(rng.integers(1, cells + 1))):
            mx, win = _edge_limit(rng)
            if ns % 4 == 1:  # only the top of the u64 range bites: long runs stay allowed
                mx = _pick(rng, EDGE_MAXIMA[4:])
            descs.append((lid, ns, q, q, mx, win))
            lid += 1
    return np.array(descs, dtype=LIMIT_DESC_DTYPE)


def spec_with_limits(descs, cls=None):
    from tests.spec_model import SpecStore
    s = (cls or SpecStore)()
    for d in descs:
        s.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
    s.clock = T0
    return s


def _edge_requests(descs, n, rng, shadow, mode, records, n_keys, monotone, big, hits, min_ctrs):
    """[(counters [(limit_id, key_lo, key_hi)], (key_lo, key_hi), delta, now)] — see edge_csr_stream.  `shadow` (a
    SpecStore) follows the stream so that clocks can be aimed at the expiry of the counter a request reads."""
    by_ns = {}
    for d in descs:
        by_ns.setdefault(int(d["ns_id"]), []).append(d)
    nss = sorted(by_ns)
    out, t, i = [], shadow.clock, 0
    while len(out) < n:
        ns = int(rng.choice(nss))
        lims = by_ns[ns]
        if records or rng.random() < 0.6:
            pick = list(range(len(lims)))
        else:
            pick = sorted(rng.choice(len(lims), size=int(rng.integers(min(min_ctrs, len(lims)) or 1, len(lims) + 1)),
                                     replace=False).tolist())
            if rng.random() < 0.3:
                rng.shuffle(pick)
        key, vkeys, ctrs = (int(rng.integers(1, n_keys + 1)), int(rng.integers(0, 2))), {}, []
        for j in pick:
            d = lims[j]
            vs = int(d["varset_id"]) if d["qualified"] else 0
            if vs not in vkeys:
                vkeys[vs] = key if records else (int(rng.integers(1, n_keys + 1)), int(rng.integers(0, 2)))
            ctrs.append((int(d["limit_id"]), *(vkeys[vs] if d["qualified"] else (0, 0))))
        # the clock: small steps, half a second +-1, or exactly expiry - 1 / expiry / expiry + 1 of the first counter
        t += _pick(rng, [0, 0, 0, 1, 2, 1000, 499_999, 500_000, 500_001])
        now = t if monotone or rng.random() < 0.7 else max(1, t - _pick(rng, [1, 2, 500_000, 1_000_000]))
        lid0, lo0, hi0 = ctrs[0]
        e = shadow.qualified.get((lid0, lo0, hi0)) if lims[pick[0]]["qualified"] else shadow.simple.get(lid0)
        if e is not None and e[1] > 2 and rng.random() < 0.25:
            now = e[1] + _pick(rng, [-1, 0, 0, 1])
            if now > t and (monotone or rng.random() < 0.5):
                t = now
        # a run: the same request again and again with one large delta (a member that differs only above bit 32)
        if rng.random() < 0.07:
            length = int(rng.integers(8, 25))
            d0 = _pick(rng, big) if hits is None else int(rng.integers(hits[0], hits[1] + 1))
            odd = int(rng.integers(1, length)) if not records and rng.random() < 0.4 else -1
            for k in range(length):
                dk = d0 ^ (1 << int(rng.integers(33, 63))) if k == odd else d0
                out.append((ctrs, key, dk, now + k // 3))
            t = max(t, now + length // 3)
        else:
            if hits is not None:
                delta = int(rng.integers(hits[0], hits[1] + 1))
            else:
                delta = _pick(rng, SMALL_DELTAS) if rng.random() < 0.6 else _pick(rng, big)
            out.append((ctrs, key, delta, now))
        for ctrs_k, _, d_k, now_k in out[i:]:
            if mode == 0:
                shadow.check_and_update(ctrs_k, d_k, False, now_k)
            elif mode == 2:
                shadow.update_counters(ctrs_k, d_k, now_k)
        i = len(out)
    shadow.clock = t
    return out[:n]


def edge_csr_stream(descs, n, seed, shadow=None, mode=0, n_keys=3, monotone=True, min_ctrs=1):
    """CSR requests over `descs` (a namespace, all or a subset of its limits, per-variable-set keys from a tiny key
    space) whose deltas mix 0 and small values with 2^31, 2^32-1, 2^32, 2^32+1, 2^62, 3*2^62, 2^63 and 2^64-1; runs of 8
    to 24 equal large deltas on one key (now and then one member differing from the others only above bit 32); clocks
    stepping by half a second +-1 and landing at expiry - 1, expiry and expiry + 1 of the counter a request reads, and
    (monotone=False) going back across them.  `shadow` (spec_with_limits) is the state the clocks aim at: pass the same
    one to every batch of a stream, with the batch's `mode` (0 check_and_update, 1 is_rate_limited, 2 update)."""
    rng = np.random.default_rng(seed)
    shadow = shadow or spec_with_limits(descs)
    reqs = _edge_requests(descs, n, rng, shadow, mode, False, n_keys, monotone, CSR_BIG_DELTAS, None, min_ctrs)
    off = np.cumsum([0] + [len(r[0]) for r in reqs]).astype(np.uint32)
    ctrs = np.array([(c[0], 0, c[1], c[2]) for r in reqs for c in r[0]], dtype=COUNTER_DTYPE)
    return (off, ctrs, np.array([r[2] for r in reqs], dtype=np.uint64), np.array([r[3] for r in reqs], dtype=np.uint64))


def edge_records(descs, n, seed, shadow=None, mode=0, n_keys=3, monotone=True, hits=None):
    """32-byte records with the clocks and runs of edge_csr_stream and hits_addend up to 2^32-1 (or, with hits=(lo, hi),
    drawn from lo..hi: 1..255 for rl_record16); 1 in 20 names a namespace without limits."""
    rng = np.random.default_rng(seed)
    shadow = shadow or spec_with_limits(descs)
    reqs = _edge_requests(descs, n, rng, shadow, mode, True, n_keys, monotone, RECORD_BIG_DELTAS, hits, 1)
    r = np.zeros(n, dtype=RECORD_DTYPE)
    ns_of = {int(d["limit_id"]): int(d["ns_id"]) for d in descs}
    r["ns_id"] = [ns_of[q[0][0][0]] for q in reqs]
    r["ns_id"][rng.random(n) < 0.05] = int(descs["ns_id"].max()) + 3
    r["hits_addend"] = [q[2] for q in reqs]
    r["key_lo"] = [q[1][0] for q in reqs]
    r["key_hi"] = [q[1][1] for q in reqs]
    r["now_us"] = [q[3] for q in reqs]
    return r


def edge_batches(descs, seed, n_batches, n, form="csr", monotone=None, **kw):
    """One edge stream as batches: [(mode, batch)], mostly check_and_update (0), every third an update_counters batch
    (2) that pushes counters past their maximum, now and then an is_rate_limited one (1).  Odd batches go back in
    time unless `monotone` is given."""
    shadow = spec_with_limits(descs)
    rng = np.random.default_rng(seed)
    gen = edge_csr_stream if form == "csr" else edge_records
    out = []
    for b in range(n_batches):
        mode = 2 if b % 3 == 1 else (1 if rng.random() < 0.15 else 0)
        mono = (b % 2 == 0) if monotone is None else monotone
        out.append((mode, gen(descs, n, seed * 1000 + b, shadow=shadow, mode=mode, monotone=mono, **kw)))
    return out


def records_as_csr(descs, recs):
    """The CSR form of 32-byte records: every limit of the namespace in registration order, keyed by the record's key
    if qualified."""
    by_ns = {}
    for d in descs:
        by_ns.setdefault(int(d["ns_id"]), []).append(d)
    off, ctrs = [0], []
    for r in recs:
        for d in by_ns.get(int(r["ns_id"]), []):
            q = int(d["qualified"])
            ctrs.append((int(d["limit_id"]), 0, int(r["key_lo"]) if q else 0, int(r["key_hi"]) if q else 0))
        off.append(len(ctrs))
    return (np.array(off, dtype=np.uint32), np.array(ctrs, dtype=COUNTER_DTYPE),
            recs["hits_addend"].astype(np.uint64), recs["now_us"].astype(np.uint64))


def _counting_spec():
    from tests.spec_model import SpecStore

    class CountingSpec(SpecStore):
        """spec_model.SpecStore that counts the edges its calls reach (self.n):
          wrapped_sums     a counter read whose value_at + delta passes 2^64
          expiry_reads     a present counter read with now == its expiry (reads as 0, inclusive bound)
          stale_flips      ... of those, reads where the expired value would have given the other verdict
          above_max_reads  a live counter read whose value is above its limit's maximum
          long_runs        >= 8 consecutive allowed increments of one counter by one delta, no window reset, that
                           add up to more than 2^32
          wrapping_runs    >= 2 such increments whose total passes 2^64 from the value the run started at
          denied_runs      >= 4 consecutive denied check_and_update calls on one counter
        Runs end at the end of a batch (end_batch), at a window reset, an update_counters call or another delta."""

        KINDS = ("wrapped_sums", "expiry_reads", "stale_flips", "above_max_reads", "long_runs", "wrapping_runs",
                 "denied_runs")

        def __init__(self):
            super().__init__()
            self.n = dict.fromkeys(self.KINDS, 0)
            self._run = {}  # counter -> [allowed?, delta, length, total, start value]

        def _key(self, lid, lo, hi):
            return (lid, lo, hi) if self.limits[lid][3] else (lid, 0, 0)

        def _entry(self, lid, lo, hi):
            return self.qualified.get((lid, lo, hi)) if self.limits[lid][3] else self.simple.get(lid)

        def _reads(self, ctrs, delta, now):
            for lid, lo, hi in ctrs:
                e, mx = self._entry(lid, lo, hi), self.limits[lid][1]
                if e is None:
                    continue
                v = self.value_at(e, now)
                self.n["wrapped_sums"] += v + delta > M64
                self.n["above_max_reads"] += v > mx
                if e[1] == now:
                    self.n["expiry_reads"] += 1
                    self.n["stale_flips"] += (((e[0] + delta) & M64) > mx) != (delta > mx)

        def _end(self, k):
            r = self._run.pop(k, None)
            if r is None:
                return
            allowed, _, length, total, v0 = r
            if allowed:
                self.n["long_runs"] += length >= 8 and total > 1 << 32
                self.n["wrapping_runs"] += length >= 2 and v0 + total > M64
            else:
                self.n["denied_runs"] += length >= 4

        def end_batch(self):
            for k in list(self._run):
                self._end(k)

        def check_and_update(self, ctrs, delta, load_counters, now):
            self._reads(ctrs, delta, now)
            before = {self._key(*c): (lambda e: None if e is None else list(e))(self._entry(*c)) for c in ctrs}
            res = super().check_and_update(ctrs, delta, load_counters, now)
            for k, e0 in before.items():
                r = self._run.get(k)
                if res[0]:
                    if r is None or r[0]:
                        self._end(k)
                        self._run[k] = r = [False, None, 0, 0, 0]
                    r[2] += 1
                elif e0 is None or e0[1] <= now:  # created or reset: a run can only start after it
                    self._end(k)
                else:
                    if r is None or not r[0] or r[1] != delta:
                        self._end(k)
                        self._run[k] = r = [True, delta, 0, 0, e0[0]]
                    r[2] += 1
                    r[3] += delta
            return res

        def is_rate_limited(self, ctrs, delta, now):
            self._reads(ctrs, delta, now)
            return super().is_rate_limited(ctrs, delta, now)

        def update_counters(self, ctrs, delta, now):
            self._reads(ctrs, delta, now)
            for c in ctrs:
                self._end(self._key(*c))
            super().update_counters(ctrs, delta, now)

    return CountingSpec


def spec_batch(s, mode, off, ctrs, delta, now, lc):
    """A CSR batch through a spec_model.SpecStore, request by request -> (limited, first limited id, remaining, ttl)
    like Oracle.batch_csr."""
    n = len(delta)
    lim, fl = np.zeros(n, dtype=np.uint8), np.full(n, NONE, dtype=np.uint32)
    rem, ttl = np.zeros(len(ctrs), dtype=np.uint64), np.zeros(len(ctrs), dtype=np.uint64)
    for i in range(n):
        cs = [(int(c["limit_id"]), int(c["key_lo"]), int(c["key_hi"])) for c in ctrs[off[i]:off[i + 1]]]
        if not cs:
            continue  # no limits apply: not limited (lib.rs:434-440)
        if mode == 0:
            limited, first, r, t = s.check_and_update(cs, int(delta[i]), lc, int(now[i]))
            if lc:
                rem[off[i]:off[i + 1]] = r
                ttl[off[i]:off[i + 1]] = t
        elif mode == 1:
            limited, first = s.is_rate_limited(cs, int(delta[i]), int(now[i]))
        else:
            s.update_counters(cs, int(delta[i]), int(now[i]))
            limited, first = False, NONE
        lim[i], fl[i] = int(limited), first
    if hasattr(s, "end_batch"):
        s.end_batch()
    return lim, fl, rem, ttl


def edge_coverage(descs, batches, form="csr"):
    """Replay [(mode, batch)] (edge_batches) through a counting spec_model -> its counts."""
    s = spec_with_limits(descs, _counting_spec())
    for mode, b in batches:
        spec_batch(s, mode, *(b if form == "csr" else records_as_csr(descs, b)), False)
    return s.n


def counting_spec(descs):
    return spec_with_limits(descs, _counting_spec())


# ---------------------------------------------------------------------------------------
# Known answers at the edges, the numbers written out (not taken from the oracle).  One qualified limit (id 0, max
# "max", window "window") and one counter (key 7); "seed" (value, t) is an update_counters(delta = value, now = t) on
# the missing counter, i.e. the state (value, t + window).  Steps: ("check", deltas, nows, verdicts, remaining, ttl),
# ("state", (value, expiry)), ("get", now, [(remaining, ttl)]) for get_counters, ("max", new max_value).
_S = 1_000_000
_T = T0
_D = 0x4000000100000003  # 2^62 + 2^32 + 3: bits above 32, so a 32-bit product k * D gets the run's sums wrong
EDGE_KATS = {
    # 2^62 + 3*2^62 wraps to 0 <= 2^63: allowed, and the value becomes 0; 3*2^62 > 2^63 then denies twice
    "wrap_allows_then_denies": dict(max=1 << 63, window=60 * _S, seed=(1 << 62, _T), steps=[
        ("check", [3 << 62] * 3, [_T + 1, _T + 2, _T + 3], [0, 1, 1], [1 << 63, 0, 0],
         [60 * _S - 1, 60 * _S - 2, 60 * _S - 3]),
        ("state", (0, _T + 60 * _S))]),
    # ten allowed increments by D from 0 (k*D passes 2^32 at once and wraps past 2^64 at k = 4 and 8) under max
    # 3*2^62 + 2^35; the eleventh, 3*2^62 + 11*2^32 + 33, is over it
    "closed_form_run_wraps": dict(max=0xC000000800000000, window=60 * _S, seed=(0, _T), steps=[
        ("check", [_D] * 11, [_T + k for k in range(1, 12)], [0] * 10 + [1],
         [0x80000006FFFFFFFD, 0x40000005FFFFFFFA, 0x4FFFFFFF7, 0xC0000003FFFFFFF4, 0x80000002FFFFFFF1,
          0x40000001FFFFFFEE, 0xFFFFFFEB, 0xBFFFFFFFFFFFFFE8, 0x7FFFFFFEFFFFFFE5, 0x3FFFFFFDFFFFFFE2, 0],
         [60 * _S - k for k in range(1, 12)]),
        ("state", (0x8000000A0000001E, _T + 60 * _S))]),
    # expiry T + 1 s: at T + 1 s - 2 and - 1 the 50 still counts; at T + 1 s it reads as 0 and the third request opens
    # a new window (1, T + 2 s); the fourth, at the same clock, adds to it
    "exact_boundary_in_a_run": dict(max=100, window=_S, seed=(50, _T), steps=[
        ("check", [1] * 4, [_T + _S - 2, _T + _S - 1, _T + _S, _T + _S], [0, 0, 0, 0], [49, 48, 99, 98],
         [2, 1, 0, _S]),
        ("state", (2, _T + 2 * _S))]),
    # 15 > max 10: delta 0 is denied and changes nothing; get_counters' remaining wraps (10 - 15); max 20 allows it
    "above_the_maximum": dict(max=10, window=60 * _S, seed=(15, _T), steps=[
        ("check", [0], [_T + 1], [1], [0], [60 * _S - 1]),
        ("state", (15, _T + 60 * _S)),
        ("get", _T + 1, [(M64 - 4, 60 * _S - 1)]),
        ("max", 20),
        ("check", [0], [_T + 2], [0], [5], [60 * _S - 2]),
        ("get", _T + 3, [(5, 60 * _S - 3)]),
        ("state", (15, _T + 60 * _S))]),
    # max 0, value 1: 1 + (2^64 - 1) wraps to 0 <= 0, allowed, and the value becomes 0
    "max_zero_wraps_to_zero": dict(max=0, window=60 * _S, seed=(1, _T), steps=[
        ("check", [M64], [_T + 1], [0], [0], [60 * _S - 1]),
        ("state", (0, _T + 60 * _S))]),
}


def edge_kat_limits(kat, max_value=None):
    mx = kat["max"] if max_value is None else max_value
    return np.array([(0, 0, 1, 1, mx, kat["window"])], dtype=LIMIT_DESC_DTYPE)


def run_edge_kat(kat, layer, batched, lc):
    """One EDGE_KATS entry through `layer`: an object with seed(value, now) (update_counters), check(deltas, nows, lc)
    -> (verdicts, remaining, ttl) on the KAT's counter, state() -> (value, expiry), get(now) -> [(remaining, ttl)] or
    None where the layer has no get_counters, set_max(max_value).  The checks go as one call per step (batched) or one
    call per request."""
    layer.seed(*kat["seed"])
    for step in kat["steps"]:
        if step[0] == "check":
            _, deltas, nows, want_lim, want_rem, want_ttl = step
            calls = [(deltas, nows)] if batched else [([d], [t]) for d, t in zip(deltas, nows)]
            got = [layer.check(d, t, lc) for d, t in calls]
            assert [v for g in got for v in g[0]] == want_lim, "verdicts"
            if lc:
                assert [v for g in got for v in g[1]] == want_rem, "remaining"
                assert [v for g in got for v in g[2]] == want_ttl, "ttl"
        elif step[0] == "state":
            assert layer.state() == step[1], "counter state"
        elif step[0] == "get":
            got = layer.get(step[1])
            assert got is None or got == step[2], "get_counters"
        else:
            layer.set_max(step[1])


@functools.cache
def emu_engine_lib():
    """tests/emu/emu_engine.cpp: the decision kernels (k_front, k_hot, k_main, the resolve kernels, k_restore,
    k_fl_step, k_wide_scatter, k_query_records, k_scan) and the peer exchange's (k_xcount .. k_xgather) compiled for
    the host under tests/emu/cuda_simt.h, driven through the engine's and the shard's call sequences."""
    L = host_lib("emu_engine.cpp", "librl_emu_engine.so")
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.emu_engine_create.restype = vp
    L.emu_engine_create.argtypes = [u32, u32, u32]
    L.emu_engine_destroy.argtypes = [vp]
    L.emu_engine_limits_set.argtypes = [vp, vp, u32]
    L.emu_engine_knobs.argtypes = [vp, u32, u32, u32, u32, u32, u32, u32, u32]
    L.emu_engine_knobs.restype = None
    L.emu_engine_interleave.argtypes = [vp, C.c_int, u64, C.c_double]
    L.emu_engine_interleave.restype = None
    L.emu_engine_report.restype = C.POINTER(C.c_ulonglong)
    L.emu_engine_report.argtypes = [vp]
    L.emu_engine_max_cells_used.restype = u32
    L.emu_engine_max_cells_used.argtypes = [vp]
    L.emu_engine_record_stride.restype = u32
    L.emu_engine_record_stride.argtypes = [vp]
    L.emu_engine_record_region.restype = C.c_int64
    L.emu_engine_record_region.argtypes = [vp, vp]
    L.emu_engine_records.argtypes = [vp, C.c_int, u32, vp, C.c_int, vp, vp, vp, vp, u64]
    L.emu_engine_csr.argtypes = [vp, C.c_int, u32, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp]
    L.emu_engine_query_records.argtypes = [vp, u32, vp, vp, vp]
    L.emu_engine_export.restype = u64
    L.emu_engine_export.argtypes = [vp, u64, vp, vp, vp, vp, vp]
    L.emu_shard_create.restype = vp
    L.emu_shard_create.argtypes = [vp, u32, u32, u32, u32]
    L.emu_shard_destroy.argtypes = [vp]
    L.emu_shard_send.argtypes = [vp, u32, u32, vp, vp]
    L.emu_shard_decide.argtypes = [vp, u32]
    L.emu_shard_collect.argtypes = [vp, u32, C.c_int]
    L.emu_shard_xwait.argtypes = [vp, u32, u32, u32, u32, vp, vp]
    L.emu_shard_xwait.restype = None
    for f in ("ctl", "set_ctl", "ctrs", "err"):
        getattr(L, f"emu_shard_{f}").argtypes = [vp, u32, vp]
        getattr(L, f"emu_shard_{f}").restype = None
    L.emu_shard_inbox.argtypes = [vp, u32, u32, u32, vp]
    L.emu_shard_inbox.restype = None
    L.emu_shard_dest.argtypes = [vp, u32, u32, vp]
    L.emu_shard_dest.restype = None
    return L


# what EmuEngine.geometry reports about the last call, in emu_engine.cpp's order
EMU_GEOMETRY = ("tiles", "tile", "merge_passes_main", "merge_passes_hot", "nparts", "items", "heavy_items", "max_w",
                "hot_in_use", "hot_candidates", "hot_max_list", "hot_sweeps", "fixed_point_rounds", "chunks", "rounds",
                "chained_chunks", "ordered_chunks", "hot_after", "max_partition", "ch", "rearmed")


class EmuEngine:
    """The engine's decision calls on the host (tests/emu/emu_engine.cpp): the same kernels the GPU runs, under the
    fiber emulator.  Knobs: chunk (128 / 256), heavy_mult, part_target, hot rows, weak grouping tags, the sharded
    geometry (tile derived from a device-side count), resident k_main blocks and the grid cap; interleave=(seed, p)
    turns cuda_simt.h's interleaving mode on.  After every call `geometry` says what the call reached."""

    def __init__(self, descs, cells, log2P, log2R, chunk=128, heavy_mult=2, part_target=128, hot=False, weak=False,
                 sharded=False, resident=1, grid_cap=132 * 16, interleave=None):
        self.L = emu_engine_lib()
        self.h = self.L.emu_engine_create(cells, log2P, log2R)
        self.cells = cells
        self.L.emu_engine_knobs(self.h, chunk, heavy_mult, part_target, int(hot), int(weak), int(sharded), resident, grid_cap)
        if interleave is not None:
            self.L.emu_engine_interleave(self.h, 1, interleave[0], interleave[1])
        self.set_limits(descs)
        self.geometry = {}

    def __del__(self):
        if getattr(self, "h", None):
            self.L.emu_engine_destroy(self.h)

    def set_limits(self, descs):
        d = np.ascontiguousarray(descs, dtype=LIMIT_DESC_DTYPE)
        assert self.L.emu_engine_limits_set(self.h, _p(d), len(d)) == 0

    @property
    def max_cells_used(self):
        return int(self.L.emu_engine_max_cells_used(self.h))

    def _report(self):
        r = self.L.emu_engine_report(self.h)
        self.geometry = {k: int(r[i]) for i, k in enumerate(EMU_GEOMETRY)}

    def region_of(self, rec):
        """The table region of a record's row (single-row namespaces), or -1."""
        r = np.ascontiguousarray(np.array([rec], dtype=RECORD_DTYPE))
        return int(self.L.emu_engine_record_region(self.h, _p(r)))

    def records(self, mode, recs, load_counters=False):
        """check_and_update (mode 0) / update_counters (mode 2) over records: limited, first-limited, remaining, ttl
        ([n * stride]) and the device error code."""
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        n = len(recs)
        stride = int(self.L.emu_engine_record_stride(self.h))
        lim = np.full(n, 0xA5, dtype=np.uint8)
        fl = np.full(n, 0xA5A5A5A5, dtype=np.uint32)
        rem = np.zeros(n * stride, dtype=np.uint64)
        ttl = np.zeros(n * stride, dtype=np.uint64)
        err = self.L.emu_engine_records(self.h, mode, n, _p(recs), int(load_counters), _p(lim), _p(fl), _p(rem), _p(ttl), 0)
        self._report()
        return lim, fl, rem, ttl, err

    def records16(self, recs16, now_us):
        """check_and_update over 16-byte records (rl_record16) stamped with one clock reading: limited, first-limited
        and the device error code."""
        from limitador_b200.engine import RECORD16_DTYPE
        recs16 = np.ascontiguousarray(recs16, dtype=RECORD16_DTYPE)
        n = len(recs16)
        lim = np.full(n, 0xA5, dtype=np.uint8)
        fl = np.full(n, 0xA5A5A5A5, dtype=np.uint32)
        assert now_us != 0  # 0 selects the 32-byte form
        err = self.L.emu_engine_records(self.h, 0, n, _p(recs16), 0, _p(lim), _p(fl), None, None, int(now_us))
        self._report()
        return lim, fl, err

    def csr(self, mode, off, ctrs, delta, now_us, load_counters=False):
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ctrs = np.ascontiguousarray(ctrs, dtype=COUNTER_DTYPE)
        delta = np.ascontiguousarray(delta, dtype=np.uint64)
        now_us = np.ascontiguousarray(now_us, dtype=np.uint64)
        n = len(delta)
        lim = np.full(n, 0xA5, dtype=np.uint8)
        fl = np.full(n, 0xA5A5A5A5, dtype=np.uint32)
        rem = np.zeros(max(len(ctrs), 1), dtype=np.uint64)
        ttl = np.zeros(max(len(ctrs), 1), dtype=np.uint64)
        err = self.L.emu_engine_csr(self.h, mode, n, _p(off), _p(ctrs), _p(delta), _p(now_us), int(load_counters),
                                    _p(lim), _p(fl), _p(rem), _p(ttl))
        self._report()
        return lim, fl, rem[:len(ctrs)], ttl[:len(ctrs)], err

    def query_records(self, recs):
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        lim = np.zeros(len(recs), dtype=np.uint8)
        fl = np.zeros(len(recs), dtype=np.uint32)
        err = self.L.emu_engine_query_records(self.h, len(recs), _p(recs), _p(lim), _p(fl))
        return lim, fl, err

    def dump(self, cap=1 << 20):
        """The table read through k_scan's export: sorted (limit_id, key_lo, key_hi, value, expiry_us)."""
        lid = np.zeros(cap, dtype=np.uint32)
        lo, hi, val, exp = (np.zeros(cap, dtype=np.uint64) for _ in range(4))
        c = int(self.L.emu_engine_export(self.h, cap, _p(lid), _p(lo), _p(hi), _p(val), _p(exp)))
        assert c <= cap
        return sorted(zip(lid[:c].tolist(), lo[:c].tolist(), hi[:c].tolist(), val[:c].tolist(), exp[:c].tolist()))


class EmuShard:
    """The namespace-sharded peer exchange on the host (tests/emu/emu_engine.cpp's emu_shard_*): one EmuEngine per rank
    and host slabs laid out as rl_shard_create lays out the device ones; send / decide / collect follow rl_shard_send,
    rl_shard_decide and rl_shard_collect launch for launch.  The caller issues them in an order in which every wait
    kernel runs after the kernels it waits for (every rank sends, then every rank decides, then every rank collects)."""

    def __init__(self, engines, cap, lag, max_batch=None):
        self.L = emu_engine_lib()
        self.engines = list(engines)
        self.world, self.cap, self.lag, self.depth = len(engines), cap, lag, lag + 2
        arr = (C.c_void_p * self.world)(*[e.h for e in self.engines])
        mb = self.world * cap if max_batch is None else max_batch
        self.h = self.L.emu_shard_create(arr, self.world, cap, lag, mb)
        assert self.h, "emu_shard_create refused its arguments"
        self._keep = {}  # (rank, step) -> (records, verdict output): the slab and the collection point at them
        self._sent = [0] * self.world

    def __del__(self):
        if getattr(self, "h", None):
            self.L.emu_shard_destroy(self.h)

    def send(self, rank, recs):
        """Returns the verdict array the step's collection fills (poisoned until then)."""
        recs = np.ascontiguousarray(recs, dtype=RECORD_DTYPE)
        out = np.full(max(len(recs), 1), 0xA5, dtype=np.uint8)
        assert self.L.emu_shard_send(self.h, rank, len(recs), _p(recs), _p(out)) == 0
        self._keep[(rank, self._sent[rank])] = (recs, out)
        self._sent[rank] += 1
        return out[:len(recs)]

    def decide(self, rank):
        """The device error code of the call; the engine's `geometry` says what it reached."""
        err = self.L.emu_shard_decide(self.h, rank)
        self.engines[rank]._report()
        return err

    def collect(self, rank, flush=False):
        return int(self.L.emu_shard_collect(self.h, rank, int(flush)))

    def ctl(self, rank):
        """Control words as [buffer, peer, (cnt, rflag, vflag, pad)]."""
        out = np.zeros(self.depth * self.world * 4, dtype=np.uint32)
        self.L.emu_shard_ctl(self.h, rank, _p(out))
        return out.reshape(self.depth, self.world, 4)

    def set_ctl(self, rank, words):
        w = np.ascontiguousarray(words, dtype=np.uint32).reshape(-1)
        assert len(w) == self.depth * self.world * 4
        self.L.emu_shard_set_ctl(self.h, rank, _p(w))

    def xwait(self, rank, buf, step, n_max):
        """k_xwait alone: (seg_prefix[0..world], n_dev, error words)."""
        seg = np.zeros(40, dtype=np.uint32)
        err = np.zeros(8, dtype=np.uint32)
        self.L.emu_shard_xwait(self.h, rank, buf, step, n_max, _p(seg), _p(err))
        return seg[:self.world + 1], int(seg[36]), err

    def inbox(self, owner, buf, src):
        out = np.zeros(self.cap, dtype=RECORD_DTYPE)
        self.L.emu_shard_inbox(self.h, owner, buf, src, _p(out))
        return out

    def dest(self, rank, buf):
        out = np.zeros(self.cap, dtype=np.uint32)
        self.L.emu_shard_dest(self.h, rank, buf, _p(out))
        return out

    def ctrs(self, rank):
        out = np.zeros(4, dtype=np.uint32)
        self.L.emu_shard_ctrs(self.h, rank, _p(out))
        return out

    def err(self, rank):
        out = np.zeros(8, dtype=np.uint32)
        self.L.emu_shard_err(self.h, rank, _p(out))
        return out
