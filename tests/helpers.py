"""Shared test helpers: oracle-backed CounterStorage, table assignment mirroring the
engine's row-group logic, the host emulator binding and random stream builders."""
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

LIMITDEV_DTYPE = np.dtype([("group", "<u4"), ("cell", "<u4"), ("ns_id", "<u4"), ("qualified", "<u4")])
CELLDESC_DTYPE = np.dtype([("max_value", "<u8"), ("window_us", "<u8"), ("limit_id", "<u4"), ("qualified", "<u4")])


def assign_tables(descs: np.ndarray, cells: int):
    """Mirror of rl_limits_set's row-group assignment (rl_engine.cu): limits of one
    (namespace, varset) share a row group, `cells` limits per group."""
    n_lim = int(descs["limit_id"].max()) + 1 if len(descs) else 1
    limits = np.zeros(n_lim, dtype=LIMITDEV_DTYPE)
    groups = [None]  # index 0 unused
    by_key = {}
    for d in descs:
        q = 1 if d["qualified"] else 0
        varset = int(d["varset_id"]) if q else 0
        key = (int(d["ns_id"]), varset)
        g = None
        for cand in by_key.get(key, []):
            if len(groups[cand]) < cells:
                g = cand
                break
        if g is None:
            g = len(groups)
            groups.append([])
            by_key.setdefault(key, []).append(g)
        cell = len(groups[g])
        groups[g].append(int(d["limit_id"]))
        limits[int(d["limit_id"])] = (g, cell, int(d["ns_id"]), q)
    desc = np.zeros(len(groups) * 8, dtype=CELLDESC_DTYPE)
    desc["limit_id"] = NONE
    by_id = {int(d["limit_id"]): d for d in descs}
    for g in range(1, len(groups)):
        for c, lid in enumerate(groups[g]):
            d = by_id[lid]
            desc[g * 8 + c] = (int(d["max_value"]), int(d["window_us"]), lid, 1 if d["qualified"] else 0)
    return limits, desc, len(groups)


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
    L.emu_set_tables.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32]
    L.emu_batch_csr.argtypes = [vp, C.c_int, C.c_int, C.c_uint32, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.emu_resolve.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, vp, C.c_uint32, vp, vp]
    L.emu_resolve.restype = C.c_int
    L.emu_dump.restype = C.c_uint64
    L.emu_dump.argtypes = [vp, C.c_uint64, vp, vp, vp, vp, vp]
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
        limits, desc, ngroups = assign_tables(descs, cells)
        self.L.emu_set_tables(self.h, _p(limits), len(limits), _p(desc), ngroups)
        self.rounds = 0

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
def mixed_limits(n_ns=6, seed=0):
    """A limits table exercising every row shape: single qualified limit, several limits on
    one variable set (one row), two variable sets (two rows), unqualified + qualified,
    unqualified only, max 0 / tiny / huge limits, 1 s .. 1 h windows."""
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
            mx = int(rng.choice([0, 1, 2, 3, 5, 8, 20, 1 << 40]))
            win = int(rng.choice([1, 2, 10, 60, 3600])) * 1_000_000
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


def wide_limits(seed, sizes=(20, 33, 64, 3), small=True):
    """Namespaces of `sizes` limits, qualified (three variable sets) and unqualified interleaved in registration order,
    with small maxima so that the limits bite."""
    rng = np.random.default_rng(seed)
    descs, lid = [], 0
    for ns, size in enumerate(sizes):
        for _ in range(size):
            q = 1 if rng.random() < 0.7 else 0
            varset = int(rng.integers(1, 4)) if q else 0
            mx = int(rng.choice([0, 1, 2, 3, 5, 8, 20, 1 << 40])) if small else (1 << 62)
            win = int(rng.choice([1, 2, 10, 60, 3600])) * 1_000_000
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
    return L


class EmuCrdt:
    """The CRDT kernels on the host (same interface as limitador_b200.crdt.CrdtTable)."""

    def __init__(self, capacity_rows, actors, self_actor, simt=False):
        from limitador_b200 import crdt as CR
        self.CR = CR
        self.L = emu_maint_lib(simt)
        self.actors, self.self_actor = actors, self_actor
        self.h = self.L.emu_crdt_create(capacity_rows, actors, self_actor)
        self.capacity = capacity_rows

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
        return self.L.emu_crdt_inc(self.h, n, _p(keys), _p(a), _p(inc), _p(win), now_us)

    def merge(self, ups, actors, values, now_us):
        ups = np.ascontiguousarray(ups, dtype=self.CR.UPDATE_DTYPE)
        actors = np.ascontiguousarray(actors, dtype=np.uint32)
        values = np.ascontiguousarray(values, dtype=np.uint64)
        return self.L.emu_crdt_merge(self.h, len(ups), _p(ups), _p(actors), _p(values), len(values), now_us)

    def read(self, keys, now_us):
        keys = np.ascontiguousarray(keys, dtype=self.CR.KEY_DTYPE)
        val = np.zeros(len(keys), dtype=np.uint64)
        exp = np.zeros(len(keys), dtype=np.uint64)
        assert self.L.emu_crdt_read(self.h, len(keys), _p(keys), now_us, _p(val), _p(exp)) == 0
        return val, exp

    def export(self, now_us, cap=1 << 16):
        k = np.zeros(cap, dtype=self.CR.KEY_DTYPE)
        val = np.zeros(cap, dtype=np.uint64)
        exp = np.zeros(cap, dtype=np.uint64)
        n = self.L.emu_crdt_scan(self.h, 0, now_us, cap, _p(k), _p(val), _p(exp), None)
        return sorted(zip(k["lo"][:n].tolist(), k["hi"][:n].tolist(), val[:n].tolist(), exp[:n].tolist()))

    def dump(self, cap=1 << 16):
        k = np.zeros(cap, dtype=self.CR.KEY_DTYPE)
        exp = np.zeros(cap, dtype=np.uint64)
        vals = np.zeros(cap * self.actors, dtype=np.uint64)
        n = self.L.emu_crdt_scan(self.h, 1, 0, cap, _p(k), None, _p(exp), _p(vals))
        v = vals[:n * self.actors].reshape(n, self.actors)
        return sorted((int(k["lo"][i]), int(k["hi"][i]), int(exp[i]), tuple(v[i].tolist())) for i in range(n))
