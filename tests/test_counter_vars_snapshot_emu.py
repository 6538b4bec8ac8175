"""Counter variable snapshots (include/rl_rls.h: rl_rls_counter_vars_export / _import) without a GPU: the export, check
and import kernels of limitador_b200/csrc/rl_cvars_dev.cuh under tests/emu/cuda_shim.h (tests/emu/emu_cvars_snap.cpp),
over dictionaries the RLS and HTTP plans recorded.  The export must be the Python map of the decoded requests limited
to the live counters; an import into an empty dictionary must give the same lookups; every corrupted entry must be
refused at its index with nothing changed.  Under the fiber emulator 256 threads of one block race to import one key
twice.  The check parser runs once more under ASan + UBSan (tests/san/san_cvars_snap.cpp)."""
import ctypes as C
import functools
import os
import struct

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import http_corpora as HC
from tests import rls_corpora as RC
from tests.test_counter_vars_emu import Dict, Limits, T0, _emu, blob, expected, http_contexts, rls_contexts
from tests.test_rls_device_emu import matcher_image

RL_OK, RL_TRANSIENT, RL_FATAL = 0, 1, 2
VARSET, LENGTH, TRAILING, VALUE, DIGEST, DUPLICATE = 1, 2, 3, 4, 5, 6


@functools.cache
def _snap(simt=False):
    """tests/emu/emu_cvars_snap.cpp (which includes emu_cvars.cpp) under the host shim or the fiber emulator."""
    L = H.host_lib("emu_cvars_snap.cpp", "librl_emu_cvars_snap_simt.so" if simt else "librl_emu_cvars_snap.so",
                   ["EMU_SIMT"] if simt else [])
    E = _emu(simt)
    for name in ("emu_cv_seed", "emu_cv_create", "emu_cv_destroy", "emu_cv_stats", "emu_cv_plan_record", "emu_cv_dump",
                 "emu_cv_arena", "emu_cv_lookup", "emu_cv_gc") + (("emu_cv_interleave",) if simt else ()):
        f, g = getattr(L, name), getattr(E, name)
        f.argtypes, f.restype = g.argtypes, g.restype
    vp, u64 = C.c_void_p, C.c_uint64
    L.emu_cvs_export.restype = u64
    L.emu_cvs_export.argtypes = [vp, vp, u64, vp, vp, vp, u64, u64, vp, vp, vp, vp, vp, C.POINTER(u64)]
    L.emu_cvs_import.restype = C.c_int
    L.emu_cvs_import.argtypes = [vp, vp, u64, vp, vp, vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
    L.emu_cvs_check_entry.restype = C.c_uint32
    L.emu_cvs_check_entry.argtypes = [vp, C.c_uint32, u64, u64, vp, u64]
    return L


class SnapDict(Dict):
    def __init__(self, max_keys=1 << 14, arena_bytes=1 << 20, simt=False):
        self.L = _snap(simt)
        self.h = self.L.emu_cv_create(max_keys, arena_bytes)
        self.interleave = None

    def export(self, m, live):
        """-> (varset, key_lo, key_hi, blob_off, blobs) of the entries the live counters [(limit_id, lo, hi)] reference."""
        img, _ = matcher_image(m)
        lid = np.ascontiguousarray([c[0] for c in live] or [0], np.uint32)
        lo = np.ascontiguousarray([c[1] for c in live] or [0], np.uint64)
        hi = np.ascontiguousarray([c[2] for c in live] or [0], np.uint64)
        nb = C.c_uint64()
        k = self.L.emu_cvs_export(self.h, img.ctypes.data, len(live), lid.ctypes.data, lo.ctypes.data, hi.ctypes.data, 0, 0,
                                  None, None, None, None, None, C.byref(nb))
        vs, klo, khi = np.zeros(max(k, 1), np.uint32), np.zeros(max(k, 1), np.uint64), np.zeros(max(k, 1), np.uint64)
        off, b = np.zeros(k + 1, np.uint64), np.zeros(max(nb.value, 1), np.uint8)
        if k:
            assert self.L.emu_cvs_export(self.h, img.ctypes.data, len(live), lid.ctypes.data, lo.ctypes.data, hi.ctypes.data, k,
                                         nb.value, vs.ctypes.data, klo.ctypes.data, khi.ctypes.data, off.ctypes.data,
                                         b.ctypes.data, C.byref(nb)) == k
        return vs[:k], klo[:k], khi[:k], off, b[:nb.value]

    def import_(self, m, vs, lo, hi, off, b):
        """-> (status, added, bad word)."""
        img, _ = matcher_image(m)
        vs, lo, hi = (np.ascontiguousarray(x, t) for x, t in ((vs, np.uint32), (lo, np.uint64), (hi, np.uint64)))
        off, b = np.ascontiguousarray(off, np.uint64), np.ascontiguousarray(b, np.uint8)
        keep = [np.zeros(1, np.uint8)]
        ptr = lambda a: a.ctypes.data if len(a) else keep[0].ctypes.data  # noqa: E731
        added, bad = C.c_uint64(), C.c_uint64()
        st = self.L.emu_cvs_import(self.h, img.ctypes.data, len(vs), ptr(vs), ptr(lo), ptr(hi), off.ctypes.data, ptr(b),
                                   C.byref(added), C.byref(bad))
        return st, added.value, bad.value

    def snapshot(self):
        return self.entries()[0], self.stats()


def as_map(vs, lo, hi, off, b):
    raw = b.tobytes()
    return {(int(vs[i]), int(lo[i]), int(hi[i])): raw[int(off[i]):int(off[i + 1])] for i in range(len(vs))}


def from_map(entries):
    """{(varset, lo, hi): blob} (or a list of pairs, repeats kept) -> the five import arrays."""
    items = list(entries.items()) if isinstance(entries, dict) else list(entries)
    vs = np.array([k[0] for k, _ in items], np.uint32)
    lo = np.array([k[1] for k, _ in items], np.uint64)
    hi = np.array([k[2] for k, _ in items], np.uint64)
    off = np.zeros(len(items) + 1, np.uint64)
    off[1:] = np.cumsum([len(v) for _, v in items])
    return vs, lo, hi, off, np.frombuffer(b"".join(v for _, v in items), np.uint8).copy()


def _recorded(http, name_or_ep):
    """A dictionary the plans filled, its matcher, the limits, the expected map and the plan's counters."""
    d = SnapDict()
    if http:
        rng = np.random.default_rng(30 + name_or_ep)
        h = HC.HttpHarness([])
        lims = Limits(h.m, HC.GATEWAY_LIMITS + [("esc", 9, 60, [], ["descriptors[0]['a\"b']", "descriptors[0].z"], None)])
        bodies = [HA.encode_info(*x) for x in HC.random_infos(rng, 600, users=50)]
        bodies += [HA.encode_info("esc", {"a\"b": "\x01\x7f\"\\é😀", "z": ""}, 1)]
        d.record(h.m, True, name_or_ep, bodies)
        p = h.api.plan(name_or_ep, *HA.pack_bodies(bodies), T0)
        return d, h.m, lims, expected(lims, p, http_contexts(bodies)), p
    limits, msgs = RC.corpora()[name_or_ep]
    m = MT.Matcher()
    lims = Limits(m, limits)
    svc = R.RlsService(m, None, R.HEADERS_NONE, 2)
    d.record(m, False, R.SHOULD_RATE_LIMIT, msgs)
    p = svc.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests(msgs), T0)
    return d, m, lims, expected(lims, p, rls_contexts(msgs)), p


def _cases():
    return [(False, n) for n in sorted(RC.corpora())] + [(True, ep) for ep in (HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT)]


@pytest.mark.parametrize("http,which", _cases())
def test_export_is_the_map_of_the_live_counters_and_an_import_gives_the_same_lookups(http, which):
    d, m, lims, want, p = _recorded(http, which)
    ctrs = sorted({(int(c["limit_id"]), int(c["key_lo"]), int(c["key_hi"])) for c in p["ctrs"]})
    rng = np.random.default_rng(len(ctrs))
    for live in (ctrs, [c for c in ctrs if rng.random() < 0.5], []):  # all, the ones "present at now_us", none
        got = as_map(*d.export(m, live))
        ref = {(lims.by_id[l][0], lo, hi): want[(lims.by_id[l][0], lo, hi)] for l, lo, hi in live if lims.by_id[l][0]}
        assert got == ref
        e = SnapDict()
        st, added, bad = e.import_(m, *d.export(m, live))
        assert (st, added, bad) == (RL_OK, len(ref), (1 << 64) - 1)
        looked = e.lookup(m, ctrs)
        for c, b0, b1 in zip(ctrs, d.lookup(m, ctrs), looked):
            vs = lims.by_id[c[0]][0]
            assert b1 == (b0 if not vs or (vs, c[1], c[2]) in ref else None)
        assert e.entries()[0] == ref and e.stats()["arena_used"] == sum(map(len, ref.values()))


def test_export_of_selected_namespaces():
    """The live counters are what rl_counters_export lists for ns_ids: the export follows them, nothing else."""
    h = HC.HttpHarness([])
    descs = [h.m.add_limit(*l) for l in HC.GATEWAY_LIMITS]
    lims = Limits(h.m, HC.GATEWAY_LIMITS)
    bodies = [HA.encode_info(*x) for x in HC.random_infos(np.random.default_rng(3), 500, users=40)]
    d = SnapDict()
    d.record(h.m, True, HA.CHECK_AND_REPORT, bodies)
    p = h.api.plan(HA.CHECK_AND_REPORT, *HA.pack_bodies(bodies), T0)
    want = expected(lims, p, http_contexts(bodies))
    ns_of = {int(x["limit_id"]): int(x["ns_id"]) for x in descs}
    ctrs = sorted({(int(c["limit_id"]), int(c["key_lo"]), int(c["key_hi"])) for c in p["ctrs"]})
    for ns in sorted(set(ns_of.values())):
        live = [c for c in ctrs if ns_of[c[0]] == ns]
        ref = {(lims.by_id[l][0], lo, hi): want[(lims.by_id[l][0], lo, hi)] for l, lo, hi in live if lims.by_id[l][0]}
        assert as_map(*d.export(h.m, live)) == ref


def _valid():
    """A matcher with one- and two-variable limits and a map of valid entries."""
    m = MT.Matcher()
    lims = Limits(m, [("a", 5, 60, [], ["descriptors[0].user"], None),
                      ("b", 5, 60, [], ["descriptors[0].user", "descriptors[0].app"], None),
                      ("b", 7, 30, [], ["descriptors[0].app", "descriptors[0].user"], None)])
    entries = {}
    for vs, srcs in {v[0]: v[1] for v in lims.by_id.values()}.items():
        for k in range(20):
            vals = [f"u{k}é", f"app{k % 3}"][:len(srcs)]
            entries[(vs,) + MT.counter_key(dict(zip(srcs, vals)))] = blob(vals)
    return m, lims, entries


def _patch(entries, k, blob_bytes=None, varset=None):
    items = list(entries.items())
    key, b = items[k]
    if varset is not None:
        key = (varset,) + key[1:]
    items[k] = (key, b if blob_bytes is None else blob_bytes)
    return items


def _corruptions(m, lims, entries):
    items = list(entries.items())
    k = len(items) // 2
    (vs, lo, hi), b = items[k]
    other = next(v for v, _ in lims.by_id.values() if v != vs)
    n0 = struct.unpack_from("<I", b, 0)[0]
    flip = bytearray(b)
    flip[4] ^= 0x02  # an ASCII letter stays an ASCII letter
    nul, bad8 = bytearray(b), bytearray(b)
    nul[4], bad8[4] = 0, 0xFF
    big = bytearray(b)
    struct.pack_into("<I", big, 0, 0xFFFFFFF0)
    assert n0 > 0
    return {
        "flipped byte": (_patch(entries, k, bytes(flip)), k, {DIGEST}),
        "wrong varset": (_patch(entries, k, varset=other), k, {DIGEST, LENGTH, TRAILING}),
        "unknown varset": (_patch(entries, k, varset=999), k, {VARSET}),
        "varset 0": (_patch(entries, k, varset=0), k, {VARSET}),
        "truncated": (_patch(entries, k, b[:-1]), k, {LENGTH}),
        "no bytes": (_patch(entries, k, b""), k, {LENGTH}),
        "trailing bytes": (_patch(entries, k, b + b"x"), k, {TRAILING}),
        "length near 2^32": (_patch(entries, k, bytes(big)), k, {LENGTH}),
        "NUL": (_patch(entries, k, bytes(nul)), k, {VALUE}),
        "invalid UTF-8": (_patch(entries, k, bytes(bad8)), k, {VALUE}),
        "duplicate key": (items + [items[k]], len(items), {DUPLICATE}),
    }


@pytest.mark.parametrize("case", ["flipped byte", "wrong varset", "unknown varset", "varset 0", "truncated", "no bytes",
                                  "trailing bytes", "length near 2^32", "NUL", "invalid UTF-8", "duplicate key"])
def test_each_corruption_is_refused_at_its_index_and_changes_nothing(case):
    m, lims, entries = _valid()
    items, at, reasons = _corruptions(m, lims, entries)[case]
    if case != "duplicate key":  # (a repeated key is found only once every entry passed its check)
        items = items + [((lims.by_id[0][0], 1, 2), blob(["x"]))]  # a second bad entry after it: the first is named
    d = SnapDict()
    part = dict(list(entries.items())[:5])
    assert d.import_(m, *from_map(part))[:2] == (RL_OK, 5)
    before = d.snapshot()
    st, added, bad = d.import_(m, *from_map(items))
    assert st == RL_FATAL and added == 0 and bad >> 8 == at and bad & 0xFF in reasons, (case, bad >> 8, bad & 0xFF)
    assert d.snapshot() == before


def test_blob_off_that_decreases_is_refused():
    m, _, entries = _valid()
    vs, lo, hi, off, b = from_map(entries)
    off[4] = off[5] + 1
    d = SnapDict()
    assert d.import_(m, vs, lo, hi, off, b) == (RL_FATAL, 0, 4 << 8)
    assert d.stats()["keys"] == 0


def test_keys_already_present_are_skipped():
    m, _, entries = _valid()
    items = list(entries.items())
    d = SnapDict()
    assert d.import_(m, *from_map(dict(items[:25])))[:2] == (RL_OK, 25)
    first = d.snapshot()
    assert d.import_(m, *from_map(dict(items[:25])))[:2] == (RL_OK, 0)
    assert d.snapshot() == first
    assert d.import_(m, *from_map(entries))[:2] == (RL_OK, len(items) - 25)
    assert d.entries()[0] == entries
    assert d.stats()["arena_used"] == sum(map(len, entries.values()))  # the import compacts


def test_a_dictionary_too_small_is_transient_and_unchanged():
    m, _, entries = _valid()
    items = list(entries.items())
    d = SnapDict(max_keys=16)
    assert d.import_(m, *from_map(dict(items[:10])))[:2] == (RL_OK, 10)
    before = d.snapshot()
    assert d.import_(m, *from_map(entries)) == (RL_TRANSIENT, 0, 1)  # no free slot within the probe length
    assert d.snapshot() == before
    arena = sum(len(b) for _, b in items[:10]) + 5
    d2 = SnapDict(arena_bytes=arena)
    assert d2.import_(m, *from_map(dict(items[:10])))[:2] == (RL_OK, 10)
    before = d2.snapshot()
    assert d2.import_(m, *from_map(dict(items[:11]))) == (RL_TRANSIENT, 0, 0)  # no room in the arena
    assert d2.snapshot() == before


def test_a_recorded_dictionary_keeps_its_dropped_count_through_an_import():
    h = HC.HttpHarness([])
    Limits(h.m, [("n", 5, 60, [], ["descriptors[0].user"], None)])
    d = SnapDict(max_keys=16)
    d.record(h.m, True, HA.CHECK, [HA.encode_info("n", {"user": f"u{k:03d}"}, 1) for k in range(20)])
    assert d.stats()["dropped"] == 4
    st = d.stats()
    ent = d.entries()[0]
    # its own entries again (all present) and an empty import: nothing changes, dropped included
    assert d.import_(h.m, *from_map(ent)) == (RL_OK, 0, (1 << 64) - 1) and d.stats() == st
    assert d.import_(h.m, *from_map({})) == (RL_OK, 0, (1 << 64) - 1) and d.stats() == st


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_256_threads_of_one_block_importing_one_key_twice_are_refused(seed):
    """Under the fiber emulator with every atomic switching: 256 entries naming one key race for its slot in one block;
    exactly one claims it, the others see it held, and the fresh table is not swapped in."""
    m, _, entries = _valid()
    key, b = next(iter(entries.items()))
    d = SnapDict(simt=True)
    assert d.import_(m, *from_map(dict(list(entries.items())[1:4])))[:2] == (RL_OK, 3)
    before = d.snapshot()
    d.L.emu_cv_interleave(1, seed, 1.0)
    try:
        st, added, bad = d.import_(m, *from_map([(key, b)] * 256))
    finally:
        d.L.emu_cv_interleave(0, 0, 1.0)
    assert (st, added, bad) == (RL_FATAL, 0, 1 << 8 | DUPLICATE)
    assert d.snapshot() == before
    # the same key once imports
    d.L.emu_cv_interleave(1, seed, 1.0)
    try:
        assert d.import_(m, *from_map([(key, b)]))[:2] == (RL_OK, 1)
    finally:
        d.L.emu_cv_interleave(0, 0, 1.0)


def test_check_entry_matches_the_python_rules():
    """rl_cv_check_entry on single blobs: every valid blob passes, every prefix and extension of it fails."""
    m, lims, entries = _valid()
    img, _ = matcher_image(m)
    L = _snap()
    for (vs, lo, hi), b in list(entries.items())[::7]:
        buf = np.frombuffer(b + b"\0", np.uint8).copy()
        assert L.emu_cvs_check_entry(img.ctypes.data, vs, lo, hi, buf.ctypes.data, len(b)) == 0
        for cut in range(len(b)):
            assert L.emu_cvs_check_entry(img.ctypes.data, vs, lo, hi, buf.ctypes.data, cut) in (LENGTH, TRAILING)
        assert L.emu_cvs_check_entry(img.ctypes.data, vs, lo, hi, buf.ctypes.data, len(b) + 1) == TRAILING
        assert L.emu_cvs_check_entry(img.ctypes.data, vs, lo ^ 1, hi, buf.ctypes.data, len(b)) == DIGEST
        assert L.emu_cvs_check_entry(img.ctypes.data, vs, lo, hi | 1 << 32, buf.ctypes.data, len(b)) == DIGEST


def test_check_parser_is_clean_under_asan_and_ubsan(tmp_path):
    """Random and adversarial blobs through rl_cv_check_entry, and imports of them, under ASan + UBSan."""
    from tests.test_sanitizers import build_and_run
    root = H.ROOT
    csrc = os.path.join(root, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(root, "tests", "san", "san_cvars_snap.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(root, "include")], extra=("-std=c++17",))
    assert out.startswith("ok valid=")
