"""Counter snapshots that carry the counter variables (RlsService.save_counters / load_counters,
rl_rls_counter_vars_export / _import) on the GPU: a restarted service on an engine of another shape answers GET
/counters and GET /limits byte for byte as the old one and serves the next batches identically; Engine.load_counters
alone still leaves the restored qualified counters unnamed; two services re-shard into three; every refusal changes
nothing; a million keys round-trip."""
import numpy as np
import pytest

from limitador_b200 import exchange
from limitador_b200 import http_api as HA
from limitador_b200 import rls as R
from tests.http_corpora import T0
from tests.test_zz9_counter_vars_gpu import NAMESPACES, Service, _infos, _reqs


def _traffic(s, rng, steps, now0, owned=None):
    """Mixed HTTP and RLS batches; with `owned`, only requests of those namespaces (a shard's share)."""
    now = now0
    for step in range(steps):
        now = now0 + step * 3_000_000
        infos = [x for x in _infos(rng, 1200) if owned is None or x[0] in owned]
        reqs = [x for x in _reqs(rng, 1200) if owned is None or x[0] in owned]
        if infos:
            s.http([HA.CHECK_AND_REPORT, HA.REPORT, HA.CHECK][step % 3], infos, now)
        if reqs:
            s.rls_serve([R.SHOULD_RATE_LIMIT, R.REPORT, R.CHECK_RATE_LIMIT][step % 3], reqs, now)
    return now


def _gets(s, now):
    return [(s.api.get_counters(ns, now), s.api.get_limits(ns)) for ns in NAMESPACES]


def _metrics(s):
    out = {}
    for line in s.rls.metrics().splitlines():
        if line and not line.startswith("#"):
            k, v = line.rsplit(" ", 1)
            out[k] = float(v)
    return out


def _delta(after, before):
    return {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}


@pytest.mark.gpu
def test_restart_on_another_engine_shape_answers_and_serves_as_before(tmp_path):
    rng = np.random.default_rng(11)
    a = Service()
    now = _traffic(a, rng, 6, T0)
    path = str(tmp_path / "snap.npz")
    a.rls.save_counters(path, now)
    with np.load(path) as z:
        assert {"cv_varset", "cv_key_lo", "cv_key_hi", "cv_blob_off", "cv_blobs"} <= set(z.files) and len(z["cv_varset"]) > 50
        assert (np.diff(z["cv_varset"].astype(np.int64)) >= 0).all()  # sorted by (varset, key)
    a.rls.save_counters(str(tmp_path / "again.npz"), now)  # the same state gives the same arrays
    with np.load(path) as z, np.load(str(tmp_path / "again.npz")) as z2:
        assert z.files == z2.files and all(np.array_equal(z[k], z2[k]) for k in z.files)
    b = Service(capacity_rows=1 << 13, cells_per_row=7)
    with np.load(path) as z:
        assert b.rls.load_counters(path) == len(z["cv_varset"])
    assert _gets(b, now) == _gets(a, now)
    assert all(b.api.get_counters(ns, now)[0] == 200 for ns in NAMESPACES)
    # the same next batches: the same responses, metrics deltas and listings (A swept at `now`: the state the
    # snapshot holds, where a counter whose window ended is absent rather than expired)
    a.e.sweep(now)
    b.values = a.values
    ma, mb = _metrics(a), _metrics(b)
    for step in range(3):
        t = now + (step + 1) * 2_000_000
        infos, reqs = _infos(rng, 1500), _reqs(rng, 1500)
        assert a.http(HA.CHECK_AND_REPORT, infos, t) == b.http(HA.CHECK_AND_REPORT, infos, t)
        assert a.rls_serve(R.SHOULD_RATE_LIMIT, reqs, t) == b.rls_serve(R.SHOULD_RATE_LIMIT, reqs, t)
        assert _gets(b, t) == _gets(a, t)
    assert _delta(_metrics(b), mb) == _delta(_metrics(a), ma)


@pytest.mark.gpu
def test_engine_load_counters_alone_still_leaves_the_restored_counters_unnamed(tmp_path):
    rng = np.random.default_rng(12)
    a = Service()
    now = _traffic(a, rng, 3, T0)
    path = str(tmp_path / "snap.npz")
    a.rls.save_counters(path, now)
    c = Service()
    c.e.load_counters(path)  # reads the service's file; ignores the cv_ arrays
    assert c.e.dump() == a.e.dump()
    st, _ = c.api.get_counters("api", now)
    assert st == 500 and c.api.last_unnamed > 0
    # a file Engine.save_counters wrote loads through the service as through the engine
    p2 = str(tmp_path / "engine.npz")
    a.e.save_counters(p2, now)
    d = Service()
    assert d.rls.load_counters(p2) == 0
    assert d.e.dump() == c.e.dump() and d.rls.counter_vars_stats()["keys"] == 0


def _concat(parts):
    vs = np.concatenate([p[0] for p in parts])
    lo = np.concatenate([p[1] for p in parts])
    hi = np.concatenate([p[2] for p in parts])
    offs, base = [np.zeros(1, np.uint64)], 0
    for p in parts:
        offs.append(p[3][1:] + np.uint64(base))
        base += int(p[3][-1])
    return vs, lo, hi, np.concatenate(offs), np.concatenate([p[4] for p in parts])


@pytest.mark.gpu
def test_two_services_reshard_into_three():
    ns_ids = {}
    old = [Service(), Service()]
    for d, l in zip(old[0].descs, old[0].limits):
        ns_ids[l[0]] = int(d["ns_id"])
    all_ns = np.array(sorted(set(ns_ids.values())), np.uint32)
    now = T0
    for r, s in enumerate(old):
        owned = {n for n, i in ns_ids.items() if exchange.owner_of(i, 2) == r}
        now = max(now, _traffic(s, np.random.default_rng(20 + r), 4, T0, owned))
    owner_old = {n: exchange.owner_of(i, 2) for n, i in ns_ids.items()}
    new = [Service(capacity_rows=1 << 13, cells_per_row=7) for _ in range(3)]
    for r, s in enumerate(new):
        mine = exchange.namespaces_owned(all_ns, r, 3)
        # each old rank exports the namespaces it owned (every engine holds its unqualified counters, present or not
        # served, so a namespace's counters come from its owner only)
        sel = [np.array([i for i in mine if exchange.owner_of(int(i), 2) == k], np.uint32) for k in range(2)]
        cv = _concat([o.rls.export_counter_vars(now, sel[k]) for k, o in enumerate(old)])
        s.rls.import_counter_vars(*cv)
        parts = [o.e.export_counters(now, sel[k]) for k, o in enumerate(old)]
        s.e.import_counters(*[np.concatenate([p[k] for p in parts]) for k in range(5)])
    for n, i in ns_ids.items():
        was = old[owner_old[n]].api.get_counters(n, now)
        assert was[0] == 200
        assert new[exchange.owner_of(i, 3)].api.get_counters(n, now) == was, n


def _state(s, now):
    return s.rls.counter_vars_stats(), [s.api.get_counters(ns, now) for ns in NAMESPACES]


@pytest.mark.gpu
def test_refusals_change_nothing():
    rng = np.random.default_rng(14)
    a = Service()
    now = _traffic(a, rng, 3, T0)
    vs, lo, hi, off, blobs = a.rls.export_counter_vars(now)
    assert len(vs) > 20
    b = Service()
    b.rls.import_counter_vars(vs[:10], lo[:10], hi[:10], off[:11], blobs[:int(off[10])])
    b.e.import_counters(*a.e.export_counters(now))
    before = _state(b, now)
    # an entry not held yet whose first value is not empty
    k = next(i for i in range(10, len(vs)) if int.from_bytes(blobs[int(off[i]):int(off[i]) + 4].tobytes(), "little") > 0)
    s0, s1 = int(off[k]), int(off[k + 1])

    def with_blob(new):
        items = [blobs[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(vs))]
        items[k] = new
        o = np.zeros(len(items) + 1, np.uint64)
        o[1:] = np.cumsum([len(x) for x in items])
        return vs, lo, hi, o, np.frombuffer(b"".join(items), np.uint8)

    blob = blobs[s0:s1].tobytes()
    assert len(blob) > 4 and blob[4] not in (0, 0xFF)
    flip = bytearray(blob)
    flip[-1] ^= 0x80 if flip[-1] < 0x80 else 0x01  # a different value (or invalid UTF-8): refused either way
    nul, bad8, big = bytearray(blob), bytearray(blob), bytearray(blob)
    nul[4], bad8[4] = 0, 0xFF
    big[0:4] = (0xFFFFFFF0).to_bytes(4, "little")
    vs_unknown = vs.copy()
    vs_unknown[k] = 999
    cases = {
        "flipped byte": with_blob(bytes(flip)), "truncated": with_blob(blob[:-1]), "trailing": with_blob(blob + b"x"),
        "length near 2^32": with_blob(bytes(big)), "NUL": with_blob(bytes(nul)), "invalid UTF-8": with_blob(bytes(bad8)),
        "unknown varset": (vs_unknown, lo, hi, off, blobs),
    }
    for name, arrs in cases.items():
        with pytest.raises(R.RlsError, match=f"entry {k} refused"):
            b.rls.import_counter_vars(*arrs)
        assert _state(b, now) == before, name
    # a key named twice (not held yet)
    dup = [np.concatenate([x, x[k:k + 1]]) for x in (vs, lo, hi)]
    o2 = np.concatenate([off, [off[-1] + np.uint64(s1 - s0)]])
    with pytest.raises(R.RlsError, match=f"entry {len(vs)} refused: the import names the key twice"):
        b.rls.import_counter_vars(*dup, o2, np.concatenate([blobs, blobs[s0:s1]]))
    assert _state(b, now) == before
    # keeping off: refused; the export is empty
    off_svc = Service(keep=None)
    with pytest.raises(R.RlsError, match="keeping on"):
        off_svc.rls.import_counter_vars(vs, lo, hi, off, blobs)
    assert len(off_svc.rls.export_counter_vars(now)[0]) == 0
    # a full dictionary: transient, unchanged
    small = Service(keep=(16, 1 << 16))
    small.rls.import_counter_vars(vs[:5], lo[:5], hi[:5], off[:6], blobs[:int(off[5])])
    before = small.rls.counter_vars_stats()
    with pytest.raises(R.RlsError, match="no room"):
        small.rls.import_counter_vars(vs, lo, hi, off, blobs)
    assert small.rls.counter_vars_stats() == before
    # and the whole export imports
    assert b.rls.import_counter_vars(vs, lo, hi, off, blobs) == len(vs) - 10
    assert all(b.api.get_counters(ns, now) == a.api.get_counters(ns, now) for ns in NAMESPACES)


@pytest.mark.gpu
def test_a_million_qualified_keys_round_trip(tmp_path):
    lim = [("big", 10 ** 9, 3600, [], ["descriptors[0].user"], None)]
    a = Service(limits=lim, keep=(1 << 21, 1 << 25), capacity_rows=1 << 21, cells_per_row=3, max_batch=1 << 17)
    n, batch = 1 << 20, 1 << 16
    for s in range(0, n, batch):
        bodies = [b'{"namespace":"big","values":{"user":"u%07d"},"delta":1}' % k for k in range(s, s + batch)]
        a.api.serve(HA.REPORT, *HA.pack_bodies(bodies), T0)
        assert all(r[0] == 200 for r in a.api.responses())
    st = a.rls.counter_vars_stats()
    assert st["keys"] == n and st["dropped"] == 0
    path = str(tmp_path / "big.npz")
    a.rls.save_counters(path, T0 + 1)
    b = Service(limits=lim, keep=(1 << 21, 1 << 25), capacity_rows=1 << 22, cells_per_row=1, max_batch=1 << 17)
    assert b.rls.load_counters(path) == n
    ea, eb = a.rls.export_counter_vars(T0 + 1), b.rls.export_counter_vars(T0 + 1)
    key = lambda e: {(int(v), int(l), int(h)): e[4][int(e[3][i]):int(e[3][i + 1])].tobytes()  # noqa: E731
                     for i, (v, l, h) in enumerate(zip(e[0], e[1], e[2]))}
    assert len(eb[0]) == n and key(ea) == key(eb)
    status, body = b.api.get_counters("big", T0 + 1)
    assert status == 200 and b.api.last_unnamed == 0
    assert (status, body) == a.api.get_counters("big", T0 + 1)

