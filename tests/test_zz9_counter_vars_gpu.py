"""GET /counters/{namespace} on the GPU: RLS and HTTP batches served into one service that keeps counter variables, and
the listing against the engine's counters joined with the variables the requests carried (built in Python from the
bodies), rendered by the Python restatement of serde (tests/serde_render.py).  Keeping must change nothing else."""
import re

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import http_corpora as HC
from tests import serde_render as S
from tests.http_corpora import T0

ESC = ("esc\"\\", 4, 30, [], ["descriptors[0]['a\"b']", "descriptors[0].z"], "q\"n")
LIMITS = HC.GATEWAY_LIMITS + [ESC]
_OPERAND = re.compile(r"""^descriptors\[(\d+)\](?:\.(\w+)|\[(['"])(.*)\3\])$""")


class Service:
    def __init__(self, limits=LIMITS, keep=(1 << 16, 1 << 22), **kw):
        from limitador_b200 import Engine
        self.m = MT.Matcher()
        args = dict(capacity_rows=1 << 14, cells_per_row=3, max_batch=1 << 17)
        args.update(kw)
        self.e = Engine(**args)
        self.limits = list(limits)
        self.descs = [self.m.add_limit(*l) for l in limits]
        self.e.limits_set(np.array(self.descs))
        self.rls = R.RlsService(self.m, self.e, R.HEADERS_NONE, 2)
        self.api = HA.HttpApi(self.rls)
        if keep:
            self.rls.keep_counter_vars(*keep)
        self.values = {}  # (limit_id, key_lo, key_hi) -> set_variables

    def _learn(self, ns, descs):
        """The set_variables of every counter the request may produce (descs: its descriptor maps)."""
        for d, l in zip(self.descs, self.limits):
            if l[0] != ns or not l[4]:
                continue
            sv = {}
            for v in l[4]:
                mo = _OPERAND.match(v)
                k, key = int(mo.group(1)), mo.group(2) if mo.group(2) is not None else mo.group(4)
                if k >= len(descs) or key not in descs[k]:
                    break
                sv[v] = descs[k][key]
            else:
                lo, hi = MT.counter_key(sv)
                self.values[(int(d["limit_id"]), lo, hi)] = sv

    def http(self, ep, infos, now):
        for ns, vals, _, _ in infos:
            self._learn(ns, [dict(vals)])
        self.api.serve(ep, *HA.pack_bodies([HA.encode_info(*x) for x in infos]), now)
        return self.api.responses()

    def rls_serve(self, method, reqs, now):
        for ns, vals in reqs:
            self._learn(ns, [dict(vals)])
        self.rls.serve(method, *R.pack_requests([R.encode_request(ns, [vals]) for ns, vals in reqs]), now)
        return self.rls.responses()

    def expected(self, ns, now):
        live = [(d, l) for d, l in zip(self.descs, self.limits) if l[0] == ns]
        if not live:
            return 200, b"[]"
        pos = {int(d["limit_id"]): k for k, (d, _) in enumerate(live)}
        lj = {int(d["limit_id"]): S.limit_json(l[0], int(d["max_value"]), l[2], l[5], l[3], l[4]) for d, l in live}
        rows = []
        for lid, lo, hi, rem, ttl in self.e.get_counters(list(pos), now):
            if lid in pos:
                rows.append((pos[lid], lo, hi, lj[lid], self.values[(lid, lo, hi)] if (lo, hi) != (0, 0) else {}, rem, ttl))
        return 200, S.counters_body(rows)


def _infos(rng, n, users=30):
    out = []
    for ns, vals, delta, hdr in HC.random_infos(rng, n, users):
        if rng.random() < 0.1:
            ns, vals = ESC[0], {"a\"b": ["\x01\x7f", "é\"\\", ""][int(rng.integers(0, 3))], "z": f"{int(rng.integers(0, 5))}\n"}
        out.append((ns, vals, delta, hdr))
    return out


def _reqs(rng, n, users=30):
    return [(ns, [(k, v) for k, v in vals.items()]) for ns, vals, _, _ in _infos(rng, n, users)]


NAMESPACES = ["api", "admin", ESC[0], "nobody"]


@pytest.mark.gpu
def test_mixed_traffic_lists_every_counter_with_its_variables_and_changes_nothing_else():
    rng = np.random.default_rng(1)
    on, off = Service(), Service(keep=None)
    for step in range(6):
        now = T0 + step * 7_000_000
        infos, reqs = _infos(rng, 1500), _reqs(rng, 1500)
        ep = [HA.CHECK_AND_REPORT, HA.REPORT, HA.CHECK][step % 3]
        assert on.http(ep, infos, now) == off.http(ep, infos, now)
        m = [R.SHOULD_RATE_LIMIT, R.REPORT, R.CHECK_RATE_LIMIT][step % 3]
        assert on.rls_serve(m, reqs, now) == off.rls_serve(m, reqs, now)
        for ns in NAMESPACES:
            assert on.api.get_counters(ns, now + 1) == on.expected(ns, now + 1), (step, ns)
    assert on.rls.metrics() == off.rls.metrics()
    ids = [int(d["limit_id"]) for d in on.descs]
    assert on.e.get_counters(ids, now) == off.e.get_counters(ids, now)
    assert on.rls.counter_vars_stats()["dropped"] == 0
    # keeping off: qualified counters cannot be listed
    assert off.api.get_counters("api", now)[0] == 500 and off.api.last_unnamed > 0
    assert off.api.get_counters("nobody", now) == (200, b"[]")


@pytest.mark.gpu
def test_lifecycle_expiry_sweep_gc_delete_and_update():
    rng = np.random.default_rng(2)
    s = Service()
    s.http(HA.CHECK_AND_REPORT, _infos(rng, 2000), T0)
    s.rls_serve(R.SHOULD_RATE_LIMIT, _reqs(rng, 2000), T0 + 5_000_000)
    now = T0 + 20_000_000  # the 10 s (admin) counters are gone, the rest live
    before = {ns: s.api.get_counters(ns, now) for ns in NAMESPACES}
    for ns in NAMESPACES:
        assert before[ns] == s.expected(ns, now)
    assert before["admin"] == (200, b"[]")
    keys = s.rls.counter_vars_stats()["keys"]
    s.e.sweep(now)
    gc = s.rls.counter_vars_gc(now)
    assert gc["kept"] < keys and gc["kept"] + gc["freed"] == keys
    assert s.rls.counter_vars_stats()["keys"] == gc["kept"]
    for ns in NAMESPACES:
        assert s.api.get_counters(ns, now) == before[ns]
    # update_limit: the new max_value shows in the limit and in remaining
    d = s.m.add_limit(*(("api", 50) + HC.GATEWAY_LIMITS[0][2:]))
    s.e.limits_set(np.array([d]))
    s.descs[0] = d
    assert s.api.get_counters("api", now) == s.expected("api", now)
    assert b'"max_value":50' in s.api.get_counters("api", now)[1]
    # a deleted limit's counters leave the listing
    s.m.delete_limit(int(s.descs[2]["limit_id"]))
    del s.descs[2], s.limits[2]
    assert s.api.get_counters("api", now) == s.expected("api", now)
    assert s.api.get_limits("api")[0] == 200


@pytest.mark.gpu
def test_a_full_dictionary_answers_500_only_where_a_counter_is_unnamed_and_recovers():
    rng = np.random.default_rng(3)
    s = Service(keep=(16, 1 << 16))
    s.http(HA.CHECK_AND_REPORT, _infos(rng, 3000, users=200), T0)
    st = s.rls.counter_vars_stats()
    assert st["dropped"] > 0 and st["keys"] <= 16
    assert s.api.get_counters("api", T0 + 1)[0] == 500 and s.api.last_unnamed > 0
    s.http(HA.CHECK_AND_REPORT, [("nobody", {"user": "x"}, 1, None)], T0)
    assert s.api.get_counters("nobody", T0 + 1) == (200, b"[]")
    # everything expires, GC empties the table, new traffic is recorded again
    later = T0 + 4000 * 1_000_000
    assert s.rls.counter_vars_gc(later)["kept"] == 0
    s.http(HA.CHECK_AND_REPORT, [("api", {"method": "GET", "user": f"v{k}"}, 1, None) for k in range(5)], later)
    assert s.api.get_counters("api", later + 1) == s.expected("api", later + 1)
    assert s.api.get_counters("api", later + 1)[0] == 200


@pytest.mark.gpu
def test_a_65536_request_batch_and_the_wide_engine():
    rng = np.random.default_rng(4)
    s = Service(capacity_rows=1 << 17)
    infos = [("api", {"method": "GET", "user": f"u{int(rng.integers(0, 20000))}"}, 1, None) for _ in range(65536)]
    s.http(HA.CHECK_AND_REPORT, infos, T0)
    users = {v["user"] for _, v, _, _ in infos}
    assert s.rls.counter_vars_stats()["keys"] == len(users)
    assert s.api.get_counters("api", T0 + 1) == s.expected("api", T0 + 1)
    # 50 limits in one namespace, up to 50 counters per request
    from tests import rls_corpora as RC
    w = Service(limits=RC.wide_limits(), max_counters_per_request=64)
    w.m.set_counter_cap(64)
    msgs = RC.wide_messages(5, 2000)
    w.rls.serve(R.SHOULD_RATE_LIMIT, *R.pack_requests(msgs), T0)
    for msg in msgs:
        ns, descs, _ = R.decode_request(msg)
        if descs:
            w._learn(ns, [dict(x) for x in descs])
    assert w.rls.counter_vars_stats()["dropped"] == 0
    ns = RC.wide_limits()[0][0]
    assert w.api.get_counters(ns, T0 + 1) == w.expected(ns, T0 + 1)
