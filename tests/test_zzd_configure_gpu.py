"""RlsService.configure_with on the GPU: mixed RLS and HTTP traffic through a service that keeps counter variables, with a
sequence of configurations applied between the batches (keep, raise and lower a max, rename, delete, re-add, duplicate,
empty a namespace, one refused).  The same requests and the same configure_with calls go through limiter.RateLimiter over
the CPU oracle; verdicts, response bytes, X-RateLimit-* headers, GET /counters and GET /limits bodies and the metrics
agree at every step, the counters of kept limits are untouched by every reload, and the refused one changes nothing."""
import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import limiter as LM
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import helpers as H
from tests import serde_render as S
from tests.http_corpora import T0, random_infos

GET = "descriptors[0].method == 'GET'"
POST = "descriptors[0].method == 'POST'"
USER = "descriptors[0].user"
NAMESPACES = ["api", "admin", "nobody", ""]


def L(ns, mx, secs, conds, vars_, name=None, id=None):
    return {"namespace": ns, "max_value": mx, "seconds": secs, "conditions": conds, "variables": vars_, "name": name, "id": id}


G, P, HR = L("api", 5, 60, [GET], [USER], "get"), L("api", 3, 60, [POST], [USER], "post"), L("api", 40, 3600, [], [USER], "hourly")
GL = L("api", 120, 60, ["descriptors[0].method != 'OPTIONS'"], [], "global")
AD = L("admin", 2, 10, [], [USER, "descriptors[0].path"])
PA = L("api", 2, 10, ["descriptors[0].path == '/a'"], [USER], "path-a", "pa")
BAD = L("api", 1, 60, ["descriptors[0].path.matches('x')"], [])

# (configuration, refused entry or None)
STEPS = [
    ([G, P, HR, GL, AD], None),
    ([dict(G, max_value=8), dict(P, max_value=1), dict(HR, name="hourly-2", id="h"), GL, AD], None),  # raise, lower, rename
    ([dict(G, max_value=8), dict(P, max_value=1), dict(HR, name="hourly-2", id="h"), AD, PA], None),  # delete GL, add PA
    ([dict(G, max_value=8), dict(P, max_value=1), dict(HR, name="hourly-2", id="other"), AD, PA, GL, dict(G, max_value=1)], None),
    ([dict(G, max_value=8), dict(P, max_value=1), dict(HR, name="hourly-2"), PA, GL], None),  # admin emptied
    ([G, P, BAD, HR], 2),
    ([dict(G, max_value=8), dict(P, max_value=1), dict(HR, name="hourly-2"), PA, GL, AD], None),  # admin back, fresh
]


def ident(l):
    return (l["namespace"], l["seconds"], tuple(sorted(set(l["conditions"]))), tuple(sorted(set(l["variables"]))))


class Pair:
    """The service under test and the mirror, fed the same requests and configurations."""

    def __init__(self, cap=None, **engine_kw):
        from limitador_b200 import Engine
        self.m = MT.Matcher()
        if cap:
            self.m.set_counter_cap(cap)
        self.e = Engine(capacity_rows=1 << 14, cells_per_row=3, max_batch=1 << 16, **engine_kw)
        self.rls = R.RlsService(self.m, self.e, R.HEADERS_DRAFT_VERSION_03, 2, use_limit_name_label=True)
        self.api = HA.HttpApi(self.rls)
        self.rls.keep_counter_vars(1 << 16, 1 << 22)
        clock = self.clock = {"t": T0}  # (a lambda over self would put the engine in a cycle the collector frees in any order)
        self.rl = LM.RateLimiter(H.OracleStorage(), clock=lambda: clock["t"])
        self.ids = {}    # identity -> our limit_id (dense, in order of first appearance)
        self.live = {}   # identity -> the limit as configured
        self.want_m = {}

    def configure(self, limits):
        rep = self.rls.configure_with(limits)
        first = {}
        for l in limits:
            first.setdefault(ident(l), l)  # HashSet::insert keeps the first of two equal limits
        for k in first:
            self.ids.setdefault(k, len(self.ids))
        self.live = first
        self.rl.configure_with([LM.Limit(l["namespace"], l["max_value"], l["seconds"], l["conditions"], l["variables"],
                                         l["name"], l["id"]) for l in first.values()])
        return rep

    def close(self):
        """The service before its engine: a test's frames can hold this object in a cycle, and the collector finalizes
        a cycle's objects in any order."""
        self.api.close()
        self.rls.close()
        self.e.close()

    def count(self, key, v=1):
        self.want_m[key] = self.want_m.get(key, 0) + v

    def traffic(self, rng, step, now):
        self.clock["t"] = now
        ep = [HA.CHECK_AND_REPORT, HA.CHECK, HA.REPORT][step % 3]
        infos = random_infos(rng, 600, users=5)
        self.api.serve(ep, *HA.pack_bodies([HA.encode_info(*x) for x in infos]), now)
        for (ns, values, delta, hdr), got in zip(infos, self.api.responses()):
            ctx = LM.Context({}, [dict(values)])
            if ep == HA.REPORT:
                self.rl.update_counters(ns, ctx, delta)
                assert got == (200, b"null", {})
            elif ep == HA.CHECK:
                w = self.rl.is_rate_limited(ns, ctx, delta)
                assert got == ((429, b"Too many requests") if w.limited else (200, b"null")) + ({},)
            else:
                w = self.rl.check_rate_limited_and_update(ns, ctx, delta, hdr is not None)
                assert got == (429 if w.limited else 200, b"null", w.response_header() if hdr == "DraftVersion03" else {})
                if w.limited:
                    self.count(f'limited_calls{{limitador_namespace="{ns}",limit_name="{w.limit_name or ""}"}}')
                else:
                    self.count(f'authorized_calls{{limitador_namespace="{ns}"}}')
                    self.count(f'authorized_hits{{limitador_namespace="{ns}"}}', delta)
        reqs = [(ns, [(k, v) for k, v in values.items()], delta) for ns, values, delta, _ in random_infos(rng, 600, users=5)]
        self.rls.serve(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request(ns, [d], h) for ns, d, h in reqs]), now)
        limited = 0
        for (ns, d, h), (grpc, body) in zip(reqs, self.rls.responses()):
            assert grpc == R.GRPC_OK
            if not ns:
                assert body == b""
                continue
            w = self.rl.check_rate_limited_and_update(ns, LM.Context({}, [dict(d)]), h or 1, True)
            hdrs = sorted(w.response_header().items())
            assert body == R.encode_response(R.CODE_OVER_LIMIT if w.limited else R.CODE_OK, hdrs), (ns, d)
            limited += w.limited
            if w.limited:
                self.count(f'limited_calls{{limitador_namespace="{ns}",limit_name="{w.limit_name or ""}"}}')
            else:
                self.count(f'authorized_calls{{limitador_namespace="{ns}"}}')
                self.count(f'authorized_hits{{limitador_namespace="{ns}"}}', h or 1)
        return limited

    def metrics(self):
        out = {}
        for line in self.rls.metrics().splitlines():
            if line and not line.startswith("#") and not line.startswith("limitador_up"):
                k, v = line.rsplit(" ", 1)
                out[k] = int(v)
        return out

    def _limit_json(self, l):
        j = S.limit_json(l.namespace, l.max_value, l.seconds, l.name, l.conditions, l.variables)
        return j if l.id is None else '{"id":' + S.ser_str(l.id) + j[len('{"id":null'):]

    def expected_gets(self, now):
        out = []
        for ns in NAMESPACES:
            lims = list(self.rl._limits.get(ns, {}).values())
            pos = {self.rl._limit_ids[l.identity()]: k for k, l in enumerate(lims)}
            rows = [(pos[c.limit_id], *c.key(), self._limit_json(c.limit), c.set_variables, c.remaining, c.expires_in_us)
                    for c in self.rl.get_counters(ns)]
            out.append(((200, S.counters_body(rows)), (200, ("[" + ",".join(self._limit_json(l) for l in lims) + "]").encode())))
        return out

    def gets(self, now):
        return [(self.api.get_counters(ns, now), self.api.get_limits(ns)) for ns in NAMESPACES]

    def export(self, ids=None):
        lid, lo, hi, val, exp = self.e.export_counters()
        rows = sorted(zip(lid.tolist(), lo.tolist(), hi.tolist(), val.tolist(), exp.tolist()))
        return rows if ids is None else [r for r in rows if r[0] in ids]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [{}, {"max_counters_per_request": 64, "cap": 64}, {"flags": 2}], ids=["default", "wide", "pipeline"])
def test_reloads_between_batches_match_the_mirror_and_keep_the_counters_of_kept_limits(cfg):
    s = Pair(**cfg)
    try:
        _reloads(s)
    finally:
        s.close()


def _reloads(s):
    rng = np.random.default_rng(7)
    limited = 0
    now = T0
    for step, (limits, refused) in enumerate(STEPS):
        now = T0 + step * 2_000_000
        s.clock["t"] = now
        if refused is not None:
            before = (s.export(), s.gets(now), s.rls.metrics(), s.rls.config_status())
            with pytest.raises(R.ConfigureError) as e:
                s.rls.configure_with(limits)
            assert e.value.index == refused and str(e.value).startswith(f"entry {refused}: unsupported condition")
            assert s.export() == before[0] and s.gets(now) == before[1] and s.rls.metrics() == before[2]
            assert s.rls.config_status()["config_err_since"] == 1
        else:
            new = {ident(l) for l in limits}
            kept = {s.ids[k] for k in s.live if k in new}
            gone = sum(k not in new for k in s.live)
            before = s.export(kept)
            rep = s.configure(limits)
            assert s.export(kept) == before, step
            assert (rep["kept"] + rep["updated"], rep["deleted"]) == (len(kept), gone), (step, rep)
            assert s.rls.config_status() == {"config_version": sum(r is None for _, r in STEPS[:step + 1]), "config_err_since": 0}
        assert s.gets(now) == s.expected_gets(now), step
        limited += s.traffic(rng, step, now)
        assert s.gets(now) == s.expected_gets(now), step
        assert s.metrics() == {k: v for k, v in s.want_m.items() if v}, step  # a series at 0 is not written
    assert limited > 100
    # the emptied and re-added namespace started from fresh counters, and the reload left the dictionary collectable
    assert s.rls.counter_vars_gc(now)["kept"] > 0
    assert s.gets(now) == s.expected_gets(now)


@pytest.mark.gpu
def test_report_counts_and_a_namespace_left_without_limits_makes_no_store_call():
    s = Pair()
    try:
        _emptied(s)
    finally:
        s.close()


def _emptied(s):
    s.configure([G, AD])
    s.traffic(np.random.default_rng(3), 0, T0)
    assert s.configure([G]) == {"kept": 1, "added": 0, "updated": 0, "deleted": 1}
    s.rls.serve(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request("admin", [[("user", "u1"), ("path", "/a")]])] * 5), T0 + 1)
    assert [R.decode_response(b) for _, b in s.rls.responses()] == [(R.CODE_OK, [])] * 5
    assert s.api.get_limits("admin") == (200, b"[]") and s.api.get_counters("admin", T0 + 1) == (200, b"[]")
    assert 'authorized_calls{limitador_namespace="admin"}' in s.rls.metrics()  # the series keep their values
