"""RlsService.configure_with (rl_rls_configure) on a service without an engine, where the matcher alone changes: identity,
update, delete, duplicates, order and all-or-nothing (DESIGN.md §9j), observed through GET /limits bodies, the CPU plan's
CSR and the limit ids; dry runs; the reference's four configure_with tests; and the limits-file parser."""
import os

import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests.http_corpora import T0

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GET = "descriptors[0].m == 'GET'"
POST = "descriptors[0].m == 'POST'"
APP = "descriptors[0].app"


def L(ns, mx, secs=60, conds=(GET,), vars_=(APP,), name=None, id=None):
    return {"namespace": ns, "max_value": mx, "seconds": secs, "conditions": list(conds), "variables": list(vars_),
            "name": name, "id": id}


class Svc:
    def __init__(self, dialect="table", cap=None):
        self.m = MT.Matcher(dialect)
        if cap:
            self.m.set_counter_cap(cap)
        self.rls = R.RlsService(self.m, None, R.HEADERS_DRAFT_VERSION_03, 2)
        self.api = HA.HttpApi(self.rls)

    def configure(self, limits, dry_run=False):
        return self.rls.configure_with(limits, dry_run)

    def limits(self, ns):
        return self.api.get_limits(ns)

    def plan(self, reqs=None):
        reqs = reqs or [(ns, [("m", m), ("app", "x")]) for ns in ("a", "b", "c") for m in ("GET", "POST")]
        p = self.rls.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request(ns, [v]) for ns, v in reqs]), T0)
        return p["n_store"], p["ctr_off"].tobytes(), p["ctrs"].tobytes(), p["store_index"].tobytes()

    def ids(self, ns, m="GET", app="x"):
        """limit ids of the counters one request of ns produces, in counter order."""
        p = self.rls.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request(ns, [[("m", m), ("app", app)]])]), T0)
        return [int(c["limit_id"]) for c in p["ctrs"]]

    def state(self):
        return [self.limits(ns) for ns in ("a", "b", "c")], self.plan()


def body(*limits):
    """GET /limits body of the given limits (limit tuples as L() takes them, in order)."""
    import json
    out = []
    for l in limits:
        out.append({"id": l["id"], "namespace": l["namespace"], "max_value": l["max_value"], "seconds": l["seconds"],
                    "name": l["name"], "conditions": sorted(set(l["conditions"])), "variables": sorted(set(l["variables"]))})
    return 200, json.dumps(out, separators=(",", ":"), ensure_ascii=False).encode()


# ---- the rules ---------------------------------------------------------------------------------------------------------
def test_identity_keeps_the_limit_id_and_a_kept_limit_is_untouched():
    s = Svc()
    a1, a2 = L("a", 10), L("a", 5, conds=(POST,))
    assert s.configure([a1, a2]) == {"kept": 0, "added": 2, "updated": 0, "deleted": 0}
    ids = s.ids("a"), s.ids("a", "POST")
    before = s.state()
    # the same identity written differently: conditions and variables are sets, order and repeats do not matter
    again = [dict(a1, conditions=[GET, GET]), dict(a2, variables=[APP, APP])]
    assert s.configure(again) == {"kept": 2, "added": 0, "updated": 0, "deleted": 0}
    assert s.state() == before and (s.ids("a"), s.ids("a", "POST")) == ids
    assert s.rls.config_status() == {"config_version": 2, "config_err_since": 0}


def test_update_takes_max_name_and_id_but_an_id_alone_changes_nothing():
    s = Svc()
    a = L("a", 10, name="n", id="one")
    s.configure([a])
    lid = s.ids("a")
    assert s.limits("a") == body(a)
    assert s.configure([dict(a, id="two")]) == {"kept": 1, "added": 0, "updated": 0, "deleted": 0}
    assert s.limits("a") == body(a)  # update_limit compares max_value and name only
    for change in ({"max_value": 3, "id": "three"}, {"name": "m", "id": None}, {"name": None, "id": 'q"\n'}):
        b = dict(a, **change)
        assert s.configure([b]) == {"kept": 0, "added": 0, "updated": 1, "deleted": 0}
        assert s.limits("a") == body(b) and s.ids("a") == lid
        a = b


def test_delete_and_re_add_bring_the_old_id_back_at_the_end_and_an_empty_namespace_answers_as_unknown():
    s = Svc()
    a1, a2, a3 = L("a", 1), L("a", 2, conds=(POST,)), L("a", 3, vars_=())
    b1 = L("b", 4)
    s.configure([a1, a2, a3, b1])
    ids = {k: v for k, v in zip(("a1", "a3"), s.ids("a"))}
    assert s.configure([a2, a3, b1]) == {"kept": 3, "added": 0, "updated": 0, "deleted": 1}
    assert s.limits("a") == body(a2, a3) and s.ids("a") == [ids["a3"]]
    # re-added: the old limit_id, behind the kept ones
    assert s.configure([a1, a2, a3, b1]) == {"kept": 3, "added": 1, "updated": 0, "deleted": 0}
    assert s.limits("a") == body(a2, a3, a1) and s.ids("a") == [ids["a3"], ids["a1"]]
    # namespace b emptied: no counter, no store call, and GET /limits answers []
    assert s.configure([a1]) == {"kept": 1, "added": 0, "updated": 0, "deleted": 3}
    assert s.limits("b") == (200, b"[]") == s.limits("never")
    p = s.rls.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request("b", [[("m", "GET"), ("app", "x")]]),
                                                          R.encode_request("never", [[("m", "GET")]])]), T0)
    assert p["n_store"] == 0
    s.rls.finish()
    assert [R.decode_response(b) for _, b in s.rls.responses()] == [(R.CODE_OK, [])] * 2


def test_duplicates_the_first_entry_wins():
    s = Svc()
    first, second = L("a", 7, name="first", id="1"), L("a", 9, name="second", id="2")
    assert s.configure([first, second, L("b", 1), second]) == {"kept": 0, "added": 2, "updated": 0, "deleted": 0}
    assert s.limits("a") == body(first)
    assert s.configure([second, first]) == {"kept": 0, "added": 0, "updated": 1, "deleted": 1}
    assert s.limits("a") == body(second)


def test_order_kept_limits_stay_and_added_ones_follow_in_the_given_order():
    s = Svc()
    x = [L("a", i, secs=i + 1, vars_=()) for i in range(5)]
    s.configure([x[0], x[1], x[2]])
    ids = s.ids("a")
    assert len(ids) == 3
    assert s.configure([x[4], x[2], x[3], x[0]]) == {"kept": 2, "added": 2, "updated": 0, "deleted": 1}
    assert s.limits("a") == body(x[0], x[2], x[4], x[3])
    got = s.ids("a")
    assert got[:2] == [ids[0], ids[2]] and len(set(got)) == 4 and min(got[2:]) > max(ids)
    # the draft-03 header lists the counters in that order when their remaining ties
    p = s.rls.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request("a", [[("m", "GET")]])]), T0)
    n = len(p["ctrs"])
    s.rls.finish(np.zeros(1, np.uint8), np.full(1, 0xFFFFFFFF, np.uint32), np.full(n, 5, np.uint64), np.full(n, 10**6, np.uint64))
    _, headers = R.decode_response(s.rls.responses()[0][1])
    assert dict(headers)["X-RateLimit-Limit"] == "0, 0;w=1, 2;w=3, 4;w=5, 3;w=4"


def _refusals():
    """(limits, index, reason) for every way of refusing one entry."""
    ok = [L("a", 1), L("b", 2), L("a", 3, conds=(POST,)), L("c", 4, vars_=())]
    return ok, [
        (dict(L("a", 1), conditions=["descriptors[0].m.startsWith('G')"]), "unsupported condition expression"),
        (dict(L("a", 1), variables=["a.b"]), "unsupported variable expression"),
        (dict(L("a", 1), conditions=["matches(x, 'y')"]), "unsupported condition expression"),
    ]


@pytest.mark.parametrize("pos", range(5))
def test_a_refused_entry_at_any_position_changes_nothing_and_is_named(pos):
    s = Svc()
    ok, bad = _refusals()
    s.configure([L("a", 50), L("c", 60, vars_=())])
    for entry, reason in bad:
        before = s.state()
        limits = ok[:pos] + [entry] + ok[pos:]
        with pytest.raises(R.ConfigureError) as e:
            s.configure(limits)
        assert e.value.index == pos and str(e.value).startswith(f"entry {pos}: {reason}")
        assert s.state() == before
    assert s.rls.config_status() == {"config_version": 1, "config_err_since": 3}
    s.configure(ok)
    assert s.rls.config_status() == {"config_version": 2, "config_err_since": 0}


def test_a_namespace_over_the_counter_cap_is_refused_at_the_entry_that_overflows_it():
    s = Svc(cap=3)
    many = [L("a", i, secs=i + 1) for i in range(4)]
    s.configure(many[:3])
    before = s.state()
    with pytest.raises(R.ConfigureError) as e:
        s.configure([L("b", 1)] + many)
    assert e.value.index == 4 and "more than 3 limits" in str(e.value)
    assert s.state() == before
    # a duplicate does not count twice
    assert s.configure(many[:3] + [many[0]])["kept"] == 3


def test_dry_run_checks_and_counts_and_changes_nothing():
    s = Svc()
    s.configure([L("a", 1), L("b", 2)])
    before = s.state()
    assert s.configure([L("a", 5), L("c", 3)], dry_run=True) == {"kept": 0, "added": 1, "updated": 1, "deleted": 1}
    with pytest.raises(R.ConfigureError) as e:
        s.configure([L("a", 5), dict(L("c", 3), variables=["x.y"])], dry_run=True)
    assert e.value.index == 1
    assert s.state() == before
    assert s.rls.config_status() == {"config_version": 1, "config_err_since": 0}


def test_boolean_dialect_limits_configure_too():
    s = Svc("boolean")
    c = "descriptors[0].m in ['GET', 'HEAD'] && has(descriptors[0].app)"
    s.configure([L("a", 1, conds=(c,))])
    assert len(s.ids("a")) == 1 and s.ids("a", "POST") == []


def test_limits_added_by_add_limit_are_kept_and_keep_a_null_id():
    s = Svc()
    d = s.m.add_limit("a", 10, 60, [GET], [APP], "n")
    assert s.configure([L("a", 10, name="n", id="given"), L("a", 1, conds=(POST,))])["kept"] == 1
    assert s.ids("a") == [int(d["limit_id"])]
    assert s.limits("a")[1].startswith(b'[{"id":null,')


# ---- the reference's configure_with tests (limitador/tests/integration_tests.rs:1102-1250) -----------------------------
def test_configure_with_creates_the_given_limits():
    s = Svc()
    first, second = L("first_namespace", 10), L("second_namespace", 20)
    s.configure([first, second])
    assert s.limits("first_namespace") == body(first) and s.limits("second_namespace") == body(second)


def test_configure_with_keeps_the_given_limits_and_counters_if_they_exist():
    s = Svc()
    limit = L("test_namespace", 10)
    s.configure([limit])
    lid = s.ids("test_namespace")
    s.configure([limit, L("test_namespace", 5, conds=(POST,))])
    assert s.ids("test_namespace") == lid  # the same counter (limit id, key): its count survives
    assert s.limits("test_namespace") == body(limit, L("test_namespace", 5, conds=(POST,)))


def test_configure_with_deletes_all_except_the_limits_given():
    s = Svc()
    a, b = L("test_namespace", 10), L("test_namespace", 20, conds=(POST,))
    s.configure([a, b])
    assert s.configure([a])["deleted"] == 1
    assert s.limits("test_namespace") == body(a) and s.ids("test_namespace", "POST") == []


def test_configure_with_updates_the_limits():
    s = Svc()
    limit = L("test_namespace", 10)
    s.configure([limit])
    lid = s.ids("test_namespace")
    assert s.configure([dict(limit, max_value=20)])["updated"] == 1
    assert s.limits("test_namespace") == body(dict(limit, max_value=20)) and s.ids("test_namespace") == lid


# ---- the staging path under ASan + UBSan ---------------------------------------------------------------------------------
def test_configure_is_clean_under_asan_and_ubsan(tmp_path):
    from tests.test_sanitizers import build_and_run
    csrc = os.path.join(ROOT, "limitador_b200", "csrc")
    out = build_and_run(tmp_path, "g++", [os.path.join(ROOT, "tests", "san", "san_configure.cpp"), os.path.join(csrc, "rl_rls.cpp"),
                                          os.path.join(csrc, "rl_match.cpp")],
                        [os.path.join(ROOT, "include")], extra=("-std=c++17",))
    assert out.startswith("ok configured=")
    configured, refused = (int(x.split("=")[1]) for x in out.split()[1:3])
    assert configured > 50 and refused > 50
