"""GET /limits/{namespace} and the rendering stage of GET /counters/{namespace} (include/rl_http.h) without a GPU: the
bodies must equal a Python restatement of actix Json + serde_json (tests/serde_render.py) byte for byte, on adversarial
strings, u64 extremes, a wrapped `remaining`, null and quoted names; and the outcomes (unknown namespace, unnamed counters,
deleted limits) must follow DESIGN §5."""
import json
import struct

import numpy as np

from limitador_b200 import engine as E
from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R
from tests import serde_render as S

U64 = (1 << 64) - 1
ODD = "q\"b\\s\x01\x1f\x7f é😀"
LIMITS = [("api", 5, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"),
          ("api", U64, 1, [], ["descriptors[0]['x\"y']", "descriptors[0].user"], ODD),
          ("api", 0, U64, ["descriptors[0].method != 'OPTIONS'", "descriptors[0]['\x7f é'] == 'é\"'"], [], None),
          (ODD, 3, 10, [], ["descriptors[0].k"], "\"quoted\""),
          ("", 1, 1, [], [], "")]


def _api(limits=LIMITS):
    m = MT.Matcher()
    descs = [m.add_limit(*l) for l in limits]
    api = HA.HttpApi(R.RlsService(m, None, R.HEADERS_NONE, 1))
    return m, descs, api


def _blob(values):
    return b"".join(struct.pack("<I", len(v.encode())) + v.encode() for v in values)


def test_limits_read():
    """server.rs:401-431 test_limits_read: one limit created, GET /limits/test_namespace lists exactly it."""
    lim = ("test_namespace", 10, 60, ["req_method == 'GET'"], ["app_id"], None)
    _, _, api = _api([lim])
    status, body = api.get_limits("test_namespace")
    assert status == 200
    got = json.loads(body)
    assert len(got) == 1
    assert got[0] == {"id": None, "namespace": "test_namespace", "max_value": 10, "seconds": 60, "name": None,
                      "conditions": ["req_method == 'GET'"], "variables": ["app_id"]}
    assert body == S.limits_body([lim])


def test_limits_bodies_on_adversarial_strings():
    m, descs, api = _api()
    by_ns = {}
    for l in LIMITS:
        by_ns.setdefault(l[0], []).append(l)
    for ns, ls in by_ns.items():
        assert api.get_limits(ns) == (200, S.limits_body(ls)), ns
    assert api.get_limits("nope") == (200, b"[]")
    assert api.get_limits("api\x00") == (200, b"[]")
    # a deleted limit leaves the listing; added again it comes last; update_limit shows its new max_value and name
    m.delete_limit(int(descs[0]["limit_id"]))
    assert api.get_limits("api") == (200, S.limits_body(by_ns["api"][1:]))
    m.add_limit("api", 99, 60, LIMITS[0][3], LIMITS[0][4], None)
    assert api.get_limits("api") == (200, S.limits_body(by_ns["api"][1:] + [("api", 99, 60, LIMITS[0][3], LIMITS[0][4], None)]))


def _render(api, ns, rows):
    """rows: (limit_id, key_lo, key_hi, remaining, ttl_us, values or None) -> render_counters' (status, body)."""
    ctrs = np.zeros(len(rows), E.COUNTER_DTYPE)
    blobs, off, un = b"", [0], []
    for i, (lid, lo, hi, _, _, vals) in enumerate(rows):
        ctrs[i] = (lid, 0, lo, hi)
        blobs += _blob(vals) if vals else b""
        off.append(len(blobs))
        un.append(1 if vals is None else 0)
    return api.render_counters(ns, ctrs, [r[3] for r in rows], [r[4] for r in rows], blobs, off, un)


def test_counters_bodies_on_adversarial_strings_and_u64_extremes():
    m, descs, api = _api()
    lim_json = {int(d["limit_id"]): S.limit_json(*l[:3], l[5], l[3], l[4]) for d, l in zip(descs, LIMITS)}
    vars_of = {int(d["limit_id"]): sorted(set(l[4])) for d, l in zip(descs, LIMITS)}
    values = ["", ODD, "\x00"[:0] + "\t\n\r\b\f", "\"\\", "é" * 40]
    rows, want = [], []
    rng = np.random.default_rng(3)
    for k in range(40):
        lid = int(descs[k % 3]["limit_id"])
        lo, hi = int(rng.integers(0, 1 << 63)) * 2 + (k & 1), int(rng.integers(0, 1 << 32))
        rem = [0, 1, U64, U64 - 4, 5][k % 5]  # (U64 - 4: a remaining that wrapped below zero)
        ttl = [1, 999_999, 1_000_000, 59_999_999, U64][k % 5]
        if vars_of[lid]:
            vals = [values[(k + j) % len(values)] for j in range(len(vars_of[lid]))]
        else:
            vals, lo, hi = [], 0, 0
        rows.append((lid, lo, hi, rem, ttl, vals))
        pos = [int(d["limit_id"]) for d in descs[:3]].index(lid)
        want.append((pos, lo, hi, lim_json[lid], dict(zip(vars_of[lid], vals)), rem, ttl))
    # a counter of another namespace's limit is left out
    rows.append((int(descs[3]["limit_id"]), 5, 6, 1, 1, ["x"]))
    status, body = _render(api, "api", rows)
    assert status == 200 and body == S.counters_body(want)
    assert len(json.loads(body)) == 40
    # the other namespaces
    lid3 = int(descs[3]["limit_id"])
    assert _render(api, ODD, [(lid3, 9, 1, 2, 3_000_000, [ODD])]) == (
        200, S.counters_body([(0, 9, 1, lim_json[lid3], {"descriptors[0].k": ODD}, 2, 3_000_000)]))
    lid4 = int(descs[4]["limit_id"])
    assert _render(api, "", [(lid4, 0, 0, 1, 999_999, [])]) == (200, S.counters_body([(0, 0, 0, lim_json[lid4], {}, 1, 999_999)]))
    assert _render(api, "nope", rows) == (200, b"[]")
    assert _render(api, "api", []) == (200, b"[]")


def test_unnamed_counters_answer_500_and_deleted_limits_are_left_out():
    m, descs, api = _api()
    l0, l1, l2 = (int(d["limit_id"]) for d in descs[:3])
    rows = [(l0, 1, 2, 3, 4_000_000, ["u1"]), (l2, 0, 0, 1, 1_000_000, []), (l1, 3, 4, 5, 6, None), (l0, 7, 8, 9, 10, None)]
    assert _render(api, "api", rows) == (500, b"Internal server error")
    assert api.last_unnamed == 2
    # a blob that does not hold one value per variable is no better than none
    assert _render(api, "api", [(l1, 3, 4, 5, 6, ["only-one"])])[0] == 500
    # the unnamed counters' limit deleted: they leave the listing, and the rest is served
    m.delete_limit(l1)
    assert _render(api, "api", rows[:3]) == (200, S.counters_body([
        (0, 1, 2, S.limit_json(*LIMITS[0][:3], LIMITS[0][5], LIMITS[0][3], LIMITS[0][4]), {"descriptors[0].user": "u1"}, 3, 4_000_000),
        (1, 0, 0, S.limit_json(*LIMITS[2][:3], LIMITS[2][5], LIMITS[2][3], LIMITS[2][4]), {}, 1, 1_000_000)]))
    assert api.last_unnamed == 0
