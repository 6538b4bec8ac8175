"""The HTTP API surface (include/rl_http.h) on the CPU: the JSON decoder against a strict Python restatement of the
CheckAndReportInfo rules (tests/http_corpora.py) and against Python's json module where RFC 8259 decides alone, and the
service's plan -> store -> finish stages with the CPU oracle as the store, against the reference's own HTTP tests
(limitador-server/src/http_api/server.rs:433-640) and against the Python mirror of RateLimiter called one request at a
time."""
import numpy as np
import pytest

from limitador_b200 import http_api as HA
from limitador_b200 import rls as R
from tests import helpers as H
from tests import http_corpora as HC

from tests.http_corpora import T0, HttpHarness


def _info(delta=1, headers=None):
    return HA.encode_info("test_namespace", {"req.method": "GET", "app.id": "1"}, delta, headers)


# ---- the reference's HTTP tests (server.rs:433-640) -------------------------------------------------------------------
def test_check_and_report():
    """:433-486 — limit 1: the first call is 200 without headers, the second 429."""
    h = HttpHarness([HC.REF_LIMIT])
    (s1, b1, h1), = h.call(HA.CHECK_AND_REPORT, [_info()])
    assert s1 == 200 and b1 == b"null" and h1 == {}
    (s2, b2, h2), = h.call(HA.CHECK_AND_REPORT, [_info()], T0 + 1_000_000)
    assert s2 == 429 and b2 == b"null" and h2 == {}
    assert h.last_plan["load_counters"].tolist() == [0]


def test_check_and_report_with_draftversion03_response_headers():
    """:488-565 — limit 2: remaining 1, then 0, then 429 with the headers."""
    h = HttpHarness([("test_namespace", 2) + HC.REF_LIMIT[2:]])
    body = _info(headers="DraftVersion03")
    out = [h.call(HA.CHECK_AND_REPORT, [body], T0 + k * 1_000_000)[0] for k in range(3)]
    assert [s for s, _, _ in out] == [200, 200, 429]
    assert [hd["X-RateLimit-Limit"] for _, _, hd in out] == ["2, 2;w=60"] * 3
    assert [hd["X-RateLimit-Remaining"] for _, _, hd in out] == ["1", "0", "0"]
    assert all(0 < int(hd["X-RateLimit-Reset"]) <= 60 for _, _, hd in out)
    # the same three in ONE batch: array order is the stream order
    h2 = HttpHarness([("test_namespace", 2) + HC.REF_LIMIT[2:]])
    assert [s for s, _, _ in h2.call(HA.CHECK_AND_REPORT, [body] * 3)] == [200, 200, 429]


def test_check_and_report_endpoints_separately():
    """:567-628 — check 200, report, check 429."""
    h = HttpHarness([HC.REF_LIMIT])
    assert h.call(HA.CHECK, [_info()])[0] == (200, b"null", {})
    assert h.call(HA.REPORT, [_info()])[0] == (200, b"null", {})
    assert h.call(HA.CHECK, [_info()])[0] == (429, b"Too many requests", {})
    assert "authorized_calls{" not in h.api.metrics() and "limited_calls{" not in h.api.metrics()  # only check_and_report counts


def test_outcomes_of_refused_and_unshippable_bodies():
    h = HttpHarness([HC.REF_LIMIT])
    nul = HA.encode_info("test_namespace", {"req.method": "GET", "app.id": "a\x00b"}, 1)
    for ep, err in ((HA.CHECK, b"Internal server error"), (HA.REPORT, b"Internal server error"), (HA.CHECK_AND_REPORT, b"null")):
        out = h.call(ep, [b"{", nul, _info(0)])
        assert [(s, b) for s, b, _ in out][:2] == [(400, b""), (500, err)]
        assert out[2][0] == 200
    # a failed store call answers 500 for the requests that needed it
    buf, off = HA.pack_bodies([_info(), HA.encode_info("nobody", {}, 1)])
    h.api.plan(HA.CHECK_AND_REPORT, buf, off, T0)
    out = h.api.finish(np.zeros(1, np.uint8), np.full(1, 0xFFFFFFFF, np.uint32), store_status=np.array([1], np.int32))
    assert [(s, b) for s, b, _ in out] == [(500, b"null"), (200, b"null")]


def test_delta_goes_to_the_store_as_it_is():
    h = HttpHarness([HC.REF_LIMIT])
    for ep in (HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT):
        h.call(ep, [_info(0), _info(5), _info(2**64 - 1)])
        assert h.last_plan["delta"].tolist() == [0, 5, 2**64 - 1]


def test_mixed_response_headers_split_the_store_calls():
    """load_counters follows response_headers.is_some() request by request: maximal runs of equal flags."""
    h = HttpHarness([("test_namespace", 3) + HC.REF_LIMIT[2:]])
    hd = [None, None, "DraftVersion03", "other", None, "DraftVersion03"]
    out = h.call(HA.CHECK_AND_REPORT, [_info(headers=x) for x in hd])
    assert h.last_plan["load_counters"].tolist() == [0, 0, 1, 1, 0, 1]
    assert h.runs == [(0, 2), (2, 4), (4, 5), (5, 6)]
    assert [s for s, _, _ in out] == [200, 200, 200, 429, 429, 429]
    assert [bool(x) for _, _, x in out] == [False, False, True, False, False, True]
    h.call(HA.CHECK, [_info(headers=x) for x in hd])
    assert h.runs == [(0, 6)]


# ---- the decoder -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,body,accepted", HC.CORPUS, ids=[c[0] for c in HC.CORPUS])
def test_decoder_corpus(name, body, accepted):
    want = HC.py_decode(body)
    assert (want is not None) == accepted, "the restatement disagrees with the corpus"
    try:
        got = HA.decode_body(body)
    except HA.HttpError:
        got = None
    assert got == want


def test_decoder_details():
    ns, pairs, delta, hdr = HA.decode_body(HC._ok(values='{"a":"1","b":"2","a":"3"}'))
    assert pairs == [("a", "1"), ("b", "2"), ("a", "3")]  # in body order; the matcher binds the last "a"
    assert HA.decode_body(b'{"name\\u0073pace":"n\\u00e9","values":{},"delta":1}')[0] == "né"
    assert HA.decode_body(HC._ok(extra=',"response_headers":"DraftVersion03"'))[3] == HA.HEADERS_DRAFT_VERSION_03
    assert HA.decode_body(HC._ok(extra=',"response_headers":"x"'))[3] == HA.HEADERS_OTHER
    assert HA.decode_body(b'["ns",{"k":"v"},1,null]') == ("ns", [("k", "v")], 1, HA.HEADERS_NONE)
    many = HA.encode_info("ns", {f"k{i}": "v" for i in range(300)}, 1)  # past the binding's first guess of 64 entries
    assert len(HA.decode_body(many)[1]) == 300


def test_decoder_against_the_restatement_on_mutations():
    rng = np.random.default_rng(5)
    bodies = HC.corpus_bodies(rng, 3000)
    acc = ref = 0
    for b in bodies:
        want = HC.py_decode(b)
        try:
            got = HA.decode_body(b)
        except HA.HttpError:
            got = None
        assert got == want, b
        acc += got is not None
        ref += got is None
    assert acc > 300 and ref > 1000


def _text(x):
    """a str that is valid Unicode (json.loads lets a lone surrogate escape through into a str)"""
    try:
        return isinstance(x, str) and bool(x.encode()) or x == ""
    except UnicodeEncodeError:
        return False


def test_restatement_against_json_loads_where_rfc_8259_decides():
    """Bodies that json.loads (duplicates detected, NaN refused) refuses on syntax are refused by the restatement, and a
    body it parses into the struct's plain shape decodes to the same fields."""
    rng = np.random.default_rng(6)
    checked = 0
    for b in HC.corpus_bodies(rng, 3000):
        try:
            v = HC.json_loads_strict(b)
        except (ValueError, UnicodeDecodeError, RecursionError):
            v = ValueError
        got = HC.py_decode(b)
        if v is ValueError:
            # json.loads refuses: syntax, or a lone surrogate / invalid UTF-8 it cannot decode; only the latter two may be
            # skipped strings the struct accepts
            if got is not None:
                assert b"\\u" in b or any(x >= 0x80 for x in b), b
            continue
        if isinstance(v, dict) and set(v) == set(HC.FIELDS[:3]) and isinstance(v["values"], dict) \
                and _text(v["namespace"]) and all(_text(k) and _text(x) for k, x in v["values"].items()) \
                and type(v["delta"]) is int and 0 <= v["delta"] < 2**64:
            assert got is not None and got[0] == v["namespace"] and dict(got[1]) == v["values"] and got[2] == v["delta"], b
            checked += 1
        elif not isinstance(v, (dict, list, tuple)):  # a scalar at the top level is no struct
            assert got is None
    assert checked > 20


def test_encode_info_is_what_serde_json_writes():
    assert HA.encode_info("ns", {"a": "1"}, 2) == b'{"namespace":"ns","values":{"a":"1"},"delta":2,"response_headers":null}'
    assert HA.encode_info("n\"s", {"k\n": "\x01ü/"}, 0, "DraftVersion03") == \
        '{"namespace":"n\\"s","values":{"k\\n":"\\u0001ü/"},"delta":0,"response_headers":"DraftVersion03"}'.encode()


# ---- batches against the Python mirror of RateLimiter ----------------------------------------------------------------
def _mirror(limits):
    from limitador_b200 import limiter as LM
    clock = {"t": T0}
    rl = LM.RateLimiter(H.OracleStorage(), clock=lambda: clock["t"])
    for ns, mx, secs, conds, vars_, name in limits:
        rl.add_limit(LM.Limit(ns, mx, secs, conds, vars_, name=name))
    return rl, clock, LM


@pytest.mark.parametrize("threads", [1, 4])
def test_random_batches_equal_the_mirror_called_request_by_request(threads):
    rng = np.random.default_rng(40 + threads)
    limits = HC.GATEWAY_LIMITS
    rl, clock, LM = _mirror(limits)
    h = HttpHarness(limits, threads=threads, use_limit_name_label=True)
    want_m = {}
    n_429 = 0
    for step, ep in enumerate([HA.CHECK_AND_REPORT, HA.CHECK, HA.REPORT, HA.CHECK_AND_REPORT, HA.CHECK]):
        now = T0 + step * 7_000_000
        clock["t"] = now
        infos = HC.random_infos(rng, 700)
        got = h.call(ep, [HA.encode_info(*x) for x in infos], now)
        for (ns, values, delta, hdr), (status, body, headers) in zip(infos, got):
            ctx = LM.Context({}, [dict(values)])
            if ep == HA.REPORT:
                rl.update_counters(ns, ctx, delta)
                assert (status, body, headers) == (200, b"null", {})
                continue
            if ep == HA.CHECK:
                w = rl.is_rate_limited(ns, ctx, delta)
                assert (status, body, headers) == ((429, b"Too many requests") if w.limited else (200, b"null")) + ({},)
                continue
            w = rl.check_rate_limited_and_update(ns, ctx, delta, hdr is not None)
            n_429 += w.limited
            want_h = w.response_header() if hdr == "DraftVersion03" else {}
            assert (status, body, headers) == (429 if w.limited else 200, b"null", want_h)
            c = want_m.setdefault(ns, [0, 0, 0])
            if w.limited:
                c[2] += 1
            else:
                c[0] += 1
                c[1] += delta
    assert 100 < n_429 < 3000
    text = h.api.metrics()
    for ns, (calls, hits, limited) in want_m.items():
        if calls:
            assert f'authorized_calls{{limitador_namespace="{ns}"}} {calls}\n' in text
        if hits:
            assert f'authorized_hits{{limitador_namespace="{ns}"}} {hits}\n' in text
    assert sum(int(l.rsplit(" ", 1)[1]) for l in text.splitlines() if l.startswith("limited_calls{")) == n_429
    assert H.normalise_dump(h.o.dump(), np.array(h.descs)) == H.normalise_dump(rl.storage.o.dump(), np.array(h.descs))


def test_rls_and_http_share_one_metrics_registry():
    h = HttpHarness([("a", 1, 60, [], ["descriptors[0].u"], None)])
    h.call(HA.CHECK_AND_REPORT, [HA.encode_info("a", {"u": "1"}, 1)] * 2)
    p = h.rls.plan(R.SHOULD_RATE_LIMIT, *R.pack_requests([R.encode_request("a", [[("u", "2")]], 1)]), T0)
    h.rls.finish(np.zeros(p["n_store"], np.uint8), np.full(p["n_store"], 0xFFFFFFFF, np.uint32))
    t = h.api.metrics()
    assert 'authorized_calls{limitador_namespace="a"} 2' in t and 'limited_calls{limitador_namespace="a"} 1' in t
