"""Bodies for the HTTP API tests (CPU and GPU): a strict restatement of the CheckAndReportInfo rules in plain Python, the
decoder corpus (one case per rule), mutated bodies and random batches."""
import json

import numpy as np

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R

T0 = 1_700_000_000_000_000
MODE = {HA.CHECK_AND_REPORT: 0, HA.CHECK: 1, HA.REPORT: 2}

WS = b" \t\n\r"
FIELDS = ("namespace", "values", "delta", "response_headers")
REF_LIMIT = ("test_namespace", 1, 60, ["descriptors[0]['req.method'] == 'GET'"], ["descriptors[0]['app.id']"], None)


class Refused(Exception):
    pass


class _P:
    """serde_json::from_slice::<CheckAndReportInfo>, restated: returns (namespace, [(k, v)], delta, headers) or raises."""

    def __init__(self, b):
        self.b, self.p = b, 0

    def ws(self):
        while self.p < len(self.b) and self.b[self.p] in WS:
            self.p += 1
        return self.b[self.p] if self.p < len(self.b) else None

    def eat(self, c):
        if self.ws() != c:
            raise Refused(f"expected {chr(c)} at {self.p}")
        self.p += 1

    def string(self, keep):
        self.eat(ord('"'))
        out, b = [], self.b
        while True:
            if self.p >= len(b):
                raise Refused("eof in string")
            c = b[self.p]
            self.p += 1
            if c == 0x22:
                break
            if c < 0x20:
                raise Refused("control byte")
            if c != 0x5C:
                out.append(bytes([c]))
                continue
            e = b[self.p:self.p + 1]
            self.p += 1
            simple = {b'"': '"', b"\\": "\\", b"/": "/", b"b": "\b", b"f": "\f", b"n": "\n", b"r": "\r", b"t": "\t"}
            if e in simple:
                out.append(simple[e].encode())
                continue
            if e != b"u":
                raise Refused("bad escape")
            cp = self.hex4()
            if not keep:
                continue
            if 0xDC00 <= cp <= 0xDFFF:
                raise Refused("lone trailing surrogate")
            if 0xD800 <= cp <= 0xDBFF:
                if b[self.p:self.p + 2] != b"\\u":
                    raise Refused("lone leading surrogate")
                self.p += 2
                lo = self.hex4()
                if not 0xDC00 <= lo <= 0xDFFF:
                    raise Refused("lone leading surrogate")
                cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00)
            out.append(chr(cp).encode())
        if not keep:
            return None
        try:
            return b"".join(out).decode("utf-8")
        except UnicodeDecodeError:
            raise Refused("invalid utf-8")

    def hex4(self):
        h = self.b[self.p:self.p + 4]
        if len(h) < 4 or any(c not in b"0123456789abcdefABCDEF" for c in h):
            raise Refused("bad \\u")
        self.p += 4
        return int(h, 16)

    def number(self):
        b = self.b
        start = self.p
        if b[self.p:self.p + 1] == b"-":
            self.p += 1
        d0 = self.p
        while self.p < len(b) and 0x30 <= b[self.p] <= 0x39:
            self.p += 1
        if self.p == d0 or (b[d0] == 0x30 and self.p - d0 > 1):
            raise Refused("bad integer part")
        for lead, signs in ((b".", False), (b"eE", True)):
            if self.p < len(b) and b[self.p:self.p + 1] in [bytes([x]) for x in lead]:
                self.p += 1
                if signs and b[self.p:self.p + 1] in (b"+", b"-"):
                    self.p += 1
                d = self.p
                while self.p < len(b) and 0x30 <= b[self.p] <= 0x39:
                    self.p += 1
                if self.p == d:
                    raise Refused("bad fraction / exponent")
        return b[start:self.p]

    def skip(self):  # any value; nesting kept in a Python list, as deep as the body
        stack = []
        while True:
            c = self.ws()
            if c in (ord("{"), ord("[")):
                self.p += 1
                close = ord("}") if c == ord("{") else ord("]")
                if self.ws() == close:
                    self.p += 1
                else:
                    stack.append(close)
                    if close == ord("}"):
                        self.string(False)
                        self.eat(ord(":"))
                    continue
            elif c == ord('"'):
                self.string(False)
            elif c is not None and (c == ord("-") or 0x30 <= c <= 0x39):
                self.number()
            else:
                for w in (b"true", b"false", b"null"):
                    if self.b.startswith(w, self.p):
                        self.p += len(w)
                        break
                else:
                    raise Refused("bad value")
            while True:
                if not stack:
                    return
                c = self.ws()
                if c == ord(","):
                    self.p += 1
                    if stack[-1] == ord("}"):
                        self.string(False)
                        self.eat(ord(":"))
                    break
                if c != stack[-1]:
                    raise Refused("bad container")
                self.p += 1
                stack.pop()

    def field(self, name, out):
        c = self.ws()
        if name == "namespace":
            out[name] = self.string(True)
        elif name == "values":
            self.eat(ord("{"))
            pairs = []
            if self.ws() == ord("}"):
                self.p += 1
            else:
                while True:
                    k = self.string(True)
                    self.eat(ord(":"))
                    pairs.append((k, self.string(True)))
                    c = self.ws()
                    self.p += 1
                    if c == ord("}"):
                        break
                    if c != ord(","):
                        raise Refused("values")
            out[name] = pairs
        elif name == "delta":
            if c is None or not 0x30 <= c <= 0x39:
                raise Refused("delta is not a u64")
            t = self.number()
            if not t.isdigit() or int(t) >= 1 << 64:
                raise Refused("delta is not a u64")
            out[name] = int(t)
        elif name == "response_headers":
            if self.b.startswith(b"null", self.p) and c == ord("n"):
                self.p += 4
                out[name] = None
            else:
                out[name] = self.string(True)
        else:
            self.skip()

    def info(self):
        out = {}
        c = self.ws()
        if c == ord("["):
            self.p += 1
            for k, f in enumerate(FIELDS):
                if k:
                    self.eat(ord(","))
                self.field(f, out)
            self.eat(ord("]"))
        elif c == ord("{"):
            self.p += 1
            if self.ws() == ord("}"):
                self.p += 1
            else:
                while True:
                    name = self.string(True)
                    self.eat(ord(":"))
                    if name in FIELDS:
                        if name in out:
                            raise Refused("duplicate field")
                        self.field(name, out)
                    else:
                        self.field(None, out)
                    c = self.ws()
                    self.p += 1
                    if c == ord("}"):
                        break
                    if c != ord(","):
                        raise Refused("object")
            if not all(f in out for f in FIELDS[:3]):
                raise Refused("missing field")
        else:
            raise Refused("not a struct")
        if self.ws() is not None:
            raise Refused("trailing characters")
        h = out.get("response_headers")
        state = HA.HEADERS_NONE if h is None else HA.HEADERS_DRAFT_VERSION_03 if h == "DraftVersion03" else HA.HEADERS_OTHER
        return out["namespace"], out["values"], out["delta"], state


def py_decode(body: bytes):
    """-> (namespace, values pairs, delta, headers state), or None for a refused body."""
    try:
        return _P(body).info()
    except (Refused, IndexError):
        return None


def _ok(ns="ns", values='{"a":"1"}', delta="1", extra=""):
    return f'{{"namespace":"{ns}","values":{values},"delta":{delta}{extra}}}'.encode()


# (name, body, accepted)
CORPUS = [
    ("plain", _ok(), True),
    ("whitespace", b' \t\n\r{ "namespace" : "ns" , "values" : { } , "delta" : 0 }\r\n', True),
    ("form feed is not whitespace", b"\x0c" + _ok(), False),
    ("bom", b"\xef\xbb\xbf" + _ok(), False),
    ("empty body", b"", False),
    ("only whitespace", b"  ", False),
    ("trailing garbage", _ok() + b"x", False),
    ("two values", _ok() + _ok(), False),
    ("comment", b"/*c*/" + _ok(), False),
    ("trailing comma in object", _ok(extra=","), False),
    ("trailing comma in values", _ok(values='{"a":"1",}'), False),
    ("NaN delta", _ok(delta="NaN"), False),
    ("Infinity in a skipped field", _ok(extra=',"x":Infinity'), False),
    ("leading zero in a skipped number", _ok(extra=',"x":01'), False),
    ("skipped numbers", _ok(extra=',"x":[-0,1.5e-3,2E+7,0.0,-12]'), True),
    ("array of 4", b'["ns",{"a":"1"},7,null]', True),
    ("array of 4 with headers", b'["ns",{},7,"DraftVersion03"]', True),
    ("array of 3", b'["ns",{"a":"1"},7]', False),
    ("array of 5", b'["ns",{"a":"1"},7,null,1]', False),
    ("empty array", b"[]", False),
    ("top-level string", b'"ns"', False),
    ("top-level null", b"null", False),
    ("escaped field name", b'{"name\\u0073pace":"ns","values":{},"delta":1}', True),
    ("duplicate namespace", _ok(extra=',"namespace":"x"'), False),
    ("duplicate delta", _ok(extra=',"delta":2'), False),
    ("duplicate response_headers", _ok(extra=',"response_headers":null,"response_headers":null'), False),
    ("duplicate unknown field", _ok(extra=',"x":1,"x":2'), True),
    ("repeated values key keeps the last", _ok(values='{"a":"1","b":"2","a":"3"}'), True),
    ("missing namespace", b'{"values":{},"delta":1}', False),
    ("missing values", b'{"namespace":"ns","delta":1}', False),
    ("missing delta", b'{"namespace":"ns","values":{}}', False),
    ("missing response_headers", _ok(), True),
    ("null response_headers", _ok(extra=',"response_headers":null'), True),
    ("other response_headers", _ok(extra=',"response_headers":"DraftVersion04"'), True),
    ("response_headers not a string", _ok(extra=',"response_headers":1'), False),
    ("namespace not a string", b'{"namespace":1,"values":{},"delta":1}', False),
    ("namespace null", b'{"namespace":null,"values":{},"delta":1}', False),
    ("empty namespace", b'{"namespace":"","values":{},"delta":1}', True),
    ("values not an object", _ok(values='[]'), False),
    ("values value not a string", _ok(values='{"a":1}'), False),
    ("values value null", _ok(values='{"a":null}'), False),
    ("delta -0", _ok(delta="-0"), False),
    ("delta -1", _ok(delta="-1"), False),
    ("delta 1.0", _ok(delta="1.0"), False),
    ("delta 1e0", _ok(delta="1e0"), False),
    ("delta 2^64-1", _ok(delta=str(2**64 - 1)), True),
    ("delta 2^64", _ok(delta=str(2**64)), False),
    ("delta 0", _ok(delta="0"), True),
    ("delta 01", _ok(delta="01"), False),
    ("delta as a string", _ok(delta='"1"'), False),
    ("escapes", _ok(values='{"k\\"\\\\\\/\\b\\f\\n\\r\\t":"\\u00e9\\u65e5"}'), True),
    ("surrogate pair", _ok(values='{"a":"\\ud83d\\ude00"}'), True),
    ("lone leading surrogate in a value", _ok(values='{"a":"\\ud83d"}'), False),
    ("lone trailing surrogate in a key", _ok(values='{"\\ude00":"1"}'), False),
    ("leading surrogate then a non-trailing one", _ok(values='{"a":"\\ud83d\\u0041"}'), False),
    ("lone surrogate in the namespace", _ok(ns="\\udfff"), False),
    ("lone surrogate in a skipped string", _ok(extra=',"x":"\\ud800"'), True),
    ("lone surrogate in a skipped key", _ok(extra=',"x":{"\\udc00":1}'), True),
    ("invalid utf-8 in a value", b'{"namespace":"ns","values":{"a":"\xc3\x28"},"delta":1}', False),
    ("invalid utf-8 in the namespace", b'{"namespace":"\xff","values":{},"delta":1}', False),
    ("invalid utf-8 in a field name", b'{"\xc0\x80":1,"namespace":"ns","values":{},"delta":1}', False),
    ("invalid utf-8 in a skipped string", b'{"x":"\xff\xfe","namespace":"ns","values":{},"delta":1}', True),
    ("overlong utf-8 in a key", b'{"namespace":"ns","values":{"\xe0\x80\x80":"1"},"delta":1}', False),
    ("raw utf-8", '{"namespace":"ñs","values":{"日本":"ü"},"delta":1}'.encode(), True),
    ("raw control byte in a value", b'{"namespace":"ns","values":{"a":"\x01"},"delta":1}', False),
    ("raw control byte in a skipped string", b'{"x":"\x1f","namespace":"ns","values":{},"delta":1}', False),
    ("bad escape in a skipped string", _ok(extra=',"x":"\\q"'), False),
    ("short \\u in a skipped string", _ok(extra=',"x":"\\u12"'), False),
    ("deep nesting in a skipped field", _ok(extra=',"x":' + "[{\"a\":" * 3000 + "1" + "}]" * 3000), True),
    ("deep nesting left open", _ok(extra=',"x":' + "[" * 3000 + "]" * 2999), False),
    ("mismatched brackets", _ok(extra=',"x":[1}'), False),
    ("skipped literals", _ok(extra=',"x":[true,false,null,{"y":{}}]'), True),
    ("bad literal", _ok(extra=',"x":nul'), False),
    ("NUL from \\u0000", _ok(values='{"a":"x\\u0000y"}'), True),
    ("key must be a string", b'{1:2,"namespace":"ns","values":{},"delta":1}', False),
    ("missing colon", b'{"namespace" "ns","values":{},"delta":1}', False),
]


def mutate(rng, body: bytes) -> bytes:
    b = bytearray(body)
    k = int(rng.integers(0, 4))
    if k == 0 and b:
        p = int(rng.integers(0, len(b)))
        del b[p:p + int(rng.integers(1, 4))]
    elif k == 1 and b:
        b[int(rng.integers(0, len(b)))] = int(rng.choice(list(b'{}[]",:\\ 0123456789-.eEnulltrufasx\x00\x1f\x7f\xc3\xff')))
    elif k == 2:
        p = int(rng.integers(0, len(b) + 1))
        b[p:p] = bytes(rng.choice([b",", b" ", b'"', b"\\u", b"\\ud800", b"[", b"}", b"1", b"\xef\xbb\xbf"]))
    else:
        b = b[:int(rng.integers(0, len(b) + 1))]
    return bytes(b)


def random_infos(rng, n, users=7):
    """(namespace, values, delta, response_headers) tuples over the gateway-style limits below."""
    out = []
    for _ in range(n):
        ns = "api" if rng.random() < 0.8 else str(rng.choice(["admin", "nobody", ""]))
        values = {"method": str(rng.choice(["GET", "POST", "OPTIONS"])), "user": f"u{int(rng.integers(0, users))}"}
        if rng.random() < 0.7:
            values["path"] = str(rng.choice(["/a", "/b", "/ü"]))
        hdr = [None, None, "DraftVersion03", "other"][int(rng.integers(0, 4))]
        out.append((ns, values, int(rng.choice([0, 1, 1, 2, 3])), hdr))
    return out


GATEWAY_LIMITS = [("api", 5, 60, ["descriptors[0].method == 'GET'"], ["descriptors[0].user"], "get-per-user"),
                  ("api", 3, 60, ["descriptors[0].method == 'POST'"], ["descriptors[0].user"], "post-per-user"),
                  ("api", 40, 3600, [], ["descriptors[0].user"], "hourly-per-user"),
                  ("api", 120, 60, ["descriptors[0].method != 'OPTIONS'"], [], "global"),
                  ("admin", 2, 10, [], ["descriptors[0].user", "descriptors[0].path"], None)]


def corpus_bodies(rng, n_mut=400):
    """The corpus, the reference scenario's bodies and mutations of both, in one list."""
    base = [b for _, b, _ in CORPUS]
    base += [HA.encode_info(*x) for x in random_infos(rng, 60)]
    return base + [mutate(rng, base[int(rng.integers(0, len(base)))]) for _ in range(n_mut)]


def json_loads_strict(body: bytes):
    """Python's json module with duplicates detected and NaN / Infinity refused: what RFC 8259 decides alone."""
    def pairs(kv):
        keys = [k for k, _ in kv]
        if len(set(keys)) != len(keys):
            return ("dup", kv)
        return dict(kv)

    def bad(_):
        raise ValueError("constant")
    # a signed integer (-0 included) is not a u64: kept apart from the ints
    return json.loads(body.decode("utf-8"), object_pairs_hook=pairs, parse_constant=bad,
                      parse_int=lambda t: ("signed", t) if t.startswith("-") else int(t))


class HttpHarness:
    """plan -> (the CPU oracle decides, one call per run of equal load_counters flags) -> finish."""

    def __init__(self, limits, threads=1, use_limit_name_label=False):
        from oracle import binding as ob
        self.m = MT.Matcher()
        self.o = ob.Oracle(64)
        self.descs = []
        for (ns, mx, secs, conds, vars_, name) in limits:
            d = self.m.add_limit(ns, mx, secs, conds, vars_, name)
            self.descs.append(d)
            self.o.limit_set(int(d["limit_id"]), int(d["ns_id"]), int(d["max_value"]), int(d["window_us"]), bool(d["qualified"]))
        self.rls = R.RlsService(self.m, None, R.HEADERS_NONE, threads, use_limit_name_label)
        self.api = HA.HttpApi(self.rls)

    def call(self, endpoint, bodies, now_us=T0):
        buf, off = HA.pack_bodies(bodies)
        p = self.api.plan(endpoint, buf, off, now_us)
        self.last_plan = p
        k = p["n_store"]
        co = p["ctr_off"]
        nc = int(co[-1]) if k else 0
        lim, fl = np.zeros(k, np.uint8), np.full(k, 0xFFFFFFFF, np.uint32)
        rem, ttl = np.zeros(nc, np.uint64), np.zeros(nc, np.uint64)
        self.runs = HA.store_runs(p["load_counters"])
        for j0, j1 in self.runs:
            c0, c1 = int(co[j0]), int(co[j1])
            out = self.o.batch_csr(MODE[endpoint], co[j0:j1 + 1] - c0, p["ctrs"][c0:c1], p["delta"][j0:j1], p["now_us"][j0:j1],
                                   bool(p["load_counters"][j0]))
            lim[j0:j1], fl[j0:j1], rem[c0:c1], ttl[c0:c1] = out
        return self.api.finish(lim, fl, rem, ttl)
