"""Wire corpora for the RLS plan stage: every corpus is (limits, messages), the limits as Matcher.add_limit takes them.
The device plan (rl_rls_dev.cuh) is checked against the CPU plan (rl_rls_plan) on each of them, under the host shim
(tests/test_rls_device_emu.py) and on the GPU (tests/test_zz7_rls_device_gpu.py)."""
import numpy as np

from limitador_b200 import rls as R

from tests.test_rls import _KUADRANT_LIMIT, _KUADRANT_REQ, _gateway


def _enc(ns, descs, hits=1):
    return R.encode_request(ns, descs, hits)


def reference():
    """The messages and limits of the reference's server tests (tests/test_rls.py), in one matcher."""
    limits = [_KUADRANT_LIMIT,
              ("test_namespace", 10, 60, ["descriptors[0].x == '1'"], ["descriptors[0].z"], None),
              ("test_namespace", 0, 60, ["descriptors[0].x == '1'", "descriptors[1].y == '2'"], ["descriptors[0].z"], None),
              ("test_namespace", 10, 60, ["descriptors[0].x == '1'"], ["descriptors[0].y"], "named"),
              ("ns", 3, 60, ["descriptors[0].x == '1'"], ["descriptors[0].y"], "L")]
    msgs = [_enc("test_namespace", _KUADRANT_REQ), _enc("test_namespace", [[("req.method", "GET")]]),
            _enc("", [[("req.method", "GET")]]), _enc("test_namespace", [[("x", "1"), ("z", "1")], [("y", "2")]]),
            _enc("test_namespace", [[("x", "1"), ("y", "1")]], 6), _enc("test_namespace", [[("x", "1"), ("y", "2")]], 0),
            _enc("ns", [[("x", "1"), ("y", "k")]], 2), _enc("", []), _enc("test_namespace", _KUADRANT_REQ, 20)]
    return limits, msgs * 3


def gateway(seed, n=600):
    """_gateway streams (duplicate keys: the last one wins), plus descriptors without entries, which shift the indices."""
    limits, reqs = _gateway(seed, n)
    rng = np.random.default_rng(seed)
    msgs = [_enc(ns, descs, hits) for ns, descs, hits in reqs]
    for _ in range(n // 10):
        msgs.insert(int(rng.integers(0, len(msgs))), _enc("admin", [[], [("user", "u1")], [("path", "/a")]], 1))
        msgs.insert(int(rng.integers(0, len(msgs))), _enc("api", [[], []], 0))
    return limits, msgs


def mutations(seed=3, n=1500):
    """Truncations, byte flips, wrong wire types, groups (nested to the depth bound and past it), field 0, invalid
    UTF-8 and unknown fields of every wire type."""
    limits, _ = _gateway(0, 1)
    rng = np.random.default_rng(seed)
    base = [_enc("api", [[("method", "GET"), ("user", "u1")], [("path", "/a")]], 2), _enc("admin", [[("user", "u2")], [("path", "/b")]]),
            _enc("api", [[("method", "POST"), ("user", "u3"), ("user", "u4")]], 0)]
    good = base[0]
    hand = [b"\x08\x01" + good, b"\x10\x01" + good, good + b"\x1a\x00", good + b"\x1a\x01x",  # known fields, wrong wire types
            b"\x7b\x08\x01\x7c" + good, b"\x7b" * 100 + b"\x7c" * 100 + good, b"\x7b" * 101 + b"\x7c" * 101 + good,
            b"\x7b\x84\x01" + good, b"\x7b" + good, b"\x0c" + good, b"\x7c" + good,  # groups: nested, too deep, mismatched, open, stray
            b"\x00\x01" + good, b"\x02\x00" + good,  # field 0
            b"\x0a\x02\xc3\x28" + good, b"\x0a\x03\xed\xa0\x80", b"\x0a\x02\xc0\x80",  # invalid UTF-8 in the domain
            _enc("api", [[("method", "GET")]])[:-3] + b"\xff\xfe\x01",  # ... and in a value
            b"\x7a\x01\x66" + good, b"\x81\x01" + bytes(8) + good, b"\x8d\x01" + bytes(4) + good, b"\xf8\xff\xff\xff\x0f\x05" + good,
            b"\x12\x05\x0a\x03\x12\x01\x00" + good,  # a descriptor whose entry has an empty key and a NUL value
            b"\x12\x04\x12\x02\x08\x05" + good, b"\x12\x04\x12\x02\x18\x05" + good,  # overrides: valid, unknown field
            b"", b"\x18\xff\xff\xff\xff\xff\xff\xff\xff\xff\x02", b"\x18\xff\xff\xff\xff\x0f" + good]
    msgs = list(hand)
    for it in range(n):
        b = bytearray(base[it % len(base)])
        if it % 3 == 0:
            b = b[:int(rng.integers(0, len(b) + 1))]
        else:
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        msgs.append(bytes(b))
    return limits, msgs


def nul_bytes():
    limits, _ = _gateway(0, 1)
    msgs = [_enc("a\x00pi", [[("method", "GET"), ("user", "u1")]]), _enc("api", [[("method", "GET"), ("us\x00er", "u1")]]),
            _enc("api", [[("method", "GET"), ("user", "u\x001")]]), _enc("api", [[("method", "GET"), ("user", "u1")], [("zz", "\x00")]]),
            _enc("nobody", [[("k", "\x00")]]), _enc("api", [[("method", "GET"), ("user", "u1")]]), _enc("\x00", [])]
    return limits, msgs * 4


def edges():
    """Empty domains, unknown namespaces, hits_addend 0 and large."""
    limits, _ = _gateway(0, 1)
    msgs = [_enc("", [[("method", "GET"), ("user", "u1")]]), _enc("", []), _enc("nobody", [[("method", "GET")]]),
            _enc("API", [[("method", "GET"), ("user", "u1")]]), _enc("api", [[("method", "GET"), ("user", "u1")]], 0),
            _enc("api", [[("method", "GET"), ("user", "u1")]], 2**32 - 1), _enc("admin", [[("user", "u1")]], 0),
            _enc("admin", [[("user", "u1")], [("path", "/a")]], 7), _enc("api", [])]
    return limits, msgs * 5


def corpora():
    out = {"reference": reference(), "mutations": mutations(), "nul_bytes": nul_bytes(), "edges": edges()}
    for seed in (1, 2, 3):
        out[f"gateway{seed}"] = gateway(seed)
    return out


def wide_limits():
    """A 50-limit namespace: each request matches up to 50 counters (cap 64)."""
    limits = []
    for l in range(50):
        vars_ = ["descriptors[0].user"] if l % 3 else []
        if l % 7 == 0:
            vars_ = ["descriptors[0].user", "descriptors[1].path"]
        limits.append(("wide", 2 + l % 5, 60 + l, ["descriptors[0].k == '1'"], vars_, f"l{l}" if l % 2 else None))
    limits.append(("api", 4, 60, [], ["descriptors[0].user"], "per-user"))
    return limits


def wide_messages(seed, n):
    rng = np.random.default_rng(seed)
    msgs = []
    for _ in range(n):
        ns = "wide" if rng.random() < 0.8 else "api"
        d0 = [("k", str(rng.choice(["1", "1", "2"]))), ("user", f"u{int(rng.integers(0, 6))}")]
        descs = [d0] + ([[("path", str(rng.choice(["/a", "/b"])))]] if rng.random() < 0.5 else [])
        msgs.append(_enc(ns, descs, int(rng.choice([0, 1, 2]))))
    return msgs


def over_cap_limits(n_limits):
    """n_limits limits of one namespace that all apply to a request with descriptors[0].k == '1'."""
    return [("oc", 100, 60 + l, ["descriptors[0].k == '1'"], ["descriptors[0].u"] if l % 2 else [], None) for l in range(n_limits)]


def over_cap_messages():
    return [_enc("oc", [[("k", "1"), ("u", "x")]]), _enc("oc", [[("k", "2"), ("u", "x")]]), _enc("oc", [[("k", "1")]]),
            _enc("api", [[("k", "1")]])] * 8
