"""Limits in the matcher's boolean dialect and request streams for them, shared by the CPU and GPU tests of the serving
plans (tests/test_match_boolean_emu.py, tests/test_zza_boolean_gpu.py)."""
import numpy as np

from limitador_b200 import http_api as HA
from limitador_b200 import matcher as MT
from limitador_b200 import rls as R

SIX = ("descriptors[0].method == 'PUT' || descriptors[0].method == 'PATCH' || descriptors[0].method.startsWith('DEL') || "
       "descriptors[0].method.endsWith('ST') && !descriptors[0].method.contains('O') || descriptors[0].method in []")

LIMITS = [
    ("api", 5, 60, ["descriptors[0].method in ['GET', 'HEAD']"], ["descriptors[0].user"], "read-per-user"),
    ("api", 3, 60, ["descriptors[0]['req.path'].startsWith('/api/') && descriptors[0]['req.path'] != '/api/health'"],
     ["descriptors[0].user"], "api-per-user"),
    ("api", 40, 3600, ["has(descriptors[0].user)"], [], "users"),
    ("api", 120, 60, ["!(descriptors[0].method in ['OPTIONS', 'TRACE'])", "'tier' in descriptors[1]"], ["descriptors[1].tier"], None),
    ("api", 7, 10, ["descriptors[1].tier.endsWith('-gold') || descriptors[1].tier == 'free' && !descriptors[1].tier.contains('é')"],
     ["descriptors[0].user"], "tiers"),
    ("api", 9, 30, [SIX], [], "six-atoms"),
    ("api", 50, 60, ["descriptors[0].method == 'GET'"], [], "eq-only"),
    ("admin", 2, 10, ["descriptors[0].user.startsWith('adm')", "descriptors[0].user != 'admin'"], ["descriptors[0].user"], None),
]

METHODS = ["GET", "HEAD", "POST", "PUT", "PATCH", "DELETE", "OPTIONS", "TRACE", "CAST", "POST"]
PATHS = ["/api/", "/api/health", "/api/v1/x", "/ap", "/apié", "/日本", "", "/api/healthz"]
TIERS = ["gold", "x-gold", "free", "free-é", "", "日本-gold", "-gold"]
USERS = ["u1", "u2", "adm", "admin", "admin2", "é", ""]


def wide_limits():
    """A 50-limit namespace of boolean conditions: each request matches up to 50 counters (cap 64)."""
    conds = ["descriptors[0].k in ['1', 'x']", "descriptors[0].k.startsWith('1') || descriptors[0].k == 'y'",
             "!(descriptors[0].k == '2')", "has(descriptors[0].k)"]
    limits = []
    for l in range(50):
        vars_ = ["descriptors[0].user"] if l % 3 else []
        if l % 7 == 0:
            vars_ = ["descriptors[0].user", "descriptors[1].path"]
        limits.append(("wide", 2 + l % 5, 60 + l, [conds[l % 4]], vars_, f"l{l}" if l % 2 else None))
    limits.append(("api", 4, 60, ["has(descriptors[0].user)"], ["descriptors[0].user"], "per-user"))
    return limits


def matcher(limits, cap=None):
    m = MT.Matcher(dialect="boolean")
    if cap:
        m.set_counter_cap(cap)
    for l in limits:
        m.add_limit(*l)
    return m


def descriptors(rng):
    d0 = []
    for key, pool, p in (("method", METHODS, 0.9), ("user", USERS, 0.8), ("req.path", PATHS, 0.7)):
        if rng.random() < p:
            d0.append((key, str(rng.choice(pool))))
    descs = [d0]
    if rng.random() < 0.6:
        descs.append([("tier", str(rng.choice(TIERS)))] if rng.random() < 0.8 else [("other", "1")])
    return descs


def rls_messages(seed, n):
    rng = np.random.default_rng(seed)
    return [R.encode_request(str(rng.choice(["api", "api", "api", "admin", "nobody"])), descriptors(rng), int(rng.integers(0, 3)))
            for _ in range(n)]


def http_bodies(seed, n):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        d0 = dict(descriptors(rng)[0])
        out.append(HA.encode_info(str(rng.choice(["api", "api", "admin", "nobody"])), d0, int(rng.integers(0, 3)),
                                  [None, "DraftVersion03"][int(rng.integers(0, 2))]))
    return out


def wide_messages(seed, n):
    rng = np.random.default_rng(seed)
    msgs = []
    for _ in range(n):
        d0 = [("k", str(rng.choice(["1", "1", "2", "x", "y"]))), ("user", f"u{int(rng.integers(0, 6))}")]
        descs = [d0] + ([[("path", str(rng.choice(["/a", "/b"])))]] if rng.random() < 0.5 else [])
        msgs.append(R.encode_request("wide" if rng.random() < 0.8 else "api", descs, int(rng.choice([0, 1, 2]))))
    return msgs
