"""The matcher's boolean dialect (include/rl_match.h, RL_MATCH_DIALECT_BOOLEAN) on the CPU.

Every expression the dialect accepts must give the same answer under both of the error rules a CEL implementation may
follow inside && and || (tests/cel_bool_spec.py), in every context, and the native matcher must apply the limit exactly
when that answer is true: a randomised differential test over generated expressions and contexts, through
rl_matcher_counters, _counters_batch and _counters_batch_ns.  The refusal rule is not vacuous: among the refused
expressions the generator produces, the two rules disagree on some context.  The default table dialect is unchanged
(tests/test_matcher.py pins it)."""
import numpy as np
import pytest

from limitador_b200 import matcher as MT
from tests import cel_bool_spec as S

RULES = ("commutative", "left_to_right")


def _accepts(m, cond, ns="probe"):
    try:
        m.add_limit(ns, 1, 1, [cond], [])
        return True
    except MT.MatcherError as ex:
        assert "unsupported condition expression" in str(ex)
        return False


ACCEPTED = [
    "descriptors[0].method in ['GET', 'HEAD']",
    "descriptors[0]['req.path'].startsWith('/api/') && descriptors[0]['req.path'] != '/api/health'",
    "has(descriptors[0].user)",
    "'user' in descriptors[1]",
    "x == 'a'", "'a' == x", '"a" != x', "x in []", "x in [\"a\"]", "x.endsWith('.json')", "x.contains('é')",
    "!(x == 'a')", "!x.startsWith('a')", "!!(x in ['a'])", "(x == 'a' || x == 'b') && !x.contains('c')",
    "has(descriptors[0].u) && descriptors[0].u.startsWith('a') && y != 'b'",
    "x == 'a' && y == 'b'",  # two groups, one per conjunct
    "  descriptors [ 0 ] . m  ==  'GET'  ",
    "x == '1' || x == '2' || x == '3' || x == '4' || x == '5' || x == '6'",  # the cap: 6 atoms
    "(((x == 'a')))",
]

REFUSED = [
    "a == 'x' || b == 'y'", "!(a == 'x' && b == 'y')", "!has(descriptors[0].u)", "!('u' in descriptors[0])",
    "has(descriptors[0].u) || x == 'a'", "x == '1' || x == '2' || x == '3' || x == '4' || x == '5' || x == '6' || x == '7'",
    "x.matches('a.*')", "size(x) == 1", "x.size() == 1", "x == 1", "x == true", "x == null", "x == b'a'", "x == r'a'",
    "x == '''a'''", "x == 'a\\nb'", "limit.name == 'a'", "limit.id == 'a'", "req.method == 'GET'", "!x == 'a'",
    "!'u' in descriptors[0]", "x in ['a',]", "x in ['a', 1]", "x in y", "has(x)", "has(descriptors[0]['u'])",
    "descriptors[0] == 'a'", "descriptors == 'a'", "x == 'a' &&", "(x == 'a'", "x == 'a')", "x = 'a'", "x == 'a' & x == 'b'",
    "true", "x", "x.startsWith(y)", "'' in descriptors[0]", "in == 'a'", "has == 'a'", "x == 'a' ? 'b' : 'c'",
    "descriptors[4294967295].u == 'a'", "x.startsWith('a', 'b')", "x.Startswith('a')", "x == 'a\nb'",
    "!" * 40 + "(x == 'a')",  # nesting deeper than the parser's bound
]


def test_the_boolean_dialect_accepts_the_listed_shapes_and_refuses_the_rest():
    b, t = MT.Matcher(dialect="boolean"), MT.Matcher()
    for c in ACCEPTED:
        assert _accepts(b, c), c
    # root bindings named like CEL words, and a literal holding a line break, are the table dialect's own business
    table_accepts = {"descriptors == 'a'", "in == 'a'", "has == 'a'", "x == 'a\nb'"}
    for c in REFUSED:
        assert not _accepts(b, c), c
        assert _accepts(t, c) == (c in table_accepts), c
    # the table dialect still refuses every new shape (tests/test_matcher.py pins what it accepts)
    for c in ACCEPTED:
        assert _accepts(t, c) == (c == "x == 'a'"), c
    with pytest.raises(MT.MatcherError):
        MT.Matcher(dialect="cel")


def test_the_dialect_governs_only_later_limits():
    m = MT.Matcher()
    with pytest.raises(MT.MatcherError):
        m.add_limit("ns", 5, 60, ["x in ['a', 'b']"], [])
    a = int(m.add_limit("ns", 5, 60, ["x == 'a'"], [])["limit_id"])
    m.set_dialect("boolean")
    b = int(m.add_limit("ns", 5, 61, ["x in ['a', 'b']"], [])["limit_id"])
    m.set_dialect("table")
    with pytest.raises(MT.MatcherError):
        m.add_limit("ns", 5, 62, ["x in ['a', 'b']"], [])
    ns = m.namespace_id("ns")
    assert m.counters(ns, {"x": "a"})["limit_id"].tolist() == [a, b]
    assert m.counters(ns, {"x": "b"})["limit_id"].tolist() == [b]
    # the identity is the source text: the same condition added again in either dialect is the same limit
    assert int(m.add_limit("ns", 9, 60, ["x == 'a'"], [])["limit_id"]) == a


def test_an_equality_only_matcher_gives_the_same_image_in_both_dialects():
    from tests.test_rls_device_emu import matcher_image
    from tests import rls_corpora as RC
    for limits in (RC.wide_limits(), [(f"ns{i}", 10, 60, ["descriptors[0].method == 'GET'", "x != 'y'"], ["descriptors[0].user"])
                                      for i in range(20)]):
        t, b = MT.Matcher(), MT.Matcher(dialect="boolean")
        for l in limits:
            t.add_limit(*l)
            b.add_limit(*l)
        assert np.array_equal(matcher_image(t)[0], matcher_image(b)[0])


# ---- the randomised differential test ---------------------------------------------------------------------------------
KEYS = ["m", "u", "path"]
LITS = ["GET", "/api/", "/api/health", "", "a", "é", "日本", "aé", "/", "x y"]
VALUES = LITS + ["/api/v1", "/ap", "GE", "ET", "/api/healthz", "éa", "日本語", "a/api/", "HEAD", "b"]


def gen_operand(rng, root_ok=True):
    r = rng.random()
    if root_ok and r < 0.25:
        return (None, str(rng.choice(KEYS)))
    k = str(rng.choice(KEYS + ["req.path"])) if r > 0.9 else str(rng.choice(KEYS))
    return (int(rng.integers(0, 3)), k)


def gen_atom(rng, operand):
    op = str(rng.choice(["eq", "eq", "prefix", "suffix", "contains", "in"]))
    if op == "in":
        lits = [str(x) for x in rng.choice(LITS, size=int(rng.integers(0, 4)))]
    else:
        lits = [str(rng.choice(LITS))]
    return ("atom", operand, op, lits, op == "eq" and rng.random() < 0.4)


def gen_group(rng, operand, n_atoms, depth=0):
    if n_atoms == 1:
        a = gen_atom(rng, operand)
        return ("not", a) if rng.random() < 0.2 else a
    k = int(rng.integers(1, n_atoms))
    e = (str(rng.choice(["and", "or"])), gen_group(rng, operand, k, depth + 1), gen_group(rng, operand, n_atoms - k, depth + 1))
    return ("not", e) if rng.random() < 0.2 else e


def gen_has(rng):
    return ("has", int(rng.integers(0, 3)), str(rng.choice(KEYS)), str(rng.choice(["has", "in"])))


def gen_condition(rng):
    """Mostly shapes of the dialect; about a third break one of its rules."""
    parts = []
    for _ in range(int(rng.integers(1, 4))):
        parts.append(gen_has(rng) if rng.random() < 0.25 else gen_group(rng, gen_operand(rng), int(rng.integers(1, 5))))
    r = rng.random()
    if r < 0.12:  # || or ! across two operands
        a, b = gen_group(rng, gen_operand(rng), 1), gen_group(rng, gen_operand(rng), int(rng.integers(1, 3)))
        parts.append(("or", a, b) if rng.random() < 0.6 else ("not", ("and", a, b)))
    elif r < 0.22:  # presence under ! or ||
        parts.append(("not", gen_has(rng)) if rng.random() < 0.4 else ("or", gen_has(rng), gen_group(rng, gen_operand(rng), 1)))
    elif r < 0.28:  # more than 6 atoms in one group
        parts.append(gen_group(rng, gen_operand(rng), 7))
    e = parts[0]
    for p in parts[1:]:
        e = ("and", e, p)
    return e


def gen_context(rng):
    root = {k: str(rng.choice(VALUES)) for k in KEYS if rng.random() < 0.5}
    descs = []
    for _ in range(int(rng.integers(0, 4))):
        descs.append({k: str(rng.choice(VALUES)) for k in KEYS + ["req.path"] if rng.random() < 0.6})
    return root, descs


@pytest.mark.parametrize("seed", range(4))
def test_accepted_expressions_do_not_depend_on_the_error_rule_and_match_natively(seed):
    rng = np.random.default_rng(100 + seed)
    m = MT.Matcher(dialect="boolean")
    m.set_counter_cap(64)
    limits = []  # (namespace, limit id, [trees], variables)
    n_refused = n_disagree = 0
    contexts = [gen_context(rng) for _ in range(300)]
    for i in range(150):
        trees = [gen_condition(rng) for _ in range(int(rng.integers(1, 3)))]
        srcs = [S.render(t, int(rng.integers(0, 2))) for t in trees]
        vars_ = [S.render_operand(gen_operand(rng))] if rng.random() < 0.3 else []
        ns = f"ns{i % 5}"
        want = all(S.accepted(t) for t in trees)
        try:
            d = m.add_limit(ns, 10, 60 + i, srcs, vars_)
            got = True
        except MT.MatcherError:
            got = False
        assert got == want, srcs
        if got:
            limits.append((ns, int(d["limit_id"]), trees, vars_))
            continue
        n_refused += 1
        if any(any(S.test(t, r, ds, RULES[0]) != S.test(t, r, ds, RULES[1]) for r, ds in contexts) for t in trees if not S.accepted(t)):
            n_disagree += 1
    assert len(limits) > 60 and n_refused > 20
    assert n_disagree > 0  # refused shapes on which the two error rules do give different answers

    def applies(tr, vars_, root, descs):
        a = [all(S.test(t, root, descs, rule) for t in tr) for rule in RULES]
        assert a[0] == a[1], [S.render(t) for t in tr]
        return a[0] and all(_bound(_parse_var(v), root, descs) for v in vars_)

    names = [f"ns{int(rng.integers(0, 5))}" for _ in contexts]
    want_ids = [[lid for ns, lid, tr, vs in limits if ns == names[j] and applies(tr, vs, *contexts[j])] for j in range(len(contexts))]
    assert sum(map(len, want_ids)) > 100 and sum(1 for w in want_ids if not w) > 10
    ns_ids = [m.namespace_id(n) for n in names]
    off, ctrs = m.counters_batch(ns_ids, contexts)
    off2, ctrs2, status = m.counters_batch_ns(names, contexts)
    assert (status == 0).all() and np.array_equal(off, off2) and ctrs.tobytes() == ctrs2.tobytes()
    for j, (root, descs) in enumerate(contexts):
        got = ctrs[off[j]:off[j + 1]]
        assert got["limit_id"].tolist() == want_ids[j], (names[j], root, descs)
        assert m.counters(ns_ids[j], root, descs).tobytes() == got.tobytes()


def _bound(operand, root, descs):
    d, k = operand
    return k in root if d is None else d < len(descs) and k in descs[d]


def _parse_var(src):
    if src.startswith("descriptors["):
        d = int(src[len("descriptors["):src.index("]")])
        rest = src[src.index("]") + 1:]
        return (d, rest[1:] if rest.startswith(".") else rest[2:-2])
    return (None, src)


def test_the_parser_survives_random_noise_over_its_alphabet():
    """Noise built from the dialect's tokens: nothing crashes, and some of it is accepted."""
    rng = np.random.default_rng(7)
    pieces = ["x", "descriptors", "[", "]", "0", ".", "u", "'a'", '"b"', "==", "!=", "&&", "||", "!", "(", ")", "in", "has",
              "startsWith", "endsWith", "contains", ",", " ", "'é'", "''", "\\", "'", "1"]
    m = MT.Matcher(dialect="boolean")
    n_acc = 0
    for i in range(3000):
        if rng.random() < 0.5:  # an accepted expression with one piece inserted or one character dropped
            s = str(rng.choice(ACCEPTED))
            k = int(rng.integers(0, len(s) + 1))
            s = s[:k] + str(rng.choice(pieces)) + s[k:] if rng.random() < 0.5 else s[:k] + s[k + 1:]
        else:
            s = "".join(str(rng.choice(pieces)) for _ in range(int(rng.integers(1, 12))))
        n_acc += _accepts(m, s, f"noise{i}")
    assert n_acc > 100


def test_the_dialect_header_is_exported_and_bound():
    """include/rl_match_dialect.h (included by rl_match.h): every call it declares is exported and bound in Python."""
    from tests.test_abi import declared_functions
    lib = MT._lib()
    names = declared_functions("rl_match_dialect.h")
    assert names == sorted(MT.DIALECT_SYMBOLS)
    for n in names:
        assert hasattr(lib, n)
