"""A specification of the matcher's boolean dialect (include/rl_match.h, RL_MATCH_DIALECT_BOOLEAN), written from CEL's
semantics rather than from the native code.

Expressions are trees:
  ("atom", operand, op, lits, negated)  operand = (descriptor index or None for a root binding, key); op one of
                                        "eq", "prefix", "suffix", "contains", "in"; negated only with "eq" (!=)
  ("has", index, key, style)            has(descriptors[index].key) (style "has") or 'key' in descriptors[index] ("in")
  ("not", x), ("and", a, b), ("or", a, b)
`render` writes one as CEL source.  `test` is the reference's Predicate::test (limit/cel.rs:321-339) under one of two
rules for errors inside && and ||:
  "commutative"    the CEL specification: false && error = error && false = false, true || error = error || true = true
  "left_to_right"  the first operand that errors decides: error && false = error, error || true = error
with the precheck that an unbound root variable makes the predicate false, and an error (a missing key, a descriptor
index past the end of the list) making it false.  `accepted` is the dialect's acceptance rule on the tree.
"""
from __future__ import annotations

ERR = "error"
MAX_ATOMS = 6


def render_operand(operand, style=0):
    d, k = operand
    if d is None:
        return k
    return f"descriptors[{d}].{k}" if style == 0 and k.isidentifier() and k.isascii() else f"descriptors[{d}]['{k}']"


def _q(s, dq=False):
    return f'"{s}"' if dq else f"'{s}'"


def render(e, style=0) -> str:
    kind = e[0]
    if kind == "atom":
        _, operand, op, lits, neg = e
        x = render_operand(operand, style)
        if op == "eq":
            sym = "!=" if neg else "=="
            return f"{_q(lits[0], style)} {sym} {x}" if style == 1 else f"{x} {sym} {_q(lits[0], style)}"
        if op == "in":
            return f"{x} in [{', '.join(_q(l, style) for l in lits)}]"
        fn = {"prefix": "startsWith", "suffix": "endsWith", "contains": "contains"}[op]
        return f"{x}.{fn}({_q(lits[0], style)})"
    if kind == "has":
        _, d, k, how = e
        return f"has(descriptors[{d}].{k})" if how == "has" else f"'{k}' in descriptors[{d}]"
    if kind == "not":
        inner = e[1]
        if inner[0] == "has" and inner[3] == "has" or inner[0] == "atom" and inner[2] in ("prefix", "suffix", "contains"):
            return "!" + render(inner, style)
        return f"!({render(inner, style)})"
    a, b = render(e[1], style), render(e[2], style)
    if kind == "and":
        a = f"({a})" if e[1][0] == "or" else a
        b = f"({b})" if e[2][0] in ("or", "and") else b
        return f"{a} && {b}"
    b = f"({b})" if e[2][0] == "or" else b
    return f"{a} || {b}"


def atoms(e):
    if e[0] == "atom":
        return [e]
    if e[0] == "has":
        return []
    return [x for c in e[1:] for x in atoms(c)]


def has_presence(e):
    if e[0] == "has":
        return True
    if e[0] == "atom":
        return False
    return any(has_presence(c) for c in e[1:])


def conjuncts(e):
    return conjuncts(e[1]) + conjuncts(e[2]) if e[0] == "and" else [e]


def accepted(e) -> bool:
    """The dialect's rule: a top-level && of presence tests and operand groups (one operand, at most 6 atoms)."""
    for c in conjuncts(e):
        if c[0] == "has":
            continue
        if has_presence(c):
            return False
        at = atoms(c)
        if len(at) > MAX_ATOMS or len({a[1] for a in at}) != 1:
            return False
    return True


def _lookup(operand, root, descs):
    d, k = operand
    if d is None:
        return root[k]  # the precheck has ruled out an unbound root
    if d >= len(descs) or k not in descs[d]:
        return ERR  # NoSuchKey / index out of range
    return descs[d][k]


def _atom(e, root, descs):
    _, operand, op, lits, neg = e
    v = _lookup(operand, root, descs)
    if v is ERR:
        return ERR
    if op == "eq":
        return (v == lits[0]) != neg
    if op == "in":
        return v in lits
    if op == "prefix":
        return v.startswith(lits[0])
    if op == "suffix":
        return v.endswith(lits[0])
    return lits[0] in v


def evaluate(e, root, descs, rule):
    kind = e[0]
    if kind == "atom":
        return _atom(e, root, descs)
    if kind == "has":
        return e[1] < len(descs) and e[2] in descs[e[1]]
    if kind == "not":
        v = evaluate(e[1], root, descs, rule)
        return ERR if v is ERR else not v
    stop = kind == "or"  # the value that decides: true for ||, false for &&
    a = evaluate(e[1], root, descs, rule)
    if rule == "left_to_right":
        if a is ERR or a == stop:
            return a
        return evaluate(e[2], root, descs, rule)
    b = evaluate(e[2], root, descs, rule)
    if a is not ERR and a == stop or b is not ERR and b == stop:
        return stop
    if a is ERR or b is ERR:
        return ERR
    return not stop


def roots(e):
    if e[0] == "atom":
        return {e[1][1]} if e[1][0] is None else set()
    if e[0] == "has":
        return set()
    return set().union(*(roots(c) for c in e[1:]))


def test(e, root, descs, rule) -> bool:
    """Predicate::test: false on an unbound root variable or an error, else the expression's value."""
    if not roots(e) <= set(root):
        return False
    v = evaluate(e, root, descs, rule)
    return False if v is ERR else bool(v)
