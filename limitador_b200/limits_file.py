"""Limitador's limits file: the YAML list of limits `limitador-server` reads at start and applies again on every change
(limitador-server/src/main.rs:187-213, serde_yaml into `Vec<Limit>`, limitador/src/limit.rs:31-48).

Each entry is a mapping:
  namespace   required string
  seconds     required u64
  max_value   u64, default 0
  name, id    optional strings (null = absent)
  conditions  required sequence of strings (null = empty, as in the reference's examples/limits.yaml)
  variables   required sequence of strings (null = empty)
Other keys are ignored (the reference has no deny_unknown_fields).

The file is read with PyYAML's BaseLoader at the node level, so that no scalar is reinterpreted (`on`, `yes` or `010` stay
the strings they are) and every field is converted and type-checked here; where this differs from serde_yaml, DESIGN.md
§5 says so.  PyYAML is imported only when a file is parsed.  The result feeds RlsService.configure_with, which checks the
expressions against the matcher's dialect.
"""
from __future__ import annotations

import re
from typing import Dict, List, Optional

_NULL = ("", "~", "null", "Null", "NULL")
_U64 = re.compile(r"^\+?(?:0x[0-9a-fA-F]+|0o[0-7]+|0b[01]+|[0-9]+)$")


class LimitsFileError(ValueError):
    pass


def _yaml():
    try:
        import yaml
    except ImportError as e:  # pragma: no cover - depends on the environment
        raise LimitsFileError("reading a limits file needs PyYAML") from e
    return yaml


def _is_null(node) -> bool:
    return node.tag == "tag:yaml.org,2002:null" or (type(node).__name__ == "ScalarNode" and node.style is None
                                                     and node.value in _NULL)


def _where(node) -> str:
    return f"line {node.start_mark.line + 1}, column {node.start_mark.column + 1}"


def _string(node, field: str) -> str:
    if type(node).__name__ != "ScalarNode" or _is_null(node):
        raise LimitsFileError(f"{field}: expected a string at {_where(node)}")
    return node.value


def _u64(node, field: str) -> int:
    if type(node).__name__ != "ScalarNode" or node.style is not None or not _U64.match(node.value):
        raise LimitsFileError(f"{field}: expected an unsigned 64-bit integer at {_where(node)}")
    v = node.value.lstrip("+")
    n = int(v[2:], {"x": 16, "o": 8, "b": 2}[v[1]]) if len(v) > 2 and v[0] == "0" and v[1] in "xob" else int(v, 10)
    if n >= 1 << 64:
        raise LimitsFileError(f"{field}: {node.value} does not fit in 64 bits at {_where(node)}")
    return n


def _strings(node, field: str) -> List[str]:
    if _is_null(node):
        return []
    if type(node).__name__ != "SequenceNode":
        raise LimitsFileError(f"{field}: expected a sequence of strings at {_where(node)}")
    return [_string(x, field) for x in node.value]


def _limit(node, i: int) -> Dict:
    if type(node).__name__ != "MappingNode":
        raise LimitsFileError(f"limit {i}: expected a mapping at {_where(node)}")
    fields = {}
    for k, v in node.value:
        key = _string(k, f"limit {i}: key")
        if key in fields:
            raise LimitsFileError(f"limit {i}: duplicate field `{key}` at {_where(k)}")
        fields[key] = v
    for req in ("namespace", "seconds", "conditions", "variables"):
        if req not in fields:
            raise LimitsFileError(f"limit {i}: missing field `{req}` at {_where(node)}")

    def opt(key) -> Optional[str]:
        v = fields.get(key)
        return None if v is None or _is_null(v) else _string(v, f"limit {i}: {key}")

    return {
        "namespace": _string(fields["namespace"], f"limit {i}: namespace"),
        "max_value": _u64(fields["max_value"], f"limit {i}: max_value") if "max_value" in fields else 0,
        "seconds": _u64(fields["seconds"], f"limit {i}: seconds"),
        "name": opt("name"),
        "id": opt("id"),
        "conditions": _strings(fields["conditions"], f"limit {i}: conditions"),
        "variables": _strings(fields["variables"], f"limit {i}: variables"),
    }


def parse_limits(text) -> List[Dict]:
    """A limits file's text (str or bytes) -> one dict per limit (namespace, max_value, seconds, name, id, conditions,
    variables), in file order.  Raises LimitsFileError for anything serde would refuse."""
    yaml = _yaml()
    try:
        root = yaml.compose(text, Loader=yaml.BaseLoader)
    except yaml.YAMLError as e:
        raise LimitsFileError(f"not YAML: {e}") from e
    if root is None or type(root).__name__ != "SequenceNode":
        raise LimitsFileError("a limits file is a sequence of limits")
    return [_limit(x, i) for i, x in enumerate(root.value)]


def load_limits_file(path: str) -> List[Dict]:
    with open(path, "rb") as f:
        return parse_limits(f.read())
