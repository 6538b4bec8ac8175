"""The limits-file parser (limitador_b200/limits_file.py) against the reference's example file and serde's rules for
`Vec<Limit>` (limit.rs:31-48).  Skipped where PyYAML is not importable."""
import os

import pytest

yaml = pytest.importorskip("yaml")
from limitador_b200 import limits_file as LF  # noqa: E402
from limitador_b200 import matcher as MT  # noqa: E402
from limitador_b200 import rls as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_the_reference_example_file():
    path = os.path.join(ROOT, "tests", "golden", "limits_example.yaml")
    assert LF.load_limits_file(path) == [
        {"namespace": "test_namespace", "max_value": 1000000, "seconds": 60, "name": None, "id": None, "conditions": [], "variables": []},
        {"namespace": "test_namespace", "max_value": 5, "seconds": 60, "name": None, "id": None,
         "conditions": ["descriptors[0]['req.method'] == 'POST'"], "variables": ["descriptors[0]['user_id']"]},
    ]
    s = R.RlsService(MT.Matcher(), None)
    assert s.load_limits_file(path) == {"kept": 0, "added": 2, "updated": 0, "deleted": 0}
    assert s.load_limits_file(path, dry_run=True) == {"kept": 2, "added": 0, "updated": 0, "deleted": 0}


def test_scalars_stay_strings_and_numbers_are_checked():
    text = """
- namespace: on
  seconds: 010
  max_value: 0x10
  name: yes
  id: "007"
  conditions: ["x == 'on'"]
  variables: [no]
  unknown_key: [1, 2]
- {namespace: '010', seconds: +3, conditions: ~, variables: null}
"""
    assert LF.parse_limits(text) == [
        {"namespace": "on", "max_value": 16, "seconds": 10, "name": "yes", "id": "007", "conditions": ["x == 'on'"], "variables": ["no"]},
        {"namespace": "010", "max_value": 0, "seconds": 3, "name": None, "id": None, "conditions": [], "variables": []},
    ]


@pytest.mark.parametrize("text,what", [
    ("", "sequence of limits"),
    ("namespace: a", "sequence of limits"),
    ("- [a]", "expected a mapping"),
    ("- {seconds: 1, conditions: [], variables: []}", "missing field `namespace`"),
    ("- {namespace: a, conditions: [], variables: []}", "missing field `seconds`"),
    ("- {namespace: a, seconds: 1, variables: []}", "missing field `conditions`"),
    ("- {namespace: a, seconds: 1, conditions: []}", "missing field `variables`"),
    ("- {namespace: a, seconds: '1', conditions: [], variables: []}", "unsigned 64-bit"),
    ("- {namespace: a, seconds: -1, conditions: [], variables: []}", "unsigned 64-bit"),
    ("- {namespace: a, seconds: 1.5, conditions: [], variables: []}", "unsigned 64-bit"),
    ("- {namespace: a, seconds: 18446744073709551616, conditions: [], variables: []}", "64 bits"),
    ("- {namespace: a, seconds: 1, max_value: ~, conditions: [], variables: []}", "unsigned 64-bit"),
    ("- {namespace: ~, seconds: 1, conditions: [], variables: []}", "namespace: expected a string"),
    ("- {namespace: [a], seconds: 1, conditions: [], variables: []}", "namespace: expected a string"),
    ("- {namespace: a, seconds: 1, conditions: x, variables: []}", "sequence of strings"),
    ("- {namespace: a, seconds: 1, conditions: [[x]], variables: []}", "expected a string"),
    ("- {namespace: a, seconds: 1, conditions: [~], variables: []}", "expected a string"),
    ("- {namespace: a, seconds: 1, name: [x], conditions: [], variables: []}", "name: expected a string"),
    ("- {namespace: a, namespace: b, seconds: 1, conditions: [], variables: []}", "duplicate field"),
    ("- {namespace: a\n", "not YAML"),
    ("- {namespace: a, seconds: 1, conditions: [], variables: []}\n---\n- {}", "not YAML"),
])
def test_what_serde_refuses_is_refused(text, what):
    with pytest.raises(LF.LimitsFileError, match=what):
        LF.parse_limits(text)
