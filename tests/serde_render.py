"""A Python restatement of what actix's Json + serde_json write for GET /limits and GET /counters
(limitador-server/src/http_api/request_types.rs: Limit, Counter): compact, fields in declaration order, strings with the
short escapes and lower-case \\u00XX for the other control characters (Python's json.dumps with ensure_ascii=False
escapes exactly so), everything else raw; set_variables a BTreeMap (sorted by source bytes)."""
import json


def ser_str(s: str) -> str:
    return json.dumps(s, ensure_ascii=False)


def limit_json(ns, max_value, seconds, name, conditions, variables) -> str:
    return ('{"id":null,"namespace":%s,"max_value":%d,"seconds":%d,"name":%s,"conditions":[%s],"variables":[%s]}'
            % (ser_str(ns), max_value, seconds, "null" if name is None else ser_str(name),
               ",".join(ser_str(c) for c in sorted(set(conditions), key=str.encode)),
               ",".join(ser_str(v) for v in sorted(set(variables), key=str.encode))))


def counter_json(limit: str, set_variables: dict, remaining: int, ttl_us: int) -> str:
    sv = ",".join("%s:%s" % (ser_str(k), ser_str(set_variables[k])) for k in sorted(set_variables, key=str.encode))
    return '{"limit":%s,"set_variables":{%s},"remaining":%d,"expires_in_seconds":%d}' % (limit, sv, remaining, ttl_us // 1_000_000)


def limits_body(limits) -> bytes:
    """limits: (ns, max_value, seconds, conditions, variables, name) in counter order."""
    return ("[" + ",".join(limit_json(ns, mx, s, name, c, v) for ns, mx, s, c, v, name in limits) + "]").encode()


def counters_body(rows) -> bytes:
    """rows: (limit position, key_lo, key_hi, limit json, set_variables, remaining, ttl_us); sorted here."""
    rows = sorted(rows, key=lambda r: r[:3])
    return ("[" + ",".join(counter_json(r[3], r[4], r[5], r[6]) for r in rows) + "]").encode()
