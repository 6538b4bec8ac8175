"""limitador_b200 — H100-native batched rate-limit engine for Kuadrant/limitador's
check_rate_limited_and_update hot path (see DESIGN.md)."""
from .engine import Engine, EngineError, Front, ShardBatch, owner_of, RECORD_DTYPE, COUNTER_DTYPE, LIMIT_DESC_DTYPE, NONE  # noqa: F401
from .limiter import (Authorization, CheckResult, Context, Counter, GpuCounterStorage, Limit,  # noqa: F401
                      RateLimiter)
from .matcher import Matcher, MatcherError, counter_key  # noqa: F401
from .rls import RlsService, RlsError  # noqa: F401
from .http_api import HttpApi, HttpError  # noqa: F401
from .crdt import CrdtTable, CrdtError  # noqa: F401

__all__ = ["Engine", "EngineError", "Front", "ShardBatch", "owner_of", "RateLimiter", "Limit", "Counter", "Context", "CheckResult",
           "Authorization", "GpuCounterStorage", "Matcher", "MatcherError", "counter_key", "RlsService", "RlsError", "HttpApi", "HttpError", "CrdtTable", "CrdtError", "RECORD_DTYPE", "COUNTER_DTYPE",
           "LIMIT_DESC_DTYPE", "NONE"]
