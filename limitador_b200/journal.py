"""Persistent counters: a journal on disk that brings an engine's or a service's counters back after a crash.

The engine keeps its counters in HBM only.  A CounterJournal drains what changed from the device (Engine.drain_changes,
and RlsService.drain_counter_vars for the variable values GET /counters names counters by) and writes it to a
directory:
  base-<generation>.npz   a save_counters file, written on every full drain (the first one, and the first after any call
                          that moves rows or re-maps cells: a limit set or deleted, counters deleted, a compaction, an
                          import, a configure_with); temporary file, fsync, rename, fsync of the directory
  log-<generation>.bin    one record per delta drain, appended and fsynced: a fixed header (magic, format version,
                          sequence number, counter entries, variable entries, payload bytes), the little-endian arrays,
                          then a CRC32 of header and payload
recover(directory, target) loads the newest base and replays every complete record after it.

When to drain is the caller's policy (after every serve call, or every N ms): a crash loses at most the increments
since the last completed drain.  The reference's disk store writes every update through RocksDB's write-ahead log and
loses none on a process crash (limitador/src/storage/disk/rocksdb_storage.rs).  Drains are serialised with the decision
calls, as every maintenance call is.
"""
from __future__ import annotations

import os
import re
import struct
import zlib

import numpy as np

from .engine import Engine

MAGIC = b"RLJ1"
FORMAT_VERSION = 1
# magic, format version, reserved, sequence number, counter entries, variable entries, payload bytes
HEADER = struct.Struct("<4sHHQQQQ")
CRC = struct.Struct("<I")
_BASE = re.compile(r"^base-(\d{16})\.npz$")

_COUNTER_COLS = ((np.uint32, "limit_id"), (np.uint64, "key_lo"), (np.uint64, "key_hi"), (np.uint64, "value"),
                 (np.uint64, "expiry_us"))
_EMPTY_VARS = (np.zeros(0, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(1, np.uint64),
               np.zeros(0, np.uint8))


def _base_name(gen: int) -> str:
    return f"base-{gen:016d}.npz"


def _log_name(gen: int) -> str:
    return f"log-{gen:016d}.bin"


def _fsync_dir(directory: str):
    fd = os.open(directory, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _split(target):
    """-> (engine, service or None)"""
    if isinstance(target, Engine):
        return target, None
    return target._engine, target


def encode_record(seq: int, counters, cvars=_EMPTY_VARS) -> bytes:
    """One log record: the header, the five counter columns, the five variable columns (export_counter_vars' layout),
    all little-endian, then the CRC32 of everything before it."""
    cols = [np.ascontiguousarray(c, dtype=t).astype(np.dtype(t).newbyteorder("<"), copy=False)
            for c, (t, _) in zip(counters, _COUNTER_COLS)]
    vs, lo, hi, off, blobs = cvars
    off = np.ascontiguousarray(off, dtype="<u8")
    n, m = len(cols[0]), len(vs)
    if any(len(c) != n for c in cols) or len(lo) != m or len(hi) != m or len(off) != m + 1:
        raise ValueError("encode_record: the counter columns need one length, the variable columns m and m + 1")
    payload = b"".join([c.tobytes() for c in cols] + [
        np.ascontiguousarray(vs, dtype="<u4").tobytes(), np.ascontiguousarray(lo, dtype="<u8").tobytes(),
        np.ascontiguousarray(hi, dtype="<u8").tobytes(), off.tobytes(),
        np.ascontiguousarray(blobs, dtype=np.uint8)[:int(off[-1])].tobytes()])
    head = HEADER.pack(MAGIC, FORMAT_VERSION, 0, seq, n, m, len(payload))
    return head + payload + CRC.pack(zlib.crc32(head + payload))


def decode_records(data: bytes, first_seq: int = 1):
    """-> (records, good_bytes): every complete record of a log in order, as (seq, counters, cvars), and the bytes they
    take.  The replay ends at the first record that is short, fails its CRC, has another magic or format version, or
    does not carry the next sequence number; what follows is a torn or corrupt tail."""
    out, at, seq = [], 0, first_seq
    while at + HEADER.size <= len(data):
        magic, ver, _, s, n, m, plen = HEADER.unpack_from(data, at)
        end = at + HEADER.size + plen
        if magic != MAGIC or ver != FORMAT_VERSION or s != seq or end + CRC.size > len(data):
            break
        if CRC.unpack_from(data, end)[0] != zlib.crc32(data[at:end]):
            break
        fixed = 36 * n + 28 * m + 8
        if plen < fixed:
            break
        p, cols = at + HEADER.size, []
        for t, _ in _COUNTER_COLS:
            w = np.dtype(t).itemsize * n
            cols.append(np.frombuffer(data, dtype=np.dtype(t).newbyteorder("<"), count=n, offset=p).astype(t))
            p += w
        vs = np.frombuffer(data, dtype="<u4", count=m, offset=p).astype(np.uint32)
        p += 4 * m
        lo = np.frombuffer(data, dtype="<u8", count=m, offset=p).astype(np.uint64)
        p += 8 * m
        hi = np.frombuffer(data, dtype="<u8", count=m, offset=p).astype(np.uint64)
        p += 8 * m
        off = np.frombuffer(data, dtype="<u8", count=m + 1, offset=p).astype(np.uint64)
        p += 8 * (m + 1)
        blobs = np.frombuffer(data, dtype=np.uint8, count=end - p, offset=p).copy()
        if off[0] != 0 or np.any(np.diff(off.astype(np.int64)) < 0) or int(off[-1]) != len(blobs):
            break
        out.append((s, tuple(cols), (vs, lo, hi, off, blobs)))
        at = end + CRC.size
        seq += 1
    return out, at


class CounterJournal:
    """Drains `target` (an Engine or an RlsService) into `directory`.  Turns change tracking on: the engine keeps one
    more copy of its table in HBM, and the first drain writes a base.  Call drain() between serve calls, as often as
    the increments a crash may lose are worth: a crash loses at most those since the last completed drain."""

    def __init__(self, target, directory: str):
        self._engine, self._service = _split(target)
        self.directory = directory
        os.makedirs(directory, exist_ok=True)
        gens = [int(m.group(1)) for f in os.listdir(directory) if (m := _BASE.match(f))]
        self.generation = max(gens, default=0)
        self.seq = 0
        self._log = None
        self._engine.track_changes(True)

    def close(self):
        if self._log is not None:
            self._log.close()
            self._log = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def checkpoint(self):
        """A full drain now: a new base, and the log starts again."""
        self._engine.track_changes(True)
        return self.drain()

    def drain(self) -> dict:
        """Drain the device and make it durable -> {'full': bool, 'counters': entries, 'vars': entries, 'bytes': written}."""
        full, counters = self._engine.drain_changes()
        vfull, cvars = (False, _EMPTY_VARS) if self._service is None else self._service.drain_counter_vars()
        if full or vfull or self._log is None:
            written = self._write_base()
            return {"full": True, "counters": len(counters[0]), "vars": 0, "bytes": written}
        rec = encode_record(self.seq + 1, counters, cvars)
        self._log.write(rec)
        self._log.flush()
        os.fsync(self._log.fileno())
        self.seq += 1
        return {"full": False, "counters": len(counters[0]), "vars": len(cvars[0]), "bytes": len(rec)}

    def _write_base(self) -> int:
        gen = self.generation + 1
        path = os.path.join(self.directory, _base_name(gen))
        tmp = path + ".tmp"
        if self._service is not None:
            # The base holds the entries its counters reference.  The GC leaves exactly those in the dictionary, so a
            # key recorded later is recorded again, and a delta carries it.  now_us = 1: every present counter counts.
            self._service.counter_vars_gc(1)
            self._service.drain_counter_vars()  # the next delta starts here
        (self._service or self._engine).save_counters(tmp)
        with open(tmp, "rb") as f:
            os.fsync(f.fileno())
        os.replace(tmp, path)
        _fsync_dir(self.directory)
        self.close()
        self._log = open(os.path.join(self.directory, _log_name(gen)), "wb")
        os.fsync(self._log.fileno())
        _fsync_dir(self.directory)
        self.generation, self.seq = gen, 0
        for f in os.listdir(self.directory):  # the older bases and logs, and temporaries a crash left behind
            m = re.match(r"^(?:base|log)-(\d{16})\.(?:npz|bin)(?:\.tmp)?$", f)
            if m and (int(m.group(1)) < gen or f.endswith(".tmp")):
                os.remove(os.path.join(self.directory, f))
        _fsync_dir(self.directory)
        return os.path.getsize(path)


def _merge_counters(base_cols, records):
    """Per counter the last value wins; within a record the absents (value = expiry = 0) come first."""
    parts = [list(base_cols)]
    for _, cols, _ in records:
        absent = (cols[3] == 0) & (cols[4] == 0)
        order = np.concatenate([np.flatnonzero(absent), np.flatnonzero(~absent)])
        parts.append([c[order] for c in cols])
    cols = [np.concatenate([p[k] for p in parts]).astype(t) for k, (t, _) in enumerate(_COUNTER_COLS)]
    if not len(cols[0]):
        return cols
    rank = np.arange(len(cols[0]))
    order = np.lexsort((rank, cols[2], cols[1], cols[0]))
    s = [c[order] for c in cols]
    last = np.ones(len(order), bool)
    last[:-1] = (s[0][1:] != s[0][:-1]) | (s[1][1:] != s[1][:-1]) | (s[2][1:] != s[2][:-1])
    return [c[last] for c in s]


def _merge_vars(base_vars, records):
    """Every entry once (one key's values are the same wherever it comes from: they digest to the key)."""
    seen, vs, lo, hi, blobs = set(), [], [], [], []
    for v in [base_vars] + [r[2] for r in records]:
        V, L, H, O, B = v
        for i in range(len(V)):
            k = (int(V[i]), int(L[i]), int(H[i]))
            if k in seen:
                continue
            seen.add(k)
            vs.append(k[0])
            lo.append(k[1])
            hi.append(k[2])
            blobs.append(bytes(B[int(O[i]):int(O[i + 1])]))
    off = np.zeros(len(blobs) + 1, np.uint64)
    np.cumsum([len(b) for b in blobs], out=off[1:])
    return (np.array(vs, np.uint32), np.array(lo, np.uint64), np.array(hi, np.uint64), off,
            np.frombuffer(b"".join(blobs), np.uint8).copy())


def read_journal(directory: str, truncate: bool = True):
    """The newest base and every complete record after it -> (limits, counter columns, variable columns, info).  The
    merged state is what rl_counters_export(NULL, 0) listed at the last completed drain.  truncate: cut a torn or
    corrupt tail off the log (fsynced), so that a journal reopened on the directory never appends after it."""
    gens = [int(m.group(1)) for f in os.listdir(directory) if (m := _BASE.match(f))]
    if not gens:
        raise FileNotFoundError(f"{directory}: no journal base")
    gen = max(gens)
    with np.load(os.path.join(directory, _base_name(gen))) as z:
        limits = z["limits"]
        cols = [z[k] for _, k in _COUNTER_COLS]
        bvars = tuple(z[k] for k in ("cv_varset", "cv_key_lo", "cv_key_hi", "cv_blob_off", "cv_blobs")) if "cv_varset" in z \
            else _EMPTY_VARS
    log = os.path.join(directory, _log_name(gen))
    data = b""
    if os.path.exists(log):
        with open(log, "rb") as f:
            data = f.read()
    records, good = decode_records(data)
    if truncate and good < len(data):
        with open(log, "r+b") as f:
            f.truncate(good)
            os.fsync(f.fileno())
    merged = _merge_counters(cols, records)
    info = {"generation": gen, "records": len(records), "truncated_bytes": len(data) - good}
    return limits, merged, _merge_vars(bvars, records), info


def recover(directory: str, target, now_us: int = 0) -> dict:
    """Load a journal into `target` (an Engine or an RlsService with the same limits registered, as load_counters
    needs): the variable entries first (import_counter_vars; keeping must be on), then the counters through the limit
    checks of Engine.load_counters and import_counters.  Absent qualified counters are dropped before the import, and
    with now_us > 0 the qualified counters expired at now_us as well.  A crash loses at most the increments since the
    last completed drain.  -> {'generation', 'records', 'truncated_bytes', 'counters', 'vars'}."""
    engine, service = _split(target)
    limits, cols, cvars, info = read_journal(directory)
    qualified = np.zeros(int(limits["limit_id"].max()) + 1 if len(limits) else 1, bool)
    qualified[limits["limit_id"][limits["qualified"] != 0]] = True
    q = qualified[np.minimum(cols[0], len(qualified) - 1)] & (cols[0] < len(qualified))
    drop = q & (cols[4] == 0)
    if now_us:
        drop |= q & (cols[4] <= now_us)
    cols = [c[~drop] for c in cols]
    if service is not None and len(cvars[0]):
        service.import_counter_vars(*cvars)
    engine.import_snapshot(limits, cols, directory)
    return dict(info, counters=len(cols[0]), vars=len(cvars[0]))
