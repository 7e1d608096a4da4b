"""Plain restatement of K5's wire form (csrc/agr_k5_json.cu) for the edge tests of tests/test_k5_edges_gpu.py.

Built only from what a test feeds the engine: the record fields, the flattened request and response headers, and the
outcomes in the order they were applied.  The string, map and record rules are oracle/gojson.py's.  Added here:
  - the flattened-header parse the kernel implements: lines end in "\\n", the first ":" of a line separates key and
    value, exactly one following space is dropped;
  - an RFC 3339 time formatter built on `datetime` (not on civil-from-days, which gojson.go_time and the kernel share);
  - the record state that decides which strings are written in their round-tripped ("touched") form;
  - builders that place a chosen byte sequence at a chosen lane of a chosen 32-byte step of a string.
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import datetime as _dt
import random
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

from oracle import gojson as G

STEP = 32                                   # bytes per warp step: one input byte per lane
EPOCH = _dt.datetime(1970, 1, 1)
MAX_NS = (1 << 63) - 1                      # time.Unix(0, ns): Go's UnixNano is signed


# ------------------------------------------------------------------------------------------------ headers
def parse_headers(flat: bytes) -> List[Tuple[bytes, bytes]]:
    """The flattened form "Key: Value\\n"... as (key, value) pairs in order."""
    if not flat:
        return []
    if not flat.endswith(b"\n"):
        raise ValueError("a flattened header segment ends in a newline")
    out = []
    for line in flat[:-1].split(b"\n"):
        i = line.find(b":")
        if i < 0:
            raise ValueError(f"header line without a separator: {line!r}")
        k, v = line[:i], line[i + 1:]
        out.append((k, v[1:] if v.startswith(b" ") else v))
    return out


def _raw(x) -> bytes:
    return x if isinstance(x, bytes) else x.encode("utf-8")


def header_map(flat: bytes, touched: bool) -> dict:
    """The map[string]string the reference marshals.  K5 writes the lines in their order, so a test must feed keys that are
    distinct and in sorted order in the form being written (a round trip can change the order of keys with invalid UTF-8)."""
    pairs = parse_headers(flat)
    conv = G.go_decode if touched else bytes
    m = {conv(k): conv(v) for k, v in pairs}
    keys = [_raw(k) for k in m]
    if len(m) != len(pairs) or keys != sorted(keys):
        raise ValueError(f"header keys must be distinct and sorted: {flat!r}")
    return m


def flat_headers(pairs: Sequence[Tuple[bytes, bytes]]) -> bytes:
    return b"".join(k + b": " + v + b"\n" for k, v in pairs)


# ------------------------------------------------------------------------------------------------ time
def rfc3339(ns: int) -> bytes:
    """time.Unix(0, ns).UTC().MarshalJSON() through datetime: seconds as a calendar date, then the fraction with its
    trailing zeros dropped."""
    if not 0 <= ns <= MAX_NS:
        raise ValueError("outside Go's UnixNano domain")
    secs, frac = divmod(ns, 1_000_000_000)
    t = EPOCH + _dt.timedelta(seconds=secs)
    s = f"{t.year:04d}-{t.month:02d}-{t.day:02d}T{t.hour:02d}:{t.minute:02d}:{t.second:02d}"
    if frac:
        s += "." + f"{frac:09d}".rstrip("0")
    return ('"' + s + 'Z"').encode()


def _ns(y, mo, d, h=0, mi=0, s=0, frac=0) -> int:
    return int((_dt.datetime(y, mo, d, h, mi, s) - EPOCH).total_seconds()) * 1_000_000_000 + frac


def time_cases(n_random: int = 100_000, seed: int = 1) -> List[int]:
    """Every month's first and last nanosecond 1970-2262, the leap-day edges, the domain's ends, every
    trailing-zero count of the fraction, and n_random values drawn uniformly from [0, 2^63)."""
    out = [0, 1, MAX_NS]
    for y in range(1970, 2263):
        for mo in range(1, 13):
            first = _ns(y, mo, 1)
            last = _ns(y + (mo == 12), mo % 12 + 1, 1) - 1
            out += [t for t in (first, last) if t <= MAX_NS]
    for (y, mo, d) in [(2000, 2, 29), (2000, 3, 1), (2100, 2, 28), (2100, 3, 1), (2200, 2, 28), (2200, 3, 1),
                       (2004, 2, 29), (2096, 2, 29), (2104, 2, 29), (2200, 12, 31), (2262, 4, 11)]:
        out += [_ns(y, mo, d), _ns(y, mo, d, 12, 34, 56, 7)]
    base = _ns(2024, 2, 29, 23, 59, 59)
    for tz in range(10):                       # a fraction with exactly tz trailing zeros (9 digits before trimming)
        out.append(base + 123456789 // 10 ** tz * 10 ** tz if tz < 9 else base)
        out.append(base + 10 ** tz if tz < 9 else base + 1)
    rng = random.Random(seed)
    out += [rng.randrange(0, 1 << 63) for _ in range(n_random)]
    return out


# ------------------------------------------------------------------------------------------------ string builders
def at_lane(seq: bytes, lane: int, step: int = 0, length: Optional[int] = None, fill: bytes = b"a") -> bytes:
    """`fill` bytes with `seq` starting at lane `lane` of step `step`; `length` cuts or pads the whole (default: the string
    ends right after seq)."""
    at = STEP * step + lane
    s = fill * at + seq
    if length is None:
        return s
    return (s + fill * max(0, length - len(s)))[:length]


def lane_sweep(lane: int, values: Sequence[int] = range(256), fill: bytes = b"a") -> bytes:
    """One step per value: step k holds values[k] at `lane` and `fill` elsewhere."""
    return b"".join(at_lane(bytes([v]), lane, length=STEP, fill=fill) for v in values)


# ------------------------------------------------------------------------------------------------ records
@dataclass
class Rec:
    """One stored record as fed, and the outcomes applied to it (through agr_complete_ex, so every outcome carries its bytes)."""
    agent: bytes
    method: str
    path: bytes
    headers: bytes               # flattened, as fed
    body: bytes
    created: int                 # Unix nanoseconds
    max_retries: int = 3
    rid: bytes = bytes(16)       # 16 raw bytes: fed in hash mode, returned by the ingest in mint mode
    stored: bool = True
    status: str = "pending"
    retry: int = 0
    responded: bool = False
    ptime: int = 0
    code: int = 0
    resp_hdr: bytes = b""
    resp_body: bytes = b""
    resp_rt: bool = False        # the Response has been through a later Unmarshal + Marshal
    err: bytes = b""
    err_rt: bool = False         # the Error has been through a later Unmarshal + Marshal

    def __post_init__(self):
        if self.max_retries == 0:    # the record layout's 0 means the reference's default of 3 (requests.go:95)
            self.max_retries = 3

    def error(self, text: bytes = b"") -> None:
        """MarkRequestFailed; an empty text reads "transport error" (the engine stores no text)."""
        self.retry = min(self.retry + 1, 255)          # the state word's 8-bit counter saturates
        self.status = "pending" if self.retry < self.max_retries else "failed"
        self.err, self.err_rt = text, False
        if self.responded:
            self.resp_rt = True

    def response(self, code: int, hdr: bytes, body: bytes, t: int) -> None:
        """StoreResponse with the flattened headers and body of the response, at time t."""
        self.status, self.responded, self.ptime, self.code = "completed", True, t, code
        self.resp_hdr, self.resp_body, self.resp_rt = hdr, body, False
        if self.retry:
            self.err_rt = True

    def wire(self, roundtrip: bool = False) -> bytes:
        """json.Marshal(requests.Request) of the record as the engine holds it; roundtrip: after one more json.Unmarshal."""
        if not self.stored:
            return b"null"
        touched = self.responded or self.retry > 0 or roundtrip

        def s(b, t):
            return G.go_decode(b) if t else b
        r = {"id": G.format_uuid(self.rid), "agent_id": s(self.agent, touched), "method": self.method,
             "path": s(self.path, touched), "headers": header_map(self.headers, touched), "body": self.body,
             "status": self.status, "retry_count": self.retry, "max_retries": self.max_retries, "created_at": self.created,
             "processed_at": None, "response": None, "error": ""}
        if self.responded:
            rt = self.resp_rt or roundtrip
            r["processed_at"] = self.ptime
            r["response"] = {"status_code": self.code, "headers": header_map(self.resp_hdr, rt), "body": self.resp_body,
                             "received_at": self.ptime}
        if self.retry:
            r["error"] = s(self.err or b"transport error", self.err_rt or roundtrip)
        return G.marshal_request(r)


def wire_rows(recs: Sequence[Rec], as_array: bool = False, roundtrip: bool = False) -> Tuple[bytes, List[int]]:
    """What agr_rows_json writes for these rows and its offsets[n + 1].  In array form a record's piece carries the "[" or
    "," before it, and the last one the "]"."""
    pieces = [r.wire(roundtrip) for r in recs]
    if as_array:
        if not pieces:
            return b"null", [0]
        pieces = [(b"[" if i == 0 else b",") + p for i, p in enumerate(pieces)]
        pieces[-1] += b"]"
    offs = [0]
    for p in pieces:
        offs.append(offs[-1] + len(p))
    return b"".join(pieces), offs
