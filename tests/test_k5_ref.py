"""tests/k5ref.py, the plain restatement the K5 edge tests check against, on hand-worked cases; and oracle/gojson.py's
civil-from-days time formatter against k5ref's datetime-based one over the whole domain of Go's signed UnixNano."""
import json

import pytest

import k5ref as kr
from oracle import gojson as G


def test_header_parse():
    assert kr.parse_headers(b"") == []
    assert kr.parse_headers(b"A: b\n") == [(b"A", b"b")]
    assert kr.parse_headers(b"A:b\n") == [(b"A", b"b")]
    assert kr.parse_headers(b"A:  b\n") == [(b"A", b" b")]              # exactly one space is dropped
    assert kr.parse_headers(b"A: b:c: d\n") == [(b"A", b"b:c: d")]      # the first ":" separates
    assert kr.parse_headers(b"A:\nB: \nC:: \n") == [(b"A", b""), (b"B", b""), (b"C", b": ")]
    assert kr.parse_headers(b": v\n") == [(b"", b"v")]
    for bad in (b"A: b", b"A b\n", b"A: b\n\n"):
        with pytest.raises(ValueError):
            kr.parse_headers(bad)


def test_header_map_needs_sorted_distinct_keys():
    assert kr.header_map(b"A: 1\nB: 2\n", False) == {b"A": b"1", b"B": b"2"}
    assert kr.header_map(b"k\xff: \xfe\n", True) == {"k\ufffd": "\ufffd"}
    for bad in (b"B: 1\nA: 2\n", b"A: 1\nA: 2\n"):
        with pytest.raises(ValueError):
            kr.header_map(bad, False)
    # two keys that are distinct and sorted as fed, equal after a round trip
    kr.header_map(b"k\xfe: 1\nk\xff: 2\n", False)
    with pytest.raises(ValueError):
        kr.header_map(b"k\xfe: 1\nk\xff: 2\n", True)


def test_time_kats():
    """Hand-derived: the epoch, one nanosecond, Go's last UnixNano instant, a leap day, and the fraction's trailing zeros."""
    assert kr.rfc3339(0) == b'"1970-01-01T00:00:00Z"'
    assert kr.rfc3339(1) == b'"1970-01-01T00:00:00.000000001Z"'
    assert kr.rfc3339(kr.MAX_NS) == b'"2262-04-11T23:47:16.854775807Z"'
    assert kr.rfc3339(951_868_800 * 10 ** 9 - 1) == b'"2000-02-29T23:59:59.999999999Z"'
    assert kr.rfc3339(4_107_542_400 * 10 ** 9 + 120_000_000) == b'"2100-03-01T00:00:00.12Z"'
    assert kr.rfc3339(1_700_000_000 * 10 ** 9 + 500) == b'"2023-11-14T22:13:20.0000005Z"'
    with pytest.raises(ValueError):
        kr.rfc3339(1 << 63)


def test_time_cases_cover_the_edges():
    ts = kr.time_cases(n_random=1000)
    assert min(ts) == 0 and max(ts) == kr.MAX_NS
    months = {kr.rfc3339(t)[1:8] for t in ts}
    assert len({m for m in months if b"1970" <= m[:4] <= b"2262"}) >= (2262 - 1970) * 12 + 4
    assert {len(kr.rfc3339(t)) for t in ts} == {22} | {23 + d for d in range(1, 10)}     # no fraction, and 1..9 digits
    for d in (b'"2000-02-29T', b'"2100-02-28T', b'"2100-03-01T', b'"2200-03-01T'):
        assert any(kr.rfc3339(t).startswith(d) for t in ts)


def test_go_time_matches_datetime_over_the_domain():
    """gojson.go_time (civil-from-days, the kernel's algorithm) and k5ref.rfc3339 (datetime) agree on every month's first and
    last instant 1970-2262, the leap-day edges, 0 and 2^63 - 1, every trailing-zero count, and 10^5 random values."""
    ts = kr.time_cases(n_random=100_000, seed=2)
    assert len(ts) > 100_000
    bad = [t for t in ts if G.go_time(t) != kr.rfc3339(t)]
    assert not bad, [(t, G.go_time(t), kr.rfc3339(t)) for t in bad[:5]]


def test_builders():
    s = kr.at_lane(b"\xe2\x82\xac", 30, step=1)
    assert len(s) == 65 and s[62:] == b"\xe2\x82\xac" and set(s[:62]) == {ord("a")}     # the last byte at lane 0 of step 2
    assert kr.at_lane(b"xyz", 31, length=33) == b"a" * 31 + b"xy"
    assert kr.at_lane(b"x", 0, step=2, length=70) == b"a" * 64 + b"x" + b"a" * 5
    sw = kr.lane_sweep(7)
    assert len(sw) == 256 * 32 and all(sw[32 * v + 7] == v for v in range(256))
    assert sw.count(b"a") == 256 * 31 + 1                                             # (and the step that holds "a" itself)
    assert kr.flat_headers([(b"A", b"1"), (b"B", b"")]) == b"A: 1\nB: \n"


def _rec(**kw):
    d = dict(agent=b"agent-1", method="POST", path=b"/p\xff", headers=b"K: v\xe2\x82\n", body=b"\x00\x01\x02\x03",
             created=1_700_000_000_000_000_000, max_retries=2, rid=bytes(range(16)))
    d.update(kw)
    return kr.Rec(**d)


HEAD = (b'{"id":"00010203-0405-0607-0809-0a0b0c0d0e0f","agent_id":"agent-1","method":"POST",')


def test_record_forms_hand_worked():
    r = _rec()
    assert r.wire() == HEAD + (b'"path":"/p\\ufffd","headers":{"K":"v\\ufffd\\ufffd"},"body":"AAECAw==","status":"pending",'
                               b'"retry_count":0,"max_retries":2,"created_at":"2023-11-14T22:13:20Z"}')
    assert r.wire(roundtrip=True) == HEAD + (b'"path":"/p\xef\xbf\xbd","headers":{"K":"v\xef\xbf\xbd\xef\xbf\xbd"},"body":"AAECAw==",'
                                             b'"status":"pending","retry_count":0,"max_retries":2,"created_at":"2023-11-14T22:13:20Z"}')
    r.error(b"e\xff")                                  # the request's strings are touched; the error text is fresh
    assert b'"path":"/p\xef\xbf\xbd"' in r.wire() and r.wire().endswith(b',"error":"e\\ufffd"}')
    assert b'"status":"pending","retry_count":1' in r.wire()
    r.response(404, b"R: \xff\n", b"ok", 1_700_000_000_000_000_001)      # the error text now touched, the response fresh
    w = r.wire()
    assert (b'"status":"completed","retry_count":1,"max_retries":2,"created_at":"2023-11-14T22:13:20Z",'
            b'"processed_at":"2023-11-14T22:13:20.000000001Z","response":{"status_code":404,"headers":{"R":"\\ufffd"},'
            b'"body":"b2s=","received_at":"2023-11-14T22:13:20.000000001Z"},"error":"e\xef\xbf\xbd"}') in w
    r.error(b"f\xff")                                  # the response touched, the new error text fresh, retry == max: failed
    w = r.wire()
    assert b'"headers":{"R":"\xef\xbf\xbd"}' in w and w.endswith(b'"error":"f\\ufffd"}') and b'"status":"failed","retry_count":2' in w
    r.error(b"")                                       # no text stored: what the proxy passes
    assert r.wire().endswith(b'"error":"transport error"}')
    json.loads(r.wire())


def test_retry_counter_saturates():
    r = _rec(max_retries=255)
    for _ in range(300):
        r.error()
    assert r.retry == 255 and r.status == "failed"
    assert b'"retry_count":255,"max_retries":255' in r.wire()


def test_rows_framing():
    a, b = _rec(), _rec(stored=False)
    one = a.wire()
    assert kr.wire_rows([a, b]) == (one + b"null", [0, len(one), len(one) + 4])
    assert kr.wire_rows([a, b], as_array=True) == (b"[" + one + b",null]", [0, len(one) + 1, len(one) + 7])
    assert kr.wire_rows([], as_array=True) == (b"null", [0])
    assert json.loads(kr.wire_rows([a, b, a], as_array=True)[0])[1] is None
