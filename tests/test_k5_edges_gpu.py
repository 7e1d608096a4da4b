"""The JSON wire form (K5, csrc/agr_k5_json.cu) against the plain restatement of tests/k5ref.py at the edges of its lane-level
code: a byte's lane in its 32-byte step, UTF-8 sequences and escapes that cross a step, the header parser's carries
across steps, the 32 base64 groups of a step, both timestamps (formatted on even and odd lanes), the per-warp stage and
its 768 B flushes, records that share 16-byte words, and the chunk scan's rounds of 1024 chunks.

Every read is checked whole, with every offset, after the output buffer has been filled with other bytes: `check` first
encodes a row whose wire form is at least as long and made of "~" almost everywhere, then makes one agr_rows_json call
whose capacity is the reference's length.  A store that the emit pass skips leaves a wrong byte; a length that the
measure pass gets wrong fails the call."""
import ctypes as C
import random

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k5ref as kr
from agentainer_lab_b200 import constants as K

pytestmark = pytest.mark.gpu

LAYOUTS = {"fixed": 0, "var": K.AGR_CFG_VARLEN}
IDS = {"hash": 0, "mint": K.AGR_CFG_MINT_IDS}
SECRET = 0x6b35_6b35
AGENT = b"agent-k5"
METHODS = list(K.METHOD_CODES)
TIMES = kr.time_cases(n_random=3000, seed=5)
PAYLOAD = {"fixed": K.AGR_PAYLOAD_BYTES, "var": K.AGR_VAR_MAX_RECORD - K.AGR_HEADER_BYTES}

# UTF-8 sequences: valid ones of every length and at the range edges, the escaped separators, a real U+FFFD, then the
# forms utf8.DecodeRune rejects (overlong, surrogates, above U+10FFFF, bytes that never start a sequence, lone
# continuation bytes) and sequences cut off by the next byte
VALID = [b"\xc2\x80", b"\xc3\xa9", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xe2\x82\xac", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xef\xbf\xbf",
         b"\xf0\x90\x80\x80", b"\xf0\x9f\x98\x80", b"\xf3\xbf\xbf\xbf", b"\xf4\x8f\xbf\xbf", b"\xe2\x80\xa8", b"\xe2\x80\xa9",
         b"\xef\xbf\xbd"]
INVALID = [b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf0\x80\x80\x80",
           b"\xf0\x8f\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8\x88\x80\x80\x80", b"\xfe", b"\xff", b"\x80",
           b"\xbf", b"\x80\x80\x80\x80", b"\xc2\x41", b"\xe2\x82\x41", b"\xf0\x9f\x98\x41", b"\xe2\x80\xa8\x80"]
PROBE_LANES = (0, 1, 2, 3, 28, 29, 30, 31)


def probes():
    """Short strings, each with one sequence at a chosen lane of its second step, or cut off at the string's end, or of one of
    the lengths around the step size."""
    out = []
    for seq in VALID + INVALID:
        for lane in PROBE_LANES:
            out.append(kr.at_lane(seq, lane, step=1) + b"zz")
        for m in range(1, len(seq)):                          # cut off at the end of the string
            out.append(kr.at_lane(seq[:m], 31 - m + 1, step=1))
    for n in (0, 1, 31, 32, 33, 63, 64, 65):
        out.append(b"L" * n)
        if n:
            out += [b"L" * (n - 1) + b"\xe2", b"L" * (n - 1) + b'"', b"\x01" * n]
    return out


def _outs(ops):
    outs = np.zeros(len(ops), dtype=A.outcome_dtype)
    segs, hl = [], np.zeros(len(ops), dtype=np.uint32)
    for j, (rec, kind, code, seq, hdr, body) in enumerate(ops):
        outs[j]["request_id"] = np.frombuffer(rec.rid, dtype=np.uint8)
        outs[j]["agent_id"] = rec.agent
        outs[j]["kind"], outs[j]["http_status"], outs[j]["seq"] = kind, code, seq
        segs.append(hdr + body)
        hl[j] = len(hdr)
    return outs, segs, hl


class Rig:
    """One engine, the records fed to it (k5ref.Rec) and a poison row that fills the output buffer before every checked read."""

    def __init__(self, layout="fixed", ids="hash", rows=1 << 14, resp=96 << 20, extra=0, max_agents=1024, setup=True):
        self.layout, self.var = layout, layout == "var"
        self.eng = A.Engine(slab_rows=rows, max_agents=max_agents, flags=K.AGR_CFG_PERSISTENCE | LAYOUTS[layout] | IDS[ids] | extra,
                            vslab_bytes=64 << 20, resp_bytes=resp, id_secret=SECRET)
        self.lib, self.h = self.eng.lib, self.eng.h
        self.batch = min(4096, rows // 2)                       # (a ring engine takes at most half its rows per call)
        self.rng = random.Random(f"{layout}-{ids}")
        self.agents = set()
        self.t = 0
        if setup:
            self.setup()

    def setup(self):
        """The anchor (the record that "null" rows replay) and the poison row."""
        self.anchor = self.mk(path=b"/anchor")
        self.anchor_row = self.ingest([self.anchor])
        self.poison_rec = self.mk(path=b"~" * 200, agent=b"agent-~~~~~~~~~~~~~~~~~~~~~~~~~")
        self.poison_row = self.ingest([self.poison_rec])
        self.poison_len = 0

    def close(self):
        self.eng.close()

    def agent(self, name: bytes):
        if name not in self.agents:
            assert self.lib.agr_set_agent_state(self.h, name, K.AGR_AGENT_STOPPED) >= 0, self.lib.agr_last_error()
            self.agents.add(name)

    def time(self, k=0):
        self.t += 1
        return TIMES[(self.t * 7 + k * len(TIMES) // 2) % len(TIMES)]

    def mk(self, path=b"/p", headers=b"", body=b"", agent=AGENT, max_retries=3, stored=True):
        i = self.rng.randrange(1 << 30)
        return kr.Rec(agent=agent, method=METHODS[i % len(METHODS)], path=path, headers=headers, body=body, created=self.time(),
                      max_retries=max_retries, rid=self.rng.randbytes(16), stored=stored)

    def ingest(self, recs):
        """Feeds the records in order (rows not stored are replays of the anchor); returns the first row.  Mint mode: the
        records take the ids the engine returns."""
        for r in recs:
            self.agent(r.agent)
            assert len(r.path) + len(r.headers) + len(r.body) <= PAYLOAD[self.layout], r
        n, first = len(recs), None
        for lo in range(0, n, self.batch):
            part = recs[lo:lo + self.batch]
            if self.var:
                blob, offs = [], [0]
                for r in part:
                    h = np.zeros(1, dtype=A.header_dtype)
                    self._head(h[0], r)
                    pay = r.path + r.headers + r.body
                    blob.append(h.tobytes() + pay + bytes(-len(pay) % 16))
                    offs.append(offs[-1] + len(blob[-1]))
                _, ids, f = self.eng.ingest_var(np.frombuffer(b"".join(blob), dtype=np.uint8).copy(), np.array(offs, dtype=np.uint32))
            else:
                arr = np.zeros(len(part), dtype=A.record_dtype)
                for i, r in enumerate(part):
                    self._head(arr[i], r)
                    pay = r.path + r.headers + r.body
                    arr[i]["payload"][: len(pay)] = np.frombuffer(pay, dtype=np.uint8)
                ids = np.zeros((len(part), 16), dtype=np.uint8)
                f = self.eng.ingest_ex(arr, np.zeros(len(part), dtype=A.verdict_dtype), ids)
            first = f if first is None else first
            for r, i in zip(part, ids):
                if r.stored and self.eng.mint:
                    r.rid = bytes(i)
        return first

    def _head(self, h, r):
        h["request_id"] = np.frombuffer(r.rid, dtype=np.uint8)
        h["agent_id"] = r.agent
        h["seq"] = r.created
        h["flags"] = K.METHOD_CODES[r.method] << K.AGR_F_METHOD_SHIFT
        h["path_len"], h["hdr_len"], h["body_len"] = len(r.path), len(r.headers), len(r.body)
        h["status"], h["max_retries"] = K.AGR_ST_PENDING, r.max_retries
        if not r.stored:                                        # a replay of a stored record: the row holds no record
            h["flags"] |= K.AGR_F_REPLAY
            h["replay_of"] = np.frombuffer(self.anchor.rid, dtype=np.uint8)

    def apply(self, ops, batch=4096):
        """ops: ("resp", rec, code, hdr, body) | ("err", rec, text), applied in order through agr_complete_ex and to the records."""
        rows = []
        for op in ops:
            if op[0] == "resp":
                _, rec, code, hdr, body = op
                t = self.time(1)
                if t == rec.created:
                    t = self.time(1)
                rows.append((rec, K.AGR_OUT_RESPONSE, code, t, hdr, body))
                rec.response(code, hdr, body, t)
            else:
                _, rec, text = op
                rows.append((rec, K.AGR_OUT_ERROR, 0, 0, b"", text))
                rec.error(text)
        batch = min(batch, self.batch)
        for lo in range(0, len(rows), batch):
            rc, res = self.eng.complete_ex(*_outs(rows[lo:lo + batch]))
            assert rc == 0 and (res == 0).all()

    def poison(self, need):
        """Fills the output buffer with at least `need` bytes of another row's wire form (array form: every byte one place
        further on), "~" almost everywhere."""
        if self.poison_len < need + 64:
            self.poison_len = max(2 * self.poison_len, need + 64)
            self.apply([("err", self.poison_rec, b"~" * self.poison_len)])
        assert self.eng.rows_json(self.poison_row, 1, as_array=True, fetch=False) >= need

    def read(self, first, n, as_array=False, roundtrip=False, cap=0):
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.uint64)
        ln = C.c_uint64()
        rc = self.lib.agr_rows_json(self.h, first, n, int(as_array) | (2 if roundtrip else 0), C.c_void_p(out.ctypes.data), cap,
                                    C.byref(ln), C.c_void_p(offs.ctypes.data))
        return rc, out[: ln.value].tobytes(), [int(o) for o in offs], ln.value

    def check(self, first, recs, as_array=False, roundtrip=False):
        want, woffs = kr.wire_rows(recs, as_array, roundtrip)
        self.poison(len(want))
        rc, got, offs, ln = self.read(first, len(recs), as_array, roundtrip, cap=len(want))
        assert rc == 0 and ln == len(want), (rc, ln, len(want), self.lib.agr_last_error())
        if got != want or offs != woffs:
            bad = next(i for i in range(len(recs)) if offs[i + 1] != woffs[i + 1] or got[woffs[i]:woffs[i + 1]] != want[woffs[i]:woffs[i + 1]])
            at = next((j for j in range(woffs[bad], woffs[bad + 1]) if got[j:j + 1] != want[j:j + 1]), None)
            raise AssertionError(f"row {bad} of {len(recs)} (as_array={as_array}, roundtrip={roundtrip}), first wrong byte at "
                                 f"{at}: got {got[woffs[bad]:woffs[bad + 1]]!r}\nwant {want[woffs[bad]:woffs[bad + 1]]!r}\n{recs[bad]}")
        return woffs

    def check_all_forms(self, first, recs):
        woffs = self.check(first, recs)
        self.check(first, recs, roundtrip=True)
        self.check(first, recs, as_array=True)
        return woffs


@pytest.fixture(params=[(lay, ids) for lay in LAYOUTS for ids in IDS], ids=lambda p: f"{p[0]}-{p[1]}")
def rig(request):
    r = Rig(*request.param)
    yield r
    r.close()


def _state_ops(rig, recs, states, rhdr=lambda i: b"", rbody=lambda i: b"", etext=lambda i: b""):
    """Outcome sequences that put a record's strings in each of their forms, by record index modulo len(states):
    0 none; 1 error then response (error text touched, response fresh); 2 response then error (response touched, error text
    fresh); 3 error, response, error (the error text fresh again after it was touched)."""
    ops = [[] for _ in range(4)]
    for i, r in enumerate(recs):
        s = states[i % len(states)]
        if s == 1:
            ops[0].append(("err", r, etext(i))); ops[1].append(("resp", r, 200 + i % 300, rhdr(i), rbody(i)))
        elif s == 2:
            ops[0].append(("resp", r, 201, rhdr(i), rbody(i))); ops[1].append(("err", r, etext(i)))
        elif s == 3:
            ops[0].append(("err", r, b"first \xff")); ops[1].append(("resp", r, 500, rhdr(i), rbody(i))); ops[2].append(("err", r, etext(i)))
    rig.apply([op for rnd in ops for op in rnd])


def _with_nulls(rig, recs, every=7):
    """Rows that hold no record ("null", 4 B) between the others, so that neighbouring warps share 16-byte words."""
    out = []
    for i, r in enumerate(recs):
        if i % every == 3:
            out.append(rig.mk(stored=False))
        out.append(r)
    return out


# ------------------------------------------------------------------------------------------------------------ strings
def test_request_strings_every_byte_at_every_lane(rig):
    """Every byte value at every lane, one per step, in the path, a request header's key (but ":" and newline) and its value
    (but newline); records fresh, after an error, after a response, and read with roundtrip."""
    per = 4 if not rig.var else 64                       # steps per field and record
    sweeps = {f: [kr.lane_sweep(l, [v for v in range(256) if v not in skip]) for l in range(32)]
              for f, skip in (("path", ()), ("key", (0x0a, 0x3a)), ("val", (0x0a,)))}
    recs = []
    for lane in range(32):
        n = max(len(sweeps[f][lane]) for f in sweeps) // (32 * per) + 1
        for c in range(n):
            part = {f: sweeps[f][lane][32 * per * c: 32 * per * (c + 1)] for f in sweeps}
            recs.append(rig.mk(path=part["path"], headers=part["key"] + b": " + part["val"] + b"\n"))
    recs = _with_nulls(rig, recs)
    first = rig.ingest(recs)
    _state_ops(rig, [r for r in recs if r.stored], (0, 1, 0, 2))
    woffs = rig.check_all_forms(first, recs)
    assert {o % 16 for o in woffs} == set(range(16))


def test_outcome_strings_every_byte_at_every_lane(rig):
    """Every byte value at every lane in a response header's key and value and in the error text, in each of their forms."""
    keys = [kr.lane_sweep(l, [v for v in range(256) if v not in (0x0a, 0x3a)]) for l in range(32)]
    vals = [kr.lane_sweep(l, [v for v in range(256) if v != 0x0a]) for l in range(32)]
    errs = [kr.lane_sweep(l) for l in range(32)]
    plan = [(l, s) for l in range(32) for s in ((1, 2, 3) if l in PROBE_LANES else (1, 2))]
    recs = [rig.mk() for _ in plan]
    first = rig.ingest(recs)
    for s in (1, 2, 3):
        sel = [i for i, p in enumerate(plan) if p[1] == s]
        _state_ops(rig, [recs[i] for i in sel], (s,), rhdr=lambda j: keys[plan[sel[j]][0]] + b": " + vals[plan[sel[j]][0]] + b"\n",
                   etext=lambda j: errs[plan[sel[j]][0]])
    rig.check(first, recs)
    rig.check(first, recs, roundtrip=True)


def test_sequences_across_steps_and_string_ends(rig):
    """UTF-8 sequences whose lead byte sits at lanes 28-31 (the rest in the next step) or at lanes 0-3, invalid forms, sequences
    cut off at the string's end and the lengths around one and two steps, in every string field and every form."""
    ps = probes()
    fields = 6
    recs = []
    for state in range(4):
        for i in range(len(ps)):
            p = [ps[(i + k) % len(ps)] for k in range(fields)]
            recs.append(rig.mk(path=p[0], headers=p[1] + b": " + p[2] + b"\n"))
            recs[-1].probe = (p[3], p[4], p[5], state)
    recs = _with_nulls(rig, recs, every=11)
    first = rig.ingest(recs)
    live = [r for r in recs if r.stored]
    states = [r.probe[3] for r in live]
    ops = [[] for _ in range(3)]
    for r, s in zip(live, states):
        hdr, text = r.probe[0] + b": " + r.probe[1] + b"\n", r.probe[2]
        if s == 1:
            ops[0].append(("err", r, text)); ops[1].append(("resp", r, 200, hdr, b""))
        elif s == 2:
            ops[0].append(("resp", r, 200, hdr, b"b")); ops[1].append(("err", r, text))
        elif s == 3:
            ops[0].append(("err", r, b"x\xff")); ops[1].append(("resp", r, 200, hdr, b"")); ops[2].append(("err", r, text))
    rig.apply([op for rnd in ops for op in rnd])
    rig.check_all_forms(first, recs)


def test_agent_ids(rig):
    """Agent ids of 1 and 31 bytes (the registration limit): every byte value at every lane, and sequences cut off at the
    id's end; fresh and touched."""
    names = [bytes([v]) for v in range(1, 256)]
    names += [bytes((v + k) % 255 + 1 for k in range(31)) for v in range(255)]
    for seq in VALID + INVALID:
        for lane in range(max(0, 31 - len(seq) - 1), 31):
            names.append(kr.at_lane(seq, lane, length=31))
    names = list(dict.fromkeys(n for n in names if len(n) <= 31 and b"\0" not in n))
    recs = [rig.mk(agent=n, path=b"/agent/" + n) for n in names]
    first = rig.ingest(recs)
    _state_ops(rig, recs, (0, 1))
    rig.check(first, recs)
    rig.check(first, recs, roundtrip=True)


# ------------------------------------------------------------------------------------------------------------ headers
def header_blobs():
    """Flattened header segments at the parser's edges (keys distinct and sorted)."""
    k31 = b"k" * 31
    hs = [
        k31 + b": v\n",                                        # ":" at lane 31, its space at lane 0 of the next step
        k31 + b":v\n", k31 + b":  v\n", k31 + b":\n", k31 + b": \n",
        b"k" * 30 + b": v\n",                                  # the space at lane 31
        b"a: " + b"v" * 28 + b"\nb: w\n",                      # newline at lane 31
        b"a: " + b"v" * 29 + b"\nb: w\n",                      # newline at lane 0
        b"a: " + b"v" * 28 + b":x\nb: w\n",                    # ":" in a value at lane 31
        b"a: " + b"v" * 29 + b":x\nb:y: z\n",                  # ":" in a value at lane 0 of the next step
        b"a: " + b"v" * 40 + b":" + b"w" * 40 + b": :\n",       # colons in a value two and three steps after its separator
        b"a:  v\nb: \nc:\nd:: \n",                             # a value that starts with a space, empty values, a value ":"
        b"K" * 70 + b": " + b"V" * 80 + b"\n" + b"L" * 33 + b":" + b"W" * 64 + b"\n",     # keys and values over 2-3 steps
        b"".join(bytes([c]) + b":\n" for c in range(0x21, 0x7f) if c != 0x3a),            # 93 lines of 3 bytes
        b"".join(bytes([c]) + b": " + bytes([c]) + b"\n" for c in range(0x41, 0x5b)),
        b"k\xc3\xa9: \xc3\xa9v\xe2\x82\xac\n\xf0\x9f\x98\x80: \xf0\x9f\x98\x80\n",          # sequences next to ": " and newline
        b"k\xe2\x80\xa8: \xe2\x80\xa9\n",
        b"a: \x80\xe2\n" + b"k\xe2\x82: \x82v\xe2\x82\n",      # cut sequences and lone continuations next to ": " and newline
        b"k\xff: \xff\n",
    ]
    out = []
    for h in hs:
        for shift in (0, 5, 13, 29, 30, 31, 33, 34):           # a first line (its key sorts first) moves the rest along the steps
            out.append(b" " * (shift - 4) + b": x\n" + h if shift else h)
    return out


def test_headers(rig):
    """Request and response headers at the parser's edges, each shifted across a step boundary; responses whose segment is all
    headers; every form."""
    blobs = header_blobs()
    recs = []
    for h in blobs:
        for s in range(3):
            recs.append(rig.mk(path=b"/h", headers=h if len(h) <= PAYLOAD[rig.layout] - 2 else b""))
            recs[-1].blob = (h, s)
    recs = _with_nulls(rig, recs)
    first = rig.ingest(recs)
    live = [r for r in recs if r.stored]
    _state_ops(rig, live, (0, 1, 2), rhdr=lambda i: live[i].blob[0],
               rbody=lambda i: b"" if i % 2 else b"body")
    rig.check_all_forms(first, recs)


# ------------------------------------------------------------------------------------------------------------ base64
def sextets(shift):
    """64 groups whose four 6-bit values are v, v+shift, v+2*shift, v+3*shift (mod 64): every value in every position."""
    return b"".join((((v << 18) | (((v + shift) % 64) << 12) | (((v + 2 * shift) % 64) << 6) | ((v + 3 * shift) % 64))).to_bytes(3, "big")
                    for v in range(64))


def test_base64(rig):
    """Request and response bodies of every length 0-200 and 96k-1..96k+1 (k = 1..4), and every 6-bit value in each of the four
    positions of a group; with varlen rows an 8 KiB body."""
    rng = random.Random(7)
    lens = list(range(201)) + [96 * k + d for k in range(1, 5) for d in (-1, 0, 1)]
    bodies = [rng.randbytes(n) for n in lens] + [sextets(s) for s in (0, 1, 5, 63)] + [sextets(1)[:n] for n in (190, 191)]
    if rig.var:
        bodies.append(rng.randbytes(PAYLOAD["var"] - 2))
    recs = [rig.mk(path=b"/b", body=b) for b in bodies]
    recs = _with_nulls(rig, recs)
    first = rig.ingest(recs)
    live = [r for r in recs if r.stored]
    _state_ops(rig, live, (0, 1), rhdr=lambda i: b"Content-Type: x\n", rbody=lambda i: bodies[-1 - i % len(bodies)])
    rig.check_all_forms(first, recs)


# ------------------------------------------------------------------------------------------------------------ numbers and times
def test_retry_counts_and_times(rig):
    """max_retries 0, 9, 10, 99, 100, 255 against retry counts crossing 9->10 and 99->100 and saturating at 255; every
    record's created_at and processed_at differ and come from the time cases (month ends 1970-2262, leap days, 2^63-1, every
    fraction length)."""
    recs, ops = [], []
    for mr in (0, 9, 10, 99, 100, 255):
        for ne in (0, 1, 9, 10, 11, 99, 100, 101, 254, 255, 256, 300):
            r = rig.mk(max_retries=mr)
            recs.append(r)
            ops += [("err", r, b"" if k % 2 else b"e%d" % k) for k in range(ne)]
            if ne % 3 == 1:
                ops.append(("resp", r, 7 if ne < 100 else 65535, b"", b""))
    first = rig.ingest(recs)
    rig.apply(ops, batch=3000)
    rig.check(first, recs)
    # every time case as a created_at; processed_at (drawn from the same cases, a different one) on two records in three
    recs = [rig.mk() for _ in TIMES]
    for r, t in zip(recs, TIMES):
        r.created = t
    first = rig.ingest(recs)
    rig.apply([("resp", r, 200, b"", b"") for i, r in enumerate(recs) if i % 3])
    rig.check(first, recs)


# ------------------------------------------------------------------------------------------------------------ stage and framing
def test_long_records_and_small_neighbours(rig):
    """A record of more than 60 KiB of output (an all-escaped error text: dozens of 768 B flushes) between "null" rows and
    short records; ranges of 1, 2, 255, 256 and 257 rows from every start residue mod 16, in both forms; the array's "[" and
    "]" in different chunks."""
    recs = []
    for i in range(700):
        recs.append(rig.mk(stored=(i % 3 != 1), path=b"/" + b"x" * (i % 37)))
    first = rig.ingest(recs)
    live = [r for r in recs if r.stored]
    big = live[5]
    rig.apply([("err", big, bytes(range(1, 32)) * 400)] +
              [("resp", r, 200, b"", b"q" * (i % 50)) for i, r in enumerate(live[6:40])] +
              [("resp", live[300], 200, b"A: " + b"\x01" * 3000 + b"\n", b"z" * 5000)])
    assert len(big.wire()) > 60 << 10
    woffs = rig.check_all_forms(first, recs)
    starts = {}
    for i in range(len(recs)):
        starts.setdefault(woffs[i] % 16, i)
    assert len(starts) == 16
    for n in (1, 2, 255, 256, 257):
        for a in sorted(set(starts.values()))[:16]:
            if a + n <= len(recs):
                rig.check(first + a, recs[a:a + n])
        a = recs.index(big)
        rig.check(first + a, recs[a:a + n], as_array=True)


def test_response_over_64k_and_get_record_json(rig):
    """A response over 64 KiB stored through agr_complete_ex; agr_get_record_json grows its buffer (AGR_ECAP) and returns it."""
    rng = random.Random(3)
    recs = [rig.mk(path=b"/big") for _ in range(3)]
    first = rig.ingest(recs)
    rig.apply([("resp", recs[0], 200, b"Content-Type: application/octet-stream\n", rng.randbytes(70 << 10)),
               ("err", recs[1], bytes(range(256)) * 64),
               ("resp", recs[2], 200, b"".join(b"H%05d: %s\n" % (k, b"\x7f<>&" * 8) for k in range(900)), b"")])
    for r in recs:
        assert len(r.wire()) > 64 << 10
        assert rig.eng.get_record_json(r.agent.decode(), r.rid) == r.wire()
    rig.check(first, recs)


@pytest.mark.parametrize("ids", sorted(IDS))
def test_rows_across_the_ring_end(ids):
    """AGR_CFG_RING: rows on both sides of the slab's physical end, read as one range.  A batch never wraps: the rows it skips
    at the end of a lap hold no record and read as null."""
    rig = Rig("fixed", ids, rows=1024, extra=K.AGR_CFG_RING, setup=False)
    try:
        old = [rig.mk(path=b"/old") for _ in range(700)]
        for r in old:
            r.created = 1000
        rig.ingest(old)
        assert rig.eng.expire(10 ** 6, 1000) == 700
        rig.eng.reclaim()
        rig.setup()
        rows, first = [], None
        for b in range(6):
            new = [rig.mk(path=b"/n" + b"w" * (i % 40), stored=i % 5 != 2) for i in range(100)]
            for r in new:
                r.created = 2 * 10 ** 6
            f = rig.ingest(new)
            first = f if first is None else first
            rows += [rig.mk(stored=False) for _ in range(f - first - len(rows))] + new      # the rows skipped at the lap's end
        assert first < 1024 < first + len(rows) and len(rows) > 600
        rig.apply([("resp", r, 200, b"A: b\n", b"x" * (i % 20)) for i, r in enumerate(rows) if r.stored and i % 3 == 0])
        rig.check_all_forms(first, rows)
    finally:
        rig.close()


# ------------------------------------------------------------------------------------------------------------ scan rounds
def test_scan_rounds_against_the_c_restatement():
    """More than 262 144 records (two rounds of k5_scan's 1024 chunks of 256): every record's wire form and offset from one
    agr_rows_json call, and one agent's pending list of more than 262 144 rows (agr_pending_json, whose selection runs again
    with a larger capacity), against oracle/cpu_ref.c."""
    from oracle.cpu_ref import CRef, record_dtype as cref_record
    n = 1024 * 256 + 8 * 256 + 77
    recs = A.synth_fill_host(0, n, seed=13, n_agents=1)
    name = A.synth_agent_id(0)
    rng = np.random.default_rng(5)
    with A.Engine(slab_rows=1 << 19, max_agents=8, flags=K.AGR_CFG_PERSISTENCE) as eng, CRef() as c:
        eng.set_agent_state(name, K.AGR_AGENT_STOPPED)
        c.set_agent_state(name, "stopped")
        first = eng.ingest_ex(recs, np.zeros(n, dtype=A.verdict_dtype), np.zeros((n, 16), dtype=np.uint8))
        c.ingest(recs.astype(cref_record))
        pick = rng.permutation(n)[:2000]
        outs = np.zeros(len(pick), dtype=A.outcome_dtype)
        outs["request_id"] = recs["request_id"][pick]; outs["agent_id"] = recs["agent_id"][pick]
        is_resp = np.arange(len(pick)) % 2 == 0
        outs["kind"] = np.where(is_resp, K.AGR_OUT_RESPONSE, K.AGR_OUT_ERROR)
        outs["http_status"] = np.where(is_resp, 200, 0)
        outs["seq"] = 1_700_000_000_000_000_000 + np.arange(len(pick))
        assert (eng.complete(outs) == 0).all()
        c.complete(outs)
        pieces = [c.get_json(name, recs["request_id"][i].tobytes()) for i in range(n)]
        want = b"".join(pieces)
        woffs = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.uint64)
        lib, h = eng.lib, eng.h
        # the same rows in array form first: longer, and every byte a place or more further on
        assert eng.rows_json(first, n, as_array=True, fetch=False) > len(want)
        out = np.zeros(len(want), dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.uint64)
        ln = C.c_uint64()
        assert lib.agr_rows_json(h, first, n, 0, C.c_void_p(out.ctypes.data), len(want), C.byref(ln), C.c_void_p(offs.ctypes.data)) == 0
        assert ln.value == len(want) and (offs == woffs).all()
        assert out.tobytes() == want
        want = c.pending_json(name)
        cnt_want = len(c.list(name, K.AGR_LIST_PENDING, cap=1 << 19))
        assert cnt_want > 262144
        assert eng.rows_json(first, n, fetch=False) > len(want)
        out = np.zeros(len(want), dtype=np.uint8)
        cnt = C.c_uint32()
        assert lib.agr_pending_json(h, name.encode(), C.c_void_p(out.ctypes.data), len(want), C.byref(ln), C.byref(cnt)) == 0
        assert cnt.value == cnt_want and ln.value == len(want)
        assert out.tobytes() == want
