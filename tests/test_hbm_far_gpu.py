"""Every byte region of the engine addressed past 4 GiB, against the plain references.

The engine keeps three byte-addressed regions in HBM: the 512-byte row slab (row p at byte 512 p), the record byte slab of a
variable-length engine (voff / vlen per row) and the response / error byte slab (resp_off / err_off per row).  A deployment's
slab is tens of GiB, and the default byte slabs pass 4 GiB at 4 M rows (records) and 64 M rows (responses).  A 32-bit
truncation of any of these offsets would not fault: it would alias into the low 4 GiB of the same allocation and overwrite
another row's bytes, and a round trip through the same truncated writer and reader would still pass.

So every case here keeps ALIASING PAIRS alive: items whose offsets differ by exactly 2^32 bytes (rows by 2^23), each with its
own random content, written through the path under test.  Truncating the writer or the reader makes one item's bytes show up
in place of the other's.  Each case checks placement twice: the per-row offsets (agr_debug_read) and raw device reads at the
predicted physical offset must equal the reference, and every read-back (agr_get_record(_var), agr_pending, the replay scan
with records, agr_rows_json / agr_pending_json, agr_get_response_body, agr_get_record_json, agr_verify with corruption planted
on both sides of 2^32) must equal the plain reference (tests/k1ref.py, k1vref.py, k5ref.py, verifyref.py, mintref.py).

The filler between the two items of a pair is written on the device (agr_synth_fill_rows + agr_ingest_rows, or one pinned
buffer reused for the responses), so the host never holds 4 GiB.  Each engine needs about 6 to 8 GiB of HBM; one is alive at a
time, and a case skips when the card does not have that much free."""
import ctypes as C

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1ref
import k1vref
import k5ref
import verifyref as VR
from agentainer_lab_b200 import constants as K
from mintref import mint_many

pytestmark = pytest.mark.gpu

P, M, V, CB = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_COMBINE
SECRET = 0x4C4F_4E47_0FF5_E701
G4 = 1 << 32                              # byte 2^32
R23 = 1 << 23                             # row 2^23 = byte 2^32 of the fixed slab
S_FAR = (1 << 23) + (1 << 16) + 5         # rows: not a multiple of 4 or 32, so K1's tiles straddle row 2^23 and the slab's end
BYTES_FAR = (1 << 32) + (1 << 28) + 48    # byte slabs a little above 2^32 + 2^28, not a multiple of 32
CHUNK = 1 << 20                           # rows per device-side filler step (max_batch)
REC = 512
TAG = "agent-far-tag"                     # every record a case reads back belongs to this agent
FILL = [A.synth_agent_id(k) for k in range(4)]   # the filler's agents, stopped: the filler stays out of the replay scan
FSEED = 17
METHODS = {v: k for k, v in K.METHOD_CODES.items()}
_rt = C.CDLL("libcudart.so")


def dev_read(ptr, n):
    out = np.zeros(max(n, 1), dtype=np.uint8)
    assert _rt.cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(n), 2) == 0
    return out[:n]


def dev_write(ptr, b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    assert _rt.cudaMemcpy(C.c_void_p(ptr), C.c_void_p(b.ctypes.data), C.c_size_t(len(b)), 1) == 0


def flip(ptr, mask=0x5A):
    dev_write(ptr, dev_read(ptr, 1) ^ np.uint8(mask))


def need_hbm(gib):
    free, total = C.c_size_t(), C.c_size_t()
    assert _rt.cudaMemGetInfo(C.byref(free), C.byref(total)) == 0
    if free.value < gib * (1 << 30):
        pytest.skip(f"need {gib} GiB, free {free.value / (1 << 30):.1f} GiB")


def engine(flags, **kw):
    kw.setdefault("max_agents", 64)
    e = A.Engine(device=0, flags=flags, id_secret=SECRET, **kw)
    e.set_agent_state(TAG, "stopped")
    for a in FILL:
        e.set_agent_state(a, "stopped")
    return e


def device_fill(eng, n):
    """n more rows reserved, filled on the device with the synthetic stream (index = row) and decided by K1; returns the first"""
    first = None
    for a in range(0, n, CHUNK):
        k = min(CHUNK, n - a)
        f = eng.reserve_rows(k)
        first = f if first is None else first
        eng.synth_fill_rows(f, f, k, seed=FSEED, n_agents=len(FILL))
        eng.ingest_rows(f, k, want_verdicts=False)
    return first


def tagged(n, rng, seq0):
    """n fixed records of TAG whose payload is random after a fixed path: every row's 512 bytes are its own"""
    r = np.zeros(n, dtype=A.record_dtype)
    path = f"/agent/{TAG}/far".encode()
    r["request_id"] = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    r["request_id"][:, 0] |= 1
    r["agent_id"] = TAG.encode()
    r["seq"] = seq0 + np.arange(n, dtype=np.uint64)
    r["flags"] = K.AGR_M_POST << K.AGR_F_METHOD_SHIFT
    r["path_len"], r["hdr_len"], r["body_len"] = len(path), 0, K.AGR_PAYLOAD_BYTES - len(path)
    r["max_retries"] = 3
    r["payload"] = rng.integers(0, 256, (n, K.AGR_PAYLOAD_BYTES), dtype=np.uint8)
    r["payload"][:, :len(path)] = np.frombuffer(path, dtype=np.uint8)
    return r


def ids_of(eng, recs, first):
    """Request.ID of rows [first, +n) as the reference knows it"""
    return mint_many(first, len(recs), SECRET) if eng.mint else np.ascontiguousarray(recs["request_id"])


def wire_rec(rec, rid):
    """k5ref.Rec of one stored 512-byte record (never completed)"""
    pl, hl, bl = int(rec["path_len"]), int(rec["hdr_len"]), int(rec["body_len"])
    pay = rec["payload"].tobytes()
    return k5ref.Rec(agent=rec["agent_id"], method=METHODS[(int(rec["flags"]) >> K.AGR_F_METHOD_SHIFT) & 0xFF], path=pay[:pl],
                     headers=pay[pl:pl + hl], body=pay[pl + hl:pl + hl + bl], created=int(rec["seq"]),
                     max_retries=int(rec["max_retries"]), rid=bytes(rid))


def fixed_readback(recs, state, ids):
    """the records as agr_get_record / agr_pending / the replay scan return them"""
    blob = np.ascontiguousarray(recs).view(np.uint8).ravel()
    offs = np.arange(len(recs) + 1, dtype=np.int64) * REC
    return k1vref.readback(blob, offs, state, np.zeros(len(recs), np.uint32), ids).view(A.record_dtype)


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero((got != want).reshape(len(got), -1).any(axis=1))[0] if got.ndim else []
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(got)} differ, first at {bad[:6].tolist()}"


# ---------------------------------------------------------------------------------------------- fixed 512-byte rows
FIXED_PATHS = ("ingest", "ingest_ex", "fill_rows", "synth_async", "tickets")


class FixedRig:
    """a fixed-stride engine of S_FAR rows and its K1 reference; tagged batches are checked as they land"""

    def __init__(self, mint):
        self.e = engine(P | CB | (M if mint else 0), slab_rows=S_FAR)
        slots = {a: self.e.agent_slot(a) for a in [TAG] + FILL}
        self.slot = slots[TAG]
        self.ref = k1ref.Ref({a: (s, K.AGR_AGENT_STOPPED) for a, s in slots.items()}, mint=mint, secret=SECRET)
        self.rows = {}                                        # row -> (expected slab bytes as a record, id, is TAG's)
        self.rng = np.random.default_rng(3 + mint)

    def used(self):
        return self.e.stats()["rows_used"]

    def batch(self, path, n):
        e, first = self.e, self.used()
        if path == "synth_async":
            recs = A.synth_fill_host(first, n, seed=FSEED + 1, n_agents=len(FILL))
        else:
            recs = tagged(n, self.rng, seq0=1000 + first)
        before = e.stats()
        iu0 = None if self.ref.mint else int(e.debug_read("index_used", 0, 1)[0])
        if path == "ingest":
            v, f = e.ingest(recs)
        elif path == "ingest_ex":
            v, ids = np.zeros(n, A.verdict_dtype), np.zeros((n, 16), np.uint8)
            f = e.ingest_ex(recs, v, ids)
            _same(ids, ids_of(e, recs, f), "ingest_ex ids")
        elif path == "fill_rows":
            f = e.reserve_rows(n)
            e.fill_rows(f, recs)
            v = e.ingest_rows(f, n)
        elif path == "synth_async":
            f = e.reserve_rows(n)
            e.synth_fill_rows(first, f, n, seed=FSEED + 1, n_agents=len(FILL))
            e.ingest_rows_async(f, n)
            e.sync()
            v = e.debug_read("verdict", f, n)
        else:                                                 # one ticket at a time through the service kernel (k_svc)
            res = [e.poll(e.submit_ingest(recs[i])) for i in range(n)]
            f = res[0]["rid"]
            assert [r["rid"] for r in res] == list(range(f, f + n)) and all(r["result"] == 0 for r in res)
            v = np.concatenate([r["verdict"] for r in res])
            _same(np.array([np.frombuffer(r["request_id"], np.uint8) for r in res]), ids_of(e, recs, f), "ticket ids")
        assert f == first
        c0, i0 = dict(self.ref.ctr), self.ref.index_used()
        out = self.ref.ingest(recs, f)
        _same(v.view("<u8"), out["verdict"].view("<u8"), f"{path} verdicts")
        _same(e.debug_read("verdict", f, n).view("<u8"), out["verdict"].view("<u8"), f"{path} verdict words")
        _same(e.debug_read("route", f, n), out["route"], f"{path} route")
        _same(e.debug_read("state", f, n), out["state"], f"{path} state")
        _same(e.debug_read("cksum", f, n), out["cksum"], f"{path} checksum")
        after = e.stats()
        for k in k1ref.COUNTERS:
            assert after[k] - before[k] == self.ref.ctr[k] - c0[k], (path, k)
        if iu0 is not None:                                   # the filler's ids are in the index too: compare what the batch added
            assert int(e.debug_read("index_used", 0, 1)[0]) - iu0 == self.ref.index_used() - i0, path
        ids = ids_of(e, recs, f)
        for i in range(n):
            self.rows[f + i] = (recs[i], ids[i], path != "synth_async")
        return f


@pytest.mark.parametrize("edge", [-17, -1])
@pytest.mark.parametrize("mint", [False, True])
def test_fixed_rows_past_row_2_23(mint, edge):
    """Rows [0, 200) and [2^23 + edge, +185) hold TAG's records written by all five ingest paths, the first K1 tile of the
    paths' rows starting at 2^23 + edge; rows p and p + 2^23 alias at byte 2^32.  The slab is filled to its last row, which
    holds one more tagged batch."""
    need_hbm(8)
    rig = FixedRig(mint)
    e = rig.e
    try:
        rig.batch("ingest", 200)
        assert device_fill(e, R23 + edge - 200) == 200
        starts = [rig.batch(p, 37 if p != "tickets" else 20) for p in FIXED_PATHS]
        assert starts[0] == R23 + edge and starts[-1] > R23
        device_fill(e, S_FAR - 37 - rig.used())
        last = rig.batch("ingest", 37)
        assert last + 37 == S_FAR == rig.used()
        rows = sorted(rig.rows)

        # raw reads at byte 512 p: what was sent, on both sides of every alias pair
        base = e.slab_ptr(0)
        assert e.slab_ptr(R23) == base + G4 and e.slab_ptr(S_FAR - 1) == base + (S_FAR - 1) * REC
        with pytest.raises(A.AgrError):
            e.debug_read("voff", 0, 1)                       # a fixed-stride engine has no record byte slab
        pairs = [p for p in rows if p >= R23 and p - R23 in rig.rows]
        assert len(pairs) >= 150
        for lo, hi in ((0, 200), (R23 + edge, R23 + edge + 168), (S_FAR - 37, S_FAR)):
            got = dev_read(base + lo * REC, (hi - lo) * REC).view(A.record_dtype)
            _same(got, np.array([rig.rows[p][0] for p in range(lo, hi)]), f"slab bytes of rows [{lo}, {hi})")

        # read-backs: agr_get_record, agr_pending, the JSON wire form, then the replay scan with records
        mine = [p for p in rows if rig.rows[p][2]]
        recs = np.array([rig.rows[p][0] for p in mine])
        ids = np.array([rig.rows[p][1] for p in mine])
        want = fixed_readback(recs, rig.ref.state[mine], ids if mint else None)
        got = np.array([e.get_record(TAG, ids[i].tobytes()) for i in range(len(mine))])
        _same(got.view(np.uint8).reshape(len(mine), -1), want.view(np.uint8).reshape(len(mine), -1), "agr_get_record")
        assert rig.ref.pending_rows(rig.slot) == mine
        _same(e.pending(TAG).view(np.uint8).reshape(len(mine), -1), want.view(np.uint8).reshape(len(mine), -1), "agr_pending")
        wires = [wire_rec(r, i) for r, i in zip(recs, ids)]
        js, cnt = e.pending_json(TAG)
        assert cnt == len(mine) and js == k5ref.wire_rows(wires, as_array=True, roundtrip=True)[0]
        for lo, n in ((R23 + edge, 168), (S_FAR - 37, 37), (0, 200)):
            js, _ = e.rows_json(lo, n)
            exp = [wire_rec(rig.rows[p][0], rig.rows[p][1]) for p in range(lo, lo + n)]
            assert js == k5ref.wire_rows(exp)[0], f"agr_rows_json of rows [{lo}, +{n})"
        e.set_agent_state(TAG, "running")
        disp, got = e.replay_scan(cap=len(mine))
        assert disp["rid"].tolist() == mine and (disp["agent_slot"] == rig.slot).all()
        _same(disp["request_id"], ids, "dispatch ids")
        _same(got.view(np.uint8).reshape(len(mine), -1), want.view(np.uint8).reshape(len(mine), -1), "replay scan records")

        # the integrity sweep: clean, then corruption at bytes 2^32 - 16, 2^32, 2^32 + 496 and in the last physical row
        assert e.verify() == (S_FAR, 0)
        for b in (G4 - 16, G4, G4 + 496, (S_FAR - 1) * REC + 300):
            flip(base + b)
        hit = np.array([R23 - 1, R23, S_FAR - 1])
        slab = np.concatenate([dev_read(base + int(p) * REC, REC) for p in hit])
        cks = np.concatenate([e.debug_read("cksum", int(p), 1) for p in hit])
        ref = VR.sweep(np.full(3, VR.ST_STORED, np.uint32), cks, slab, span=3, ring=False)
        assert len(ref.bad) == 3
        assert e.verify() == (S_FAR, len(ref.bad))
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------- variable-length records
VAR_LENS = [96, 512, 4096, 8192] * 10     # B's fourth record (an 8 KiB one) starts at byte 2^32 - 16
VAR_FORMS = {"staged": 0, "lsu": 0x20, "tickets": 0}


S_RING = (1 << 23) + (1 << 21) + 5        # a variable-length ring: rows for a second lap of 512-byte slots next to the first


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("form", list(VAR_FORMS))
@pytest.mark.parametrize("mint", [False, True])
def test_record_bytes_past_2_32(mint, form, ring):
    """A variable-length engine, append-only or a ring: blob A at byte 0, 4 GiB of 512-byte slots decided on the device, a
    pad record, then blob B (same lengths) through K1v in its staged or LSU form or through the service kernel (k_svc_var),
    its records beginning below byte 2^32 and ending above it, then reserved 512-byte slots above 2^32.  B's bytes past 2^32
    alias A's.  On the ring, everything before B's fifth record then expires and is released, so the byte ring's tail lies
    past 2^32; the next reservation skips the end of the lap (which lies past 2^32) to byte 0, and the ring is filled up to
    that tail exactly: 16 bytes more do not fit."""
    need_hbm(9)
    rng = np.random.default_rng(11 + mint + 2 * ring)
    e = engine(P | V | (M if mint else 0) | (CB if form == "tickets" else 0) | (K.AGR_CFG_RING if ring else 0),
               slab_rows=S_RING if ring else S_FAR, vslab_bytes=BYTES_FAR, k1_variant=VAR_FORMS[form])
    try:
        items = []                                           # (first row, blob, offsets, byte offset of the blob)

        def var(lens, seq0, split=None, seq_head=None):
            h = k1vref.headers(len(lens), [TAG], rng, seq0=seq0)
            if seq_head is not None:                         # the first records expire with everything before them
                h["seq"][:len(seq_head)] = seq_head
            k1vref.fit_lens(h, lens, rng)
            blob, offs = k1vref.blob_from(h, lens, rng)
            at = e.stats()["rows_used"]
            vb = vused
            parts = [(0, len(lens))] if split is None else [(0, split), (split, len(lens))]
            for a, b in parts:                               # n <= 32 in the compact form: one ticket per record
                sub = np.ascontiguousarray(blob[offs[a]: offs[b]])
                ops = e.stats()["svc_ops"]
                v, ids, f = e.ingest_var(sub, (offs[a: b + 1] - offs[a]).astype(np.uint32))
                # the service kernel decided exactly the calls that had to go through it
                assert e.stats()["svc_ops"] - ops == (b - a if form == "tickets" and b - a <= 32 else 0)
                assert f == at + a
                assert (v["code"] == K.AGR_V_QUEUED).all() and (v["flags"] == K.AGR_VF_STORED | K.AGR_VF_TRACKED).all()
                want_ids = mint_many(f, b - a, SECRET) if mint else h["request_id"][a:b]
                _same(ids, want_ids, "ingest_var ids")
            items.append((at, blob, offs, vb, h))
            return vb + int(offs[-1])

        vused = 0
        vused = var(VAR_LENS, 1)                             # A
        target = G4 - 16 - sum(VAR_LENS[:3])                 # where B must begin
        k = (target - vused - 600) // REC
        device_fill(e, k)                                    # (synthetic records: seq = row + 1 < 2^24)
        vused += REC * k
        vused = var([target - vused], 10_000)               # one pad record up to B
        assert vused == target
        vused = var(VAR_LENS, 1 << 24, split=20 if form == "tickets" else None, seq_head=[5] * 4)   # B
        # reserved 512-byte slots, filled from the host, above 2^32
        slots = tagged(37, rng, seq0=(1 << 24) + 1000)
        f = e.reserve_rows(37)
        e.fill_rows(f, slots)
        v = e.ingest_rows(f, 37)
        assert (v["flags"] == K.AGR_VF_STORED | K.AGR_VF_TRACKED).all()
        sblob = slots.view(np.uint8).ravel()
        soffs = (np.arange(38) * REC).astype(np.uint32)
        items.append((f, sblob, soffs, vused, slots.view(np.uint8).reshape(37, REC)[:, :96].copy().view(A.header_dtype).ravel()))
        vused += 37 * REC

        base = e.slab_ptr(0)
        a_first = items[0][0]
        b_first, _, b_offs, b_at, _ = items[2]
        assert b_at + int(b_offs[3]) == G4 - 16 and b_at + int(b_offs[-1]) > G4 + 60_000
        assert items[3][3] > G4
        live = []
        for first, blob, offs, at, h in items:
            n = len(offs) - 1
            _same(e.debug_read("voff", first, n), at + offs[:-1].astype(np.uint64), f"voff of rows [{first}, +{n})")
            _same(e.debug_read("vlen", first, n), np.diff(offs.astype(np.int64)).astype(np.uint32), f"vlen of rows [{first}, +{n})")
            _same(e.debug_read("cksum", first, n), k1vref.cksum(blob, offs), f"checksums of rows [{first}, +{n})")
            raw = dev_read(base + at, int(offs[-1]))
            assert (raw == blob).all(), f"byte slab at [{at}, +{int(offs[-1])}) differs from the records sent"
            state = k1vref.stored_state(h, np.zeros(n, bool))
            _same(e.debug_read("state", first, n), state, "state")
            ids = mint_many(first, n, SECRET) if mint else np.ascontiguousarray(h["request_id"])
            want = k1vref.readback(blob, offs, state, np.zeros(n, np.uint32), ids if mint else None)
            for i in range(n):
                got = e.get_record_var(TAG, ids[i].tobytes())
                assert got is not None and (got == want[offs[i]: offs[i + 1]]).all(), f"agr_get_record_var of row {first + i}"
            live.append((first, n, want, offs, ids))
        # a pair at distance 2^32: A's record 0 and the bytes of B that lie past 2^32
        assert e.debug_read("voff", a_first, 1)[0] == 0

        # the replay scan with records (k_var_copy): TAG's rows, in row order
        e.set_agent_state(TAG, "running")
        disp, blob, offs = e.replay_scan_var(blob_cap=1 << 21)
        rids = np.concatenate([np.arange(f, f + n) for f, n, _, _, _ in live])
        assert disp["rid"].tolist() == rids.tolist()
        _same(disp["request_id"], np.concatenate([x[4] for x in live]), "dispatch ids")
        want = np.concatenate([w for _, _, w, _, _ in live])
        assert len(blob) == len(want) and (blob == want).all(), "agr_replay_scan_var records"

        # the integrity sweep: clean, then corruption at 2^32 - 16, 2^32, 2^32 + 496 (all in B's fourth record), in A's first
        # record (at the alias of 2^32) and in the last slot
        used = e.stats()["rows_used"]
        assert e.verify() == (used, 0)
        last = items[3][0] + 36
        for b in (G4 - 16, G4, G4 + 496, 0, items[3][3] + 36 * REC + 511):
            flip(base + b)
        hit = [a_first, b_first + 3, last]
        vo = np.concatenate([e.debug_read("voff", r, 1) for r in hit]).astype(np.int64)
        vl = np.concatenate([e.debug_read("vlen", r, 1) for r in hit]).astype(np.int64)
        slab = np.concatenate([dev_read(base + int(o), int(l)) for o, l in zip(vo, vl)])
        loc = np.concatenate([[0], np.cumsum(vl)[:-1]])
        cks = np.concatenate([e.debug_read("cksum", r, 1) for r in hit])
        ref = VR.sweep(np.full(3, VR.ST_STORED, np.uint32), cks, slab, span=3, ring=False, voff=loc, vlen=vl)
        assert len(ref.bad) == 3
        assert e.verify() == (used, len(ref.bad))
        if not ring:
            return

        e.set_agent_state(TAG, "stopped")
        # release: everything before B's fifth record expires; the new tail is that record's voff (k_first_live, reclaim_apply)
        assert e.expire(1 << 24, 1) == used - 36 - 37
        assert e.reclaim() == b_first + 4
        tail = b_at + int(b_offs[4])
        assert tail > G4
        # the lap ends past 2^32: a reservation that does not fit before it skips to byte 0 (vbytes_fit / vbytes_take)
        n0 = 1 << 19
        assert vused < BYTES_FAR < vused + n0 * REC
        f0 = device_fill(e, n0)
        assert e.debug_read("voff", f0, 1)[0] == 0
        vused = BYTES_FAR + n0 * REC                         # logical: the second lap
        # fill up to the tail with slots, then records: 16 bytes more do not fit, the exact amount does
        free = tail + BYTES_FAR - vused
        while free > (CHUNK + 64) * REC:
            device_fill(e, CHUNK)
            vused += CHUNK * REC
            free -= CHUNK * REC
        m = free // REC - 32
        device_fill(e, m)
        vused += m * REC
        free -= m * REC
        lens = [400] * 33 + [free - 400 * 33]                # more than 32 records: one locked batch, all or nothing
        assert 96 <= lens[-1] <= 8192 and lens[-1] % 16 == 0
        with pytest.raises(A.AgrError) as ex:
            over = lens[:-1] + [lens[-1] + 16]
            h = k1vref.headers(len(over), [TAG], rng, seq0=1 << 25)
            k1vref.fit_lens(h, over, rng)
            blob, offs = k1vref.blob_from(h, over, rng)
            e.ingest_var(blob, offs)
        assert ex.value.code == K.AGR_ENOSPC
        at = vused
        vused = var(lens, 1 << 25)
        assert vused == tail + BYTES_FAR
        first, _, offs, _, _ = items[-1]
        _same(e.debug_read("voff", first, len(lens)), (at - BYTES_FAR) + offs[:-1].astype(np.uint64), "voff of the last records")
        with pytest.raises(A.AgrError) as ex:
            var([96] * 33, 1 << 25)
        assert ex.value.code == K.AGR_ENOSPC
        # B's live records past 2^32 are untouched by the second lap, which ends right below them
        bf, bn, bwant, boffs, bids = live[2]
        for i in range(4, bn):
            got = e.get_record_var(TAG, bids[i].tobytes())
            assert got is not None and (got == bwant[boffs[i]: boffs[i + 1]]).all(), f"agr_get_record_var of row {bf + i}"
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------- response / error bytes
SEG = (1 << 16) - 5                       # filler segment: rounds up to 64 KiB in the slab
SEGS_PER_CALL = 2048                      # one pinned buffer of 128 MiB, reused call after call


def r16(x):
    return (int(x) + 15) & ~15


def segments(rng, n, lo, hi):
    """n response segments (flattened headers, body) of random lengths: odd lengths, so the sources sit at every residue mod 16"""
    out = []
    for i in range(n):
        hdr = f"X-Far: {i}\n".encode() if i % 3 else b""
        body = rng.integers(0, 256, int(rng.integers(lo, hi)) | 1, dtype=np.uint8).tobytes()
        out.append((hdr, body))
    return out


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("mint", [False, True])
def test_response_bytes_past_2_32(mint, ring):
    """Responses of rows [0, 64) at byte 0 of the response slab (agr_complete_ex), 4 GiB of responses of other rows from one
    pinned buffer, then responses and error texts below, across and above byte 2^32 through agr_complete_ex (one batch across
    2^32, one wholly above it), single-slot and multi-slot tickets (k_svc) and agr_store_response / agr_store_error_text.  The
    rows at byte 2^32 + x alias those at x.  On the ring, the first rows of [0, 64) then expire and are released while the live
    responses still span more than 4 GiB, so the new tail (k_bytes_span) is the offset of the oldest live one; the rest of the
    lap is filled, and a batch that skips the end of the lap (past 2^32) to byte 0 fits exactly up to that tail."""
    need_hbm(7)
    rng = np.random.default_rng(23 + mint + 2 * ring)
    nrows = 70_000
    e = engine(P | CB | (M if mint else 0) | (K.AGR_CFG_RING if ring else 0), slab_rows=1 << 17, resp_bytes=BYTES_FAR, log_entries=1 << 18)
    pin = None
    try:
        recs = tagged(nrows, rng, seq0=1)
        for a in range(0, nrows, 1 << 14):
            e.ingest(np.ascontiguousarray(recs[a: a + (1 << 14)]))
        ids = ids_of(e, recs, 0)
        wires = [wire_rec(recs[i], ids[i]) for i in range(nrows)]
        used = 0
        stored = {}                                          # row -> expected (resp_off, bytes, hdr_len) of its response
        errs = {}                                            # row -> expected (err_off, text)

        def outcomes(rows, kinds, t):
            o = np.zeros(len(rows), dtype=A.outcome_dtype)
            o["request_id"] = ids[rows]
            o["agent_id"] = TAG.encode()
            o["kind"] = kinds
            o["http_status"] = 200 + np.arange(len(rows)) % 300
            o["seq"] = t
            return o

        def complete(rows, segs, kinds, t):
            nonlocal used
            rows = np.asarray(rows)
            flat = [h + b for h, b in segs]
            rc, res = e.complete_ex(outcomes(rows, kinds, t), flat, np.array([len(h) for h, _ in segs], np.uint32))
            assert rc == 0 and (res == 0).all()
            for i, r in enumerate(rows.tolist()):
                if kinds[i] == K.AGR_OUT_RESPONSE:
                    stored[r] = (used, flat[i], len(segs[i][0]))
                    wires[r].response(200 + i % 300, segs[i][0], segs[i][1], int(np.broadcast_to(t, len(rows))[i]))
                else:
                    errs[r] = (used, flat[i])
                    wires[r].error(flat[i])
                used += r16(len(flat[i]))

        # A: rows [0, 64) at the start of the slab, six of them error texts
        kinds_a = np.where(np.arange(64) % 11 == 5, K.AGR_OUT_ERROR, K.AGR_OUT_RESPONSE)
        sa = segments(rng, 64, 100, 4000)
        sa = [(b"", h + b) if k == K.AGR_OUT_ERROR else (h, b) for (h, b), k in zip(sa, kinds_a)]
        complete(np.arange(64), sa, kinds_a, 100 + np.arange(64))          # last-SET times 100..163: they expire row by row
        a_off = {r: (stored[r] if r in stored else errs[r])[0] for r in range(64)}
        # filler: rows from 64 on, SEG bytes each, until B's region straddles 2^32
        nfill = (G4 - used - 30_000) // r16(SEG)
        pin = e.pinned(SEGS_PER_CALL * SEG, np.uint8)
        buf = pin.array
        buf[:] = rng.integers(0, 256, len(buf), dtype=np.uint8)
        offs = (np.arange(SEGS_PER_CALL + 1, dtype=np.uint64) * SEG)
        row = 64
        while row < 64 + nfill:
            k = min(SEGS_PER_CALL, 64 + nfill - row)
            rows = np.arange(row, row + k)
            tags = buf[: SEGS_PER_CALL * SEG].reshape(SEGS_PER_CALL, SEG)[:k, :8]
            tags[:] = rows.astype("<u8").view(np.uint8).reshape(k, 8)   # each segment starts with its row
            rc, res = e.complete_ex(outcomes(rows, K.AGR_OUT_RESPONSE, 1000), (buf, offs[: k + 1].copy()))
            assert rc == 0 and (res == 0).all()
            used += k * r16(SEG)
            for r in rows.tolist():
                wires[r].status = "completed"
            row += k
        assert G4 - 100_000 < used < G4 - 29_000
        last_fill = row - 1
        last_bytes = buf[(k - 1) * SEG: k * SEG].copy()
        # B: 64 rows through agr_complete_ex from below 2^32 to above it
        rb = np.arange(row, row + 64)
        sb = segments(rng, 64, 2000, 4000)
        kinds_b = np.where(np.arange(64) % 13 == 7, K.AGR_OUT_ERROR, K.AGR_OUT_RESPONSE)
        sb = [(b"", h + b) if k == K.AGR_OUT_ERROR else (h, b) for (h, b), k in zip(sb, kinds_b)]
        b0 = used
        complete(rb, sb, kinds_b, 2000)
        assert b0 < G4 < used
        row += 64
        # C: 40 more rows through agr_complete_ex, the whole batch above 2^32
        sc = segments(rng, 40, 500, 3000)
        c0 = used
        complete(np.arange(row, row + 40), sc, np.full(40, K.AGR_OUT_RESPONSE), 2500)
        assert G4 < c0
        row += 40
        # tickets: single-slot (agr_submit_complete_ex) and multi-slot (agr_submit_complete_large), above 2^32
        for j, (hl, bl, large) in enumerate([(0, 300, False), (11, 429, False), (0, 441, True), (20, 5000, True), (0, 16384, True),
                                             (7, 1, False)]):
            r = row + j
            hdr = b"X-T: " + b"a" * (hl - 6) + b"\n" if hl else b""
            body = rng.integers(0, 256, bl, dtype=np.uint8).tobytes()
            o = outcomes(np.array([r]), K.AGR_OUT_RESPONSE, 3000)
            t = (e.submit_complete_large if large else e.submit_complete_ex)(o[0], hdr, body)
            assert e.wait(t) == 0
            stored[r] = (used, hdr + body, hl)
            wires[r].response(200, hdr, body, 3000)
            used += r16(hl + bl)
        row += 6
        # agr_store_response over an A row and a B row, agr_store_error_text over a failed A row
        for r, (hdr, body) in zip((3, int(rb[9])), segments(rng, 2, 50, 700)):
            assert e.store_response(TAG, ids[r].tobytes(), hdr, body)
            stored[r] = (used, hdr + body, len(hdr))
            wires[r].resp_hdr, wires[r].resp_body = hdr, body
            used += r16(len(hdr) + len(body))
        text = b"dial tcp: far away " * 5
        assert e.store_error_text(TAG, ids[5].tobytes(), text)
        errs[5] = (used, text)
        wires[5].err = text
        used += r16(len(text))
        assert used > G4 + 20_000

        # placement: every per-row offset and length is the reference's
        rs = sorted(stored)
        for lo in (0, int(rb[0])):
            n = 110 if lo else 64
            off, ln = e.debug_read("resp_off", lo, n), e.debug_read("resp_len", lo, n)
            eo, el = e.debug_read("err_off", lo, n), e.debug_read("err_len", lo, n)
            for i in range(n):
                r = lo + i
                if r in stored:
                    assert (int(off[i]), int(ln[i])) == (stored[r][0], len(stored[r][1])), f"response of row {r}"
                else:
                    assert ln[i] == 0, f"row {r} has no response"
                if r in errs:
                    assert (int(eo[i]), int(el[i])) == (errs[r][0], len(errs[r][1])), f"error text of row {r}"
        assert max(stored[r][0] for r in rs) > G4 and min(stored[r][0] for r in rs) == 0
        assert any(stored[r][0] < G4 < stored[r][0] + len(stored[r][1]) for r in rs) or \
            any(errs[r][0] < G4 < errs[r][0] + len(errs[r][1]) for r in errs), "no segment straddles 2^32"
        # read-backs: the stored bytes and the JSON wire form (K5), on both sides of 2^32
        for r in rs:
            assert e.get_response_body(TAG, ids[r].tobytes()) == stored[r][1], f"agr_get_response_body of row {r}"
        assert e.get_response_body(TAG, ids[last_fill].tobytes()) == last_bytes.tobytes()
        for r in rs + sorted(errs):
            assert e.get_record_json(TAG, ids[r].tobytes()) == wires[r].wire(), f"agr_get_record_json of row {r}"
        for lo, n in ((0, 64), (int(rb[0]), 110)):
            js, _ = e.rows_json(lo, n)
            assert js == k5ref.wire_rows(wires[lo: lo + n])[0], f"agr_rows_json of rows [{lo}, +{n})"
        got = e.pending(TAG, cap=nrows)
        pend = [r for r in range(nrows) if wires[r].status == "pending"]
        _same(got["request_id"], ids[pend], "agr_pending ids")
        assert e.verify() == (nrows, 0)
        if not ring:
            return

        # release rows [0, k): the oldest live bytes are then row k's, more than 4 GiB behind the head
        k = min(r for r in range(64) if a_off[r] >= 70_000)
        tail = a_off[k]
        assert used - tail > G4
        assert e.expire(100 + k, 1) == k
        assert e.reclaim() == k
        # the rest of the lap (it ends past 2^32) in SEG segments: then less than a segment is left, less than the tail
        nl, done = (BYTES_FAR - used) // r16(SEG), 0
        while done < nl:
            kk = min(SEGS_PER_CALL, nl - done)
            rc, res = e.complete_ex(outcomes(np.arange(64 + done, 64 + done + kk), K.AGR_OUT_RESPONSE, 4000), (buf, offs[: kk + 1].copy()))
            assert rc == 0 and (res == 0).all()
            done += kk
        used += nl * r16(SEG)
        assert 0 < BYTES_FAR - used < tail

        def fill_to(need, first):
            """segments of odd lengths whose 16-byte rounded region is exactly `need` bytes, for rows first.."""
            lens = [4095] * (need // 4096) + ([need % 4096 - 1] if need % 4096 else [])
            return np.arange(first, first + len(lens)), [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in lens]

        # a batch that skips the end of the lap to byte 0 fits exactly up to the tail, 16 bytes more do not
        rows, segs = fill_to(tail + 16, row)
        rc, _ = e.complete_ex(outcomes(rows, K.AGR_OUT_RESPONSE, 5000), segs)
        assert rc == K.AGR_ENOSPC
        row += len(rows)
        rows, segs = fill_to(tail, row)
        rc, res = e.complete_ex(outcomes(rows, K.AGR_OUT_RESPONSE, 5000), segs)
        assert rc == 0 and (res == 0).all()
        row += len(rows)
        want_off = np.cumsum([0] + [r16(len(b)) for b in segs])[:-1].astype(np.uint64)
        _same(e.debug_read("resp_off", int(rows[0]), len(rows)), want_off, "offsets of the batch after the wrap")
        for r, b in zip(rows.tolist(), segs):
            assert e.get_response_body(TAG, ids[r].tobytes()) == b, f"agr_get_response_body of row {r}"
        rc, _ = e.complete_ex(outcomes(np.array([row]), K.AGR_OUT_RESPONSE, 5000), [b"x"])
        assert rc == K.AGR_ENOSPC
        # the live responses on both sides of 2^32 kept their bytes
        for r in sorted(stored):
            if r >= k:
                assert e.get_response_body(TAG, ids[r].tobytes()) == stored[r][1], f"agr_get_response_body of row {r}"
    finally:
        if pin is not None:
            pin.free()
        e.close()
