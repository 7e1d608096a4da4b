"""The engine far along its arrival counter.  A ring shard (AGR_CFG_RING) counts arrivals in 64 bits and runs indefinitely, but a
minted id holds 40 bits of its row and a single-request answer 48.  agr_debug_skip_arrivals puts a fresh engine at 2^32, 2^40,
2^48 and just below the 2^52 bound, and these tests check it there against the plain references: the model (scenario.run_oracle),
the id restatement (tests/mintref.py, not the engine's agr_mint_ids) and the K3 restatement (tests/k3ref.py).  The last test
checks the hook itself against an engine that really ingested 2^32 records."""
import ctypes as C
import json
import uuid

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.binding import _ptr
from k3rig import Rig, layout
from mintref import ROW_LIMIT, decode, mint_bytes, mint_many, split
from scenario import assert_same, random_scenario, run_engine, run_oracle

pytestmark = pytest.mark.gpu

SECRET = 0x1234567890ABCDEF
R = 4097
MINT_RING = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING


def padded_start(edge):
    """(start, ring rows): the start sits 5 rows before the end of the ring, so the first batch gets end-of-ring padding, and the
    rows after the padding reach the edge within 200 rows."""
    r = R
    while not 10 <= edge % r <= 200:
        r += 1
    return (edge // r) * r - 5, r


STARTS = {"0": (0, R), "2^32-37": (2**32 - 37, R), "2^40-37": (2**40 - 37, R), "2^40+3R+11": (2**40 + 3 * R + 11, R),
          "2^40-pad": padded_start(2**40), "2^48-37": (2**48 - 37, R), "2^48-pad": padded_start(2**48),
          "bound": (ROW_LIMIT - 4 * R - 5, R)}


def far_engine(start, rows, flags=MINT_RING, **kw):
    eng = A.Engine(device=0, slab_rows=rows, max_agents=64, flags=flags, id_secret=SECRET, **kw)
    eng.skip_arrivals(start)
    st = eng.stats()
    assert st["rows_used"] == start and st["rows_tail"] == start
    return eng


def next_first(end, n, rows):
    at = end % rows
    return end + (rows - at if at + n > rows else 0)


class RefIds:
    """The engine as run_engine sees it, with the ids taken from the reference instead of agr_mint_ids.  Every id and row the
    engine hands out itself is checked against the reference, and every batch must land where the padding rule puts it."""

    def __init__(self, eng, start, rows, tickets=False):
        self.eng, self.rows, self.tickets = eng, rows, tickets
        self.mint, self.varlen = eng.mint, eng.varlen
        self.end = start
        self.last = None
        self.batches = 0

    def __getattr__(self, k):
        return getattr(self.eng, k)

    def _landed(self, first, n):
        assert first == next_first(self.end, n, self.rows), (first, self.end, n)
        self.end = first + n
        self.batches += 1

    def mint_ids(self, first, n):
        if self.last is not None and self.last[0] == first and len(self.last[1]) == n:
            return self.last[1]
        return mint_many(first, n, SECRET)

    def ingest(self, recs):
        n = len(recs)
        if self.tickets and self.batches % 2:
            return self._ingest_tickets(recs)
        verdicts = np.zeros(n, dtype=A.verdict_dtype)
        ids = np.zeros((n, 16), dtype=np.uint8)
        first = self.eng.ingest_ex(np.ascontiguousarray(recs), verdicts, ids)
        if not self.tickets:
            self._landed(first, n)
            assert np.array_equal(ids, mint_many(first, n, SECRET)), f"ingest_ex ids differ from the reference at row {first}"
        else:
            # through the single-request ring one call's records may land in two dispatcher batches, with end-of-ring padding
            # between them: each id must be the reference's id of a row, the rows rising from first_rid
            rows = [decode(*split(x), SECRET, 0, 1, self.end, self.end + 2 * self.rows) for x in ids]
            assert rows[0] == first >= self.end and None not in rows and rows == sorted(set(rows)), (first, self.end, rows)
            assert rows[-1] - first < n + self.rows
            self.end = rows[-1] + 1
            self.batches += 1
        self.last = (first, ids)
        return verdicts, first

    def _ingest_tickets(self, recs):
        lib, n = self.eng.lib, len(recs)
        out = np.zeros(n, dtype=A.verdict_dtype)
        tks = []
        for i in range(n):
            rec = np.ascontiguousarray(recs[i: i + 1])
            t = C.c_uint64()
            while True:
                rc = lib.agr_submit_ingest(self.eng.h, _ptr(rec), C.byref(t))
                if rc != K.AGR_EAGAIN:
                    assert rc == 0, rc
                    break
            tks.append(t.value)
        rows, ids = [], []
        for i, t in enumerate(tks):
            res = (C.c_uint8 * 40)()
            assert lib.agr_wait(self.eng.h, C.c_uint64(t), C.cast(res, C.c_void_p)) == 0
            raw = bytes(res)
            out[i:i + 1] = np.frombuffer(raw[:8], dtype=A.verdict_dtype)
            row = int.from_bytes(raw[24:32], "little")
            assert int.from_bytes(raw[32:36], "little", signed=True) == 0
            assert raw[8:24] == mint_bytes(row, SECRET), f"ticket id of row {row} differs from the reference"
            rows.append(row)
            ids.append(raw[8:24])
        assert rows[0] >= self.end and rows == sorted(set(rows)), rows
        self.end = rows[-1] + 1
        self.batches += 1
        assert rows[-1] - rows[0] < n + self.rows                    # (end-of-ring padding may fall between two tickets)
        self.last = (rows[0], np.frombuffer(b"".join(ids), dtype=np.uint8).reshape(n, 16))
        return out, rows[0]

    def ingest_var(self, blob, offs):
        verdicts, ids, first = self.eng.ingest_var(blob, offs)
        self._landed(first, len(offs) - 1)
        assert np.array_equal(ids, mint_many(first, len(offs) - 1, SECRET)), f"ingest_var ids differ from the reference at row {first}"
        return verdicts, ids, first


MODES = {"tma": dict(flags=MINT_RING),
         "varlen": dict(flags=MINT_RING | K.AGR_CFG_VARLEN, vslab_bytes=R * 1024),
         "combine": dict(flags=MINT_RING | K.AGR_CFG_COMBINE)}
CASES = [(m, s) for m in MODES for s in STARTS if not (m == "combine" and s.endswith("pad"))]
CASES += [("hash", "2^32-37"), ("hash", "2^40-37"), ("hash", "2^40+3R+11")]


@pytest.mark.parametrize("mode,start", CASES)
def test_model_parity_far_along_the_counter(mode, start):
    """random_scenario streams with replays (rows of earlier batches and of the same batch) through run_engine and run_oracle,
    from a start whose first batches straddle the edge; the ids run_engine maps to the model's come from the reference."""
    s0, rows = STARTS[start]
    kw = dict(flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_RING) if mode == "hash" else dict(MODES[mode])
    flags = kw.pop("flags")
    for seed in (1, 2):
        eng = far_engine(s0, rows, flags=flags, **kw)
        try:
            events = random_scenario(seed * 31 + len(start), n_events=260, n_agents=5, p_replay=0.3, p_manual=0.05)
            drv = RefIds(eng, s0, rows, tickets=mode == "combine") if mode != "hash" else eng
            got = run_engine(drv, events, max_batch=32 if mode == "combine" else 1 << 30, rng=np.random.default_rng(seed))
            assert_same(run_oracle(events), got)
            if mode != "hash":
                assert drv.end > s0 + 100 and drv.batches > 3
                if start != "0" and start != "bound":
                    assert drv.end > s0 + 37 + 5                    # the stream passed the edge
        finally:
            eng.close()


def uuid_str(b):
    return str(uuid.UUID(bytes=bytes(b)))


@pytest.mark.parametrize("mode", ["tma", "varlen"])
@pytest.mark.parametrize("start", ["2^32-37", "2^40-37", "2^40-pad", "2^48-37", "bound"])
def test_ids_and_resolution_far_along_the_counter(mode, start):
    """Every id the engine emits equals the reference's id of its arrival (ingest, dispatch, gathered records, agr_get_record,
    K5's JSON); live ids resolve; ids of released rows, one 2^40 period off and with one bit flipped do not, and change nothing."""
    s0, rows = STARTS[start]
    kw = dict(MODES[mode])
    eng = far_engine(s0, rows, flags=kw.pop("flags"), **kw)
    drv = RefIds(eng, s0, rows)
    try:
        agents = [f"agent-{1700000000000000000 + 1000003 * k}" for k in range(3)]
        for a in agents:
            eng.set_agent_state(a, "stopped")
        from scenario import Req, make_records, make_var_batch
        seq = 0

        def batch(n):
            nonlocal seq
            reqs = [Req(agents[(seq + i) % 3], bytes(16), seq + i + 1) for i in range(n)]
            seq += n
            if mode == "varlen":
                blob, offs = make_var_batch(reqs)
                _, _, first = drv.ingest_var(blob, offs)
            else:
                _, first = drv.ingest(make_records(reqs))
            return first

        firsts = [(batch(40), 40), (batch(60), 60)]
        # release the first batch: everything due, reclaim up to the second batch
        eng.expire(41, 1)                                             # (a record's time is its seq: 1..40, then 41..100)
        released = eng.reclaim()
        assert released >= 40
        live = list(range(firsts[1][0], firsts[1][0] + 60))
        dead = list(range(firsts[0][0], firsts[0][0] + 40))
        st = eng.stats()
        assert st["rows_tail"] == firsts[1][0] and st["rows_used"] == firsts[1][0] + 60
        # dispatch and gathered records (all agents stopped: nothing dispatched, so start them)
        for a in agents:
            eng.set_agent_state(a, "running")
        if mode == "varlen":
            disp, vblob, voffs = eng.replay_scan_var()
            heads = [bytes(vblob[int(voffs[j]): int(voffs[j]) + 16]) for j in range(len(disp))]
        else:
            disp, recs = eng.replay_scan(with_records=True)
            heads = [bytes(r["request_id"]) for r in recs]
        assert sorted(int(r) for r in disp["rid"]) == live
        for d, h in zip(disp, heads):
            assert bytes(d["request_id"]) == mint_bytes(int(d["rid"]), SECRET) == h
        # agr_get_record and K5's JSON
        for row in live[:5] + live[-5:]:
            a = agents[(row - live[0] + 40) % 3]
            idb = mint_bytes(row, SECRET)
            rec = eng.get_record_var(a, idb) if mode == "varlen" else eng.get_record(a, idb)
            assert rec is not None and bytes(rec[:16] if mode == "varlen" else rec["request_id"]) == idb
            js = eng.get_record_json(a, idb)
            assert js is not None and json.loads(js)["id"] == uuid_str(idb)
        if mode != "varlen":
            text, offs = eng.rows_json(live[0], 60)
            for j in range(60):
                assert json.loads(text[int(offs[j]): int(offs[j + 1])])["id"] == uuid_str(mint_bytes(live[j], SECRET))
        # resolution: wrong ids first (nothing may change), then every live id completes
        before = (eng.debug_read("state", live[0], 60).copy(), eng.debug_read("route", live[0], 60).copy())
        misses0 = eng.stats()["completion_misses"]
        agent_of = {r: agents[(r - live[0] + 40) % 3] for r in live + dead}
        bad = [(mint_bytes(r, SECRET), agent_of[r]) for r in dead]        # each id with the agent its row had: only the id is wrong
        bad += [(mint_bytes(r + k * 2**40, SECRET), agent_of[r]) for r in live[::7] for k in (-1, 1, 2) if r + k * 2**40 >= 0]
        for r in live[::11]:
            idb = mint_bytes(r, SECRET)
            for bit in (0, 9, 40, 51, 63, 64, 100, 127):
                x = bytearray(idb); x[bit // 8] ^= 1 << (bit % 8)
                bad.append((bytes(x), agent_of[r]))
        bad_ids = [b for b, _ in bad]
        outs = np.zeros(len(bad), dtype=A.outcome_dtype)
        outs["request_id"] = np.frombuffer(b"".join(bad_ids), dtype=np.uint8).reshape(-1, 16)
        outs["agent_id"] = [a.encode() for _, a in bad]
        outs["kind"], outs["http_status"] = K.AGR_OUT_RESPONSE, 200
        res = eng.complete(outs)
        assert (res == K.AGR_ENOTFOUND).all(), res
        assert eng.stats()["completion_misses"] - misses0 == len(bad_ids)
        assert np.array_equal(eng.debug_read("state", live[0], 60), before[0])
        assert np.array_equal(eng.debug_read("route", live[0], 60), before[1])
        for idb in bad_ids[:20]:
            for a in agents:
                assert (eng.get_record_var(a, idb) if mode == "varlen" else eng.get_record(a, idb)) is None
        outs = np.zeros(60, dtype=A.outcome_dtype)
        outs["request_id"] = mint_many(live[0], 60, SECRET)
        outs["agent_id"] = [agents[(r - live[0] + 40) % 3].encode() for r in live]
        outs["kind"], outs["http_status"] = K.AGR_OUT_RESPONSE, 200
        assert (eng.complete(outs) == 0).all()
        for a in agents:
            assert len(eng.list(a, K.AGR_LIST_COMPLETED)) == 20
    finally:
        eng.close()


def test_skip_arrivals_contract():
    with A.Engine(device=0, slab_rows=R, max_agents=8, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS) as eng:
        with pytest.raises(A.AgrError) as e:
            eng.skip_arrivals(5)                                      # append-only
        assert e.value.code == K.AGR_EINVAL
    eng = far_engine(0, R)
    try:
        with pytest.raises(A.AgrError):
            eng.skip_arrivals(ROW_LIMIT + 1)
        eng.skip_arrivals(ROW_LIMIT - 1000)                           # up to the bound is fine
        eng.set_agent_state("agent-x", "stopped")
        rec = np.zeros(1, dtype=A.record_dtype)
        rec["agent_id"] = b"agent-x"
        rec["seq"] = 1
        _, first = eng.ingest(rec)
        assert first == ROW_LIMIT - 1000
        with pytest.raises(A.AgrError) as e:
            eng.skip_arrivals(1)                                      # a live row
        assert e.value.code == K.AGR_EINVAL
        eng.expire(10, 1)
        assert eng.reclaim() == 1
        first = eng.reserve_rows(3)
        with pytest.raises(A.AgrError):
            eng.skip_arrivals(1)                                      # reserved rows not ingested yet
        eng.fill_rows(first, np.ascontiguousarray(np.repeat(rec, 3)))
        eng.ingest_rows(first, 3)
        eng.expire(10, 1)
        assert eng.reclaim() == 3
        left = ROW_LIMIT - eng.stats()["rows_used"]
        with pytest.raises(A.AgrError):
            eng.skip_arrivals(left + 1)                               # past the bound
        eng.skip_arrivals(left)
        assert eng.stats()["rows_used"] == ROW_LIMIT
        with pytest.raises(A.AgrError) as e:
            eng.ingest(rec)                                           # row ids stop at 2^52
        assert e.value.code == K.AGR_ENOSPC
    finally:
        eng.close()


@pytest.mark.parametrize("use_async", [False, True])
def test_k3_laps_across_2_40(use_async):
    """Several laps of ingest / complete / expire / reclaim on a 4097-row ring whose window moves across 2^40, compared with
    the K3 restatement after every step (dispatch rows and order, pending, all three lists, gathered records byte for byte)."""
    base = 2**40 - 2 * R - 123
    rig = Rig(slab_rows=R, max_agents=64, flags=MINT_RING, base=base, id_secret=SECRET,
              mint_ids=lambda first, n: mint_many(first, n, SECRET))
    try:
        rig.register(40)
        for lap in range(5):
            sizes = [300, 511, 97, 1024][lap % 4:] + [300, 511, 97, 1024][: lap % 4]
            k = 0
            while True:
                b = sizes[k % len(sizes)]
                n_abs = base + rig.ref.n
                first_abs = next_first(n_abs, b, R)
                if first_abs + b - (base + rig.ref.tail) > R:
                    break
                first = rig.ingest(layout("uniform", b, len(rig.names), rig.rng, rig.ref.n))
                assert first + base == first_abs
                k += 1
            rig.check()
            rig.random_outcomes(0.3)
            rig.check()
            seqs = rig.recs["seq"][rig.ref.tail: rig.ref.n].astype(np.int64)
            live = seqs[seqs > 0]
            cut = int(live[int(len(live) * 0.7)])
            rows = np.flatnonzero((seqs > 0) & (seqs <= cut)) + rig.ref.tail
            assert rig.eng.expire(cut + 1, 1) == rig.ref.expire(rows)
            rig.check()
            if use_async:
                got = rig.eng.reclaim_async()                        # what the previous scan found ...
                got += rig.eng.reclaim()                             # ... and the rest
                assert got == rig.ref.reclaim()
            else:
                assert rig.eng.reclaim() == rig.ref.reclaim()
            rig.check()
        assert base + rig.ref.tail > 2**40                           # the window really moved across the edge
    finally:
        rig.close()


def test_restore_past_2_40(tmp_path):
    s0 = 2**40 + 3 * R + 11
    eng = far_engine(s0, R)
    path = str(tmp_path / "snap")
    try:
        eng.set_agent_state("agent-a", "stopped")
        recs = np.zeros(50, dtype=A.record_dtype)
        recs["agent_id"] = b"agent-a"
        recs["seq"] = np.arange(1, 51)
        recs["status"], recs["max_retries"] = K.AGR_ST_PENDING, 3
        _, first = eng.ingest(recs)
        assert first == next_first(s0, 50, R)
        eng.snapshot(path)
    finally:
        eng.close()
    eng = A.Engine(device=0, slab_rows=R, max_agents=64, flags=MINT_RING, restore_from=path)
    try:
        for r in (first, first + 17, first + 49):
            rec = eng.get_record("agent-a", mint_bytes(r, SECRET))
            assert rec is not None and bytes(rec["request_id"]) == mint_bytes(r, SECRET)
        assert eng.get_record("agent-a", mint_bytes(first - 2**40, SECRET)) is None
        out = np.zeros(10, dtype=A.verdict_dtype)
        ids = np.zeros((10, 16), dtype=np.uint8)
        f2 = eng.ingest_ex(np.ascontiguousarray(recs[:10]), out, ids)
        assert f2 == next_first(first + 50, 10, R)
        assert np.array_equal(ids, mint_many(f2, 10, SECRET))
        o = np.zeros(1, dtype=A.outcome_dtype)
        o["request_id"] = np.frombuffer(mint_bytes(first + 3, SECRET), dtype=np.uint8)
        o["agent_id"], o["kind"], o["http_status"] = b"agent-a", K.AGR_OUT_RESPONSE, 200
        assert eng.complete(o)[0] == 0
    finally:
        eng.close()


def test_hook_matches_an_engine_that_ingested_2_32_records():
    """Real traffic past 2^32: device-synthesised 1 Mi batches through an 8 Mi-row ring with the TTL sweep and agr_reclaim_async,
    like the bench's sustained_ring, for 4097 steps.  A second engine skips to the same arrival with the hook; both get the same
    batch and must agree on verdicts, ids, dispatch and JSON bytes."""
    B, RR = 1 << 20, 8 << 20
    steps = (2**32 + B - 1) // B + 1
    kw = dict(device=0, slab_rows=RR, max_agents=1024, max_batch=B, flags=MINT_RING, id_secret=SECRET)
    real = A.Engine(**kw)
    names = [A.synth_agent_id(k, agent_nanos0=1700000000000000000) for k in range(256)]
    synth = dict(seed=11, n_agents=256, agent_nanos0=1700000000000000000)
    try:
        real.set_agent_states(names, ["stopped"] * 256)
        for s in range(steps):
            first = real.reserve_rows(B)
            real.synth_fill_rows(s * B, first, B, **synth)
            real.ingest_rows_async(first, B)
            real.expire((s + 1) * B, 4 * B, want_count=False)
            real.reclaim_async()
        real.sync()
        real.expire(2**62, 1)
        real.reclaim()
        real.reclaim()
        st = real.stats()
        at = st["rows_used"]
        assert st["rows_tail"] == at and at > 2**32
        hook = A.Engine(**kw)
        try:
            hook.skip_arrivals(at)
            hook.set_agent_states(names, ["running" if k % 3 else "stopped" for k in range(256)])
            real.set_agent_states(names, ["running" if k % 3 else "stopped" for k in range(256)])
            n = 5000
            got = []
            for eng in (real, hook):
                f = eng.reserve_rows(n)
                assert f == at
                eng.synth_fill_rows(steps * B, f, n, dup_permille=100, mint_base=f, **synth)
                v = eng.ingest_rows(f, n)
                disp, recs = eng.replay_scan(with_records=True)
                text, offs = eng.rows_json(f, n)
                got.append((v.tobytes(), disp.tobytes(), recs.tobytes(), text))
                assert all(bytes(d["request_id"]) == mint_bytes(int(d["rid"]), SECRET) for d in disp[:2000])
                assert json.loads(text[int(offs[0]): int(offs[1])])["id"] == uuid_str(mint_bytes(at, SECRET))
            assert got[0] == got[1]
            assert len(got[0][1]) > 0
        finally:
            hook.close()
    finally:
        real.close()
