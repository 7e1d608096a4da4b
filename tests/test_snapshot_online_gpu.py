"""AGR_CFG_ONLINE_SNAPSHOT: agr_snapshot holds the engine only for the device-side cut and writes the file while other calls go
on.  The file is written into a named pipe, so the writer blocks on the full pipe after the header (which is written only
once the cut has run) while the test drives traffic into the same engine.  The file must then be what a blocking snapshot of
an identical engine without the flag writes at the cut, and restore to the same state."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from jsoncase import make_requests, records_array, var_batch
from snapfile import HEADER, WORDS, parse, referenced

pytestmark = pytest.mark.gpu

SLAB_ROWS = 1 << 12
RING_ROWS, RESP, VSLAB = 512, 64 << 10, 1 << 20
SEC = 1_000_000_000
T0, STEP = 1_700_000_000 * SEC, 3600 * SEC
SECRET = 0x5EED_1234_ABCD_0002
AGENTS = ["agent-1700000000000000001", "agent-1700000000000000002", "agent-1700000000000000003", "agent-1700000000000000004"]
STATUS = ["running", "running", "stopped", "running"]
P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
MODES = {"hash": P, "mint": P | M, "var": P | V | M, "ring": P | M | R, "var_ring": P | V | M | R,
         "ring_combine": P | M | R | K.AGR_CFG_COMBINE}
JOIN_S = 120                                  # the traffic during a write finishes long before this unless the writer holds the engine


def outcomes(rows):
    outs = np.zeros(len(rows), dtype=A.outcome_dtype)
    for j, (rid, agent, kind, http, seq) in enumerate(rows):
        outs[j]["request_id"] = np.frombuffer(rid, dtype=np.uint8)
        outs[j]["agent_id"] = agent.encode()
        outs[j]["kind"], outs[j]["http_status"], outs[j]["seq"] = kind, http, seq
    return outs


def engine_kw(flags, online):
    ring, var = bool(flags & R), bool(flags & V)
    return dict(slab_rows=RING_ROWS if ring else SLAB_ROWS, max_agents=16, id_secret=SECRET,
                flags=flags | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0),
                vslab_bytes=VSLAB if ring else 8 << 20, resp_bytes=RESP if ring else 0)


class Driver:
    """Seeded calls, applied the same way to every engine it drives; remembers every stored record's id."""

    def __init__(self, flags, seed):
        self.flags, self.rng = flags, np.random.default_rng(seed)
        self.var, self.ring = bool(flags & V), bool(flags & R)
        self.ids = {}                                              # logical row -> (agent, Request.ID)
        self.round = 0

    def batch(self, engines, n, rnd):
        now = T0 + rnd * STEP
        batch = make_requests(50 + rnd, n, AGENTS, max_payload=1000 if self.var else 416, big_bodies=self.var)
        for k, r in enumerate(batch):
            r.now = now + k * SEC
        firsts = []
        for eng in engines:
            if self.var:
                blob, offs = var_batch(batch)
                _, got, first = eng.ingest_var(blob, offs)
            else:
                got = np.zeros((n, 16), dtype=np.uint8)
                first = eng.ingest_ex(records_array(batch), np.zeros(n, dtype=A.verdict_dtype), got)
            firsts.append((first, [bytes(x) for x in got]))
        assert all(f == firsts[0] for f in firsts)                  # same rows and ids everywhere (same id_secret)
        first, got = firsts[0]
        rows = []
        for k, r in enumerate(batch):
            self.ids[first + k] = (r.agent_id, got[k] if self.flags & M else r.rid)
            rows.append(first + k)
        return rows, now

    def complete(self, engines, rows, now, body_max):
        t = now + 600 * SEC
        ops, segs, hlens, failing = [], [], [], []
        for j, k in enumerate(self.rng.permutation(len(rows))[: len(rows) * 2 // 3]):
            agent, rid = self.ids[rows[int(k)]]
            if j % 3 == 0:
                failing.append((agent, rid))
            elif j % 7 == 1:
                ops.append((rid, agent, K.AGR_OUT_DIAL_ERR, 0, t)); segs.append(b""); hlens.append(0)
            else:
                hdr = b"Content-Type: text/plain\n" if j % 2 else b""
                body = bytes(self.rng.integers(0, 256, int(self.rng.integers(0, body_max)), dtype=np.uint8))
                ops.append((rid, agent, K.AGR_OUT_RESPONSE, 200, t)); segs.append(hdr + body); hlens.append(len(hdr))
        texts = [[bytes(self.rng.integers(0, 256, int(self.rng.integers(1, 60)), dtype=np.uint8)) for _ in failing] for _ in range(3)]
        for eng in engines:
            assert eng.complete_ex(outcomes(ops), segs, np.array(hlens, dtype=np.uint32))[0] == 0
            for tx in texts:                                       # three rounds: out of retries, into the failed log
                assert eng.complete_ex(outcomes([(rid, a, K.AGR_OUT_ERROR, 0, t) for a, rid in failing]), tx)[0] == 0

    def build(self, engines, rounds):
        """State before the cut: in ring modes until rows, response bytes and record bytes have gone round, with expiry and
        release of everything older than the previous round; then one more batch that stays untouched."""
        for eng in engines:
            for a, s in zip(AGENTS, STATUS):
                eng.set_agent_state(a, s)
        for rnd in range(rounds):
            if self.ring and rnd:
                for eng in engines:
                    eng.expire(T0 + rnd * STEP, STEP + STEP // 2)
                    eng.reclaim()
            rows, now = self.batch(engines, 120, rnd)
            self.complete(engines, rows, now, 100 if self.ring else 300)
        self.round = rounds
        self.batch(engines, 40, rounds)


def submit_ingest(eng, rec):
    t = C.c_uint64()
    while True:
        rc = eng.lib.agr_submit_ingest(eng.h, C.c_void_p(rec.ctypes.data), C.byref(t))
        if rc != K.AGR_EAGAIN:
            assert rc == 0
            return int(t.value)


class PipeSnapshot:
    """agr_snapshot into a named pipe from a thread: after header() the cut has run and the writer is blocked on the pipe."""

    def __init__(self, eng, tmp_path):
        self.path = str(tmp_path / "snap.fifo")
        os.mkfifo(self.path)
        self.err = None
        self.thread = threading.Thread(target=self._run, args=(eng,), daemon=True)
        self.thread.start()
        self.f = open(self.path, "rb", buffering=0)
        self.head = self._read(HEADER.itemsize)

    def _run(self, eng):
        try:
            eng.snapshot(self.path)
        except Exception as e:                                     # noqa: BLE001 (reported by drain)
            self.err = e

    def _read(self, n):
        out = bytearray()
        while len(out) < n:
            b = self.f.read(n - len(out))
            assert b, "snapshot writer closed the pipe early"
            out += b
        return bytes(out)

    def drain(self) -> bytes:
        chunks = [self.head]
        while True:
            b = self.f.read(1 << 20)
            if not b:
                break
            chunks.append(b)
        self.f.close()
        self.thread.join(JOIN_S)
        assert not self.thread.is_alive()
        if self.err:
            raise self.err
        return b"".join(chunks)


def while_writing(snap, fn):
    """Runs fn in a thread while the writer is blocked.  If it does not finish (the writer would be holding the engine), the
    pipe is drained so that nothing stays blocked, and the test fails."""
    box = {}

    def run():
        try:
            box["out"] = fn()
        except BaseException as e:                                 # noqa: BLE001
            box["err"] = e
    t = threading.Thread(target=run, daemon=True)
    t.start()
    t.join(JOIN_S)
    if t.is_alive():
        snap.drain()
        t.join(JOIN_S)
        pytest.fail("calls did not complete while the snapshot was being written")
    if "err" in box:
        snap.drain()
        raise box["err"]
    return box.get("out")


def assert_same_engine(back, twin, drv, used, var):
    assert back.verify()[1] == 0
    for a in AGENTS:
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert np.array_equal(back.list(a, which), twin.list(a, which)), (a, which)
        if not var:
            assert back.pending(a).tobytes() == twin.pending(a).tobytes()
    for L, (a, rid) in drv.ids.items():
        if L >= used:
            continue
        assert back.get_record_json(a, rid) == twin.get_record_json(a, rid), L
        assert back.get_response_body(a, rid) == twin.get_response_body(a, rid), L
    if var:
        got, want = back.replay_scan_var(), twin.replay_scan_var()
        assert all(np.array_equal(x, y) for x, y in zip(got, want))
    else:
        got, want = back.replay_scan(), twin.replay_scan()
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_online_file_is_the_cut_and_restores_like_the_twin(mode, tmp_path):
    flags = MODES[mode]
    var, ring, combine = bool(flags & V), bool(flags & R), bool(flags & K.AGR_CFG_COMBINE)
    drv = Driver(flags, seed=5)
    with A.Engine(**engine_kw(flags, True)) as eng, A.Engine(**engine_kw(flags, False)) as twin:
        drv.build([eng, twin], 6 if ring else 2)
        twin_path = str(tmp_path / "twin.snap")
        twin.snapshot(twin_path)                                   # the twin stays as it is at the cut from here on

        snap = PipeSnapshot(eng, tmp_path)
        st0 = eng.stats()

        def traffic():
            rnd = drv.round + 1
            now = T0 + rnd * STEP
            eng.complete_ex(outcomes([(drv.ids[L][1], drv.ids[L][0], K.AGR_OUT_RESPONSE, 200, now)
                                      for L in sorted(drv.ids)[-30:]]), [b"after the cut %d" % i for i in range(30)])
            eng.expire(now + 10 * STEP, STEP)                       # everything is due
            if ring:
                eng.reclaim()
                eng.reclaim_async()
                eng.reclaim_async()
            rows, _ = drv.batch([eng], 24, rnd)                     # ring: lands on rows released before the cut
            drv.complete([eng], rows, now, 50)
            eng.drop_agent(AGENTS[1])
            eng.set_agent_state("agent-after-the-cut", "running")
            if combine:
                ops0 = eng.stats()["svc_ops"]
                recs = records_array(make_requests(90, 8, AGENTS))
                deadline = time.monotonic() + 30
                tickets = [submit_ingest(eng, recs[k: k + 1]) for k in range(8)]
                assert [eng.wait(t) for t in tickets] == [0] * 8   # (result field: 0 for an accepted record)
                assert time.monotonic() < deadline
                assert eng.stats()["svc_ops"] >= ops0 + 8
            return eng.stats()

        st1 = while_writing(snap, traffic)
        data = snap.drain()

        ref = open(twin_path, "rb").read()
        hd, agents, sec = parse(data)
        hd_t, agents_t, sec_t = parse(ref)
        assert data[: HEADER.itemsize] == ref[: HEADER.itemsize] == snap.head
        assert agents == agents_t
        for name in WORDS + ("completed_log", "failed_log"):
            assert np.array_equal(sec[name], sec_t[name]), name
        slab_m, resp_m, live = referenced(sec, hd, var)
        assert len(live) > 30 and resp_m.sum() > 1000
        assert np.array_equal(sec["slab"][slab_m], sec_t["slab"][slab_m])
        assert np.array_equal(sec["resp"][resp_m], sec_t["resp"][resp_m])
        if not ring and not var:                                    # append-only fixed rows: every row was written
            assert sec["slab"].tobytes() == sec_t["slab"].tobytes()

        # the traffic did change what the shadow protects: words, logs and the window moved on after the cut
        S, used = int(hd["slab_rows"]), int(hd["rows_used"])
        n = min(used, S)
        lo = used - n
        now_state = np.roll(eng.debug_read("state", lo, n), lo % S) if ring else eng.debug_read("state", 0, n)
        assert not np.array_equal(now_state, sec["state"])
        assert (st1["completed_log_len"], st1["failed_log_len"]) != (int(hd["log_len"][0]), int(hd["log_len"][1]))
        assert st1["rows_used"] > st0["rows_used"] == used

        # restored from the online file: the same state as the twin
        with A.Engine(restore_from=_save(tmp_path, data), **engine_kw(flags, False)) as back:
            assert_same_engine(back, twin, drv, used, var)


def _save(tmp_path, data):
    p = str(tmp_path / "online.snap")
    with open(p, "wb") as f:
        f.write(data)
    return p


# ---- the pins: a ring does not reuse the cut's window while its file is written
def _requests(seed, n, now):
    reqs = make_requests(seed, n, AGENTS)
    for r in reqs:
        r.now = now
    return records_array(reqs)


def _pin_engine(online):
    eng = A.Engine(slab_rows=512, max_agents=16, resp_bytes=16 << 10, id_secret=SECRET,
                   flags=P | M | R | K.AGR_CFG_COMBINE | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0))
    for a in AGENTS:
        eng.set_agent_state(a, "running")
    recs = _requests(7, 200, T0)                                   # rows 0..199, 48 B of response bytes each
    ids = np.zeros((200, 16), dtype=np.uint8)
    eng.ingest_ex(recs, np.zeros(200, dtype=A.verdict_dtype), ids)
    for k in range(200):
        assert eng.store_response(recs[k]["agent_id"].decode(), bytes(ids[k]), b"", bytes(40))
    return eng


def _attempt(fn):
    try:
        fn()
        return 0, ""
    except A.AgrError as e:
        return e.code, str(e)


def _pin_steps(eng, recs):
    """Expire + reclaim release every row and byte of the first fill; rows 200..511 are then taken, and the steps that
    follow need the released ones: 40 rows, one ticket, 4 x 2 KiB of response bytes (the first fill's 9600 B plus 8 KiB pass
    16 KiB).  Returns (code, message) per step and the ids of rows 200..349."""
    eng.expire(T0 + 100 * STEP, STEP)
    eng.reclaim()
    ids = np.zeros((312, 16), dtype=np.uint8)
    for a, b in ((0, 150), (150, 300), (300, 312)):
        eng.ingest_ex(recs[a:b], np.zeros(b - a, dtype=A.verdict_dtype), ids[a:b])
    out = [_attempt(lambda: eng.ingest_ex(recs[312:352], np.zeros(40, dtype=A.verdict_dtype), np.zeros((40, 16), dtype=np.uint8)))]
    out.append((eng.wait(submit_ingest(eng, recs[352:353])), ""))
    store = [_attempt(lambda k=k: eng.store_response(recs[k]["agent_id"].decode(), bytes(ids[k]), b"", bytes(2048))) for k in range(4)]
    out.append(min(store))
    return out, ids


def test_pins_hold_the_window_until_the_file_is_written(tmp_path):
    recs = _requests(8, 400, T0 + 200 * STEP)
    with _pin_engine(False) as ctl:                                # no write in progress: every step succeeds
        got, _ = _pin_steps(ctl, recs)
        assert [c for c, _ in got] == [0, 0, 0], got
    with _pin_engine(True) as eng:
        snap = PipeSnapshot(eng, tmp_path)
        got, ids = while_writing(snap, lambda: _pin_steps(eng, recs))
        assert [c for c, _ in got] == [K.AGR_ENOSPC] * 3, got
        assert "snapshot" in got[0][1] and "snapshot" in got[2][1]
        snap.drain()
        # the file is written: the same reservations go through
        eng.ingest_ex(recs[312:352], np.zeros(40, dtype=A.verdict_dtype), np.zeros((40, 16), dtype=np.uint8))
        assert eng.wait(submit_ingest(eng, recs[352:353])) == 0
        assert eng.store_response(recs[3]["agent_id"].decode(), bytes(ids[3]), b"", bytes(2048))


def test_pins_hold_the_byte_ring(tmp_path):
    def batch(seed, now):                                          # 64 records of 496 B: 31744 B, under half the 64 KiB ring
        reqs = make_requests(seed, 64, AGENTS)
        for r in reqs:
            r.path, r.headers, r.body, r.now = b"/x", {}, bytes(398), now
        return var_batch(reqs)

    def make(online):
        eng = A.Engine(slab_rows=4096, max_agents=16, vslab_bytes=64 << 10, id_secret=SECRET,
                       flags=P | M | R | V | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0))
        for a in AGENTS:
            eng.set_agent_state(a, "running")
        for rnd in range(12):                                      # the byte ring goes round; ~800 rows make the file outgrow a pipe
            eng.expire(T0 + rnd * STEP, STEP // 2)
            eng.reclaim()
            eng.ingest_var(*batch(30 + rnd, T0 + rnd * STEP))
        return eng

    def steps(eng):
        """Everything is released, then two more batches: the second needs bytes of the cut's window."""
        eng.expire(T0 + 100 * STEP, STEP)
        eng.reclaim()
        return [_attempt(lambda k=k: eng.ingest_var(*batch(60 + k, T0 + 200 * STEP))) for k in range(2)]

    with make(False) as ctl:
        got = steps(ctl)
        assert [c for c, _ in got] == [0, 0], got
    with make(True) as eng:
        snap = PipeSnapshot(eng, tmp_path)
        got = while_writing(snap, lambda: steps(eng))
        assert [c for c, _ in got] == [0, K.AGR_ENOSPC] and "byte slab" in got[1][1] and "snapshot" in got[1][1], got
        snap.drain()
        eng.ingest_var(*batch(62, T0 + 200 * STEP))


def test_unopenable_path_fails_cleanly_and_leaves_no_pin(tmp_path):
    with _pin_engine(True) as eng:
        with pytest.raises(A.AgrError) as e:
            eng.snapshot(str(tmp_path / "no-such-dir" / "x.snap"))
        assert e.value.code == K.AGR_EINVAL
        got, _ = _pin_steps(eng, _requests(8, 400, T0 + 200 * STEP))
        assert [c for c, _ in got] == [0, 0, 0], got
        eng.snapshot(str(tmp_path / "ok.snap"))
        with A.Engine(restore_from=str(tmp_path / "ok.snap"), slab_rows=512, max_agents=16, resp_bytes=16 << 10,
                      flags=P | M | R) as back:
            assert back.stats()["rows_used"] == eng.stats()["rows_used"] and back.verify()[1] == 0


def test_cut_time_is_reported(tmp_path):
    with A.Engine(slab_rows=1 << 16, max_agents=16, flags=P | M | K.AGR_CFG_TIMING | K.AGR_CFG_ONLINE_SNAPSHOT) as eng:
        eng.ingest(A.synth_fill_host(0, 50_000, seed=3, n_agents=4))
        with pytest.raises(A.AgrError):
            eng.op_time(3)                                         # no cut yet
        eng.snapshot(str(tmp_path / "t.snap"))
        assert eng.op_time(3) > 0
