"""Variable-length records through the single-request ring (AGR_CFG_COMBINE | AGR_CFG_VARLEN): agr_submit_ingest of one record,
and agr_ingest_var of n <= 32 records in the compact form, go through the pinned request ring as record spans of up to 16 slots
and are decided by the service kernel (k_svc_var).  Checked against a twin AGR_CFG_VARLEN engine fed the same operations in the
front end's event order through the locked calls (verdicts, ids, rows, per-row words, stored bytes, JSON, lists, replay scan,
stats), at the length edges of the slot layout, with threads against oracle/model.py, with duplicates and replays, at the byte
ring's edges, and across blocking, online, delta and relocating snapshots."""
import random
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from oracle import gojson as G
from oracle import model as M
from scenario import Req, make_var_batch, _outcomes_array

pytestmark = pytest.mark.gpu
VAR = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN
COMBINE = VAR | K.AGR_CFG_COMBINE
AGENTS = ["agent-1700000000000000001", "agent-1700000000000000002", "agent-1700000000000000003"]
EDGES = [96, 112, 496, 512, 528, 1008, 1024, 1040, 4192, 8176, 8192]
SECRET = 0x5EC2E7
WORDS = ("state", "route", "aux", "cksum", "verdict", "mtime")      # agr_debug_read words 0-5
STAT_SKIP = ("k1_launches", "k2_launches", "k3_launches", "k4_launches", "k5_launches", "svc_batches", "svc_ops")   # accounting


def engine(flags, **kw):
    kw.setdefault("slab_rows", 1 << 12)
    kw.setdefault("max_agents", 64)
    kw.setdefault("vslab_bytes", 8 << 20)
    return A.Engine(flags=flags, id_secret=SECRET, **kw)


def twins(flags, **kw):
    """(locked VARLEN engine, COMBINE | VARLEN engine) with the same configuration and agents"""
    a, b = engine(flags, **kw), engine(flags | K.AGR_CFG_COMBINE, **kw)
    for e in (a, b):
        for k, ag in enumerate(AGENTS):
            e.set_agent_state(ag, K.AGR_AGENT_RUNNING if k != 1 else K.AGR_AGENT_STOPPED)
    return a, b


def var_rec(agent, rid, seq, length, rng, replay_of=None, body_len=None):
    """one variable-length record of stored length `length` (no path, no headers): its body_len rounds up to that length, or
    is body_len (a header whose lengths exceed the record)"""
    h = np.zeros(1, dtype=A.header_dtype)
    h["request_id"] = np.frombuffer(rid, dtype=np.uint8)
    if replay_of is not None:
        h["replay_of"] = np.frombuffer(replay_of, dtype=np.uint8)
    h["agent_id"] = agent.encode()
    h["seq"] = seq
    h["flags"] = (K.AGR_F_REPLAY if replay_of is not None else 0) | (K.METHOD_CODES["POST"] << K.AGR_F_METHOD_SHIFT)
    p = length - K.AGR_HEADER_BYTES
    blen = body_len if body_len is not None else (p - rng.randrange(16) if p else 0)
    h["body_len"], h["status"], h["max_retries"] = blen, K.AGR_ST_PENDING, 3
    body = bytes(rng.randrange(32, 127) for _ in range(min(blen, p)))
    rec = np.frombuffer(h.tobytes() + body + bytes(p - len(body)), dtype=np.uint8).copy()
    assert A.var_record_len(rec) == len(rec)
    return rec


def chat_rec(agent, rid, seq, rng, replay_of=None):
    """a record as a chat request carries it: path, headers, a log-uniform 128 B - 4 KiB body (BASELINE config 5)"""
    n = int(np.exp(rng.uniform(np.log(128), np.log(4096))))
    r = Req(agent, rid, seq, replay=replay_of is not None, replay_of=replay_of or bytes(16), body=rng.integers(32, 127, n, dtype=np.uint8).tobytes())
    blob, _ = make_var_batch([r])
    return blob


def blob_of(recs, pad=0):
    """one blob of the records; pad: 16 zero bytes after every record shorter than 8 KiB (offsets no longer compact)"""
    parts = [np.concatenate([r, np.zeros(pad if len(r) < K.AGR_VAR_MAX_RECORD else 0, np.uint8)]) for r in recs]
    offs = np.zeros(len(recs) + 1, dtype=np.uint32)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.concatenate(parts), offs


def answers_locked(eng, recs, pad=0):
    blob, offs = blob_of(recs, pad)
    v, ids, first = eng.ingest_var(blob, offs)
    return [(tuple(v[i].tolist()), bytes(ids[i]), first + i, 0) for i in range(len(recs))]


def answers_tickets(eng, recs):
    tickets = [eng.submit_ingest(r) for r in recs]                    # all in flight together, then collected in order
    out = []
    for t in tickets:
        x = eng.poll(t)
        out.append((tuple(x["verdict"][0].tolist()), x["request_id"], x["rid"], x["result"]) if x["result"] == 0 else
                   (None, None, None, x["result"]))
    return out


def json_of(eng, first, n):
    return eng.rows_json(first, n)[0] if n else b""


def assert_twins(a, b, ids_by_agent):
    sa, sb = a.stats(), b.stats()
    assert {k: v for k, v in sa.items() if k not in STAT_SKIP} == {k: v for k, v in sb.items() if k not in STAT_SKIP}
    first, n = sa["rows_tail"], sa["rows_used"] - sa["rows_tail"]
    for w in WORDS:
        assert np.array_equal(a.debug_read(w, first, n), b.debug_read(w, first, n)), w
    assert json_of(a, first, n) == json_of(b, first, n)
    for ag in AGENTS:
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert np.array_equal(a.list(ag, which), b.list(ag, which)), (ag, which)
    da, ba, oa = a.replay_scan_var()
    db, bb, ob = b.replay_scan_var()
    assert np.array_equal(da, db) and np.array_equal(ba, bb) and np.array_equal(oa, ob)
    for ag, ids in ids_by_agent.items():
        for rid in ids:
            x, y = a.get_record_var(ag, rid), b.get_record_var(ag, rid)
            assert (x is None and y is None) or np.array_equal(x, y)
    assert a.verify()[1] == 0 and b.verify()[1] == 0


class Stream:
    """random operations for both twins: records (chat bodies, length edges, replays of stored ids, in-batch duplicate ids in
    hash mode), outcomes of stored records"""

    def __init__(self, seed, mint):
        self.rng, self.mint, self.seq, self.stored, self.ids = random.Random(seed), mint, 0, [], {}

    def records(self, n):
        recs = []
        for _ in range(n):
            self.seq += 1
            ag = self.rng.choice(AGENTS)
            rid = self.rng.randbytes(16)
            u = self.rng.random()
            if u < 0.1 and not self.mint and recs:                      # an id already in flight in this call (hash mode)
                rid = bytes(recs[-1][:16])
            replay = None
            if u > 0.85 and self.stored:
                ag, replay = self.rng.choice(self.stored)
            if self.rng.random() < 0.3:
                recs.append(var_rec(ag, rid, self.seq, self.rng.choice(EDGES), self.rng, replay_of=replay))
            else:
                recs.append(chat_rec(ag, rid, self.seq, np.random.default_rng(self.seq), replay_of=replay))
        return recs

    def note(self, recs, answers):
        for r, (v, rid, row, res) in zip(recs, answers):
            ag = bytes(r[32:64]).rstrip(b"\0").decode()
            if res == 0 and v[1] & K.AGR_VF_STORED:
                self.stored.append((ag, rid))
                self.ids.setdefault(ag, []).append(rid)

    def outcomes(self, n, now):
        ops = []
        for _ in range(min(n, len(self.stored))):
            ag, rid = self.rng.choice(self.stored)
            kind = self.rng.choice([K.AGR_OUT_RESPONSE, K.AGR_OUT_RESPONSE, K.AGR_OUT_ERROR])
            ops.append((rid, ag, kind, 200, now))
        return _outcomes_array(ops) if ops else None


def feed(a, b, st, round_, now):
    """one round: records through a path of b's chosen by the round, the same records through a's locked call, then outcomes"""
    path = ("tickets", "ring", "locked", "noncompact")[round_ % 4]
    recs = st.records(st.rng.randrange(1, 33) if path in ("ring", "noncompact") else st.rng.randrange(1, 49))
    pad = 16 if path == "noncompact" else 0
    if pad and all(len(r) == K.AGR_VAR_MAX_RECORD for r in recs):
        recs.append(var_rec(AGENTS[0], st.rng.randbytes(16), st.seq, 112, st.rng))
    ops0 = b.stats()["svc_ops"]
    want = answers_locked(a, recs, pad)
    if path == "tickets":
        got = answers_tickets(b, recs)
    else:
        if path == "locked" and len(recs) <= 32:
            recs += st.records(33 - len(recs))
            want += answers_locked(a, recs[len(want):], pad)
        got = answers_locked(b, recs, pad)
    assert got == want, path
    # compact records of n <= 32 went through the ring, everything else did not
    assert b.stats()["svc_ops"] - ops0 == (len(recs) if path in ("tickets", "ring") else 0), path
    st.note(recs, want)
    outs = st.outcomes(st.rng.randrange(0, 40), now)
    if outs is not None:
        for k in range(0, len(outs), 32):
            assert np.array_equal(a.complete(outs[k:k + 32]), b.complete(outs[k:k + 32]))


@pytest.mark.parametrize("ring", [False, True], ids=["append", "ring"])
@pytest.mark.parametrize("mode", ["hash", "mint"])
def test_twins(mode, ring):
    """Tickets, blocking ring calls, locked and non-compact calls against the locked twin; with AGR_CFG_RING agr_expire +
    agr_reclaim after every round, so rows and the byte ring (1 MiB: it wraps, with a skip at the end of each lap) are reused."""
    flags = VAR | (K.AGR_CFG_MINT_IDS if mode == "mint" else 0) | (K.AGR_CFG_RING if ring else 0)
    st = Stream(11 + ring + 2 * (mode == "mint"), mode == "mint")
    a, b = twins(flags, vslab_bytes=(1 << 20) if ring else (8 << 20))
    with a, b:
        for r in range(16 if ring else 8):
            now = (r + 1) * 1000
            st.seq = max(st.seq, now)
            feed(a, b, st, r, now)
            if ring:
                assert a.expire(now, 1500) == b.expire(now, 1500)
                assert a.reclaim() == b.reclaim()
                live = {(ag, rid) for ag, rid in st.stored if a.get_record_var(ag, rid) is not None}
                st.stored = [x for x in st.stored if x in live]
                st.ids = {ag: [rid for (g, rid) in st.stored if g == ag] for ag in AGENTS}
            assert_twins(a, b, st.ids)
        if ring:
            assert a.stats()["rows_tail"] > 0


def test_length_edges():
    """Every edge length alone, all of them in one blocking call, and next to agr_submit_complete_large spans in flight at the
    same time; a header whose lengths exceed 8 KiB is AGR_VF_BAD_LEN as through the locked call.  Stored bytes read back."""
    rng = random.Random(5)
    a, b = twins(VAR, resp_bytes=4 << 20)
    with a, b:
        seq = 0

        def recs_of(lengths):
            nonlocal seq
            out = []
            for L in lengths:
                seq += 1
                over = L == "over"
                out.append(var_rec(AGENTS[seq % 3], rng.randbytes(16), seq, 8192 if over else L, rng, body_len=9000 if over else None))
            return out

        alone = recs_of(EDGES + ["over"])
        for r in alone:
            assert answers_tickets(b, [r]) == answers_locked(a, [r])
        together = recs_of(EDGES + ["over"])
        assert answers_locked(b, together) == answers_locked(a, together)
        over = recs_of(["over"])
        bad = answers_locked(a, over)
        assert answers_tickets(b, over) == bad and bad[0][0][1] & K.AGR_VF_BAD_LEN
        # records in flight next to large completions of stored records (their order does not matter: different rows)
        stored = [(bytes(r[32:64]).rstrip(b"\0").decode(), bytes(r[:16])) for r in alone + together]
        stored = [s for s, r in zip(stored, alone + together) if A.var_record_len(r) < 8192 or int(np.frombuffer(r[80:84].tobytes(), "<u4")[0]) < 9000]
        mixed = recs_of(EDGES * 2)
        segs = [(b"Content-Type: text/plain\n", rng.randbytes(rng.choice([0, 441, 4096, 16000]))) for _ in stored]
        outs = _outcomes_array([(rid, ag, K.AGR_OUT_RESPONSE, 201, 9) for ag, rid in stored])
        tickets = []
        for k in range(max(len(mixed), len(stored))):
            if k < len(mixed):
                tickets.append(("r", b.submit_ingest(mixed[k])))
            if k < len(stored):
                tickets.append(("o", b.submit_complete_large(outs[k], segs[k][0], segs[k][1])))
        got_r = []
        for kind, t in tickets:
            if kind == "r":
                x = b.poll(t)
                got_r.append((tuple(x["verdict"][0].tolist()), x["request_id"], x["rid"], x["result"]))
            else:
                assert b.wait(t) == 0
        assert got_r == answers_locked(a, mixed)
        rc, res = a.complete_ex(outs, [h + body for h, body in segs], np.array([len(h) for h, _ in segs], dtype=np.uint32))
        assert rc == 0 and (res == 0).all()
        for (ag, rid), (h, body) in zip(stored, segs):
            assert a.get_response_body(ag, rid) == b.get_response_body(ag, rid) == h + body
        for r in alone + together + mixed:
            ag, rid = bytes(r[32:64]).rstrip(b"\0").decode(), bytes(r[:16])
            got = b.get_record_var(ag, rid)
            if got is not None:
                assert len(got) == len(r) and got[96:].tobytes() == r[96:].tobytes() and got[:84].tobytes() == r[:84].tobytes()
        assert_twins(a, b, {ag: [bytes(r[:16]) for r in alone + together + mixed if bytes(r[32:64]).rstrip(b"\0").decode() == ag] for ag in AGENTS})


@pytest.mark.parametrize("mode", ["mint", "hash"])
def test_threads_one_request_at_a_time_against_the_model(mode):
    """Threads each ingest one chat request at a time through a ticket and complete it; every record ends as
    oracle/model.py says."""
    flags = COMBINE | (K.AGR_CFG_MINT_IDS if mode == "mint" else 0)
    T, per = 6, 40
    rng = np.random.default_rng(3)
    reqs = []
    for i in range(T * per):
        n = int(np.exp(rng.uniform(np.log(128), np.log(4096))))
        reqs.append(Req(AGENTS[0], bytes(rng.integers(0, 256, 16, dtype=np.uint8)), i + 1, body=bytes(rng.integers(32, 127, n, dtype=np.uint8))))
    with engine(flags) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        errors, ids = [], [None] * len(reqs)

        def worker(t):
            try:
                for i in range(t, len(reqs), T):
                    x = eng.poll(eng.submit_ingest(make_var_batch([reqs[i]])[0]))
                    assert x["result"] == 0 and x["verdict"][0]["code"] == K.AGR_V_FORWARD
                    if mode == "hash":
                        assert x["request_id"] == reqs[i].rid
                    ids[i] = x["request_id"]
                    if i % 3:
                        o = _outcomes_array([(ids[i], AGENTS[0], K.AGR_OUT_RESPONSE if i % 3 == 1 else K.AGR_OUT_ERROR, 200, reqs[i].seq + 1)])
                        assert eng.wait(eng.submit_complete(o[0])) == 0
            except Exception as ex:                              # noqa: BLE001 (re-raised in the main thread)
                errors.append(ex)

        th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors[0]
        mgr = M.Manager(M.MiniRedis())
        for i, r in enumerate(reqs):
            mgr.store_request(r.agent_id, M.HttpRequest(r.method, r.path, dict(r.headers), r.body, new_id=G.format_uuid(ids[i]), now=r.seq))
            if i % 3 == 1:
                mgr.store_response(r.agent_id, G.format_uuid(ids[i]), M.HttpResponse(200, {}, b"", now=r.seq + 1))
            elif i % 3 == 2:
                mgr.mark_request_failed(r.agent_id, G.format_uuid(ids[i]), b"transport error")
        for i, r in enumerate(reqs):
            want = G.marshal_request(mgr.redis.get(f"agent:{r.agent_id}:requests:{G.format_uuid(ids[i])}"))
            assert eng.get_record_json(r.agent_id, ids[i]) == want
        assert eng.stats()["svc_ops"] == len(reqs) + sum(1 for i in range(len(reqs)) if i % 3)


def test_no_room_then_reclaim():
    """A small byte ring: records refused with AGR_ENOSPC leave rows and bytes as they were and go through once agr_expire +
    agr_reclaim released the tail; a record above half the byte ring is AGR_EINVAL, as through the locked call."""
    flags = VAR | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING
    rng = random.Random(8)
    a, b = twins(flags, vslab_bytes=32 << 10)
    with a, b:
        seq, refused = 0, None
        for k in range(64):
            seq += 1
            r = var_rec(AGENTS[0], rng.randbytes(16), seq, 4096, rng)
            before = b.stats()
            x = answers_tickets(b, [r])[0]
            if x[3] == K.AGR_ENOSPC:
                assert b.stats()["rows_used"] == before["rows_used"]
                with pytest.raises(A.AgrError) as e:
                    answers_locked(a, [r])
                assert e.value.code == K.AGR_ENOSPC and a.stats()["rows_used"] == before["rows_used"]
                refused = r
                break
            assert [x] == answers_locked(a, [r])
        assert refused is not None
        assert a.expire(10 ** 9, 1) == b.expire(10 ** 9, 1) and a.reclaim() == b.reclaim()
        assert answers_tickets(b, [refused]) == answers_locked(a, [refused])
        big = var_rec(AGENTS[0], rng.randbytes(16), seq + 1, 8192 + 0, rng)
        with engine(flags | K.AGR_CFG_COMBINE, vslab_bytes=12 << 10) as small, engine(flags, vslab_bytes=12 << 10) as small_a:
            for e in (small, small_a):
                e.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
            assert answers_tickets(small, [big])[0][3] == K.AGR_EINVAL
            with pytest.raises(A.AgrError) as e:
                answers_locked(small_a, [big])
            assert e.value.code == K.AGR_EINVAL
            # records that fit: batches end before half the byte ring instead of being refused
            recs = [var_rec(AGENTS[0], rng.randbytes(16), seq + 2 + i, 2048, rng) for i in range(4)]
            got = answers_tickets(small, recs)
            assert [g[3] for g in got] == [0] * 4
        assert_twins(a, b, {})
        assert b.stats()["rows_tail"] > 0


@pytest.mark.parametrize("kind", ["blocking", "online", "delta"])
def test_snapshots(tmp_path, kind):
    """Snapshots of a COMBINE | VARLEN engine restore to the twin's state, in place and relocated into a ring of another size;
    online snapshots are written while tickets are in flight."""
    flags = VAR | K.AGR_CFG_RING | (K.AGR_CFG_ONLINE_SNAPSHOT if kind != "blocking" else 0) | (K.AGR_CFG_DELTA_SNAPSHOT if kind == "delta" else 0)
    st = Stream(21, False)
    a, b = twins(flags, vslab_bytes=4 << 20)
    paths = [str(tmp_path / f"s{k}.agr") for k in range(2)]
    with a, b:
        for r in range(3):
            feed(a, b, st, r, (r + 1) * 1000)
        b.snapshot(paths[0])
        if kind == "online":
            # tickets in flight while the file is written: the snapshot holds the rows decided before its cut
            extra = st.records(200)
            got = []

            def traffic():
                for r in extra:
                    got.append(answers_tickets(b, [r])[0])
            th = threading.Thread(target=traffic)
            th.start()
            b.snapshot(paths[1])
            th.join()
            assert got == answers_locked(a, extra)
            st.note(extra, got)
            # the rows' words as the cut saw them: records only have come since, and they change no earlier row
            sa = a.stats()
            at_cut = [a.debug_read(w, sa["rows_tail"], sa["rows_used"] - sa["rows_tail"]) for w in WORDS]
        for r in range(3, 5):
            feed(a, b, st, r, (r + 1) * 1000)
        if kind != "online":
            b.snapshot(paths[1])
        assert_twins(a, b, st.ids)
        sa = a.stats()
        first, n = sa["rows_tail"], sa["rows_used"] - sa["rows_tail"]
        want_json = json_of(a, first, n)
        want_words = [a.debug_read(w, first, n) for w in WORDS]
    for cfg in (dict(), dict(slab_rows=1 << 13, vslab_bytes=6 << 20)):
        kw = dict(slab_rows=1 << 12, max_agents=64, vslab_bytes=4 << 20)
        kw.update(cfg)
        with A.Engine(flags=flags | K.AGR_CFG_COMBINE, id_secret=SECRET, restore_from=paths[1], **kw) as c:
            if kind == "online":
                sc = c.stats()
                m = sc["rows_used"] - first
                assert sc["rows_tail"] == first and 0 < m <= n
                assert all(np.array_equal(c.debug_read(w, first, m), x[:m]) for w, x in zip(WORDS, at_cut))
            else:
                assert json_of(c, first, n) == want_json
                assert all(np.array_equal(c.debug_read(w, first, n), x) for w, x in zip(WORDS, want_words))
            assert c.verify()[1] == 0
            # the restored engine keeps serving tickets
            more = st.records(5)
            assert [x[3] for x in answers_tickets(c, more)] == [0] * 5
