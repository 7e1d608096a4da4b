"""agr_complete_ex / agr_submit_complete_ex: outcomes that carry the bytes StoreResponse / MarkRequestFailed keep
(requests.go:134-175,244), stored in the same call.

Checked two ways: against the Go-JSON restatement (oracle/model.py's Manager read through oracle/gojson.py), and against the
sequential API the call is defined by — agr_complete(n = 1) followed, when it returned 0, by agr_store_response /
agr_store_error_text — on a second engine fed the same stream."""
import json
import random
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from oracle import gojson as G
from jsoncase import AWKWARD, make_requests, make_script, records_array, run_model, var_batch

pytestmark = pytest.mark.gpu
MODES = {"hash": K.AGR_CFG_PERSISTENCE, "mint": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS,
         "var": K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN | K.AGR_CFG_MINT_IDS}
AGENTS = ["agent-1700000000000000001", "agent-1700000000000000002", "agent-1700000000000000003"]
SECRET = 0x5eed5eed


def engine(flags, **kw):
    kw.setdefault("slab_rows", 1 << 12)
    kw.setdefault("resp_bytes", 8 << 20)
    return A.Engine(max_agents=64, flags=flags, vslab_bytes=8 << 20, id_secret=SECRET, **kw)


def ingest(eng, reqs, batch=64):
    """Registers the agents and ingests reqs; fills r.rid with the ids the engine knows them by; returns the first row."""
    for k, a in enumerate(AGENTS):
        eng.set_agent_state(a, K.AGR_AGENT_RUNNING if k != 1 else K.AGR_AGENT_STOPPED)
    first = None
    for lo in range(0, len(reqs), batch):
        chunk = reqs[lo:lo + batch]
        if eng.varlen:
            blob, offs = var_batch(chunk)
            _, ids, rid0 = eng.ingest_var(blob, offs)
        else:
            out = np.zeros(len(chunk), dtype=A.verdict_dtype)
            ids = np.zeros((len(chunk), 16), dtype=np.uint8)
            rid0 = eng.ingest_ex(records_array(chunk), out, ids)
        first = rid0 if first is None else first
        for r, i in zip(chunk, ids):
            r.rid = bytes(i)
    return first


def flat(headers):
    return b"".join(k + b": " + v + b"\n" for k, v in sorted(headers.items()))


# an op: (request id, agent, kind, http status, seq, headers, body); an error's text is its body
def arrays(ops):
    outs = np.zeros(len(ops), dtype=A.outcome_dtype)
    for j, (rid, agent, kind, http, seq, _, _) in enumerate(ops):
        outs[j]["request_id"] = np.frombuffer(rid, dtype=np.uint8)
        outs[j]["agent_id"] = agent.encode()
        outs[j]["kind"], outs[j]["http_status"], outs[j]["seq"] = kind, http, seq
    return outs, [op[5] + op[6] for op in ops], np.array([len(op[5]) for op in ops], dtype=np.uint32)


def apply_batched(eng, ops, batch):
    results = []
    for lo in range(0, len(ops), batch):
        outs, segs, hl = arrays(ops[lo:lo + batch])
        rc, res = eng.complete_ex(outs, segs, hl)
        assert rc == 0
        results += list(res)
    return results


def apply_sequential(eng, ops):
    """What agr_complete_ex is defined as: per outcome agr_complete(n = 1), then the byte store if that returned 0."""
    results = []
    for op in ops:
        rid, agent, kind = op[:3]
        r = int(eng.complete(arrays([op])[0])[0])
        results.append(r)
        if r != 0 or rid == bytes(16):
            continue
        if kind == K.AGR_OUT_RESPONSE:
            assert eng.store_response(agent, rid, op[5], op[6])
        elif kind == K.AGR_OUT_ERROR:
            assert eng.store_error_text(agent, rid, op[6])
    return results


def script_ops(reqs, script):
    ops = []
    for op in script:
        r = reqs[op[1]]
        if op[0] == "resp":
            ops.append((r.rid, r.agent_id, K.AGR_OUT_RESPONSE, op[2], op[5], flat(op[3]), op[4]))
        else:
            ops.append((r.rid, r.agent_id, K.AGR_OUT_ERROR, 0, 0, b"", op[2]))
    return ops


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("seed", [1, 2])
def test_wire_form_against_the_oracle(mode, seed):
    var = mode == "var"
    reqs = make_requests(seed, 200, AGENTS, max_payload=7000 if var else 416, big_bodies=var)
    script = make_script(seed, len(reqs), 420)
    script.sort(key=lambda op: op[1] % 23)                     # neighbours often name one record: several per batch
    with engine(MODES[mode]) as eng:
        first = ingest(eng, reqs)
        redis, mgr = run_model(reqs, script)
        ops = script_ops(reqs, script)
        assert len({op[0] for op in ops[:11]}) < 11
        assert all(r == 0 for r in apply_batched(eng, ops, 11))
        every = []
        for r in reqs:
            want = redis.get(f"agent:{r.agent_id}:requests:{G.format_uuid(r.rid)}")
            every.append(want)
            assert eng.get_record_json(r.agent_id, r.rid) == G.marshal_request(want), r
        for a in AGENTS:
            got, cnt = eng.pending_json(a)
            assert got == G.marshal_list(mgr.get_pending_requests(a))
        got, _ = eng.rows_json(first, len(reqs), as_array=True)
        assert got == G.marshal_list(every)
        got, offs = eng.rows_json(first, len(reqs), as_array=False)
        for i, rec in enumerate(every):
            assert got[int(offs[i]):int(offs[i + 1])] == G.marshal_request(rec)
        import copy
        for arr in (True, False):
            got, offs = eng.rows_json(first, len(reqs), as_array=arr, roundtrip=True)
            rt = [G.unmarshal_strings(copy.deepcopy(r)) for r in every]
            if arr:
                assert got == G.marshal_list(rt)
            else:
                assert all(got[int(offs[i]):int(offs[i + 1])] == G.marshal_request(x) for i, x in enumerate(rt))


def awkward_bytes(rng, lens=(0, 1, 15, 16, 17, 100, 300, 440, 441, 1000)):
    return (rng.choice(AWKWARD) + bytes(rng.randrange(256) for _ in range(rng.choice(lens))))


def mixed_stream(reqs, seed, n_ops, t0=1_700_000_000_000_000_000, lens=(0, 1, 15, 16, 17, 100, 300, 440, 441, 1000)):
    """Responses and errors with awkward bytes, plus every case that stores nothing: unknown ids and agents, dial errors, zero
    ids; empty response segments that clear an earlier response; runs of a dozen outcomes of one record."""
    rng = random.Random(seed)
    ops = []
    for k in range(n_ops):
        r = reqs[0] if k % 97 < 12 else rng.choice(reqs)       # > 8 outcomes of one row in a batch: k2_apply_one's fallback walk
        rid, agent, x, seq = r.rid, r.agent_id, rng.random(), t0 + k
        if x < 0.04:
            ops.append((bytes(rng.randrange(256) for _ in range(16)), agent, K.AGR_OUT_RESPONSE, 200, seq, b"", b"miss"))
        elif x < 0.06:
            ops.append((rid, "agent-unknown", K.AGR_OUT_ERROR, 0, seq, b"", b"unknown agent"))
        elif x < 0.10:
            ops.append((rid, agent, K.AGR_OUT_DIAL_ERR, 0, seq, b"", b""))
        elif x < 0.13:
            ops.append((bytes(16), agent, K.AGR_OUT_RESPONSE, 200, seq, b"X-Zero: id\n", b"zero id"))
        elif x < 0.18:
            ops.append((rid, agent, K.AGR_OUT_RESPONSE, 204, seq, b"", b""))
        elif x < 0.55:
            hdr = flat({k_: rng.choice(AWKWARD).replace(b"\n", b" ") for k_ in rng.sample([b"Content-Type", b"Server", b"X-A", b"Set-Cookie"], rng.randrange(3))})
            ops.append((rid, agent, K.AGR_OUT_RESPONSE, rng.choice([200, 404, 500]), seq, hdr, awkward_bytes(rng, lens)))
        else:
            ops.append((rid, agent, K.AGR_OUT_ERROR, 0, seq, b"", awkward_bytes(rng, lens)[:300]))
    return ops


STAT_KEYS = ["rows_used", "ingested", "stored", "completions", "completion_misses", "failures", "dead_lettered", "dial_errors",
             "completed_log_len", "failed_log_len", "rows_tail", "log_overflow"]


def assert_same(a, b, reqs, first, n_rows):
    ja, oa = a.rows_json(first, n_rows)
    jb, ob = b.rows_json(first, n_rows)
    assert ja == jb and (oa == ob).all()
    for r in reqs:
        assert a.get_response_body(r.agent_id, r.rid) == b.get_response_body(r.agent_id, r.rid)
    for ag in AGENTS:
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert (a.list(ag, which) == b.list(ag, which)).all()
    sa, sb = a.stats(), b.stats()
    assert {k: sa[k] for k in STAT_KEYS} == {k: sb[k] for k in STAT_KEYS}


@pytest.mark.parametrize("mode", sorted(MODES))
def test_equals_the_sequential_api(mode):
    var = mode == "var"
    reqs = make_requests(11, 150, AGENTS, max_payload=7000 if var else 416, big_bodies=var)
    with engine(MODES[mode]) as ea:
        first = ingest(ea, reqs)
        ops = mixed_stream(reqs, 5, 1500)                     # (after the ingest: mint mode filled in the ids)
        want = apply_sequential(ea, ops)
        assert want.count(K.AGR_ENOTFOUND) > 50 and want.count(0) > 1000
        for batch in (1, 7, 64, 4096):
            with engine(MODES[mode]) as eb:
                ingest(eb, make_requests(11, 150, AGENTS, max_payload=7000 if var else 416, big_bodies=var))
                assert apply_batched(eb, ops, batch) == want
                assert_same(ea, eb, reqs, first, len(reqs))


def test_byte_ring_wraps_under_expire_and_reclaim():
    """AGR_CFG_RING with a response slab a few steps long: the byte ring wraps several times while agr_expire + agr_reclaim
    release rows and bytes; the batched engine equals the sequential one after every step."""
    flags = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING
    per, steps, ttl, resp = 32, 40, 2000, 32 << 10
    with engine(flags, slab_rows=1024, resp_bytes=resp) as ea, engine(flags, slab_rows=1024, resp_bytes=resp) as eb:
        stored, live = 0, []
        for s in range(steps):
            now = (s + 1) * 1000
            chunk_a = make_requests(100 + s, per, AGENTS)
            chunk_b = make_requests(100 + s, per, AGENTS)
            for r in chunk_a + chunk_b:
                r.now = now
            fa, fb = ingest(ea, chunk_a), ingest(eb, chunk_b)
            assert fa == fb
            live = (live + chunk_a)[-2 * per:]
            ops = mixed_stream(live, 1000 + s, 48, t0=now, lens=(0, 1, 17, 100, 250))
            assert apply_batched(eb, ops, 16) == apply_sequential(ea, ops)
            stored += sum(len(op[5]) + len(op[6]) for op in ops)
            assert ea.expire(now, ttl) == eb.expire(now, ttl)
            assert ea.reclaim() == eb.reclaim()
            sa = ea.stats()
            assert_same(ea, eb, live, sa["rows_tail"], sa["rows_used"] - sa["rows_tail"])
        assert stored > 3 * resp


@pytest.mark.parametrize("ring", [False, True])
def test_no_room_stores_no_byte_of_the_batch(ring):
    flags = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | (K.AGR_CFG_RING if ring else 0)
    reqs = make_requests(3, 4, AGENTS[:1])
    with engine(flags, slab_rows=1024, resp_bytes=4096) as eng:
        ingest(eng, reqs)
        ops = [(r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 201, 5, b"A: b\n", bytes([65 + i]) * 1500) for i, r in enumerate(reqs[:3])]
        outs, segs, hl = arrays(ops)
        rc, res = eng.complete_ex(outs, segs, hl)
        assert rc == K.AGR_ENOSPC and (res == 0).all()
        assert b"response byte slab" in A.load_library().agr_last_error()
        for r in reqs[:3]:
            d = json.loads(eng.get_record_json(r.agent_id, r.rid))
            assert d["status"] == "completed" and d["response"]["status_code"] == 201
            assert eng.get_response_body(r.agent_id, r.rid) == b""
        assert eng.stats()["completions"] == 3
        ops = [(reqs[3].rid, reqs[3].agent_id, K.AGR_OUT_ERROR, 0, 6, b"", b"small enough")]
        rc, res = eng.complete_ex(*arrays(ops))
        assert rc == 0 and res[0] == 0
        assert json.loads(eng.get_record_json(reqs[3].agent_id, reqs[3].rid))["error"] == "small enough"
        # a dial error carries no bytes
        ops = [(reqs[3].rid, reqs[3].agent_id, K.AGR_OUT_DIAL_ERR, 0, 7, b"", b"x")]
        with pytest.raises(A.AgrError) as e:
            eng.complete_ex(*arrays(ops))
        assert e.value.code == K.AGR_EINVAL


def test_snapshot_restore_after_complete_ex(tmp_path):
    reqs = make_requests(4, 120, AGENTS)
    flags = MODES["mint"]
    with engine(flags) as eng:
        first = ingest(eng, reqs)
        apply_batched(eng, mixed_stream(reqs, 9, 400), 64)
        want, _ = eng.rows_json(first, len(reqs), as_array=True)
        bodies = [eng.get_response_body(r.agent_id, r.rid) for r in reqs]
        assert sum(len(b) for b in bodies) > 10000
        path = str(tmp_path / "snap.agr")
        eng.snapshot(path)
    with engine(flags, restore_from=path) as eng2:
        got, _ = eng2.rows_json(first, len(reqs), as_array=True)
        assert got == want
        assert [eng2.get_response_body(r.agent_id, r.rid) for r in reqs] == bodies


def test_tickets_with_inline_bytes():
    """AGR_CFG_COMBINE: threads ingest and complete one request at a time.  A third of the outcomes go in tickets with their bytes
    inline, a third as plain agr_submit_complete, and a third carry a body above AGR_OUT_INLINE_BYTES and take
    agr_complete_ex(n = 1).  Every record ends with its own response, and its wire form equals the model's."""
    flags = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_COMBINE
    T, per = 6, 60
    reqs = make_requests(21, T * per, AGENTS[:1])
    rng = random.Random(4)
    plan = []
    for i, r in enumerate(reqs):
        hdr = flat({b"Content-Type": rng.choice(AWKWARD).replace(b"\n", b" ")})
        body = bytes(rng.randrange(256) for _ in range(rng.choice([0, 5, 200, 440 - len(hdr)])))
        if i % 3 == 1:
            hdr, body = b"", b""
        elif i % 3 == 2:
            body = bytes(rng.randrange(256) for _ in range(rng.choice([441, 900, 3000])))
        plan.append((hdr, body, 200 + i % 5, r.now + 1))
    with engine(flags, slab_rows=1 << 12) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        o = np.zeros(1, dtype=A.outcome_dtype)
        o["agent_id"], o["kind"] = AGENTS[0].encode(), K.AGR_OUT_RESPONSE
        with pytest.raises(A.AgrError) as e:
            eng.submit_complete_ex(o, b"", bytes(441))
        assert e.value.code == K.AGR_EINVAL
        errors = []

        def worker(t):
            try:
                for i in range(t, len(reqs), T):
                    r = reqs[i]
                    out, ids = np.zeros(1, dtype=A.verdict_dtype), np.zeros((1, 16), dtype=np.uint8)
                    eng.ingest_ex(records_array([r]), out, ids)
                    r.rid = bytes(ids[0])
                    hdr, body, code, seq = plan[i]
                    op = (r.rid, r.agent_id, K.AGR_OUT_RESPONSE, code, seq, hdr, body)
                    outs, segs, hl = arrays([op])
                    if i % 3 == 0:
                        assert eng.wait(eng.submit_complete_ex(outs[0], hdr, body)) == 0
                    elif i % 3 == 1:
                        assert eng.wait(eng.submit_complete(outs[0])) == 0
                    else:
                        rc, res = eng.complete_ex(outs, segs, hl)
                        assert rc == 0 and res[0] == 0
            except Exception as ex:                              # noqa: BLE001 (re-raised in the main thread)
                errors.append(ex)

        th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors[0]
        from oracle import model as M
        redis = M.MiniRedis()
        mgr = M.Manager(redis)
        for r, (hdr, body, code, seq) in zip(reqs, plan):
            mgr.store_request(r.agent_id, M.HttpRequest(r.method, r.path, dict(r.headers), r.body, new_id=G.format_uuid(r.rid), now=r.now))
            hmap = dict(l.split(b": ", 1) for l in hdr.split(b"\n") if l)
            mgr.store_response(r.agent_id, G.format_uuid(r.rid), M.HttpResponse(code, hmap, body, now=seq))
        for r, (hdr, body, _, _) in zip(reqs, plan):
            assert eng.get_response_body(r.agent_id, r.rid) == hdr + body
            assert eng.get_record_json(r.agent_id, r.rid) == G.marshal_request(redis.get(f"agent:{r.agent_id}:requests:{G.format_uuid(r.rid)}"))
        st = eng.stats()
        assert st["completions"] == len(reqs) and st["svc_ops"] >= len(reqs) + 2 * len(reqs) // 3
