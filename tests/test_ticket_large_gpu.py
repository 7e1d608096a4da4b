"""agr_submit_complete_large: one single-request ticket whose response or error text (up to AGR_OUT_TICKET_MAX_BYTES) spreads
over consecutive ring slots.  Checked against oracle/model.py read through oracle/gojson.py, and against the sequential API
(agr_complete(n = 1) followed by agr_store_response / agr_store_error_text) on a second engine fed the same stream."""
import ctypes as C
import json
import random
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from oracle import gojson as G
from oracle import model as M
from jsoncase import make_requests, records_array
from test_complete_bytes_gpu import AGENTS, apply_sequential, arrays, assert_same, engine, flat, ingest

pytestmark = pytest.mark.gpu
COMBINE = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_COMBINE
SIZES = [0, 440, 441, 951, 952, 953, 4096, 16384]          # headers + body: one slot, the slot's edges, the longest span
HDR = flat({b"Content-Type": b"application/json"})


def segment(rng, size):
    """headers + body of exactly size bytes (no headers when they would not fit)"""
    hdr = HDR if size >= len(HDR) else b""
    return hdr, rng.randbytes(size - len(hdr))


def model_of(reqs):
    mgr = M.Manager(M.MiniRedis())
    for r in reqs:
        mgr.store_request(r.agent_id, M.HttpRequest(r.method, r.path, dict(r.headers), r.body, new_id=G.format_uuid(r.rid), now=r.now))
    return mgr


def model_apply(mgr, op):
    rid, agent, kind, code, seq, hdr, body = op
    if kind == K.AGR_OUT_RESPONSE:
        hmap = dict(l.split(b": ", 1) for l in hdr.split(b"\n") if l)
        mgr.store_response(agent, G.format_uuid(rid), M.HttpResponse(code, hmap, body, now=seq))
    else:                                                  # no text: the proxy's own "transport error" (server.go:608)
        mgr.mark_request_failed(agent, G.format_uuid(rid), body or b"transport error")


def wire(mgr, r):
    return G.marshal_request(mgr.redis.get(f"agent:{r.agent_id}:requests:{G.format_uuid(r.rid)}"))


@pytest.mark.parametrize("mode", ["mint", "hash"])
def test_threads_one_request_at_a_time_against_the_model(mode):
    """Threads ingest and complete one request at a time.  Most outcomes go through agr_submit_complete_large at every size of
    SIZES, responses and error texts; the others as inline tickets (agr_submit_complete_ex) and plain agr_submit_complete."""
    flags = COMBINE | (K.AGR_CFG_MINT_IDS if mode == "mint" else 0)
    T, per = 6, 48
    reqs = make_requests(31, T * per, AGENTS[:1])
    rng = random.Random(7)
    plan = []                                              # (call, kind, headers, body, http status, seq)
    for i, r in enumerate(reqs):
        j = i % 12
        kind = K.AGR_OUT_ERROR if (i // 12) % 3 == 2 else K.AGR_OUT_RESPONSE
        if j < len(SIZES):
            call, (hdr, body) = "large", segment(rng, SIZES[j])
        elif j < 10:
            call, (hdr, body) = "inline", segment(rng, rng.choice([0, 100, 440]))
        else:
            call, hdr, body, kind = "plain", b"", b"", K.AGR_OUT_RESPONSE
        if kind == K.AGR_OUT_ERROR:
            hdr, body = b"", hdr + body
        plan.append((call, kind, hdr, body, 200 + i % 5, r.now + 1))
    with engine(flags, slab_rows=1 << 12) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        errors = []

        def worker(t):
            try:
                for i in range(t, len(reqs), T):
                    r = reqs[i]
                    out, ids = np.zeros(1, dtype=A.verdict_dtype), np.zeros((1, 16), dtype=np.uint8)
                    eng.ingest_ex(records_array([r]), out, ids)
                    if mode == "hash":
                        assert bytes(ids[0]) == r.rid
                    r.rid = bytes(ids[0])
                    call, kind, hdr, body, code, seq = plan[i]
                    o = arrays([(r.rid, r.agent_id, kind, code, seq, hdr, body)])[0][0]
                    if call == "large":
                        assert eng.wait(eng.submit_complete_large(o, hdr, body)) == 0
                    elif call == "inline":
                        assert eng.wait(eng.submit_complete_ex(o, hdr, body)) == 0
                    else:
                        assert eng.wait(eng.submit_complete(o)) == 0
            except Exception as ex:                              # noqa: BLE001 (re-raised in the main thread)
                errors.append(ex)

        th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors[0]
        mgr = model_of(reqs)
        for r, (_, kind, hdr, body, code, seq) in zip(reqs, plan):
            model_apply(mgr, (r.rid, r.agent_id, kind, code, seq, hdr, body))
        for r, (_, kind, hdr, body, _, _) in zip(reqs, plan):
            assert eng.get_response_body(r.agent_id, r.rid) == (hdr + body if kind == K.AGR_OUT_RESPONSE else b"")
            assert eng.get_record_json(r.agent_id, r.rid) == wire(mgr, r)
        assert eng.stats()["svc_ops"] == 2 * len(reqs)                 # operations, not slots: a span counts once


def test_latest_wins_among_tickets_in_flight():
    """Several large responses and errors for one record are all handed over before any is collected: the record ends as
    the model says after applying them in ring (ticket) order — the last response's bytes and the last error's text."""
    flags = COMBINE | K.AGR_CFG_MINT_IDS
    reqs = make_requests(41, 8, AGENTS[:1])
    rng = random.Random(9)
    with engine(flags, slab_rows=1 << 10) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        ingest(eng, reqs)
        mgr = model_of(reqs)
        ops = []
        for k in range(6):
            for r in reqs:
                size = rng.choice([441, 953, 4096, 16384, 2000])
                if k % 3 == 2:
                    ops.append((r.rid, r.agent_id, K.AGR_OUT_ERROR, 0, 0, b"", rng.randbytes(size)))
                else:
                    hdr, body = segment(rng, size)
                    ops.append((r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 200 + k, r.now + k + 1, hdr, body))
        outs = arrays(ops)[0]
        tickets = [eng.submit_complete_large(outs[j], op[5], op[6]) for j, op in enumerate(ops)]
        assert tickets == sorted(tickets)
        assert [eng.wait(t) for t in tickets] == [0] * len(ops)
        for op in ops:
            model_apply(mgr, op)
        for r in reqs:
            last = [op for op in ops if op[0] == r.rid and op[2] == K.AGR_OUT_RESPONSE][-1]
            assert eng.get_response_body(r.agent_id, r.rid) == last[5] + last[6]
            assert eng.get_record_json(r.agent_id, r.rid) == wire(mgr, r)


def test_span_across_the_ring_end():
    """On a fresh engine 16 381 single-slot tickets are collected (one ingest, the rest plain completions of an unknown id),
    so a 4096 B response takes slots 16 381 .. 16 389 and wraps past the ring's last slot."""
    flags = COMBINE | K.AGR_CFG_MINT_IDS
    reqs = make_requests(51, 1, AGENTS[:1])
    assert A.load_library().agr_ring_capacity() == 16384
    with engine(flags, slab_rows=1 << 10) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        out, ids = np.zeros(1, dtype=A.verdict_dtype), np.zeros((1, 16), dtype=np.uint8)
        eng.ingest_ex(records_array(reqs), out, ids)
        r = reqs[0]
        r.rid = bytes(ids[0])
        miss = arrays([(bytes(range(1, 17)), r.agent_id, K.AGR_OUT_RESPONSE, 200, 1, b"", b"")])[0][0]
        for lo in range(1, 16381, 512):
            tickets = [eng.submit_complete(miss) for _ in range(lo, min(lo + 512, 16381))]
            assert [eng.wait(t) for t in tickets] == [K.AGR_ENOTFOUND] * len(tickets)
        hdr, body = segment(random.Random(3), 4096)
        o = arrays([(r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 201, r.now + 1, hdr, body)])[0][0]
        t = eng.submit_complete_large(o, hdr, body)
        assert t & ((1 << 63) - 1) == 16381
        assert eng.wait(t) == 0
        assert eng.get_response_body(r.agent_id, r.rid) == hdr + body
        mgr = model_of(reqs)
        model_apply(mgr, (r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 201, r.now + 1, hdr, body))
        assert eng.get_record_json(r.agent_id, r.rid) == wire(mgr, r)
        assert eng.stats()["svc_ops"] == 16382


def test_no_room_on_the_ring_path():
    """A response byte slab too small: an inline ticket and a span are applied, their ticket result is AGR_ENOSPC and no byte
    is stored; a small segment that fits afterwards is stored."""
    flags = COMBINE | K.AGR_CFG_MINT_IDS
    reqs = make_requests(61, 3, AGENTS[:1])
    rng = random.Random(5)
    with engine(flags, slab_rows=1 << 10, resp_bytes=256) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        ingest(eng, reqs)
        for r, size, call in zip(reqs[:2], (400, 4096), ("ex", "large")):
            hdr, body = segment(rng, size)
            o = arrays([(r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 202, r.now + 1, hdr, body)])[0][0]
            submit = eng.submit_complete_ex if call == "ex" else eng.submit_complete_large
            assert eng.wait(submit(o, hdr, body)) == K.AGR_ENOSPC
            d = json.loads(eng.get_record_json(r.agent_id, r.rid))
            assert d["status"] == "completed" and d["response"]["status_code"] == 202
            assert not d["response"]["body"] and not d["response"]["headers"]
            assert eng.get_response_body(r.agent_id, r.rid) == b""
        r = reqs[2]
        o = arrays([(r.rid, r.agent_id, K.AGR_OUT_ERROR, 0, 0, b"", b"small")])[0][0]
        assert eng.wait(eng.submit_complete_large(o, b"", b"small")) == 0
        assert json.loads(eng.get_record_json(r.agent_id, r.rid))["error"] == "small"
        assert eng.stats()["completions"] == 2


def test_byte_ring_expire_reclaim_snapshot(tmp_path):
    """AGR_CFG_RING: large responses and errors through tickets while agr_expire + agr_reclaim release rows and bytes and the
    byte ring wraps; equal to the sequential API on a second engine after every step, and unchanged by a snapshot / restore."""
    flags = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING
    per, steps, ttl, resp = 32, 28, 2000, 1 << 20
    rng = random.Random(11)
    path = str(tmp_path / "snap.agr")
    with engine(flags, slab_rows=1024, resp_bytes=resp) as ea, engine(flags | K.AGR_CFG_COMBINE, slab_rows=1024, resp_bytes=resp) as eb:
        stored = 0
        for s in range(steps):
            now = (s + 1) * 1000
            chunk_a, chunk_b = make_requests(200 + s, per, AGENTS), make_requests(200 + s, per, AGENTS)
            for r in chunk_a + chunk_b:
                r.now = now
            assert ingest(ea, chunk_a) == ingest(eb, chunk_b)
            assert [r.rid for r in chunk_a] == [r.rid for r in chunk_b]
            ops = []
            for r in chunk_a:
                size = rng.choice(SIZES + [2000, 8000])
                if rng.random() < 0.3:
                    ops.append((r.rid, r.agent_id, K.AGR_OUT_ERROR, 0, now, b"", rng.randbytes(size)))
                else:
                    hdr, body = segment(rng, size)
                    ops.append((r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 200, now, hdr, body))
            outs = arrays(ops)[0]
            tickets = [eb.submit_complete_large(outs[j], op[5], op[6]) for j, op in enumerate(ops)]
            assert [eb.wait(t) for t in tickets] == apply_sequential(ea, ops)
            stored += sum(len(op[5]) + len(op[6]) for op in ops)
            assert ea.expire(now, ttl) == eb.expire(now, ttl)
            assert ea.reclaim() == eb.reclaim()
            sa = ea.stats()
            assert_same(ea, eb, chunk_a, sa["rows_tail"], sa["rows_used"] - sa["rows_tail"])
        assert stored > 2 * resp
        sb = eb.stats()
        first, n = sb["rows_tail"], sb["rows_used"] - sb["rows_tail"]
        want, _ = eb.rows_json(first, n, as_array=True)
        bodies = [eb.get_response_body(r.agent_id, r.rid) for r in chunk_b]
        assert sum(len(b) for b in bodies) > 0
        eb.snapshot(path)
    with engine(flags | K.AGR_CFG_COMBINE, slab_rows=1024, resp_bytes=resp, restore_from=path) as ec:
        got, _ = ec.rows_json(first, n, as_array=True)
        assert got == want
        assert [ec.get_response_body(r.agent_id, r.rid) for r in chunk_b] == bodies


def test_rejections():
    lib = A.load_library()
    reqs = make_requests(71, 1, AGENTS[:1])
    hdr, body = b"A: b\n", bytes(K.AGR_OUT_TICKET_MAX_BYTES - 5)
    with engine(COMBINE | K.AGR_CFG_MINT_IDS, slab_rows=1 << 10) as eng:
        eng.set_agent_state(AGENTS[0], K.AGR_AGENT_RUNNING)
        ingest(eng, reqs)
        r = reqs[0]
        o = arrays([(r.rid, r.agent_id, K.AGR_OUT_RESPONSE, 200, 1, b"", b"")])[0][0]
        for h_, b_ in ((hdr, body + b"x"), (b"", bytes(K.AGR_OUT_TICKET_MAX_BYTES + 1))):
            with pytest.raises(A.AgrError) as e:
                eng.submit_complete_large(o, h_, b_)
            assert e.value.code == K.AGR_EINVAL
        dial = arrays([(r.rid, r.agent_id, K.AGR_OUT_DIAL_ERR, 0, 1, b"", b"")])[0][0]
        with pytest.raises(A.AgrError) as e:
            eng.submit_complete_large(dial, b"", b"x" * 1000)
        assert e.value.code == K.AGR_EINVAL
        assert eng.wait(eng.submit_complete_large(dial, b"", b"")) == 0      # a dial error without bytes is fine
        oa = np.ascontiguousarray(o.reshape(1))
        buf = (C.c_uint8 * 16)()
        t = C.c_uint64()
        p = lambda x: C.cast(x, C.c_void_p)                                  # noqa: E731
        assert lib.agr_submit_complete_large(None, oa.ctypes.data, p(buf), 4, p(buf), 4, C.byref(t)) == K.AGR_EINVAL
        assert lib.agr_submit_complete_large(eng.h, None, p(buf), 4, p(buf), 4, C.byref(t)) == K.AGR_EINVAL
        assert lib.agr_submit_complete_large(eng.h, oa.ctypes.data, None, 4, p(buf), 4, C.byref(t)) == K.AGR_EINVAL
        assert lib.agr_submit_complete_large(eng.h, oa.ctypes.data, p(buf), 4, None, 4, C.byref(t)) == K.AGR_EINVAL
        assert lib.agr_submit_complete_large(eng.h, oa.ctypes.data, p(buf), 4, p(buf), 4, None) == K.AGR_EINVAL
        assert eng.wait(eng.submit_complete_large(o, hdr, body)) == 0          # exactly the limit
        assert eng.get_response_body(r.agent_id, r.rid) == hdr + body
    with engine(K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS, slab_rows=1 << 10) as plain:
        with pytest.raises(A.AgrError) as e:
            plain.submit_complete_large(o, b"", b"x" * 1000)
        assert e.value.code == K.AGR_EINVAL
