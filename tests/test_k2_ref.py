"""tests/k2ref.py, the plain restatement the K2 edge tests check against, compared with oracle/model.py's Manager on seeded
outcome streams and on hand-worked orders: lists, per-record status, retry, response and error, and the wire form."""
import random

import numpy as np
import pytest

import k2ref as R
import k5ref
from jsoncase import make_requests, make_script
from oracle import gojson as G
from oracle import model as M

AGENTS = ["agent-1700000000000000001", "agent-1700000000000000002", "agent-1700000000000000003"]


class Pair:
    """The restatement and the model, fed the same records and outcomes."""

    def __init__(self, reqs, max_retries=3, log_cap=1 << 20, skip_inflight=False, running=(True, False, True)):
        self.redis = M.MiniRedis()
        self.mgr = M.Manager(self.redis)
        self.ref = R.K2Ref(log_cap, skip_inflight=skip_inflight)
        self.reqs = reqs
        for a in AGENTS:
            self.ref.register(a)
        recs = []
        for r in reqs:
            self.mgr.store_request(r.agent_id, M.HttpRequest(r.method, r.path, dict(r.headers), r.body,
                                                             new_id=G.format_uuid(r.rid), now=r.now))
            self.redis.strings[self.key(r)]["max_retries"] = max_retries or 3
            recs.append(k5ref.Rec(r.agent_id.encode(), r.method, r.path, r.flat_headers(), r.body, r.now, max_retries=max_retries, rid=r.rid))
        slots = [self.ref.slot_of(r.agent_id) for r in reqs]
        self.ref.add_rows(0, slots, np.array([list(r.rid) for r in reqs], dtype=np.uint8),
                          [running[s] for s in slots], max_retries=max_retries, recs=recs)
        self.recs = recs

    def key(self, r):
        return f"agent:{r.agent_id}:requests:{G.format_uuid(r.rid)}"

    def apply(self, ops, with_bytes=True):
        """ops: (request index or raw (id, agent), kind, http, seq, hdr, body).  Returns (results, rc) of the restatement after
        checking each op's result against the model's."""
        ids, slots, kinds, https, seqs, segs, hls, want = [], [], [], [], [], [], [], []
        for who, kind, http, seq, hdr, body in ops:
            rid, agent = (self.reqs[who].rid, self.reqs[who].agent_id) if isinstance(who, int) else who
            ids.append(list(rid)); slots.append(self.ref.slot_of(agent)); kinds.append(kind); https.append(http)
            seqs.append(seq); segs.append(hdr + body); hls.append(len(hdr))
            w = 0
            if rid != bytes(16) and kind in (R.OUT_RESPONSE, R.OUT_ERROR):
                try:
                    if kind == R.OUT_RESPONSE:
                        old = self.redis.get(f"agent:{agent}:requests:{G.format_uuid(rid)}") if not with_bytes else None
                        if old is not None and old.get("response"):
                            hmap, b = old["response"]["headers"], old["response"]["body"]
                        else:
                            hmap, b = dict(k5ref.parse_headers(hdr)), body
                        self.mgr.store_response(agent, G.format_uuid(rid), M.HttpResponse(http, hmap, b, now=seq))
                    else:
                        old = self.redis.get(f"agent:{agent}:requests:{G.format_uuid(rid)}") if not with_bytes else None
                        text = body if with_bytes else old["error"]
                        self.mgr.mark_request_failed(agent, G.format_uuid(rid), text or b"transport error")   # (K5's empty text)
                except (KeyError, M.RedisNil):
                    w = R.ENOTFOUND
            want.append(w)
        res, rc = self.ref.complete(np.array(ids, dtype=np.uint8).reshape(-1, 16), slots, kinds, https, seqs,
                                    segs if with_bytes else None, np.array(hls) if with_bytes else None)
        assert res.tolist() == want
        return res, rc

    def check(self):
        for k, r in enumerate(self.reqs):
            want = self.redis.get(self.key(r))
            rec = self.recs[k]
            assert rec.wire() == G.marshal_request(want), k
            st = self.ref.state_words([k])[0]
            assert {1: "pending", 3: "completed", 4: "failed"}[int(st & 7)] == want["status"]
            assert int(st >> R.ST_RETRY_SHIFT & 0xff) == min(want["retry_count"], 255)
            assert bool(st & R.ST_INQ) == (G.format_uuid(r.rid) in self.redis.lrange_all(f"agent:{r.agent_id}:requests:pending"))
            if want["response"]:
                assert int(self.ref.aux_words([k])[0] & 0xffff) == want["response"]["status_code"]
        for s, a in enumerate(AGENTS):
            for which, name in ((R.LIST_PENDING, "pending"), (R.LIST_COMPLETED, "completed"), (R.LIST_FAILED, "failed")):
                rows = self.ref.list(s, which)
                got = [G.format_uuid(self.reqs[r].rid) for r in rows]
                assert got == self.redis.lrange_all(f"agent:{a}:requests:{name}"), (a, name)


def script_ops(script, t0=1_000):
    ops = []
    for k, op in enumerate(script):
        if op[0] == "resp":
            ops.append((op[1], R.OUT_RESPONSE, op[2], op[5], k5ref.flat_headers(sorted(op[3].items())), op[4]))
        else:
            ops.append((op[1], R.OUT_ERROR, 0, t0 + k, b"", op[2]))
    return ops


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("batch", [1, 7, 64, 10_000])
def test_scripts_against_the_model(seed, batch):
    reqs = make_requests(seed, 60, AGENTS)
    p = Pair(reqs)
    ops = script_ops(make_script(seed, len(reqs), 400))
    ops.sort(key=lambda op: op[0] % 7)                     # many ops of one record in a call
    for lo in range(0, len(ops), batch):
        p.apply(ops[lo:lo + batch])
    p.check()
    c = p.ref.ctr
    assert c["completions"] == sum(op[1] == R.OUT_RESPONSE for op in ops) and c["log_overflow"] == 0
    assert c["completions"] + c["failures"] == len(ops)


@pytest.mark.parametrize("max_retries", [0, 1, 3, 255])
def test_plain_complete_keeps_the_stored_bytes(max_retries):
    """agr_complete carries no bytes: a later plain RESPONSE keeps the stored headers and body, a plain ERROR the text."""
    reqs = make_requests(4, 6, AGENTS[:1])
    p = Pair(reqs, max_retries=max_retries)
    p.apply([(0, R.OUT_RESPONSE, 201, 10, b"A: b\n", b"body"), (1, R.OUT_ERROR, 0, 11, b"", b"first text")])
    p.apply([(0, R.OUT_RESPONSE, 500, 12, b"", b""), (1, R.OUT_ERROR, 0, 13, b"", b""), (0, R.OUT_ERROR, 0, 14, b"", b""),
             (2, R.OUT_ERROR, 0, 15, b"", b"")], with_bytes=False)
    p.check()
    assert p.recs[0].resp_body == b"body" and p.recs[0].code == 500 and p.recs[1].err == b"first text"


def test_order_within_a_call():
    """KAT-H: MarkRequestFailed then StoreResponse is not StoreResponse then MarkRequestFailed."""
    reqs = make_requests(5, 4, AGENTS[:1])
    p = Pair(reqs, max_retries=1)
    p.apply([(0, R.OUT_ERROR, 0, 5, b"", b"e"), (0, R.OUT_RESPONSE, 200, 6, b"", b"ok"),
             (1, R.OUT_RESPONSE, 200, 7, b"", b"ok"), (1, R.OUT_ERROR, 0, 8, b"", b"e")])
    p.check()
    st = p.ref.state_words([0, 1])
    assert (st & 7).tolist() == [R.ST_COMPLETED, R.ST_FAILED]
    assert p.ref.logs == ([0, 1], [0, 1])                   # 0 failed (max 1) then completed; 1 completed then failed
    assert (p.ref.mtime[:2] == [6, 8]).all()


def test_errors_past_max_and_retry_saturation():
    reqs = make_requests(6, 3, AGENTS[:1])
    p = Pair(reqs, max_retries=255)
    ops = [(0, R.OUT_ERROR, 0, 100 + k, b"", b"x%d" % k) for k in range(254)]
    p.apply(ops)
    assert int(p.ref.retry[0]) == 254 and p.ref.status[0] == R.ST_PENDING and p.ref.logs[1] == []
    p.apply([(0, R.OUT_ERROR, 0, 1000, b"", b"last")])
    p.check()                                              # (the model's counter has not passed 255 yet)
    assert p.ref.status[0] == R.ST_FAILED and p.ref.logs[1] == [0]
    ref = p.ref
    ref.complete(np.tile(ref.ids[0], (45, 1)), [0] * 45, [R.OUT_ERROR] * 45, [0] * 45, range(2000, 2045))
    assert int(ref.retry[0]) == 255 and ref.logs[1] == [0] * 46 and ref.ctr["dead_lettered"] == 46
    # past max_retries = 3: every further ERROR pushes once more, a RESPONSE completes it again
    q = Pair(make_requests(7, 2, AGENTS[:1]))
    q.apply([(0, R.OUT_ERROR, 0, k, b"", b"e") for k in range(1, 7)] + [(0, R.OUT_RESPONSE, 200, 9, b"", b"")])
    q.check()
    assert q.ref.logs == ([0], [0, 0, 0, 0])


def test_misses_of_every_kind():
    reqs = make_requests(8, 6, AGENTS)
    p = Pair(reqs, skip_inflight=True)
    other = next(a for a in AGENTS if a != reqs[0].agent_id)
    p.ref.expire([3])
    p.redis.delete(p.key(reqs[3]))
    res, rc = p.apply([((bytes(16), reqs[0].agent_id), R.OUT_RESPONSE, 200, 1, b"", b"zero id"),
                       ((reqs[0].rid, "agent-unknown"), R.OUT_RESPONSE, 200, 2, b"", b""),
                       ((reqs[0].rid, other), R.OUT_ERROR, 0, 3, b"", b"wrong agent"),
                       ((bytes(range(16)), reqs[0].agent_id), R.OUT_ERROR, 0, 4, b"", b"unknown id"),
                       (3, R.OUT_RESPONSE, 200, 5, b"", b"expired"),
                       (4, R.OUT_DIAL_ERR, 0, 6, b"", b""),
                       ((bytes(16), reqs[0].agent_id), R.OUT_DIAL_ERR, 0, 7, b"", b"")])
    assert res.tolist() == [0, R.ENOTFOUND, R.ENOTFOUND, R.ENOTFOUND, R.ENOTFOUND, 0, 0] and rc == 0
    assert p.ref.ctr["completion_misses"] == 4 and p.ref.ctr["dial_errors"] == 2
    assert p.ref.logs == ([], [])
    # a dial error changes only the in-flight bit, and only with AGR_CFG_SKIP_INFLIGHT
    for skip in (False, True):
        q = Pair(reqs, skip_inflight=skip, running=(True, True, True))
        before = q.ref.state_words(range(6))
        q.apply([(k, R.OUT_DIAL_ERR, 0, 9, b"", b"") for k in range(6)])
        after = q.ref.state_words(range(6))
        assert ((before ^ after) == (R.ST_INFLIGHT if skip else 0)).all()
        assert (q.ref.mtime[:6] == 0).all() and q.ref.ctr["dial_errors"] == 6
    # a dropped agent's records keep their keys (Q17): its outcomes still apply
    q = Pair(reqs)
    q.ref.drop(reqs[0].agent_id)
    q.apply([(0, R.OUT_RESPONSE, 200, 9, b"", b"after drop")])
    assert q.ref.status[0] == R.ST_COMPLETED and q.ref.logs[0] == [0]


def test_bytes_with_empty_segments():
    """The last RESPONSE's segment of a call is the response (an empty one clears it), the last ERROR's the text."""
    reqs = make_requests(9, 3, AGENTS[:1])
    p = Pair(reqs)
    p.apply([(0, R.OUT_RESPONSE, 200, 1, b"A: 1\n", b"one"), (0, R.OUT_RESPONSE, 201, 2, b"B: 2\n", b"two"),
             (1, R.OUT_ERROR, 0, 3, b"", b"first"), (1, R.OUT_ERROR, 0, 4, b"", b"")])
    p.check()
    assert (p.recs[0].resp_hdr, p.recs[0].resp_body, p.recs[1].err) == (b"B: 2\n", b"two", b"")
    p.apply([(0, R.OUT_RESPONSE, 204, 5, b"", b""), (2, R.OUT_RESPONSE, 200, 6, b"", b""), (2, R.OUT_ERROR, 0, 7, b"", b"e")])
    p.check()
    assert (p.recs[0].resp_hdr, p.recs[0].resp_body) == (b"", b"")


def test_log_cap():
    """Only the first log_cap pushes land; a call that ends exactly at the cap returns 0, one past it AGR_ENOSPC."""
    reqs = make_requests(10, 20, AGENTS[:1])
    p = Pair(reqs, max_retries=1, log_cap=5)
    _, rc = p.apply([(k, R.OUT_RESPONSE, 200, k + 1, b"", b"") for k in range(5)])
    assert rc == 0 and p.ref.logs[0] == [0, 1, 2, 3, 4]
    _, rc = p.apply([(k, R.OUT_ERROR, 0, k + 1, b"", b"") for k in range(5, 11)])
    assert rc == R.ENOSPC and p.ref.logs[1] == [5, 6, 7, 8, 9] and p.ref.ctr["log_overflow"] == 1
    _, rc = p.apply([(11, R.OUT_RESPONSE, 200, 1, b"", b"")])
    assert rc == R.ENOSPC and p.ref.logs[0] == [0, 1, 2, 3, 4] and p.ref.status[11] == R.ST_COMPLETED
    _, rc = p.apply([(12, R.OUT_DIAL_ERR, 0, 1, b"", b"")])
    assert rc == 0 and p.ref.ctr["log_overflow"] == 2


def test_bulk_path_is_fast_and_equals_the_loop():
    """2^20 single-op rows take the vectorised path; the same ops one at a time give the same rows, logs and counters."""
    n = 1 << 20
    rng = np.random.default_rng(3)
    ids = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    slots = rng.integers(0, 3, size=n)
    a = R.K2Ref(3 * n)
    for s in range(3):
        a.register(AGENTS[s])
    a.add_rows(0, slots, ids, slots != 1, max_retries=rng.integers(0, 4, size=n))
    kinds = rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=n)
    seqs = rng.integers(0, 1 << 40, size=n).astype(np.uint64)
    perm = rng.permutation(n)
    import time
    t = time.perf_counter()
    res, rc = a.complete(ids[perm], slots[perm], kinds, rng.integers(100, 600, size=n), seqs)
    assert time.perf_counter() - t < 30 and rc == 0 and (res == 0).all()
    assert len(a.logs[0]) == int((kinds == R.OUT_RESPONSE).sum())
    # a small slice against the one-op-at-a-time path
    b = R.K2Ref(3 * n)
    for s in range(3):
        b.register(AGENTS[s])
    m = 2000
    b.add_rows(0, slots[:m], ids[:m], slots[:m] != 1, max_retries=3)
    c = R.K2Ref(3 * n)
    for s in range(3):
        c.register(AGENTS[s])
    c.add_rows(0, slots[:m], ids[:m], slots[:m] != 1, max_retries=3)
    pick = rng.integers(0, m, size=3 * m)                  # chains: the multi-op path
    k2 = rng.choice([R.OUT_RESPONSE, R.OUT_ERROR], size=3 * m)
    b.complete(ids[pick], slots[pick], k2, np.full(3 * m, 200), np.arange(3 * m, dtype=np.uint64))
    for j in range(3 * m):
        c.complete(ids[pick[j:j + 1]], slots[pick[j:j + 1]], k2[j:j + 1], [200], [j])
    assert (b.state_words(range(m)) == c.state_words(range(m))).all() and b.logs == c.logs
    assert {k: v for k, v in b.ctr.items()} == {k: v for k, v in c.ctr.items()}


def test_random_outcome_streams():
    """Random kinds, misses and chains, many small calls: restatement and model agree after every call."""
    rng = random.Random(11)
    reqs = make_requests(11, 40, AGENTS)
    p = Pair(reqs, max_retries=2)
    for step in range(60):
        ops = []
        for _ in range(rng.randrange(1, 30)):
            k = rng.randrange(len(reqs))
            x = rng.random()
            if x < 0.45:
                ops.append((k, R.OUT_RESPONSE, rng.choice([200, 404]), step * 100 + len(ops), b"", bytes(rng.randrange(3))))
            elif x < 0.85:
                ops.append((k, R.OUT_ERROR, 0, step * 100 + len(ops), b"", b"t%d" % rng.randrange(3)))
            elif x < 0.95:
                ops.append(((reqs[k].rid, AGENTS[(AGENTS.index(reqs[k].agent_id) + 1) % 3]), R.OUT_RESPONSE, 200, 1, b"", b""))
            else:
                ops.append((k, R.OUT_DIAL_ERR, 0, 1, b"", b""))
        p.apply(ops)
        p.check()
