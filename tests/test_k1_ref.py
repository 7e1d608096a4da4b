"""The plain dedupe-hit reference (tests/k1ref.py) on hand-worked batches that cover the in-batch and earlier-batch cases, with
ids from the id reference (tests/mintref.py).  The GPU test of K1's replay decision runs the same batches.  CPU only."""
import copy

import numpy as np
import pytest

import k1ref
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.binding import record_dtype
from mintref import mint_many
from scenario import Req, make_records, rid_of

SECRET = 0x5eed1234
AGENTS = {"agent-run": "running", "agent-other": "running", "agent-stop": "stopped", "agent-drop": "running"}
REGISTERED = ("agent-run", "agent-other", "agent-stop")      # agent-drop is dropped after registration, agent-nobody never exists


def hand_batch(first, ids):
    """one batch at row `first` covering the in-batch cases (ids: the minted ids of rows first, first + 1, ...); returns
    (records, expected KNOWN per row with persistence on)"""
    rid = lambda k: bytes(ids[k])
    R = lambda k, a, **kw: Req(a, rid_of(first + k), first + k, **kw)
    reqs, known = [], []

    def add(req, hit):
        reqs.append(req); known.append(hit)
    add(R(0, "agent-run"), False)                                               # 0: stored
    add(R(1, "agent-run", replay=True, replay_of=rid(0)), True)                 # 1: earlier row, same agent
    add(R(2, "agent-other", replay=True, replay_of=rid(0)), False)              # 2: earlier row, other agent
    add(R(3, "agent-run"), False)                                               # 3: too long for its row (below): not stored
    add(R(4, "agent-run", replay=True, replay_of=rid(3)), False)                # 4: target with a bad length
    add(R(5, "agent-run", replay=True, replay_of=rid(0)), True)                 # 5: replay-flagged (and itself a hit)
    add(R(6, "agent-run", replay=True, replay_of=rid(5)), False)                # 6: target is replay-flagged
    add(R(7, "agent-run", replay=True, replay_of=rid(8)), False)                # 7: target is a later row
    add(R(8, "agent-run"), False)
    add(R(9, "agent-run", replay=True, replay_of=rid(9)), False)                # 9: names itself
    add(R(10, "agent-stop"), False)                                             # 10: stored, queued
    add(R(11, "agent-stop", replay=True, replay_of=rid(10)), True)              # 11: stopped agent
    add(R(12, "agent-nobody"), False)                                           # 12: unknown agent: not stored
    add(R(13, "agent-nobody", replay=True, replay_of=rid(12)), False)           # 13: not found itself
    add(R(14, "agent-drop"), False)                                             # 14: removed agent
    add(R(15, "agent-drop", replay=True, replay_of=rid(14)), False)
    add(R(16, "agent-run", replay=True, replay_of=rid_of(99)), False)           # 16: id the engine never minted
    add(R(17, "agent-other", replay=True, replay_of=rid(18)), False)
    add(R(18, "agent-other"), False)
    add(R(19, "agent-other", replay=True, replay_of=rid(18)), True)             # 19: earlier row of another agent, same agent
    add(R(20, "agent-run", replay=True), False)                                 # 20: untracked replay (no id)
    recs = make_records(reqs)
    recs[3]["body_len"] = 400                                                   # path + headers + body > 416 B
    return recs, np.array(known)


def hand_stream(ids):
    """two hand batches at rows 0 and 21 (ids: the minted ids of rows 0..41), the second with replays naming rows of the first;
    returns ([records of each batch], [expected KNOWN of each batch])"""
    r0, k0 = hand_batch(0, ids)
    r1, k1 = hand_batch(len(r0), ids[len(r0):])
    r1[20]["flags"] |= K.AGR_F_REPLAY
    r1[20]["replay_of"] = ids[0]                                                # earlier batch, stored, same agent
    k1[20] = True
    r1[17]["replay_of"] = ids[2]                                                # earlier batch, a replay: not stored
    return [r0, r1], [k0, k1]


@pytest.mark.parametrize("persistence", [True, False])
@pytest.mark.parametrize("nb", [1, 2])
def test_hand_batches(nb, persistence):
    ids = mint_many(0, 64, SECRET)
    batches, exp = hand_stream(ids)
    recs = np.concatenate(batches[:nb])
    known, stored = k1ref.dedupe_hits(recs, ids[:len(recs)], REGISTERED, persistence)
    if persistence:
        assert known.tolist() == np.concatenate(exp[:nb]).tolist()
        assert np.nonzero(stored[:21])[0].tolist() == [0, 8, 10, 18]
    else:
        assert not known.any() and not stored.any()                            # nothing is stored, nothing is known


# ------------------------------------------------------------------------------------------------------- k1ref.Ref
STATUS = {"agent-run": K.AGR_AGENT_RUNNING, "agent-other": K.AGR_AGENT_RUNNING, "agent-stop": K.AGR_AGENT_STOPPED}


def _ref(mint=False, persistence=True, dropped=("agent-drop",)):
    table = {a: (k, STATUS.get(a, K.AGR_AGENT_RUNNING)) for k, a in enumerate(AGENTS)}
    for a in dropped:
        table[a] = (table[a][0], "dropped")
    return k1ref.Ref(table, mint=mint, secret=SECRET, persistence=persistence)


def _rec(recs, k, agent, rid=None, replay_of=None, seq=None):
    recs[k]["agent_id"] = agent.encode()
    recs[k]["request_id"] = np.frombuffer(rid if rid is not None else rid_of(1000 + k), dtype=np.uint8)
    recs[k]["flags"] = 2 << K.AGR_F_METHOD_SHIFT
    if replay_of is not None:
        recs[k]["flags"] |= K.AGR_F_REPLAY
        recs[k]["replay_of"] = np.frombuffer(replay_of, dtype=np.uint8)
    recs[k]["path_len"], recs[k]["hdr_len"], recs[k]["body_len"] = 10, 10, 10
    recs[k]["max_retries"] = 5
    recs[k]["seq"] = 100 + k if seq is None else seq


def test_hand_rows_caller_ids():
    """each rule on hand-worked rows: the defect triple (A < B carry id X, R > A replays X), a zero id, a 416 / 417 B payload,
    max_retries 0, a stopped agent, a dropped and an unknown agent, a replay of a later row"""
    X, Y = rid_of(1), rid_of(2)
    recs = np.zeros(12, dtype=record_dtype)
    _rec(recs, 0, "agent-run", X)                          # A: owns X
    _rec(recs, 1, "agent-run", replay_of=X)                # R: hit (A is stored, same agent)
    _rec(recs, 2, "agent-other", X)                        # B: X again -> DUP_ID
    _rec(recs, 3, "agent-run", bytes(16))                  # zero id -> DUP_ID, not stored
    _rec(recs, 4, "agent-stop", Y)                         # stopped: stored, queued
    recs[4]["max_retries"] = 0                             #   max_retries 0 reads 3
    _rec(recs, 5, "agent-run"); recs[5]["body_len"] = 396  # 10 + 10 + 396 = 416: stored
    _rec(recs, 6, "agent-run"); recs[6]["body_len"] = 397  # 417: BAD_LEN
    _rec(recs, 7, "agent-drop")                            # dropped: not found
    _rec(recs, 8, "agent-nobody")                          # unknown: not found
    _rec(recs, 9, "agent-stop", replay_of=rid_of(1011))    # replay of a later row: tracked, not a hit, queued
    _rec(recs, 10, "agent-other", replay_of=X)             # replay of X by another agent: not a hit
    _rec(recs, 11, "agent-run")
    recs[11]["request_id"] = np.frombuffer(rid_of(1011), dtype=np.uint8)
    ref = _ref()
    out = ref.ingest(recs)
    v = out["verdict"]
    S, T, R, KN, D, B = (K.AGR_VF_STORED, K.AGR_VF_TRACKED, K.AGR_VF_REPLAY, K.AGR_VF_KNOWN, K.AGR_VF_DUP_ID, K.AGR_VF_BAD_LEN)
    assert v["flags"].tolist() == [S | T, R | T | KN, D, D, S | T, S | T, B, 0, 0, R | T, R | T, S | T]
    F, Q, U, NF = K.AGR_V_FORWARD, K.AGR_V_QUEUED, K.AGR_V_UNAVAILABLE, K.AGR_V_NOT_FOUND
    assert v["code"].tolist() == [F, F, F, F, Q, F, F, NF, NF, Q, F, F]
    assert v["http_status"].tolist() == [0, 0, 0, 0, 202, 0, 0, 404, 404, 202, 0, 0]
    assert v["agent_slot"].tolist() == [0, 0, 1, 0, 2, 0, 0, 0x7FFFFF, 0x7FFFFF, 2, 1, 0]
    run = 1 | 0x8 | 0x20 | 0x10
    assert out["state"].tolist() == [run | 5 << 16, 0, 0, 0, (1 | 0x8 | 0x20) | 3 << 16, run | 5 << 16, 0, 0, 0, 0, 0, run | 5 << 16]
    assert (out["route"] == (np.where(v["agent_slot"] == 0x7FFFFF, 0x7FFFFF, v["agent_slot"]).astype(np.int64)
                             | v["code"].astype(np.int64) << 23 | v["flags"].astype(np.int64) << 26)).all()
    assert ref.ctr == dict(ingested=12, stored=4, replay_flagged=3, dedupe_hits=1, forwarded=8, queued=2, unavailable=0,
                           not_found=2, dup_ids=2, malformed=1)
    assert ref.index_used() == 4                           # X, Y, rid_of(1005), rid_of(1011): B's X is no new key
    assert ref.pending_rows(0) == [0, 5, 11] and ref.pending_rows(2) == [4]
    # a second batch: X again (an earlier batch owns it), and a replay of X that is now a hit for agent-run
    r2 = np.zeros(2, dtype=record_dtype)
    _rec(r2, 0, "agent-run", X); _rec(r2, 1, "agent-run", replay_of=X)
    o2 = ref.ingest(r2)
    assert o2["verdict"]["flags"].tolist() == [D, R | T | KN] and o2["first"] == 12


def test_hand_rows_expire_reclaim():
    """the ring's sweep drops stored rows whose created_at is ttl or more before now; reclaim moves the tail to the first row
    still stored and (caller ids) rebuilds the index from the rows left, only when it released something"""
    recs = np.zeros(4, dtype=record_dtype)
    for k, t in enumerate((10, 50, 90, 20)):
        _rec(recs, k, "agent-run", seq=t)
    ref = _ref()
    ref.ingest(recs)
    assert ref.expire(60, 40) == 2 and ref.stored_rows().tolist() == [1, 2]       # 60 - t >= 40 for rows 0 and 3
    assert ref.index_used() == 4
    assert ref.reclaim() == 1 and ref.tail == 1 and ref.index_used() == 2          # row 3 is expired but not released
    assert ref.expire(60, 40) == 0 and ref.reclaim() == 0 and ref.index_used() == 2
    assert ref.expire(100, 40) == 1 and ref.reclaim() == 1 and ref.index_used() == 1
    assert ref.expire(200, 40) == 1 and ref.reclaim() == 2 and ref.index_used() == 0 and ref.tail == 4


def test_hand_rows_restore_index():
    """the index a restore leaves: Z (expires), P (completed later, so it does not), A carrying X (expires behind P); the
    release stops at P and leaves A out of the index; C carries X again and is stored.  A ring's restore rebuilds the index
    from the rows that hold a record (C owns X; the ids of A and Y, expired but not released, are gone); an append-only
    engine's comes back as it was"""
    X, Y, W = rid_of(1), rid_of(2), rid_of(3)
    recs = np.zeros(5, dtype=record_dtype)
    _rec(recs, 0, "agent-run", rid_of(9), seq=10)         # Z
    _rec(recs, 1, "agent-run", W, seq=10)                  # P
    _rec(recs, 2, "agent-run", X, seq=10)                  # A
    _rec(recs, 3, "agent-stop", Y, seq=10)                 # expires behind P, its id never comes back
    _rec(recs, 4, "agent-run", rid_of(8), seq=95)          # stays stored
    ref = _ref()
    ref.ingest(recs)
    ref.touch([1], 90)                                     # P's StoreResponse
    assert ref.expire(100, 50) == 3 and ref.stored_rows().tolist() == [1, 4]
    assert ref.reclaim() == 1 and ref.tail == 1 and ref.index_used() == 2     # the index of P onward: W and rid_of(8)
    c = np.zeros(3, dtype=record_dtype)
    _rec(c, 0, "agent-run", X, seq=100)                    # C: X is free again
    _rec(c, 1, "agent-run", replay_of=X, seq=100)          # names C: a hit
    _rec(c, 2, "agent-other", X, seq=100)                  # X again: DUP_ID
    S, T, KN, D, RP = K.AGR_VF_STORED, K.AGR_VF_TRACKED, K.AGR_VF_KNOWN, K.AGR_VF_DUP_ID, K.AGR_VF_REPLAY
    assert ref.ingest(c)["verdict"]["flags"].tolist() == [S | T, RP | T | KN, D]
    assert ref.owner[X] == 5 and ref.index_used() == 3
    flat = copy.deepcopy(ref)
    assert ref.restore(ring=True) == 3 and ref.owner == {W: 1, rid_of(8): 4, X: 5}
    assert flat.restore(ring=False) == 3 and flat.owner == ref.owner
    # after a ring restore: Y is free, X still names C; a later release leaves the same index as the restore did
    r2 = np.zeros(3, dtype=record_dtype)
    _rec(r2, 0, "agent-stop", Y, seq=100)
    _rec(r2, 1, "agent-run", X, seq=100)
    _rec(r2, 2, "agent-run", replay_of=X, seq=100)
    assert ref.ingest(r2)["verdict"]["flags"].tolist() == [S | T, D, RP | T | KN]
    assert ref.owner[Y] == 8 and ref.owner[X] == 5
    # an id of a row that expired after the last release: in the index of an engine that never restarted, not after a
    # ring restore
    live = _ref()
    live.ingest(recs[:3])
    live.expire(100, 50)
    assert live.index_used() == 3 and live.restore(ring=True) == 0
    again = _ref()
    again.ingest(recs[:3])
    again.expire(100, 50)
    assert again.restore(ring=False) == 3                   # append-only: X, W and rid_of(9) stay


def test_hand_rows_minted_ids():
    """minted ids: the target is the row the id was minted for, if it is in the window [tail, head) and earlier"""
    ids = mint_many(0, 8, SECRET)
    recs = np.zeros(6, dtype=record_dtype)
    _rec(recs, 0, "agent-run")
    _rec(recs, 1, "agent-run", replay_of=bytes(ids[0]))       # hit
    _rec(recs, 2, "agent-run", replay_of=bytes(ids[2]))       # itself: no
    _rec(recs, 3, "agent-run", replay_of=bytes(ids[4]))       # a later row: no
    _rec(recs, 4, "agent-run", bytes(16))                     # zero caller id: ignored with minted ids, stored
    _rec(recs, 5, "agent-run", replay_of=bytes(ids[7]))       # beyond the batch: no
    ref = _ref(mint=True)
    out = ref.ingest(recs)
    assert out["known"].tolist() == [False, True, False, False, False, False] and out["stored"].tolist() == [1, 0, 0, 0, 1, 0]
    assert ref.expire(1 << 40, 1) == 2 and ref.reclaim() == 6
    r2 = np.zeros(1, dtype=record_dtype)
    _rec(r2, 0, "agent-run", replay_of=bytes(ids[0]))         # released: no
    assert not ref.ingest(r2)["known"][0]


def test_cksum_hand():
    r = np.zeros(3, dtype=record_dtype)
    w = r.view(np.uint8).reshape(3, 512).view("<u4")
    w[0, 0] = 1
    w[1, 127] = 0xFFFFFFFF
    w[2, :] = 0x01000001
    c = k1ref.cksum(r)
    assert c[0] == (1 << 32) | 1
    assert c[1] == ((128 * 0xFFFFFFFF) % (1 << 32)) << 32 | 0xFFFFFFFF
    assert c[2] == ((0x01000001 * 128 * 129 // 2) % (1 << 32)) << 32 | ((0x01000001 * 128) % (1 << 32))


def test_hashes_and_grid():
    from mintref import fmix64
    rng = np.random.default_rng(3)
    x = rng.integers(0, 1 << 63, 50, dtype=np.uint64)
    assert k1ref.fmix64(x).tolist() == [fmix64(int(v)) for v in x]
    ids = rng.integers(0, 256, (20, 16), dtype=np.uint8)
    M = (1 << 64) - 1
    for i in range(20):
        lo, hi = int.from_bytes(bytes(ids[i, :8]), "little"), int.from_bytes(bytes(ids[i, 8:]), "little")
        assert int(k1ref.hash_id(ids[i:i + 1])[0]) == fmix64(lo ^ ((hi * 0x9E3779B97F4A7C15) & M))
    name = b"agent-x"
    w = [int.from_bytes((name + bytes(32))[8 * k:8 * k + 8], "little") for k in range(4)]
    h = (w[0] * 0x9E3779B97F4A7C15) & M
    h ^= ((w[1] + 0x165667B19E3779F9) & M) * 0xC2B2AE3D27D4EB4F & M
    h ^= ((w[2] + 0x27D4EB2F165667C5) & M) * 0xFF51AFD7ED558CCD & M
    h ^= ((w[3] + 0x85EBCA77C2B2AE63) & M) * 0xC4CEB9FE1A85EC53 & M
    assert int(k1ref.hash_agent([name])[0]) == fmix64(h)
    assert k1ref.grid(1, 132) == (1, 14) and k1ref.grid(32 * 14 * 132, 132) == (132, 1848)
    assert k1ref.grid(32 * 14 * 132 + 1, 132) == (132, 1848) and k1ref.grid(32 * 15, 132) == (2, 28)
    warp, rnd = k1ref.schedule(32 * 1849, 132)
    assert warp[-1] == 0 and rnd[-1] == 1 and rnd[:-1].max() == 0


def _stream(seed, n, dups):
    """n requests over the AGENTS (and one never registered), unique ids or (dups) ids repeated by the same agent, and
    replay-flagged requests naming an earlier id, a later id, an unknown id, or none"""
    from scenario import Req
    rng = np.random.default_rng(seed)
    names = list(AGENTS) + ["agent-nobody"]
    reqs = []
    for k in range(n):
        a = names[int(rng.choice(len(names), p=[0.35, 0.3, 0.2, 0.05, 0.1]))]
        rid = rid_of(seed * 100000 + k)
        u = rng.random()
        if dups and u < 0.1 and reqs:
            j = int(rng.integers(0, len(reqs)))
            if not reqs[j].replay:
                a, rid = reqs[j].agent_id, reqs[j].rid
        if 0.1 <= u < 0.3:
            kind = int(rng.integers(0, 4))
            tgt = (reqs[int(rng.integers(0, len(reqs)))].rid if reqs and kind == 0 else rid_of(seed * 100000 + k + 5) if kind == 1
                   else rid_of(7) if kind == 2 else bytes(16))
            if kind == 0 and rng.random() < 0.8:
                a = next((r.agent_id for r in reqs if r.rid == tgt), a)
            reqs.append(Req(a, rid, k + 1, replay=True, replay_of=tgt))
        else:
            reqs.append(Req(a, rid, k + 1))
    return reqs


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("persistence", [True, False])
def test_against_model(seed, persistence):
    """seeded streams with unique ids through oracle/model.py (proxyToAgentHandler + StoreRequest): every code, HTTP status,
    stored and tracked bit, and every pending list, in several batches"""
    from scenario import make_records, run_oracle
    reqs = _stream(seed, 600, dups=False)
    ev = [("agent", a, "running" if STATUS.get(a, 1) == 1 else "stopped") for a in AGENTS] + [("remove", "agent-drop")]
    ev += [("req", r, ("dial",)) for r in reqs]             # a dial error leaves a stored request pending
    obs = run_oracle(ev, persistence)
    recs = make_records(reqs)
    ref = _ref(persistence=persistence)
    outs = [ref.ingest(recs[a:b]) for a, b in ((0, 1), (1, 250), (250, 600))]
    v = np.concatenate([o["verdict"] for o in outs])
    got = [(int(x["code"]), int(x["http_status"]), bool(x["flags"] & K.AGR_VF_STORED), bool(x["flags"] & K.AGR_VF_TRACKED)) for x in v]
    assert got == [tuple(t) for t in obs.verdicts]
    for a in ("agent-run", "agent-other", "agent-stop"):
        rows = ref.pending_rows(AGENTS_INDEX[a])
        assert [reqs[r].rid.hex() for r in rows] == [h.replace("-", "") for h in obs.lists[a]["pending"]], a


AGENTS_INDEX = {a: k for k, a in enumerate(AGENTS)}


@pytest.mark.parametrize("seed", [4, 5])
def test_against_cref(seed):
    """caller-id streams with duplicate fresh ids and replays naming them, one record at a time through the C restatement:
    codes, HTTP statuses and flags agree wherever an id is fresh; a repeated id is DUP_ID (the C port stores it again, its pending
    list then holds the id twice, the reference's only the first); a replay is a dedupe hit exactly when the C port holds the
    record it names for that agent"""
    from oracle.cpu_ref import CRef
    from scenario import make_records
    reqs = _stream(seed, 800, dups=True)
    recs = make_records(reqs)
    ref = _ref()
    with CRef(K.AGR_CFG_PERSISTENCE) as c:
        for a in AGENTS:
            c.set_agent_state(a, "running" if STATUS.get(a, 1) == 1 else "stopped")
        c.drop_agent("agent-drop")
        cv, known = [], []
        for k in range(len(recs)):
            if reqs[k].replay and reqs[k].replay_of != bytes(16):
                known.append(c.get_record(reqs[k].agent_id, reqs[k].replay_of) is not None)
            else:
                known.append(False)
            cv.append(c.ingest(recs[k:k + 1])[0][0])
        cv = np.array(cv)
        out = ref.ingest(recs)
        v = out["verdict"]
        dup = (v["flags"] & K.AGR_VF_DUP_ID) != 0
        assert dup.sum() > 10 and out["known"].sum() > 10
        same = ~dup
        assert (v["code"][same] == cv["code"][same]).all() and (v["http_status"][same] == cv["http_status"][same]).all()
        assert ((v["flags"][same] & 7) == (cv["flags"][same] & 7)).all()
        assert (cv["flags"][dup] & K.AGR_VF_STORED).all() and not (v["flags"][dup] & K.AGR_VF_STORED).any()
        assert out["known"].tolist() == known
        found = v["code"] != K.AGR_V_NOT_FOUND
        assert (v["agent_slot"][found] == cv["agent_slot"][found]).all()
        for a in ("agent-run", "agent-other", "agent-stop"):
            theirs = [bytes(r) for r in c.list(a, K.AGR_LIST_PENDING)]
            first = list(dict.fromkeys(theirs))
            assert [reqs[r].rid for r in ref.pending_rows(AGENTS_INDEX[a])] == first, a
