"""Engine-minted ids: the TMA K1 kernel decides every replay's dedupe hit itself, including replays that name an earlier row of
their own batch, and a batch ingested without outputs is one K1 launch (no k1_post).  Consecutive K1 launches overlap through
programmatic dependent launch.  Every verdict and counter is checked against the LSU K1 kernel, which leaves every tracked
replay to k1_post, and against agr_ingest_ex on the same engine kind."""
import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from scenario import Req, make_records, rid_of

pytestmark = pytest.mark.gpu

MINT = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS
SECRET = 0x5eed1234
TMA, LSU = 4, 5                      # k1_variant: 14 x 1 TMA kernel (the default) / LSU kernel + k1_post over every row
COUNTERS = ("ingested", "stored", "replay_flagged", "dedupe_hits", "forwarded", "queued", "unavailable", "not_found", "dup_ids")
AGENTS = {"agent-run": "running", "agent-other": "running", "agent-stop": "stopped", "agent-drop": "running"}


def _engine(variant, flags=MINT, rows=1 << 14, batch=1 << 12, agents=AGENTS):
    eng = A.Engine(slab_rows=rows, max_agents=512, max_batch=batch, k1_variant=variant, flags=flags, id_secret=SECRET)
    for a, s in agents.items():
        eng.set_agent_state(a, s)
    if "agent-drop" in agents:
        eng.drop_agent("agent-drop")
    return eng


def _ids(first, n):
    with A.Engine(slab_rows=64, max_agents=4, flags=MINT, id_secret=SECRET) as e:
        return e.mint_ids(first, n)


def _rows_no_outputs(eng, batches):
    """agr_ingest_rows_async per batch (no verdicts, no ids), verdicts read back from the route words afterwards"""
    firsts = []
    for recs in batches:
        first = eng.reserve_rows(len(recs))
        eng.fill_rows(first, recs)
        eng.ingest_rows_async(first, len(recs))
        firsts.append(first)
    eng.sync()
    return [eng.debug_read("verdict", f, len(r)) for f, r in zip(firsts, batches)]


def _ingest_ex(eng, batches):
    out = []
    for recs in batches:
        v = np.zeros(len(recs), dtype=A.verdict_dtype)
        eng.ingest_ex(recs, v, np.zeros((len(recs), 16), dtype=np.uint8))
        out.append(v)
    return out


def _check_paths(batches, flags=MINT):
    """the same stream through: TMA K1 without outputs (one launch per batch), TMA K1 + k1_post with outputs, LSU K1 + k1_post"""
    with _engine(TMA, flags) as e0, _engine(TMA, flags) as e1, _engine(LSU, flags) as e2:
        v0, v1, v2 = _rows_no_outputs(e0, batches), _ingest_ex(e1, batches), _ingest_ex(e2, batches)
        for b in range(len(batches)):
            assert v0[b].tobytes() == v1[b].tobytes(), b
            assert v0[b].tobytes() == v2[b].tobytes(), b
        s0, s1, s2 = e0.stats(), e1.stats(), e2.stats()
        for c in COUNTERS:
            assert s0[c] == s1[c] == s2[c], c
        assert s0["k1_launches"] == len(batches)                  # no k1_post
        assert s1["k1_launches"] == 2 * len(batches)
        return v0, s0


def _hand_batch(first):
    """one batch at row `first` covering the in-batch cases; returns (records, expected KNOWN per row)"""
    ids = _ids(first, 32)
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


@pytest.mark.parametrize("flags", [MINT, K.AGR_CFG_MINT_IDS], ids=["persistence", "no_persistence"])
def test_in_batch_replays_batch0_row0(flags):
    """batch 0 starts at row 0: the in-K1 decision covers it too"""
    recs, known = _hand_batch(0)
    v, s = _check_paths([recs], flags)
    got = (v[0]["flags"] & K.AGR_VF_KNOWN) != 0
    if flags & K.AGR_CFG_PERSISTENCE:
        assert (got == known).all(), np.nonzero(got != known)[0]
    else:
        assert not got.any()                                                    # nothing is stored, nothing is known
    assert s["dedupe_hits"] == int(got.sum())


def test_in_batch_and_earlier_batch_replays():
    """a second batch with the same cases, plus replays naming rows of the first"""
    r0, k0 = _hand_batch(0)
    r1, k1 = _hand_batch(len(r0))
    ids0 = _ids(0, len(r0))
    r1[20]["flags"] |= K.AGR_F_REPLAY
    r1[20]["replay_of"] = ids0[0]                                               # earlier batch, stored, same agent
    k1[20] = True
    r1[17]["replay_of"] = ids0[2]                                               # earlier batch, a replay: not stored
    v, s = _check_paths([r0, r1])
    assert (((v[0]["flags"] & K.AGR_VF_KNOWN) != 0) == k0).all()
    assert (((v[1]["flags"] & K.AGR_VF_KNOWN) != 0) == k1).all()
    assert s["dedupe_hits"] == int(k0.sum() + k1.sum())


def test_c3_shaped_stream():
    """several 64 Ki batches of the C3 mix (Zipf agents, 10 % replay-flagged duplicates) — many replays name rows of their own
    batch — against the other K1 paths and the C restatement of the reference"""
    from oracle.cpu_ref import CRef
    B, nb, na = 1 << 16, 4, 256
    agents = {A.synth_agent_id(k): ("stopped" if k % 5 == 1 else "running") for k in range(na)}
    with _engine(TMA, agents={}) as m:                        # duplicates name the ids the engines mint
        big = A.synth_fill_host(0, nb * B, seed=7, n_agents=na, zipf_milli=1200, dup_permille=100, mint=(m, 0))
    big["request_id"] = _ids(0, nb * B)
    batches = [np.ascontiguousarray(big[b * B:(b + 1) * B]) for b in range(nb)]
    engines = [_engine(v, rows=nb * B + 1024, batch=B, agents=agents) for v in (TMA, TMA, LSU)]
    try:
        v0, v1, v2 = _rows_no_outputs(engines[0], batches), _ingest_ex(engines[1], batches), _ingest_ex(engines[2], batches)
        hits = 0
        with CRef() as ref:
            for a, st in agents.items():
                ref.set_agent_state(a, st)
            for b in range(nb):
                assert v0[b].tobytes() == v1[b].tobytes() == v2[b].tobytes(), b
                vr, _ = ref.ingest(batches[b])
                assert (v0[b]["code"] == vr["code"]).all() and ((v0[b]["flags"] & 0x7) == (vr["flags"] & 0x7)).all(), b
                assert (v0[b]["agent_slot"] == vr["agent_slot"]).all(), b
                hits += int(((v0[b]["flags"] & K.AGR_VF_KNOWN) != 0).sum())
        st = [e.stats() for e in engines]
        for c in COUNTERS:
            assert st[0][c] == st[1][c] == st[2][c], c
        assert st[0]["dedupe_hits"] == hits > nb * B // 40
        assert st[0]["k1_launches"] == nb
    finally:
        for e in engines:
            e.close()


def test_kernel_between_batches_is_waited_for():
    """a synth_fill_rows kernel writes the next batch's rows between two ingest_rows_async calls: K1 must see its records"""
    B, na = 1 << 14, 16
    agents = {A.synth_agent_id(k): "running" for k in range(na)}
    synth = dict(seed=9, n_agents=na, zipf_milli=1200, dup_permille=100)
    with _engine(TMA, rows=4 * B, batch=B, agents=agents) as e0, _engine(TMA, rows=4 * B, batch=B, agents=agents) as e1:
        f0 = e0.reserve_rows(3 * B)
        for k in range(3):                                        # back to back: fill, ingest, fill, ingest, ...
            e0.synth_fill_rows(k * B, f0 + k * B, B, mint_base=f0, **synth)
            e0.ingest_rows_async(f0 + k * B, B)
        e0.sync()
        f1 = e1.reserve_rows(3 * B)
        for k in range(3):                                        # every fill done and synchronised before any ingest
            e1.synth_fill_rows(k * B, f1 + k * B, B, mint_base=f1, **synth)
        e1.sync()
        for k in range(3):
            e1.ingest_rows(f1 + k * B, B, want_verdicts=False)
        assert f0 == f1
        assert e0.debug_read("cksum", f0, 3 * B).tobytes() == e1.debug_read("cksum", f1, 3 * B).tobytes()
        assert e0.debug_read("cksum", f0, 3 * B).all()
        assert e0.debug_read("verdict", f0, 3 * B).tobytes() == e1.debug_read("verdict", f1, 3 * B).tobytes()
        assert (e0.debug_read("verdict", f0, 3 * B)["code"] == K.AGR_V_FORWARD).all()
        s0, s1 = e0.stats(), e1.stats()
        for c in COUNTERS:
            assert s0[c] == s1[c], c
        assert s0["dedupe_hits"] > 0
