"""Engine-minted ids: the TMA K1 kernel decides every replay's dedupe hit itself, including replays that name an earlier row of
their own batch, and a batch ingested without outputs is one K1 launch (no k1_post).  Consecutive K1 launches overlap through
programmatic dependent launch.  The same stream runs through the two TMA paths (no outputs, and agr_ingest_ex with k1_post),
which must agree with each other; AGR_VF_KNOWN and dedupe_hits are checked against the plain reference of the rule
(tests/k1ref.py), and the C3-shaped stream's verdicts against the C restatement of the reference."""
import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1ref
from agentainer_lab_b200 import constants as K
from test_k1_ref import AGENTS, REGISTERED, SECRET, hand_batch, hand_stream

pytestmark = pytest.mark.gpu

MINT = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS
COUNTERS = ("ingested", "stored", "replay_flagged", "dedupe_hits", "forwarded", "queued", "unavailable", "not_found", "dup_ids")


def _engine(flags=MINT, rows=1 << 14, batch=1 << 12, agents=AGENTS):
    eng = A.Engine(slab_rows=rows, max_agents=512, max_batch=batch, flags=flags, id_secret=SECRET)
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
    """the same stream through TMA K1 without outputs (one launch per batch) and TMA K1 + k1_post with outputs: identical
    verdicts and counters, KNOWN and dedupe_hits as the reference has them"""
    with _engine(flags) as e0, _engine(flags) as e1:
        v0, v1 = _rows_no_outputs(e0, batches), _ingest_ex(e1, batches)
        for b in range(len(batches)):
            assert v0[b].tobytes() == v1[b].tobytes(), b
        s0, s1 = e0.stats(), e1.stats()
        for c in COUNTERS:
            assert s0[c] == s1[c], c
        assert s0["k1_launches"] == len(batches)                  # no k1_post
        assert s1["k1_launches"] == 2 * len(batches)
        recs = np.concatenate(batches)
        known, _ = k1ref.dedupe_hits(recs, _ids(0, len(recs)), REGISTERED, bool(flags & K.AGR_CFG_PERSISTENCE))
        got = (np.concatenate(v0)["flags"] & K.AGR_VF_KNOWN) != 0
        assert (got == known).all(), np.nonzero(got != known)[0]
        assert s0["dedupe_hits"] == int(known.sum())
        return v0


@pytest.mark.parametrize("flags", [MINT, K.AGR_CFG_MINT_IDS], ids=["persistence", "no_persistence"])
def test_in_batch_replays_batch0_row0(flags):
    """batch 0 starts at row 0: the in-K1 decision covers it too"""
    recs, known = hand_batch(0, _ids(0, 32))
    v = _check_paths([recs], flags)
    got = (v[0]["flags"] & K.AGR_VF_KNOWN) != 0
    if flags & K.AGR_CFG_PERSISTENCE:
        assert (got == known).all(), np.nonzero(got != known)[0]
    else:
        assert not got.any()                                                    # nothing is stored, nothing is known


def test_in_batch_and_earlier_batch_replays():
    """a second batch with the same cases, plus replays naming rows of the first"""
    batches, known = hand_stream(_ids(0, 64))
    v = _check_paths(batches)
    for b in range(2):
        assert (((v[b]["flags"] & K.AGR_VF_KNOWN) != 0) == known[b]).all(), b


def test_c3_shaped_stream():
    """several 64 Ki batches of the C3 mix (Zipf agents, 10 % replay-flagged duplicates) — many replays name rows of their own
    batch — through both TMA paths, against the dedupe-hit reference and the C restatement of the reference"""
    from oracle.cpu_ref import CRef
    B, nb, na = 1 << 16, 4, 256
    agents = {A.synth_agent_id(k): ("stopped" if k % 5 == 1 else "running") for k in range(na)}
    with _engine(agents={}) as m:                             # duplicates name the ids the engines mint
        big = A.synth_fill_host(0, nb * B, seed=7, n_agents=na, zipf_milli=1200, dup_permille=100, mint=(m, 0))
    big["request_id"] = _ids(0, nb * B)
    batches = [np.ascontiguousarray(big[b * B:(b + 1) * B]) for b in range(nb)]
    known, _ = k1ref.dedupe_hits(big, big["request_id"], agents)
    engines = [_engine(rows=nb * B + 1024, batch=B, agents=agents) for _ in range(2)]
    try:
        v0, v1 = _rows_no_outputs(engines[0], batches), _ingest_ex(engines[1], batches)
        with CRef() as ref:
            for a, st in agents.items():
                ref.set_agent_state(a, st)
            for b in range(nb):
                assert v0[b].tobytes() == v1[b].tobytes(), b
                vr, _ = ref.ingest(batches[b])
                assert (v0[b]["code"] == vr["code"]).all() and ((v0[b]["flags"] & 0x7) == (vr["flags"] & 0x7)).all(), b
                assert (v0[b]["agent_slot"] == vr["agent_slot"]).all(), b
                assert (((v0[b]["flags"] & K.AGR_VF_KNOWN) != 0) == known[b * B:(b + 1) * B]).all(), b
        st = [e.stats() for e in engines]
        for c in COUNTERS:
            assert st[0][c] == st[1][c], c
        assert st[0]["dedupe_hits"] == int(known.sum()) > nb * B // 40
        assert st[0]["k1_launches"] == nb
    finally:
        for e in engines:
            e.close()


def test_kernel_between_batches_is_waited_for():
    """a synth_fill_rows kernel writes the next batch's rows between two ingest_rows_async calls: K1 must see its records"""
    B, na = 1 << 14, 16
    agents = {A.synth_agent_id(k): "running" for k in range(na)}
    synth = dict(seed=9, n_agents=na, zipf_milli=1200, dup_permille=100)
    with _engine(rows=4 * B, batch=B, agents=agents) as e0, _engine(rows=4 * B, batch=B, agents=agents) as e1:
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
