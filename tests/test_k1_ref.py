"""The plain dedupe-hit reference (tests/k1ref.py) on hand-worked batches that cover the in-batch and earlier-batch cases, with
ids from the id reference (tests/mintref.py).  The GPU test of K1's replay decision runs the same batches.  CPU only."""
import numpy as np
import pytest

import k1ref
from agentainer_lab_b200 import constants as K
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
