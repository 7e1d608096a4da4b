"""Plain reference of K1's dedupe-hit rule (AGR_VF_KNOWN on a verdict, counted in dedupe_hits), written from k1_finish and
k1_post_one.  Nothing here comes from the engine.

A row is a dedupe hit when it is replay-flagged, its replay_of is non-zero, its agent is registered and not dropped, and its
replay_of names a row of EARLIER arrival that was stored, with the same agent.  A row is stored when persistence is on, it is
not replay-flagged, its agent is registered and not dropped, path_len + hdr_len + body_len <= 416, and its id is non-zero and
not the id of an earlier stored row."""
import numpy as np

from agentainer_lab_b200 import constants as K

PAYLOAD = 512 - 96             # payload bytes of a fixed-stride record


def dedupe_hits(recs, ids, registered, persistence=True):
    """recs: records in arrival order (every batch of a stream, one after the other); ids: each row's request id (the minted
    ids with AGR_CFG_MINT_IDS, else recs["request_id"]); registered: agent ids (str) that are registered and not dropped.
    Returns (known, stored), one bool per row."""
    n = len(recs)
    reg = {a.encode() for a in registered}
    idb = np.ascontiguousarray(ids, dtype=np.uint8).tobytes()
    rob = np.ascontiguousarray(recs["replay_of"]).tobytes()
    agents = recs["agent_id"].tolist()
    replay = ((recs["flags"] & K.AGR_F_REPLAY) != 0).tolist()
    fits = (recs["path_len"].astype(np.int64) + recs["hdr_len"] + recs["body_len"] <= PAYLOAD).tolist()
    zero = bytes(16)
    known, stored = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    owner = {}                                                     # id -> agent of the stored row that carries it
    for i in range(n):
        if agents[i] not in reg:
            continue
        if replay[i]:
            t = rob[16 * i:16 * i + 16]
            known[i] = t != zero and owner.get(t) == agents[i]
        elif persistence and fits[i]:
            rid = idb[16 * i:16 * i + 16]
            if rid != zero and rid not in owner:
                owner[rid] = agents[i]
                stored[i] = True
    return known, stored
