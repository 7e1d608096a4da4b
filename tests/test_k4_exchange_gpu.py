"""The multi-GPU exchange on one GPU.  (a) K4's kernels (owner hash, count matrix, k4_scan, stable owner-major scatter, the
in-place shift, k4_unpermute) bit for bit against the plain reference tests/k4ref.py, for 1..32 shards (agr_debug_k4).
(b) G engines on one device, each a shard of a simulated world (agr_debug_world), running agr_ingest_sharded_rows' own stages
(agr_debug_exchange_begin / _end) with the test carrying the records and verdicts between them, against oracle/cpu_ref.c per
owner fed the owner's merge order.  (c) A caller's flags bit 31 does not make a record of this shard a hole.  (d) The real NCCL
path at world = 1 against plain ingest / complete.  Real peer transfers and K2 over received outcomes need two GPUs
(tests/test_sharded_gpu.py)."""
import ctypes

import numpy as np
import pytest
import torch

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.sharding import make_rank_batch, owned_agents
from k4ref import expected, fnv1a64, unpermute
from oracle.cpu_ref import CRef

pytestmark = pytest.mark.gpu

GS = [1, 2, 3, 5, 8, 17, 31, 32]
NS = [0, 1, 31, 32, 33, 1000, 2049]
DISTS = ["uniform", "zipf", "one_peer", "all_me", "none_me", "alternating"]
HOLE_BIT = 0x80000000


def _id_pools(G: int, rng) -> list:
    """agent ids (32 B fields) owned by each of G shards: 1..31 bytes from 0x01..0xff (bytes >= 0x80 included), junk after the NUL"""
    pools = [[] for _ in range(G)]
    while min(len(p) for p in pools) < 4:
        ln = int(rng.integers(1, 32))
        f = rng.integers(1, 256, 32).astype(np.uint8)
        f[ln] = 0
        pools[fnv1a64(f.tobytes()) % G].append(f)
    return [np.array(p) for p in pools]


def _owners_for(dist: str, n: int, G: int, me: int, rng) -> np.ndarray:
    if dist == "uniform":
        return rng.integers(0, G, n)
    if dist == "zipf":
        return (rng.zipf(1.3, n) - 1) % G
    if dist == "one_peer":
        return np.full(n, (me + 1) % G)
    if dist == "all_me":
        return np.full(n, me)
    if dist == "none_me":
        return (me + 1 + rng.integers(0, max(G - 1, 1), n)) % G if G > 1 else np.full(n, me)
    return np.arange(n) % G                                                   # alternating: match_any groups of one


def _items(n, item_bytes, agent_off, owner, pools, rng, noise):
    raw = noise[: n * item_bytes].reshape(n, item_bytes).copy()
    for g in np.unique(owner):
        sel = np.nonzero(owner == g)[0]
        raw[sel, agent_off: agent_off + 32] = pools[g][rng.integers(0, len(pools[g]), len(sel))]
    return raw


def _check_k4(eng, raw, agent_off, G, me, inplace, rdt, ctx):
    n = len(raw)
    if rdt == np.uint64:
        loc, rem = np.arange(n, dtype=np.uint64) | (0xA5 << 40), np.arange(n, dtype=np.uint64) | (0x5A << 40) | (1 << 63)
    else:
        loc, rem = np.arange(n, dtype=np.uint32) * 2 + 1, np.arange(n, dtype=np.uint32) * 2
    got = eng.debug_k4(raw, agent_off, inplace, loc, rem)
    e = expected(raw, agent_off, G, me, inplace)
    assert np.array_equal(got["owner"], e["owner"]), ctx
    assert np.array_equal(got["gtotal"][:G], e["gtotal"]) and np.array_equal(got["goff"][: G + 1], e["goff"]), ctx
    assert np.array_equal(got["perm"], e["perm"]), ctx
    assert np.array_equal(got["send"], e["send"]), ctx            # shipped copies are the source bytes, flags word included
    assert np.array_equal(got["local"], e["local"]), ctx
    assert np.array_equal(got["items"], raw), ctx                 # K4 writes nothing into the source rows
    assert np.array_equal(got["res"], unpermute(e["owner"], e["perm"], e["goff"], me, inplace, loc, rem)), ctx


FORMS = [("records", 512, 32, True), ("outcomes", 64, 16, False)]


@pytest.mark.parametrize("form", FORMS, ids=[f[0] for f in FORMS])
@pytest.mark.parametrize("G", GS)
def test_k4_against_reference(G, form):
    """max_batch 32768: 32 warps at most, so per_warp is exactly 32 up to n = 1024 and chunk edges fall inside warps above."""
    _, ib, aoff, inplace = form
    rng = np.random.default_rng(1000 + G * 2 + inplace)
    pools = _id_pools(G, rng)
    mb = 1 << 15
    noise = rng.integers(0, 256, mb * ib, dtype=np.uint8)
    with A.Engine(slab_rows=1 << 12, max_batch=mb) as eng:
        for mi, me in enumerate(sorted({0, G // 2, G - 1})):
            eng.debug_world(me, G)
            for n in NS + [mb]:
                dists = DISTS if n in (33, 1000, 2049, mb) else ["uniform", "all_me"]
                for di, dist in enumerate(dists):
                    rdt = np.uint64 if (mi + di + inplace) % 2 else np.uint32
                    owner = _owners_for(dist, n, G, me, rng)
                    raw = _items(n, ib, aoff, owner, pools, rng, noise)
                    _check_k4(eng, raw, aoff, G, me, inplace, rdt, (G, me, n, dist))


@pytest.mark.parametrize("G", [3, 32])
def test_k4_long_warp_runs_and_full_grid(G):
    """max_batch 4096: four warps, runs of several hundred items that n does not divide.  max_batch = sm_count * 32 * 1024: the
    warp count reaches its cap (32 per SM) at n = sm_count * 32 * 32, and the runs grow past 32 above that."""
    rng = np.random.default_rng(77 + G)
    pools = _id_pools(G, rng)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for mb, ns in ((4096, [1000, 2049, 4000, 4096]), (sms * 32 * 1024, [sms * 32 * 32, sms * 32 * 32 + 4097, 3 * sms * 1024 + 5])):
        noise = rng.integers(0, 256, max(ns) * 64, dtype=np.uint8)
        with A.Engine(slab_rows=1 << 12, max_batch=mb) as eng:
            for me in (0, G - 1):
                eng.debug_world(me, G)
                for n in ns:
                    for dist in ("uniform", "zipf", "alternating"):
                        owner = _owners_for(dist, n, G, me, rng)
                        for ib, aoff, inplace in ((64, 16, False), (64, 16, True)) if n > 4096 else ((512, 32, True), (64, 16, False)):
                            raw = _items(n, ib, aoff, owner, pools, rng, noise if ib == 64 else rng.integers(0, 256, n * ib, dtype=np.uint8))
                            _check_k4(eng, raw, aoff, G, me, inplace, np.uint64 if inplace else np.uint32, (mb, G, me, n, dist))


# ------------------------------------------------------------------------------------------------ (b) simulated world
def _vkey(v):
    return int(v["code"]), int(v["flags"])


def _split_send(send, info, G, me):
    """the owner-major send buffer of rank `me` as {owner: its segment}"""
    out, o = {}, 0
    for q in range(G):
        if q != me and info.sent_to[q]:
            out[q] = send[o: o + info.sent_to[q]]
            o += info.sent_to[q]
    assert o == len(send)
    return out


def _world_step(engs, batches, G):
    """one exchange step of the simulated world; returns every rank's verdicts (caller order) and infos"""
    firsts, segs, infos = [], [], []
    for r, e in enumerate(engs):
        n = len(batches[r])
        f = e.reserve_rows(n) if n else e.stats()["rows_used"]
        if n:
            e.fill_rows(f, batches[r])
        send, info = e.debug_exchange_begin(f, n)
        assert info.n_local + info.n_sent == n and info.n_received == 0 and info.first_rid == f
        firsts.append(f); segs.append(_split_send(send, info, G, r)); infos.append(info)
    back = [dict() for _ in range(G)]
    for o, e in enumerate(engs):                                  # the owner's merge order: own batch (done), then sources by rank
        srcs = [s for s in range(G) if s != o and o in segs[s]]
        if not srcs:
            continue
        inc = np.ascontiguousarray(np.concatenate([segs[s][o] for s in srcs]))
        f2 = e.reserve_rows(len(inc))
        e.fill_rows(f2, inc)
        v = e.ingest_rows(f2, len(inc))
        k = 0
        for s in srcs:
            back[s][o] = v[k: k + len(segs[s][o])]
            k += len(segs[s][o])
    outs = []
    for r, e in enumerate(engs):
        parts = [back[r][q] for q in range(G) if q in back[r]]
        b = np.concatenate(parts) if parts else np.zeros(0, A.verdict_dtype)
        outs.append(e.debug_exchange_end(b, len(batches[r])))
    return outs, infos


def _owned_mask(b, G, r):
    return np.array([A.agent_shard(a.decode(), G) == r for a in b["agent_id"]], dtype=bool) if len(b) else np.zeros(0, bool)


WORLD_CASES = [  # (G, minted ids, every agent registered on every shard)
    (2, False, False), (3, True, False), (5, False, False), (3, False, False), (2, True, False), (5, True, False),
    (3, False, True), (5, True, True), (2, False, True),
]


@pytest.mark.parametrize("G,mint,everywhere", WORLD_CASES)
def test_simulated_world_against_cref(G, mint, everywhere):
    own = owned_agents(G, 6)
    status = lambda a: "running" if int(a[-1]) % 3 else "stopped"
    flags = K.AGR_CFG_PERSISTENCE | (K.AGR_CFG_MINT_IDS if mint else 0)
    engs = [A.Engine(slab_rows=1 << 15, max_agents=256, max_batch=4096, flags=flags) for _ in range(G)]
    refs = [CRef() for _ in range(G)]
    try:
        for r, e in enumerate(engs):
            e.debug_world(r, G)
            for q in range(G):
                if q == r or everywhere:
                    for a in own[q]:
                        e.set_agent_state(a, status(a))
            for a in own[r]:
                refs[r].set_agent_state(a, status(a))
        exp_stats = [dict(ingested=0, stored=0, forwarded=0, queued=0) for _ in range(G)]
        shipped = []
        for step, n in enumerate((700, 1, 0, 1500)):
            batches = []
            for r in range(G):
                nr = n if (n != 1 or r == 0) else 0
                b = make_rank_batch(r, G, own, nr, seed=31 + step, p_cross_replay=0.05, p_missteer=0.08, first_index=step * 10000) \
                    if nr else np.zeros(0, A.record_dtype)
                batches.append(b)
            outs, infos = _world_step(engs, batches, G)
            exp = {}
            for o in range(G):
                order = [o] + [p for p in range(G) if p != o]
                mine = [batches[p][_owned_mask(batches[p], G, o)] for p in order]
                mine = np.ascontiguousarray(np.concatenate(mine))
                if not len(mine):
                    continue
                ev, _ = refs[o].ingest(mine)
                for rec, v in zip(mine, ev):
                    exp[bytes(rec["request_id"])] = _vkey(v)
                s = exp_stats[o]
                s["ingested"] += len(mine); s["stored"] += int((ev["flags"] & K.AGR_VF_STORED).astype(bool).sum())
                s["forwarded"] += int((ev["code"] == K.AGR_V_FORWARD).sum()); s["queued"] += int((ev["code"] == K.AGR_V_QUEUED).sum())
            for r in range(G):
                assert infos[r].n_local == int(_owned_mask(batches[r], G, r).sum())
                for q in range(G):
                    assert infos[r].sent_to[q] == (0 if q == r else int(_owned_mask(batches[r], G, q).sum()))
                for i, (rec, v) in enumerate(zip(batches[r], outs[r])):
                    assert _vkey(v) == exp[bytes(rec["request_id"])], (step, r, i)
                    o = A.agent_shard(rec["agent_id"].decode(), G)
                    if o != r and (v["flags"] & K.AGR_VF_STORED):
                        shipped.append((r, o, rec.copy()))
        for r, e in enumerate(engs):
            st = e.stats()
            for k, val in exp_stats[r].items():
                assert st[k] == val, (r, k, st[k], val)
            if not mint:                                          # a shipped record leaves no index entry at the shard it left
                assert int(e.debug_read("index_used", 0, 1)[0]) == st["stored"], r
        assert shipped
        if not mint:
            for r, o, rec in shipped[:40]:
                a, rid = rec["agent_id"].decode(), bytes(rec["request_id"])
                assert engs[r].get_record(a, rid) is None
                got = engs[o].get_record(a, rid)
                assert got is not None and got.tobytes()[96:] == rec.tobytes()[96:]
            # a later fresh record at the shard a record left, for a local agent, reusing the shipped id
            r, o, rec = shipped[0]
            fresh = make_rank_batch(r, G, own, 1, seed=99, p_cross_replay=0.0, first_index=90000)
            fresh["request_id"][0] = rec["request_id"]
            v, _ = engs[r].ingest(fresh)
            ev, _ = refs[r].ingest(fresh)
            assert _vkey(v[0]) == _vkey(ev[0])
        # completions at every owner (plain K2): then the per-agent lists agree with the reference
        for r, e in enumerate(engs):
            for a in own[r]:
                pe, pr = e.list(a, 0), refs[r].list(a, 0)
                assert len(pe) == len(pr)
                if not mint:
                    assert [bytes(x) for x in pe] == [bytes(x) for x in pr]
                take = list(range(0, len(pe), 3))
                for ids, tgt in ((pe, e), (pr, refs[r])):
                    arr = np.zeros(len(take), A.outcome_dtype)
                    for j, t in enumerate(take):
                        arr[j]["request_id"] = ids[t]; arr[j]["agent_id"] = a.encode()
                        arr[j]["kind"] = K.AGR_OUT_RESPONSE if t % 2 else K.AGR_OUT_ERROR; arr[j]["http_status"] = 200
                    if len(arr):
                        res = tgt.complete(arr)
                        assert list(res) == [0] * len(arr)
            for a in own[r]:
                for w in (0, 1, 2):
                    le, lr = e.list(a, w), refs[r].list(a, w)
                    assert len(le) == len(lr), (r, a, w)
                    if not mint:
                        assert [bytes(x) for x in le] == [bytes(x) for x in lr], (r, a, w)
    finally:
        for e in engs:
            e.close()
        for c in refs:
            c.close()


def test_same_batch_replay_is_known_at_the_owner():
    """Minted ids: a replay that names an earlier row of its own exchange batch is a dedupe hit decided inside K1 (the
    same-batch path), while rows shipped away in that batch are holes."""
    G = 2
    own = owned_agents(G, 2)
    flags = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS
    with A.Engine(slab_rows=1 << 12, max_batch=1024, flags=flags) as e:
        e.debug_world(0, G)
        for a in own[0] + own[1]:
            e.set_agent_state(a, "running")
        b = np.zeros(6, A.record_dtype)
        for i, a in enumerate([own[0][0], own[1][0], own[0][0], own[0][1], own[1][0], own[0][1]]):
            b[i]["agent_id"] = a.encode(); b[i]["seq"] = 1 + i; b[i]["request_id"][0] = 1 + i
        f = e.reserve_rows(6)
        ids = e.mint_ids(f, 6)
        b[2]["flags"] = K.AGR_F_REPLAY; b[2]["replay_of"] = ids[0]          # own target, same batch: KNOWN
        b[3]["flags"] = HOLE_BIT                                              # the caller's bit 31: still this shard's record
        b[5]["flags"] = K.AGR_F_REPLAY; b[5]["replay_of"] = ids[3]          # target carries bit 31: KNOWN all the same
        e.fill_rows(f, b)
        send, info = e.debug_exchange_begin(f, 6)
        assert info.n_sent == 2 and send.tobytes() == b[[1, 4]].tobytes()
        back = np.zeros(2, A.verdict_dtype); back["code"] = [7, 9]
        v = e.debug_exchange_end(back, 6)
        assert list(v["code"][[1, 4]]) == [7, 9]
        assert v[2]["flags"] & K.AGR_VF_KNOWN and v[5]["flags"] & K.AGR_VF_KNOWN
        assert v[0]["flags"] & K.AGR_VF_STORED and v[3]["flags"] & K.AGR_VF_STORED
        st = e.stats()
        assert st["ingested"] == 4 and st["stored"] == 2 and st["dedupe_hits"] == 2


# ------------------------------------------------------------------------------------------------ (c) the caller's bit 31
def test_caller_bit31_does_not_make_a_hole():
    """A record of this shard whose caller left flags bit 31 set, in an exchange batch that ships a record away, gets the
    verdict, stored state and bytes plain agr_ingest gives it."""
    G = 2
    own = owned_agents(G, 3)
    rng = np.random.default_rng(5)
    with A.Engine(slab_rows=1 << 12, max_batch=1024) as e, A.Engine(slab_rows=1 << 12, max_batch=1024) as twin:
        e.debug_world(0, G)
        for a in own[0] + own[1]:
            e.set_agent_state(a, "running"); twin.set_agent_state(a, "running")
        b = A.synth_fill_host(0, 64, seed=3, n_agents=4)
        ag = [own[0][i % 3] for i in range(64)]
        ag[5] = ag[40] = own[1][0]                                # two records for the peer
        b["agent_id"] = [a.encode() for a in ag]
        b["flags"][rng.random(64) < 0.5] |= HOLE_BIT
        b["flags"][7] = HOLE_BIT | K.AGR_F_REPLAY; b["replay_of"][7] = b["request_id"][3]
        f = e.reserve_rows(64)
        e.fill_rows(f, b)
        send, info = e.debug_exchange_begin(f, 64)
        assert info.n_sent == 2 and send.tobytes() == b[[5, 40]].tobytes()
        v = e.debug_exchange_end(np.zeros(2, A.verdict_dtype), 64)
        mine = np.ones(64, bool); mine[[5, 40]] = False
        tv, _ = twin.ingest(np.ascontiguousarray(b[mine]))
        assert v[mine].tobytes() == tv.tobytes()
        se, st = e.stats(), twin.stats()
        for k in ("ingested", "stored", "forwarded", "queued", "dup_ids", "replay_flagged", "dedupe_hits"):
            assert se[k] == st[k], k
        for rec in b[mine]:
            a, rid = rec["agent_id"].decode(), bytes(rec["request_id"])
            ge, gt = e.get_record(a, rid), twin.get_record(a, rid)
            assert (ge is None) == (gt is None)
            if ge is not None:
                assert ge.tobytes() == gt.tobytes() and int(ge["flags"]) == int(rec["flags"])
        for a in own[0]:
            assert [bytes(x) for x in e.list(a, 0)] == [bytes(x) for x in twin.list(a, 0)]


# ------------------------------------------------------------------------------------------------ (d) NCCL at world = 1
def test_nccl_world_of_one_matches_plain_ingest():
    try:
        ctypes.CDLL("libnccl.so.2")
    except OSError as ex:
        pytest.skip(f"libnccl.so.2 cannot be loaded: {ex}")
    own = owned_agents(1, 8)
    with A.Engine(slab_rows=1 << 14, max_batch=4096) as e, A.Engine(slab_rows=1 << 14, max_batch=4096) as twin:
        e.comm_init(A.comm_unique_id(), 0, 1)
        for a in own[0]:
            s = "running" if int(a[-1]) % 3 else "stopped"
            e.set_agent_state(a, s); twin.set_agent_state(a, s)
        b1 = make_rank_batch(0, 1, own, 1500, seed=4)
        b1["flags"][::7] |= HOLE_BIT
        v, info = e.ingest_sharded(b1)
        tv, _ = twin.ingest(b1)
        assert v.tobytes() == tv.tobytes()
        assert (info.world, info.rank, info.n_local, info.n_sent, info.n_received) == (1, 0, 1500, 0, 0)
        b2 = make_rank_batch(0, 1, own, 900, seed=5, first_index=5000)
        b2["flags"][1::5] |= HOLE_BIT
        f = e.reserve_rows(900)
        e.fill_rows(f, b2)
        v, info = e.ingest_sharded_rows(f, 900, want_verdicts=True)
        tv, _ = twin.ingest(b2)
        assert v.tobytes() == tv.tobytes() and info.first_rid == f and info.n_local == 900
        outs = []
        for a in own[0]:
            for j, rid in enumerate(twin.list(a, 0)[:30]):
                outs.append((bytes(rid), a, K.AGR_OUT_RESPONSE if j % 3 else K.AGR_OUT_ERROR))
        outs.append((bytes(range(16)), own[0][0], K.AGR_OUT_RESPONSE))
        arr = np.zeros(len(outs), A.outcome_dtype)
        for j, (rid, a, kind) in enumerate(outs):
            arr[j]["request_id"] = np.frombuffer(rid, np.uint8); arr[j]["agent_id"] = a.encode(); arr[j]["kind"] = kind
            arr[j]["http_status"] = 200
        res, cinfo = e.complete_sharded(arr)
        tres = twin.complete(arr)
        assert list(res) == list(tres) and tres[-1] == K.AGR_ENOTFOUND and cinfo.n_local == len(arr) and cinfo.n_sent == 0
        for a in own[0]:
            for w in (0, 1, 2):
                assert [bytes(x) for x in e.list(a, w)] == [bytes(x) for x in twin.list(a, w)]
        se, st = e.stats(), twin.stats()
        for k in ("ingested", "stored", "forwarded", "queued", "completions", "failures", "dedupe_hits"):
            assert se[k] == st[k], k
