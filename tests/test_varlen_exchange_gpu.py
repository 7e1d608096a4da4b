"""The resident batch path and the multi-GPU exchange on variable-length engines (AGR_CFG_VARLEN).  A row that agr_reserve_rows
or the exchange hands out there owns a 512-byte slot of the byte ring, and K1v decides the slot as a variable-length record of
stored length 512.  (1) reserve_rows + fill_rows + ingest_rows against a twin fed agr_ingest_var with the same 512-byte blob,
and the JSON views against a twin fed the compact form.  (2) The byte ring: skips, a row range across a skip, refusals, pins
of an online snapshot, reclaim next to reserved rows, synth_fill_rows.  (3) G engines on one device running the exchange's
stages (agr_debug_exchange_begin / _end), against oracle/cpu_ref.c per owner.  (4) NCCL at world 1.  (5) Snapshots and
restores.  (6) Two GPUs."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.sharding import make_rank_batch, owned_agents
from oracle.cpu_ref import CRef
from slotref import SLOT, slot_layout

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
MODES = {"hash": P | V, "mint": P | V | M, "hash_ring": P | V | R, "mint_ring": P | V | M | R}
SECRET = 0x5EED_0000_C5C5_0001
NS = [0, 1, 31, 32, 33, 1000, 2049]
STAT_KEYS = ("rows_used", "rows_tail", "ingested", "stored", "replay_flagged", "dedupe_hits", "forwarded", "queued",
             "unavailable", "not_found", "dup_ids", "malformed")
AGENTS = [A.synth_agent_id(k) for k in range(8)]
STATUS = {a: ("stopped" if k % 3 == 2 else "running") for k, a in enumerate(AGENTS)}


def engine(flags, **kw):
    kw.setdefault("slab_rows", 1 << 14)
    kw.setdefault("max_agents", 64)
    kw.setdefault("max_batch", 4096)
    kw.setdefault("vslab_bytes", 16 << 20)
    kw.setdefault("id_secret", SECRET)
    return A.Engine(flags=flags, **kw)


def register(engs, agents=AGENTS, status=STATUS):
    for e in engs:
        for a in agents:
            e.set_agent_state(a, status[a])


def blob512(recs):
    n = len(recs)
    return np.ascontiguousarray(recs).view(np.uint8).reshape(-1).copy(), (np.arange(n + 1, dtype=np.uint32) * SLOT)


def compact(recs):
    """the same records in the compact variable-length form: 96 B header + payload rounded up to 16 B (a payload longer than
    the fixed form holds keeps the whole 512 B record, so that both forms refuse it alike)"""
    parts, offs = [], [0]
    for r in recs:
        pl = int(r["path_len"]) + int(r["hdr_len"]) + int(r["body_len"])
        ln = SLOT if pl > 416 else 96 + ((pl + 15) & ~15)
        parts.append(np.frombuffer(r.tobytes()[:ln], np.uint8))
        offs.append(offs[-1] + ln)
    blob = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return np.ascontiguousarray(blob), np.array(offs, dtype=np.uint32)


def make_batch(rng, n, first_index, minted, earlier, seed):
    """n records of AGENTS: ~4 % with a payload of exactly 416 B, ~4 % with 417 B, ~12 % replay-flagged records naming an earlier
    record of the same batch or of an earlier one (`earlier`: (agent, id) pairs).  minted: the ids the rows will have (minted-id
    engines), or None (the records' own request ids)."""
    b = A.synth_fill_host(first_index, n, seed=seed, n_agents=len(AGENTS))
    ids_of = (lambda j: minted[j]) if minted is not None else (lambda j: b["request_id"][j].copy())
    for i in range(n):
        u = rng.random()
        if u < 0.04:
            b[i]["path_len"], b[i]["hdr_len"], b[i]["body_len"] = 16, 0, 400
        elif u < 0.08:
            b[i]["path_len"], b[i]["hdr_len"], b[i]["body_len"] = 16, 0, 401
        if rng.random() < 0.12 and (i > 0 or earlier):
            if i > 0 and (not earlier or rng.random() < 0.5):
                j = int(rng.integers(0, i))
                a, tid = b[j]["agent_id"], ids_of(j)
            else:
                a, tid = earlier[int(rng.integers(0, len(earlier)))]
            b[i]["flags"] |= K.AGR_F_REPLAY
            b[i]["replay_of"] = np.frombuffer(bytes(tid), np.uint8)
            b[i]["agent_id"] = a
    return b


def assert_same_state(e, twin, ids, first=0):
    """stats, the per-agent lists, every row's words and every stored record's bytes, and agr_verify"""
    se, st = e.stats(), twin.stats()
    for k in STAT_KEYS:
        assert se[k] == st[k], (k, se[k], st[k])
    for a in AGENTS:
        assert [bytes(x) for x in e.list(a, 0)] == [bytes(x) for x in twin.list(a, 0)], a
    n = se["rows_used"] - first
    if n:
        for w in ("state", "route", "aux", "cksum", "verdict"):
            assert e.debug_read(w, first, n).tobytes() == twin.debug_read(w, first, n).tobytes(), w
    for a, rid in ids:
        ge, gt = e.get_record_var(a, rid), twin.get_record_var(a, rid)
        assert (ge is None) == (gt is None)
        if ge is not None:
            assert ge.tobytes() == gt.tobytes() and len(ge) == SLOT
    assert e.verify()[1] == 0


# ------------------------------------------------------------------------------------------ (1) resident path = agr_ingest_var
@pytest.mark.parametrize("mode", sorted(MODES))
def test_resident_path_equals_ingest_var(mode):
    flags = MODES[mode]
    mint = bool(flags & M)
    rng = np.random.default_rng(11 + flags)
    with engine(flags) as e, engine(flags) as twin, engine(flags) as ctwin:
        register([e, twin, ctwin])
        earlier, stored_ids, idx = [], [], 0
        for step, n in enumerate(NS):
            f = e.reserve_rows(n)
            minted = e.mint_ids(f, n) if mint else None
            b = make_batch(rng, n, idx, minted, earlier, seed=5 + step)
            idx += n
            e.fill_rows(f, b)
            if n == 1000:                                             # the asynchronous form: verdicts from the row words
                e.ingest_rows_async(f, n)
                e.sync()
                v = e.debug_read("verdict", f, n)
            else:
                v = e.ingest_rows(f, n)
            tv, tids, tf = twin.ingest_var(*blob512(b))
            cv, cids, cf = ctwin.ingest_var(*compact(b))
            assert tf == f and cf == f
            assert v.tobytes() == tv.tobytes() == cv.tobytes(), step
            if mint:
                assert e.mint_ids(f, n).tobytes() == tids.tobytes() == cids.tobytes()
            if n:
                assert int((tv["flags"] & K.AGR_VF_BAD_LEN).astype(bool).sum()) > 0 or n < 100
            ids = tids if mint else b["request_id"]
            for i in range(n):
                earlier.append((b[i]["agent_id"], bytes(ids[i])))
                stored_ids.append((b[i]["agent_id"].decode(), bytes(ids[i])))
        assert e.stats()["dedupe_hits"] > 0 and e.stats()["malformed"] > 0
        assert_same_state(e, twin, stored_ids)
        # the JSON views read a slot as the compact record it holds
        for a, rid in stored_ids:
            assert e.get_record_json(a, rid) == ctwin.get_record_json(a, rid)
        for a in AGENTS:
            assert e.pending_json(a) == ctwin.pending_json(a)
        used = e.stats()["rows_used"]
        (je, oe), (jc, oc) = e.rows_json(0, used, as_array=True), ctwin.rows_json(0, used, as_array=True)
        assert je == jc and oe.tobytes() == oc.tobytes()
        # the replay scan returns a slot as a 512-byte record
        d, blob, offs = e.replay_scan_var()
        td, tblob, toffs = twin.replay_scan_var()
        assert d.tobytes() == td.tobytes() and blob.tobytes() == tblob.tobytes() and offs.tobytes() == toffs.tobytes()


# ------------------------------------------------------------------------------------------ (2) the byte ring
def ring_engine(flags, slots=128, **kw):
    return engine(flags | R, slab_rows=4096, vslab_bytes=slots * SLOT, max_batch=2048, **kw)


def plain_batch(n, first_index, seed, created=1):
    b = A.synth_fill_host(first_index, n, seed=seed, n_agents=len(AGENTS))
    b["seq"] = created                                               # (seq is the record's created_at: what agr_expire reads)
    return b


def _code(fn):
    try:
        fn()
        return 0
    except A.AgrError as ex:
        return ex.code


@pytest.mark.parametrize("mint", [False, True], ids=["hash", "mint"])
def test_reservations_meet_the_end_of_the_byte_ring(mint):
    """Reservations take their slots where tests/slotref.py says (skip at the end of the lap, never a wrap), and what K1v
    decides there equals agr_ingest_var of the same blob at the same place."""
    flags = P | V | (M if mint else 0)
    ops = [("reserve", 40), ("reserve", 40), ("reserve", 40), ("release_all",), ("reserve", 40), ("reserve", 30),
           ("release_all",), ("reserve", 64), ("reserve", 65), ("reserve", 64), ("reserve", 1), ("release_all",), ("reserve", 17)]
    want = slot_layout(128 * SLOT, True, ops)
    with ring_engine(flags) as e, ring_engine(flags) as twin:
        register([e, twin])
        base, idx, t, ids = None, 0, 0, []
        for op, w in zip(ops, want):
            if op[0] == "release_all":
                t += 10 ** 12
                for x in (e, twin):
                    x.expire(t, 1)
                    x.reclaim()
                continue
            n = op[1]
            if isinstance(w, str):
                code = _code(lambda: e.reserve_rows(n))
                assert code == (K.AGR_ENOSPC if w == "ENOSPC" else K.AGR_EINVAL), op
                assert _code(lambda: twin.ingest_var(*blob512(plain_batch(n, 0, 1)))) == code
                continue
            f = e.reserve_rows(n)
            p = e.slab_ptr(f)
            assert p and e.slab_ptr(f + n - 1) == p + (n - 1) * SLOT
            base = p if base is None else base
            assert p - base == w, op
            b = plain_batch(n, idx, 7 + idx, created=t + 1)
            idx += n
            e.fill_rows(f, b)
            v = e.ingest_rows(f, n)
            tv, tids, tf = twin.ingest_var(*blob512(b))
            assert tf == f and v.tobytes() == tv.tobytes()
            got = tids if mint else b["request_id"]
            ids += [(b[i]["agent_id"].decode(), bytes(got[i])) for i in range(n)]
        assert_same_state(e, twin, ids, first=e.stats()["rows_tail"])


@pytest.mark.parametrize("mint", [False, True], ids=["hash", "mint"])
def test_range_across_a_skip_is_decided_as_its_reservations(mint):
    flags = P | V | (M if mint else 0)
    with ring_engine(flags) as e, ring_engine(flags) as twin:
        register([e, twin])
        for x in (e, twin):                                          # the cursor 100 slots into the lap, all released
            x.ingest_var(*blob512(plain_batch(50, 0, 1)))
            x.ingest_var(*blob512(plain_batch(50, 50, 2)))
            x.expire(10 ** 18, 1)
            x.reclaim()
        f1 = e.reserve_rows(20)                                      # slots 100..120
        f2 = e.reserve_rows(30)                                      # 8 slots skipped: slots 0..30
        assert f2 == f1 + 20 and e.slab_ptr(f2) < e.slab_ptr(f1)
        ids1 = e.mint_ids(f1, 50) if mint else None
        b = plain_batch(50, 100, 3)
        if not mint:
            ids1 = b["request_id"]
        for i, j in ((25, 3), (40, 10), (45, 30)):                   # replays across the skip and on either side of it
            b[i]["flags"] |= K.AGR_F_REPLAY
            b[i]["replay_of"] = ids1[j]
            b[i]["agent_id"] = b[j]["agent_id"]
        e.fill_rows(f1, b)                                           # one call across the skip
        # the exchange needs the batch's slots back to back
        e.debug_world(0, 2)
        assert _code(lambda: e.debug_exchange_begin(f1, 50)) == K.AGR_EINVAL
        v = e.ingest_rows(f1, 50)
        tv1, tid1, _ = twin.ingest_var(*blob512(b[:20]))
        tv2, tid2, _ = twin.ingest_var(*blob512(b[20:]))
        assert v.tobytes() == np.concatenate([tv1, tv2]).tobytes()
        assert e.stats()["dedupe_hits"] == twin.stats()["dedupe_hits"] > 0
        ids = np.concatenate([tid1, tid2]) if mint else b["request_id"]
        assert_same_state(e, twin, [(b[i]["agent_id"].decode(), bytes(ids[i])) for i in range(50)], first=f1)


@pytest.mark.parametrize("ring", [False, True], ids=["append", "ring"])
def test_full_byte_slab_refuses_and_changes_nothing(ring):
    flags = P | V | M | (R if ring else 0)
    with engine(flags, slab_rows=4096, vslab_bytes=128 * SLOT, max_batch=2048) as e:
        register([e])
        if ring:
            assert _code(lambda: e.reserve_rows(65)) == K.AGR_EINVAL
            f = e.reserve_rows(64)
            e.reserve_rows(64)
        else:
            f = e.reserve_rows(100)
            e.reserve_rows(28)
        used = e.stats()["rows_used"]
        assert _code(lambda: e.reserve_rows(1)) == K.AGR_ENOSPC
        assert e.stats()["rows_used"] == used                       # the refused call reserved no rows either
        e.fill_rows(f, plain_batch(used, 0, 4))
        e.ingest_rows(f, used)
        assert e.verify()[1] == 0 and e.stats()["stored"] > 0


def test_online_snapshot_pins_hold_the_slots(tmp_path):
    from test_snapshot_online_gpu import PipeSnapshot, while_writing, _attempt

    def batch(seed, created=1):                                      # 62 slots: 31744 B, under half the 64 KiB ring
        return plain_batch(62, seed * 100, seed, created)

    def resident(eng, b):
        f = eng.reserve_rows(len(b))
        eng.fill_rows(f, b)
        eng.ingest_rows(f, len(b))

    def make(online):
        eng = ring_engine(P | V | M | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0), slots=128)
        register([eng])
        for rnd in range(12):                                        # the byte ring goes round several times
            eng.expire(10 ** 12 * (rnd + 1), 1)
            eng.reclaim()
            resident(eng, batch(30 + rnd, 10 ** 12 * (rnd + 1) + 1))
        return eng

    def steps(eng):                                                  # everything released, then two more batches
        eng.expire(10 ** 15, 1)
        eng.reclaim()
        return [_attempt(lambda k=k: resident(eng, batch(60 + k))) for k in range(2)]

    with make(False) as ctl:
        assert [c for c, _ in steps(ctl)] == [0, 0]
    with make(True) as eng:
        snap = PipeSnapshot(eng, tmp_path)
        got = while_writing(snap, lambda: steps(eng))
        assert [c for c, _ in got] == [0, K.AGR_ENOSPC] and "byte slab" in got[1][1] and "snapshot" in got[1][1], got
        snap.drain()
        resident(eng, batch(62))
        assert eng.verify()[1] == 0


@pytest.mark.parametrize("use_async", [False, True], ids=["reclaim", "reclaim_async"])
def test_reclaim_never_releases_a_reserved_slot(use_async):
    flags = P | V | M
    with ring_engine(flags) as e:
        register([e])
        a = plain_batch(40, 0, 1)
        fa = e.reserve_rows(40)
        e.fill_rows(fa, a)
        e.ingest_rows(fa, 40)                                        # slots 0..40, decided
        b = plain_batch(40, 40, 2)
        fb = e.reserve_rows(40)                                      # slots 40..80, filled, not decided
        e.fill_rows(fb, b)
        e.expire(10 ** 18, 1)
        released = 0
        for _ in range(2):
            released += e.reclaim_async() if use_async else e.reclaim()
        assert released == 40
        # were the tail past fb's slots, 60 slots would fit at the start of the lap, on top of them
        assert _code(lambda: e.reserve_rows(60)) == K.AGR_ENOSPC
        vb = e.ingest_rows(fb, 40)
        ids = e.mint_ids(fb, 40)
        assert (vb["flags"] & K.AGR_VF_STORED).any()
        for i in np.nonzero(vb["flags"] & K.AGR_VF_STORED)[0]:               # the slots kept what fill_rows put there
            got = e.get_record_var(b[i]["agent_id"].decode(), bytes(ids[i])).tobytes()
            assert got[96:] == b[i].tobytes()[96:] and got[16:80] == b[i].tobytes()[16:80]
        assert e.verify()[1] == 0
        e.expire(10 ** 18, 1)
        e.reclaim()
        e.reclaim()
        assert e.reserve_rows(60) == fb + 40


@pytest.mark.parametrize("mint", [False, True], ids=["hash", "mint"])
def test_synth_fill_rows_into_slots(mint):
    flags = P | V | (M if mint else 0)
    with ring_engine(flags) as e, ring_engine(flags) as twin:
        register([e, twin])
        for x in (e, twin):
            x.ingest_var(*blob512(plain_batch(60, 0, 1)))
            x.ingest_var(*blob512(plain_batch(50, 0, 2)))
            x.expire(10 ** 18, 1)
            x.reclaim()
        fe = [e.reserve_rows(10), e.reserve_rows(40)]               # the second skips to the start of the lap
        ft = [twin.reserve_rows(10), twin.reserve_rows(40)]
        assert fe == ft
        e.synth_fill_rows(1234, fe[0], 50, seed=9, n_agents=len(AGENTS))
        twin.fill_rows(ft[0], A.synth_fill_host(1234, 50, seed=9, n_agents=len(AGENTS)))
        assert e.ingest_rows(fe[0], 50).tobytes() == twin.ingest_rows(ft[0], 50).tobytes()
        b = A.synth_fill_host(1234, 50, seed=9, n_agents=len(AGENTS))
        ids = e.mint_ids(fe[0], 50) if mint else b["request_id"]
        assert_same_state(e, twin, [(b[i]["agent_id"].decode(), bytes(ids[i])) for i in range(50)], first=fe[0])


# ------------------------------------------------------------------------------------------ (3) simulated worlds
def _vkey(v):
    return int(v["code"]), int(v["flags"])


def _split_send(send, info, G, me):
    out, o = {}, 0
    for q in range(G):
        if q != me and info.sent_to[q]:
            out[q] = send[o: o + info.sent_to[q]]
            o += info.sent_to[q]
    assert o == len(send)
    return out


def _world_step(engs, batches, G):
    """one exchange step: every rank's batch through its slots and the exchange's stages, the received records decided at
    their owner through reserve_rows + fill_rows + ingest_rows (the resident path)"""
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
    for o, e in enumerate(engs):
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


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("G", [2, 3, 5])
def test_simulated_world_against_cref(G, mode):
    flags = MODES[mode]
    mint = bool(flags & M)
    own = owned_agents(G, 6)
    everyone = [a for o in own for a in o]
    status = {a: ("running" if int(a[-1]) % 3 else "stopped") for a in everyone}
    engs = [engine(flags, max_agents=256) for _ in range(G)]
    refs = [CRef() for _ in range(G)]
    try:
        for r, e in enumerate(engs):
            e.debug_world(r, G)
            register([e], everyone, status)                          # every agent on every shard: holes must stay unlisted
            for a in own[r]:
                refs[r].set_agent_state(a, status[a])
        exp_stats = [dict(ingested=0, stored=0, forwarded=0, queued=0) for _ in range(G)]
        shipped = []
        for step, n in enumerate((700, 1, 0, 1500)):
            batches = []
            for r in range(G):
                nr = n if (n != 1 or r == 0) else 0
                b = make_rank_batch(r, G, own, nr, seed=41 + step, p_cross_replay=0.05, p_missteer=0.08, first_index=step * 10000) \
                    if nr else np.zeros(0, A.record_dtype)
                batches.append(b)
            outs, infos = _world_step(engs, batches, G)
            exp = {}
            for o in range(G):
                order = [o] + [p for p in range(G) if p != o]
                mine = np.ascontiguousarray(np.concatenate([batches[p][_owned_mask(batches[p], G, o)] for p in order]))
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
                for i, (rec, v) in enumerate(zip(batches[r], outs[r])):
                    assert _vkey(v) == exp[bytes(rec["request_id"])], (step, r, i)
                    o = A.agent_shard(rec["agent_id"].decode(), G)
                    if o != r and (v["flags"] & K.AGR_VF_STORED):
                        shipped.append((r, o, rec.copy()))
        for r, e in enumerate(engs):
            st = e.stats()
            for k, val in exp_stats[r].items():
                assert st[k] == val, (r, k, st[k], val)
            for q in range(G):                                       # the holes at this shard: nothing listed for peers' agents
                if q != r:
                    for a in own[q]:
                        assert len(e.list(a, 0)) == 0, (r, a)
            assert e.verify()[1] == 0
            if not mint:
                assert int(e.debug_read("index_used", 0, 1)[0]) == st["stored"], r
        assert shipped
        if not mint:
            for r, o, rec in shipped[:40]:
                a, rid = rec["agent_id"].decode(), bytes(rec["request_id"])
                assert engs[r].get_record_var(a, rid) is None
                got = engs[o].get_record_var(a, rid)
                assert got is not None and got.tobytes()[96:] == rec.tobytes()[96:]
        for r, e in enumerate(engs):
            for a in own[r]:
                pe, pr = e.list(a, 0), refs[r].list(a, 0)
                assert len(pe) == len(pr)
                if not mint:
                    assert [bytes(x) for x in pe] == [bytes(x) for x in pr]
    finally:
        for e in engs:
            e.close()
        for c in refs:
            c.close()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_same_batch_replay_is_known_at_the_owner(mode):
    flags = MODES[mode]
    mint = bool(flags & M)
    G = 2
    own = owned_agents(G, 2)
    with engine(flags) as e:
        e.debug_world(0, G)
        for a in own[0] + own[1]:
            e.set_agent_state(a, "running")
        b = np.zeros(6, A.record_dtype)
        for i, a in enumerate([own[0][0], own[1][0], own[0][0], own[0][1], own[1][0], own[0][1]]):
            b[i]["agent_id"] = a.encode(); b[i]["seq"] = 1 + i; b[i]["request_id"][0] = 1 + i
        f = e.reserve_rows(6)
        ids = e.mint_ids(f, 6) if mint else b["request_id"].copy()
        b[2]["flags"] = K.AGR_F_REPLAY; b[2]["replay_of"] = ids[0]
        b[5]["flags"] = K.AGR_F_REPLAY; b[5]["replay_of"] = ids[3]
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
        assert len(e.list(own[1][0], 0)) == 0                        # the holes are neither stored nor listed here
        assert e.verify()[1] == 0


# ------------------------------------------------------------------------------------------ (4) NCCL at world = 1
@pytest.mark.parametrize("mode", sorted(MODES))
def test_nccl_world_of_one_matches_ingest_var(mode):
    try:
        ctypes.CDLL("libnccl.so.2")
    except OSError as ex:
        pytest.skip(f"libnccl.so.2 cannot be loaded: {ex}")
    flags = MODES[mode]
    mint = bool(flags & M)
    own = owned_agents(1, 8)
    status = {a: ("running" if int(a[-1]) % 3 else "stopped") for a in own[0]}
    with engine(flags) as e, engine(flags) as twin:
        e.comm_init(A.comm_unique_id(), 0, 1)
        register([e, twin], own[0], status)
        ids = []
        b1 = make_rank_batch(0, 1, own, 1500, seed=4)
        v, info = e.ingest_sharded(b1)
        tv, tid1, _ = twin.ingest_var(*blob512(b1))
        assert v.tobytes() == tv.tobytes()
        assert (info.world, info.rank, info.n_local, info.n_sent, info.n_received) == (1, 0, 1500, 0, 0)
        ids += list(zip(b1["agent_id"], tid1 if mint else b1["request_id"]))
        b2 = make_rank_batch(0, 1, own, 900, seed=5, first_index=5000)
        f = e.reserve_rows(900)
        e.fill_rows(f, b2)
        v, info = e.ingest_sharded_rows(f, 900, want_verdicts=True)
        tv, tid2, tf = twin.ingest_var(*blob512(b2))
        assert v.tobytes() == tv.tobytes() and info.first_rid == f == tf and info.n_local == 900
        ids += list(zip(b2["agent_id"], tid2 if mint else b2["request_id"]))
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
        for k in STAT_KEYS + ("completions", "failures"):
            assert se[k] == st[k], k
        for a, rid in ids[::7]:
            ge, gt = e.get_record_var(a.decode(), bytes(rid)), twin.get_record_var(a.decode(), bytes(rid))
            assert (ge is None) == (gt is None) and (ge is None or ge.tobytes() == gt.tobytes())
        assert e.verify()[1] == 0


# ------------------------------------------------------------------------------------------ (5) durability
SNAP_KINDS = {"blocking": 0, "online": K.AGR_CFG_ONLINE_SNAPSHOT, "delta": K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT}


def _traffic(e, own, step, ids):
    """one step of every path: a batch through the exchange's stages (peer records shipped, their verdicts made up), a batch
    through the resident path, and a compact blob through agr_ingest_var"""
    b = make_rank_batch(0, 2, own, 300, seed=70 + step, p_cross_replay=0.05, p_missteer=0.05, first_index=step * 10000)
    f = e.reserve_rows(len(b))
    e.fill_rows(f, b)
    send, info = e.debug_exchange_begin(f, len(b))
    v = e.debug_exchange_end(np.zeros(info.n_sent, A.verdict_dtype), len(b))
    mine = _owned_mask(b, 2, 0)
    minted = e.mint_ids(f, len(b)) if e.mint else b["request_id"]
    ids += [(b[i]["agent_id"].decode(), bytes(minted[i])) for i in np.nonzero(mine)[0]]
    c = make_rank_batch(0, 2, own, 200, seed=80 + step, p_cross_replay=0.0, first_index=step * 10000 + 5000)
    f = e.reserve_rows(len(c))
    e.fill_rows(f, c)
    e.ingest_rows(f, len(c))
    minted = e.mint_ids(f, len(c)) if e.mint else c["request_id"]
    ids += [(c[i]["agent_id"].decode(), bytes(minted[i])) for i in range(len(c))]
    d = make_rank_batch(0, 2, own, 100, seed=90 + step, p_cross_replay=0.0, first_index=step * 10000 + 8000)
    _, did, _ = e.ingest_var(*compact(d))
    ids += [(d[i]["agent_id"].decode(), bytes(did[i] if e.mint else d[i]["request_id"])) for i in range(len(d))]


def _same_engine(back, src, ids):
    sb, ss = back.stats(), src.stats()
    for k in ("rows_used", "rows_tail"):                             # (the event counters are not part of a snapshot)
        assert sb[k] == ss[k], k
    for a, rid in ids:
        gb, gs = back.get_record_var(a, rid), src.get_record_var(a, rid)
        assert (gb is None) == (gs is None) and (gb is None or gb.tobytes() == gs.tobytes())
    for a in sorted({a for a, _ in ids}):
        assert [bytes(x) for x in back.list(a, 0)] == [bytes(x) for x in src.list(a, 0)], a
    assert back.verify()[1] == 0


@pytest.mark.parametrize("kind", sorted(SNAP_KINDS))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_snapshots_restore_in_place_and_relocated(mode, kind, tmp_path):
    flags = MODES[mode]
    own = owned_agents(2, 6)
    everyone = own[0] + own[1]
    status = {a: ("running" if int(a[-1]) % 3 else "stopped") for a in everyone}
    kw = dict(slab_rows=1 << 13, vslab_bytes=4 << 20, max_batch=1024)
    moved = dict(slab_rows=1 << 14, vslab_bytes=6 << 20, max_batch=1024)
    with engine(flags | SNAP_KINDS[kind], **kw) as e:
        e.debug_world(0, 2)
        register([e], everyone, status)
        ids = []
        paths = []
        for step in range(3 if kind == "delta" else 1):
            _traffic(e, own, step, ids)
            paths.append(str(tmp_path / f"s{step}.snap"))
            e.snapshot(paths[-1])
        assert e.verify()[1] == 0
        for where in (kw, moved):
            with engine(flags, restore_from=paths[-1], **where) as back:
                _same_engine(back, e, ids)
                # the restored engine goes on taking slots
                f = back.reserve_rows(10)
                back.fill_rows(f, make_rank_batch(0, 2, own, 10, seed=99, p_cross_replay=0.0, first_index=90000))
                back.ingest_rows(f, 10)
                assert back.verify()[1] == 0


# ------------------------------------------------------------------------------------------ (6) two GPUs
def _worker(rank, world, port, q):
    sys.path.insert(0, HERE); sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    import agentainer_lab_b200 as A
    from agentainer_lab_b200 import constants as K
    from agentainer_lab_b200.sharding import make_rank_batch, owned_agents
    from oracle.cpu_ref import CRef
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    uid = [A.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    own = owned_agents(world, 8)
    status = lambda a: "running" if int(a[-1]) % 3 else "stopped"
    eng = A.Engine(device=rank, slab_rows=1 << 16, max_agents=64, max_batch=1 << 13, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN,
                   vslab_bytes=64 << 20)
    eng.comm_init(uid[0], rank, world)
    ref = CRef()
    for a in own[rank]:
        eng.set_agent_state(a, status(a)); ref.set_agent_state(a, status(a))
    ok = True
    for step, n in enumerate((3000, 1, 0, 5000)):
        n_here = n if (n != 1 or rank == 0) else 0
        batch = make_rank_batch(rank, world, own, n_here, seed=21 + step, p_cross_replay=0.05, first_index=step * 10000) \
            if n_here else np.zeros(0, dtype=A.record_dtype)
        if step % 2:
            v, info = eng.ingest_sharded(batch)
        else:
            f = eng.reserve_rows(n_here) if n_here else eng.stats()["rows_used"]
            if n_here:
                eng.fill_rows(f, batch)
            v, info = eng.ingest_sharded_rows(f, n_here, want_verdicts=True)
        allb = [None] * world
        dist.all_gather_object(allb, batch.tobytes())
        batches = [np.frombuffer(x, dtype=A.record_dtype) for x in allb]
        order = [rank] + [p for p in range(world) if p != rank]
        mine = [x[np.array([A.agent_shard(a.decode(), world) == rank for a in x["agent_id"]], dtype=bool)] if len(x) else x
                for x in (batches[p] for p in order)]
        mine = np.ascontiguousarray(np.concatenate(mine)) if sum(len(m) for m in mine) else np.zeros(0, dtype=A.record_dtype)
        ev, _ = ref.ingest(mine) if len(mine) else (np.zeros(0, dtype=A.verdict_dtype), 0)
        ok &= info.n_local + info.n_sent == n_here and info.n_received == len(mine) - info.n_local
        alle = [None] * world
        dist.all_gather_object(alle, (mine["request_id"].tobytes(), ev["code"].tobytes(), ev["flags"].tobytes()))
        exp = {}
        for rids, codes, fl in alle:
            r_ = np.frombuffer(rids, np.uint8).reshape(-1, 16)
            for k in range(len(r_)):
                exp[r_[k].tobytes()] = (codes[k], fl[k])
        for rec, vv in zip(batch, v if v is not None else []):
            ok &= exp[bytes(rec["request_id"])] == (int(vv["code"]), int(vv["flags"]))
    for a in own[rank]:
        for w in (0, 1, 2):
            ok &= [bytes(x) for x in eng.list(a, w)] == [bytes(x) for x in ref.list(a, w)]
    ok &= eng.verify()[1] == 0
    st = eng.stats()
    q.put((rank, bool(ok), st["k4_launches"], st["stored"]))
    dist.barrier()
    dist.destroy_process_group()
    eng.close(); ref.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_varlen_exchange_two_gpus():
    import torch.multiprocessing as mp
    world, port = 2, 29561
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, k4, stored in res:
        assert ok, f"rank {rank}: the variable-length exchange differs from the oracle"
        assert k4 > 0 and stored > 0
