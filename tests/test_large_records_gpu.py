"""Variable-length records longer than AGR_VAR_MAX_RECORD (LONG records, up to agr_config.max_record_bytes), on the device,
against plain references: decisions against a fixed-stride twin fed k1vref.twin_records (pinned to oracle/model.py by
test_parity_gpu.py), checksums against tests/verifyref.py / k1vref.cksum and tests/longref.py, voff / vlen and slab bytes
from snapshot files (tests/snapfile.py), the wire form against oracle/gojson.py (through tests/k5ref.py).

  - K1v in both forms, both id modes, append-only and ring, with long records at the tile edges where K1v changes path;
  - agr_verify on corruption at a long record's first chunk, both sides of an 8 KiB piece boundary and its last chunk;
  - agr_rows_json / agr_get_record_json / agr_pending_json of long records;
  - snapshots (blocking, online, delta) restored in place, relocated, into an engine with the default limit, and the
    refused conversion to 512-byte rows;
  - the byte ring's wrap, AGR_ENOSPC and expire + reclaim with long records;
  - the single-request front end: long tickets refused, long agr_ingest_var(n = 1) next to ticket callers;
  - one long record across byte 2^32 of the byte slab."""
import hashlib
import os
import tempfile
import threading
from dataclasses import dataclass

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1vref as kr
import k5ref
import longref as L
import snapfile
import test_hbm_far_gpu as HF
import test_k1v_tiles_gpu as T
import test_k5_edges_gpu as T5
import verifyref as VR
from agentainer_lab_b200 import constants as K

pytestmark = pytest.mark.gpu

MB = 1 << 20
MAXREC = MB + 4096                       # the engines' max_record_bytes in most cases
P, V, R, CB, M = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_VARLEN, K.AGR_CFG_RING, K.AGR_CFG_COMBINE, K.AGR_CFG_MINT_IDS
ON, DELTA = K.AGR_CFG_ONLINE_SNAPSHOT, K.AGR_CFG_DELTA_SNAPSHOT


@dataclass
class Case:
    steps: list                          # T.Batch, or "expire" (expire everything + reclaim)
    rows: int
    vslab: int
    flags: int = 0
    maxrec: int = MAXREC


def _batch(lens, rng, seq0, bad=()):
    b = T._batch(lens, rng, seq0, None)
    for i in bad:                                        # headers that claim more than their stored payload
        T._make_bad(b.h, b.lens, [i], i % 2)
    b.blob, b.offs = L.blob_from(b.h, b.lens, rng)
    return b


def _to_tile(at):
    """small records (<= 8 KiB) from byte `at` up to the next tile boundary at least 96 B away"""
    gap = -(-(at + 96) // kr.TILE) * kr.TILE - at
    return list(kr.layout([("to", gap)]))


def case_mixed():
    rng = np.random.default_rng(7)
    a = list(kr.layout([("to", kr.TILE - 16)])) + [8208]                       # a long record in the last 16 B of tile 0
    a += [65536, 8208, MB]                                                         # consecutive long records
    a += _to_tile(sum(a)) + [16384] + [96] * 86 + [5008, 96]                       # 86 small starts in the tile after a long one
    b = [8208, 65536, MB, MAXREC]                                                  # only long records, the maximum exactly
    c = [96, 4000, MAXREC - 16, 112, 8192, 8208 + 16 * 5, 512]
    return Case([_batch(a, rng, 1, bad=(len(a) - 90, len(a) - 96)), _batch(b, rng, 10_000, bad=(1,)), _batch(c, rng, 20_000)],
                rows=1 << 12, vslab=16 * MB)


def case_ring():
    """a byte ring of 3 MiB: the third batch skips the end of the lap to byte 0 (after an expire + reclaim)"""
    rng = np.random.default_rng(8)
    lens = lambda: [96, 2000, MB, 512, 8208]                                       # noqa: E731
    return Case([_batch(lens(), rng, 1), _batch(lens(), rng, 100), "expire", _batch(lens(), rng, 200), _batch([MAXREC], rng, 300)],
                rows=1 << 10, vslab=3 * MB, flags=R)


CASES = {"mixed": case_mixed, "ring": case_ring}
_cases, _twins = {}, {}


def case(name):
    if name not in _cases:
        _cases[name] = CASES[name]()
    return _cases[name]


def engine(c: Case, mode, form=None, **kw):
    """form None: the fixed-stride twin"""
    flags = P | T.MODES[mode] | c.flags | (0 if form is None else V)
    if form is not None:
        kw.update(vslab_bytes=c.vslab, k1_variant=T.FORMS[form], max_record_bytes=c.maxrec)
    e = A.Engine(flags=flags, slab_rows=c.rows, max_agents=64, id_secret=T.SECRET, **kw)
    for a, s in T.AGENTS.items():
        e.set_agent_state(a, s)
    e.drop_agent("agent-drop")
    return e


def twin(name, mode):
    if (name, mode) not in _twins:
        c, out = case(name), []
        with engine(c, mode) as e:
            for b in c.steps:
                if isinstance(b, str):
                    T.expire_all(e)
                    continue
                n = len(b.lens)
                v, ids = np.zeros(n, dtype=A.verdict_dtype), np.zeros((n, 16), dtype=np.uint8)
                first = e.ingest_ex(kr.twin_records(b.blob, b.offs), v, ids)
                out.append(dict(first=first, v=v, ids=ids, state=e.debug_read("state", first, n), route=e.debug_read("route", first, n)))
            _twins[(name, mode)] = (out, e.stats())
    return _twins[(name, mode)]


_digests = {}


@pytest.mark.parametrize("mode", T.MODES)
@pytest.mark.parametrize("form", T.FORMS)
@pytest.mark.parametrize("name", CASES)
def test_k1v_with_long_records(name, form, mode):
    c = case(name)
    tw, tstats = twin(name, mode)
    ring = bool(c.flags & R)
    dig = hashlib.sha256()
    malformed = 0
    with engine(c, mode, form) as e, tempfile.TemporaryDirectory() as tmp:
        live, vused, bi = [], 0, 0
        for b in c.steps:
            if isinstance(b, str):
                T.full_check(e, c, mode, live, dig, tmp, False)
                T.expire_all(e)
                live = []
                continue
            n, nbytes = len(b.lens), int(b.offs[-1])
            if ring and vused % c.vslab + nbytes > c.vslab:
                vused += c.vslab - vused % c.vslab
            base = vused % c.vslab if ring else vused
            vused += nbytes
            launches = e.stats()["k1_launches"]
            v, ids, first = e.ingest_var(b.blob, b.offs)
            assert e.stats()["k1_launches"] - launches == 3 + 2 * bool((b.lens > K.AGR_VAR_MAX_RECORD).any())
            t = tw[bi]; bi += 1
            assert first == t["first"]
            assert v.tobytes() == t["v"].tobytes(), T._diff(v.view("<u8"), t["v"].view("<u8"), "verdicts")
            assert ids.tobytes() == t["ids"].tobytes(), "ids"
            state, route = e.debug_read("state", first, n), e.debug_read("route", first, n)
            assert (state == t["state"]).all(), T._diff(state, t["state"], "state")
            assert (route == t["route"]).all(), T._diff(route, t["route"], "route")
            ck = e.debug_read("cksum", first, n)
            want = kr.cksum(b.blob, b.offs)
            assert (ck == want).all(), T._diff(ck, want, "cksum")
            long = np.nonzero(b.lens > K.AGR_VAR_MAX_RECORD)[0]
            assert (L.piece_cksums(b.blob, b.offs)[long] == want[long]).all()
            malformed += T.plain_checks(b, v, state, mode)
            for x in (v, ids, state, route, ck):
                dig.update(x.tobytes())
            live.append((b, first, base))
        T.full_check(e, c, mode, live, dig, tmp, True)
        s = e.stats()
        for k in T.COUNTERS:
            assert s[k] == tstats[k], (k, s[k], tstats[k])
        assert s["malformed"] == malformed
        # one record 16 B over the maximum: AGR_EINVAL, no row used
        used = s["rows_used"]
        rng = np.random.default_rng(99)
        over = _batch([96, c.maxrec + 16], rng, 50_000)
        with pytest.raises(A.AgrError) as ex:
            e.ingest_var(over.blob, over.offs)
        assert ex.value.code == K.AGR_EINVAL and f"[96, {c.maxrec}]" in str(ex.value)
        assert e.stats()["rows_used"] == used
    _digests.setdefault((name, mode), set()).add(dig.hexdigest())
    assert len(_digests[(name, mode)]) == 1, "the two forms disagree"


# ---------------------------------------------------------------------------------------------- integrity sweep
def test_verify_counts_corruption_in_long_records():
    rng = np.random.default_rng(21)
    lens = [96, 3 * 8192 + 48, 512, MB, 8208, 112]
    b = _batch(lens, rng, 1)
    with A.Engine(flags=P | V, slab_rows=256, max_agents=8, vslab_bytes=8 * MB, max_record_bytes=MAXREC) as e:
        e.set_agent_state("agent-run", "running"); e.set_agent_state("agent-stop", "stopped")
        _, _, first = e.ingest_var(b.blob, b.offs)
        n = len(lens)
        base = e.slab_ptr(0)
        voff = e.debug_read("voff", first, n).astype(np.int64)
        vlen = e.debug_read("vlen", first, n).astype(np.int64)
        assert (vlen == np.diff(b.offs.astype(np.int64))).all()
        plan = {1: [0, 8192 - 16, 8192, 2 * 8192 - 16, 2 * 8192, int(vlen[1]) - 16],
                3: [0, 8192 - 4, 8192, 64 * 8192 - 1, 64 * 8192, int(vlen[3]) - 1],
                4: [0, 8192 - 1, 8192]}
        for rec, spots in plan.items():
            for at in spots:
                ptr = base + int(voff[rec]) + at
                HF.flip(ptr)
                slab = HF.dev_read(base, int(voff[-1] + vlen[-1]))
                state, ck = e.debug_read("state", first, n), e.debug_read("cksum", first, n)
                want = VR.sweep(state, ck, slab, span=n, ring=False, voff=voff, vlen=vlen)
                assert want.bad.tolist() == [rec], (rec, at)
                assert e.verify() == (want.checked, len(want.bad)), (rec, at)
                HF.flip(ptr)
        assert e.verify()[1] == 0


# ---------------------------------------------------------------------------------------------- JSON wire form
T5.PAYLOAD["long"] = MAXREC - K.AGR_HEADER_BYTES


@pytest.mark.parametrize("ids", sorted(T5.IDS))
def test_json_of_long_records(ids):
    rig = T5.Rig("var", ids, setup=False)
    rig.eng.close()
    rig.eng = A.Engine(slab_rows=1 << 12, max_agents=64, flags=P | V | T5.IDS[ids], vslab_bytes=64 * MB, resp_bytes=64 * MB,
                       id_secret=T5.SECRET, max_record_bytes=MAXREC)
    rig.lib, rig.h, rig.layout = rig.eng.lib, rig.eng.h, "long"
    try:
        rig.setup()
        rng = np.random.default_rng(5)
        pad = MAXREC - K.AGR_HEADER_BYTES
        bodies = [rng.bytes(n) for n in (8100, 70000, MB - 300, pad - 200 - 40)]
        recs = [rig.mk(path=b"/small")]
        for k, body in enumerate(bodies):
            recs.append(rig.mk(path=b"/long/%d" % k, headers=b"".join(b"X-H%d: v\n" % j for j in range(k + 1)), body=body))
            recs.append(rig.mk(path=b"/s%d" % k, body=rng.bytes(k * 50)))
        assert len(recs[-2].path) + len(recs[-2].headers) + len(recs[-2].body) > pad - 240
        first = rig.ingest(recs)
        rig.check_all_forms(first, recs)
        rig.apply([("resp", recs[3], 200, b"A: b\n", b"ok"), ("err", recs[5], b"boom")])
        rig.check_all_forms(first, recs)
        for r in recs:
            assert rig.eng.get_record_json(r.agent.decode(), r.rid) == r.wire()
        got, cnt = rig.eng.pending_json(T5.AGENT.decode())
        by_id = {r.rid: r for r in [rig.anchor, rig.poison_rec] + recs}
        pend = [by_id[bytes(i)] for i in rig.eng.list(T5.AGENT.decode(), K.AGR_LIST_PENDING)]
        assert all(recs[k] in pend for k in (1, 5, 7)) and recs[3] not in pend
        assert cnt == len(pend) and got == k5ref.wire_rows(pend, as_array=True, roundtrip=True)[0]
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------- durability
def _feed(e, rng, seq0, lens):
    b = _batch(lens, rng, seq0)
    v, ids, first = e.ingest_var(b.blob, b.offs)
    return b, v, ids, first


def _check_rows(e, items, mode):
    """every record's bytes (get_record_var), voff-independent words and verify() against the references"""
    for b, v, ids, first in items:
        n = len(b.lens)
        state, aux = e.debug_read("state", first, n), e.debug_read("aux", first, n)
        assert (e.debug_read("vlen", first, n) == np.diff(b.offs.astype(np.int64))).all()
        assert (e.debug_read("cksum", first, n) == kr.cksum(b.blob, b.offs)).all()
        want = kr.readback(b.blob, b.offs, state, aux, ids if mode == "mint" else None)
        stored = (state & T.ST_STORED) != 0
        for i in np.nonzero(stored)[0]:
            got = e.get_record_var(b.h["agent_id"][i].decode(), bytes(ids[i]))
            assert got is not None and got.tobytes() == want[b.offs[i]: b.offs[i + 1]].tobytes(), i
    assert e.verify()[1] == 0


@pytest.mark.parametrize("mode", T.MODES)
@pytest.mark.parametrize("snap", ["blocking", "online", "delta"])
def test_snapshots_of_long_records(snap, mode, tmp_path):
    extra = {"blocking": 0, "online": ON, "delta": ON | DELTA}[snap]
    flags = P | V | T.MODES[mode] | extra
    rng = np.random.default_rng(31)
    kw = dict(slab_rows=1 << 10, max_agents=64, id_secret=T.SECRET)
    with A.Engine(flags=flags, vslab_bytes=16 * MB, max_record_bytes=MAXREC, **kw) as e:
        for a, s in T.AGENTS.items():
            e.set_agent_state(a, s)
        items = [_feed(e, rng, 1, [96, MB, 8208, 704])]
        e.snapshot(str(tmp_path / "a.snap"))
        items.append(_feed(e, rng, 100, [65536, 96, MAXREC]))
        path = str(tmp_path / "b.snap")
        e.snapshot(path)
        if snap != "delta":
            with open(path, "rb") as f:
                _, _, sec = snapfile.parse(f.read())
            for b, _, _, first in items:
                n = len(b.lens)
                vo = sec["voff"][first: first + n].astype(np.int64)
                assert (sec["vlen"][first: first + n] == np.diff(b.offs.astype(np.int64))).all()
                assert sec["slab"][vo[0]: vo[0] + len(b.blob)].tobytes() == b.blob.tobytes()
        _check_rows(e, items, mode)
    for vslab, maxrec in ((16 * MB, MAXREC), (5 * MB, MAXREC), (16 * MB, 0)):     # in place, relocated, the default limit
        with A.Engine(flags=flags, vslab_bytes=vslab, max_record_bytes=maxrec, restore_from=path, **kw) as r:
            _check_rows(r, items, mode)
            b = _batch([96, MB], rng, 1000)
            if maxrec:
                r.ingest_var(b.blob, b.offs)
            else:
                with pytest.raises(A.AgrError) as ex:
                    r.ingest_var(b.blob, b.offs)
                assert ex.value.code == K.AGR_EINVAL and "[96, 8192]" in str(ex.value)
    # into the fixed 512-byte form (a ring): refused, every live record over 512 B counted
    stored = sum(int(((x[1]["flags"] & K.AGR_VF_STORED) != 0)[x[0].lens > 512].sum()) for x in items)
    with pytest.raises(A.AgrError) as ex:
        A.Engine(flags=(flags & ~V) | R, restore_from=path, **kw)
    assert ex.value.code == K.AGR_EINVAL and f"{stored} live records are longer than the 512 B rows" in str(ex.value)


# ---------------------------------------------------------------------------------------------- byte ring
def test_ring_space_and_release_of_long_records():
    rng = np.random.default_rng(41)
    with A.Engine(flags=P | V | R, slab_rows=1 << 10, max_agents=64, vslab_bytes=3 * MB, max_record_bytes=MAXREC, id_secret=T.SECRET) as e:
        for a, s in T.AGENTS.items():
            e.set_agent_state(a, s)
        items = [_feed(e, rng, 1, [MB, 96]), _feed(e, rng, 10, [MB - 4096, 8208])]
        used = e.stats()["rows_used"]
        b = _batch([MAXREC], rng, 20)
        with pytest.raises(A.AgrError) as ex:
            e.ingest_var(b.blob, b.offs)
        assert ex.value.code == K.AGR_ENOSPC and e.stats()["rows_used"] == used
        _check_rows(e, items, "hash")
        assert e.expire(1 << 60, 1) == sum(int(((x[1]["flags"] & K.AGR_VF_STORED) != 0).sum()) for x in items)
        assert e.reclaim() == used
        v, ids, first = e.ingest_var(b.blob, b.offs)                    # skips the end of the lap to byte 0
        assert e.debug_read("voff", first, 1)[0] == 0
        _check_rows(e, [(b, v, ids, first)], "hash")


# ---------------------------------------------------------------------------------------------- single requests
def _one(rng, seq, length, agent="agent-run"):
    b = T._batch([length], rng, seq, None, agent_of=np.array([T.NAMES.index(agent)]))
    b.blob, b.offs = L.blob_from(b.h, b.lens, rng)
    return b


def test_long_tickets_are_refused_and_long_calls_take_the_locked_path():
    rng = np.random.default_rng(51)
    c = Case([], rows=1 << 12, vslab=64 * MB, flags=CB, maxrec=MAXREC)
    with engine(c, "hash", "staged") as e:
        ops = e.stats()["svc_ops"]
        big = _one(rng, 1, 65536)
        with pytest.raises(A.AgrError) as ex:
            e.submit_ingest(big.blob)
        assert ex.value.code == K.AGR_EINVAL and "agr_ingest_var" in str(ex.value)
        assert e.stats()["svc_ops"] == ops and e.stats()["rows_used"] == 0
        # long agr_ingest_var(n = 1) from threads while ticket callers submit short records
        results, errors = {}, []
        lock = threading.Lock()

        def longs(k):
            r = np.random.default_rng(1000 + k)
            for j in range(6):
                b = _one(r, 10_000 * (k + 1) + j, [65536, 8208, MB][j % 3], T.NAMES[j % 3])
                v, ids, first = e.ingest_var(b.blob, b.offs)
                with lock:
                    results[first] = (b, v[0])

        def tickets(k):
            r = np.random.default_rng(2000 + k)
            for j in range(40):
                b = _one(r, 100_000 * (k + 1) + j, int(r.integers(6, 300)) * 16, T.NAMES[j % 4])
                t = e.submit_ingest(b.blob)
                a = e.poll(t)
                with lock:
                    assert a["rid"] not in results
                    results[a["rid"]] = (b, a["verdict"][0])

        def guard(f, k):
            try:
                f(k)
            except Exception as x:                                   # noqa: BLE001
                errors.append(x)
        th = [threading.Thread(target=guard, args=(longs, k)) for k in range(3)] + [threading.Thread(target=guard, args=(tickets, k)) for k in range(8)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        assert len(results) == 3 * 6 + 8 * 40 and e.stats()["svc_ops"] - ops == 8 * 40
        order = sorted(results)
        assert order == list(range(len(order)))                       # every call took rows of its own, none twice
        # the end state equals a twin engine fed the calls in the order the engine applied them
        bl = [results[r][0] for r in order]
        recs = np.concatenate([kr.twin_records(b.blob, b.offs) for b in bl])
        with engine(Case([], rows=1 << 12, vslab=0), "hash") as tw:
            tv = np.zeros(len(recs), dtype=A.verdict_dtype)
            tw.ingest_ex(recs, tv, np.zeros((len(recs), 16), dtype=np.uint8))
            got = np.array([results[r][1] for r in order], dtype=A.verdict_dtype)
            assert got.tobytes() == tv.tobytes()
            n = len(recs)
            for w in ("state", "route"):
                assert (e.debug_read(w, 0, n) == tw.debug_read(w, 0, n)).all(), w
            assert (e.debug_read("cksum", 0, n) == np.concatenate([kr.cksum(b.blob, b.offs) for b in bl])).all()
            for k in T.COUNTERS:
                assert e.stats()[k] == tw.stats()[k], k
        assert e.verify()[1] == 0


def test_default_engine_still_decides_an_over_long_ticket_bad_len():
    rng = np.random.default_rng(61)
    c = Case([], rows=1 << 10, vslab=16 * MB, flags=CB, maxrec=0)
    with engine(c, "hash", "staged") as e:
        b = _one(rng, 1, 8192)
        b.h["body_len"] = 20000
        b.blob[:96] = b.h.view(np.uint8)
        t = e.submit_ingest(b.blob)
        a = e.poll(t)
        assert int(a["verdict"]["flags"][0]) & K.AGR_VF_BAD_LEN and a["result"] == 0


# ---------------------------------------------------------------------------------------------- past byte 2^32
def test_long_record_across_byte_2_32():
    HF.need_hbm(9)
    rng = np.random.default_rng(71)
    e = HF.engine(P | V, slab_rows=HF.S_FAR, vslab_bytes=HF.BYTES_FAR, max_record_bytes=MAXREC)
    try:
        start = HF.G4 - 3 * 8192 - 16                            # a piece boundary 16 B before 2^32, the record ends 1 MiB above
        k = (start - 600) // HF.REC
        HF.device_fill(e, k)
        vused = HF.REC * k
        pad = _batch([start - vused], rng, 10_000)
        e.ingest_var(pad.blob, pad.offs)
        h = kr.headers(2, [HF.TAG], rng, seq0=1 << 24)
        lens = [MB, 8208]
        kr.fit_lens(h, lens, rng)
        blob, offs = L.blob_from(h, lens, rng)
        v, ids, first = e.ingest_var(blob, offs)
        assert (v["flags"] == K.AGR_VF_STORED | K.AGR_VF_TRACKED).all()
        assert (e.debug_read("voff", first, 2) == start + offs[:-1].astype(np.uint64)).all()
        assert (e.debug_read("vlen", first, 2) == np.diff(offs.astype(np.int64))).all()
        assert (e.debug_read("cksum", first, 2) == kr.cksum(blob, offs)).all()
        state, aux = e.debug_read("state", first, 2), e.debug_read("aux", first, 2)
        want = kr.readback(blob, offs, state, aux)
        for i in range(2):
            assert e.get_record_var(HF.TAG, bytes(h["request_id"][i])).tobytes() == want[offs[i]: offs[i + 1]].tobytes()
        assert HF.dev_read(e.slab_ptr(0) + start, len(blob)).tobytes() == blob.tobytes()
        assert e.verify()[1] == 0
    finally:
        e.close()
