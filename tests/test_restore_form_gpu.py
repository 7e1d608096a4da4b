"""agr_restore into a ring of the other record form: 512 B rows to variable-length records and back.  The converted state
against the plain reference (tests/formref.py), file for file, and the converted engine against a same-form restore of the
same file, call for call, across the restart and on through further laps of its new ring."""
import re

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from formref import NotRepresentable, bad_rows, compact_len, convert
from jsoncase import make_requests, records_array, var_batch
from oracle.gojson import format_uuid
from snapfile import parse, parse_delta
from test_restore_resize_gpu import KeyDriver, kw, run_on
from test_restore_scale_gpu import assert_file, same_reads
from test_restore_scale_gpu import source as scale_source
from test_snapshot_online_gpu import AGENTS, RESP, RING_ROWS, SEC, SECRET, STEP, T0, VSLAB, Driver, outcomes

pytestmark = pytest.mark.gpu

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
CHAIN = K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT
SOURCE_V = {"to_var": 0, "to_fixed": V}                 # the source's form, by direction
IDS = {"mint": M, "hash": 0}


def read(p):
    with open(p, "rb") as f:
        return f.read()


class FormDriver(Driver):
    """Driver whose records fit both forms (path, headers and body within 416 B), each engine fed in its own form."""

    def batch(self, engines, n, rnd):
        now = T0 + rnd * STEP
        batch = make_requests(50 + rnd, n, AGENTS)
        for k, r in enumerate(batch):
            r.now = now + k * SEC
        firsts = []
        for eng in engines:
            if eng.varlen:
                _, got, first = eng.ingest_var(*var_batch(batch))
            else:
                got = np.zeros((n, 16), dtype=np.uint8)
                first = eng.ingest_ex(records_array(batch), np.zeros(n, dtype=A.verdict_dtype), got)
            firsts.append((first, [bytes(x) for x in got]))
        assert all(f == firsts[0] for f in firsts)
        first, got = firsts[0]
        for k, r in enumerate(batch):
            self.ids[first + k] = (r.agent_id, got[k] if self.flags & M else r.rid)
        return list(range(first, first + n)), now


class FormKeyDriver(KeyDriver, FormDriver):
    """KeyDriver over FormDriver's batches"""


def own_kw(flags):
    """the capacities a source of these flags is built with (and restored in, in its own form)"""
    return kw(flags) if flags & R else kw(flags, 4096, VSLAB, 1 << 20)


def source(tmp_path, flags, seed, name="src.snap", driver=FormDriver):
    drv = driver(flags, seed)
    with A.Engine(**own_kw(flags)) as eng:
        drv.build([eng], 6 if flags & R else 3)
        path = str(tmp_path / name)
        eng.snapshot(path)
        used = eng.stats()["rows_used"]
    return path, drv, used


_SOURCES = {}


def cached_source(tmp_path_factory, flags):
    if flags not in _SOURCES:
        _SOURCES[flags] = source(tmp_path_factory.mktemp("form_src"), flags, seed=31 + flags % 89)
    return _SOURCES[flags]


def needs(hd, ag, sec, flags):
    """record bytes (variable-length target) and response bytes the live rows take once converted and packed"""
    out, _, _ = convert(hd, ag, sec, flags, 1 << 20, 1 << 40, 1 << 40)
    return int(out["vused"]), int(out["resp_used"])


# ---- 1. the file written right after the restore is the reference's
@pytest.mark.parametrize("geom", ["same", "more_rows", "fewer_rows", "npot_rows", "smaller_bytes"])
@pytest.mark.parametrize("src", ["ring", "append"])
@pytest.mark.parametrize("ids", sorted(IDS))
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_file_after_the_conversion_is_the_reference(to, ids, src, geom, tmp_path, tmp_path_factory):
    sflags = P | IDS[ids] | SOURCE_V[to] | (R if src == "ring" else 0)
    tflags = (sflags ^ V) | R
    path, _, _ = cached_source(tmp_path_factory, sflags)
    hd, ag, sec = parse(read(path))
    need_v, need_r = needs(hd, ag, sec, tflags)
    window = int(hd["rows_used"]) - int(hd["tail"])
    S, vcap, rcap = {"same": (RING_ROWS, VSLAB, RESP), "more_rows": (2 * RING_ROWS, VSLAB, RESP), "fewer_rows": (window + 3, VSLAB, RESP),
                     "npot_rows": (777, VSLAB, RESP), "smaller_bytes": (RING_ROWS, max(need_v + 100, 1 << 14), need_r + 48)}[geom]
    want = convert(hd, ag, sec, tflags, S, vcap, rcap)
    with A.Engine(restore_from=path, **kw(tflags, S, vcap, rcap)) as back:
        assert back.verify()[1] == 0
        back.snapshot(str(tmp_path / "after.snap"))
    got = parse(read(tmp_path / "after.snap"))
    assert_file(got, want, bool(tflags & V), geom)
    assert int(got[0]["vused"]) == need_v
    assert int(np.count_nonzero(got[2]["state"])) > 100


# ---- 2. the converted engine behaves like a same-form restore of the same file
def dispatch(eng):
    return (eng.replay_scan_var() if eng.varlen else eng.replay_scan(with_records=False))[0]


def same_engine(conv, twin, drv, used, tail):
    """conv (converted) and twin (restored in the file's own form) row for row: listings, wire forms, records, responses,
    the replay scan's dispatch list; each record in the variable-length engine is the fixed one's first bytes, then zeros"""
    assert conv.verify()[1] == 0 and twin.verify()[1] == 0
    for a in AGENTS:
        assert conv.pending_json(a) == twin.pending_json(a), a
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert np.array_equal(conv.list(a, which), twin.list(a, which)), (a, which)
    (jc, oc), (jt, ot) = conv.rows_json(tail, used - tail, as_array=True), twin.rows_json(tail, used - tail, as_array=True)
    assert jc == jt and np.array_equal(oc, ot)
    var_eng, fixed_eng = (conv, twin) if conv.varlen else (twin, conv)
    found = 0
    for L, (a, rid) in drv.ids.items():
        if L >= used:
            continue
        assert conv.get_record_json(a, rid) == twin.get_record_json(a, rid), L
        assert conv.get_response_body(a, rid) == twin.get_response_body(a, rid), L
        rv, rf = var_eng.get_record_var(a, rid), fixed_eng.get_record(a, rid)
        assert (rv is None) == (rf is None), L
        if rv is not None:
            raw = rf.tobytes()
            assert len(rv) == compact_len(np.frombuffer(raw, np.uint8)), L
            assert raw[: len(rv)] == rv.tobytes() and not any(raw[len(rv):]), L
            found += 1
    assert found > 100
    assert dispatch(conv).tobytes() == dispatch(twin).tobytes()


def same_by_key(conv, cd, twin, td):
    """same_engine with rows matched by arrival key (rings of other sizes put the same calls on other rows)"""
    assert conv.verify()[1] == 0 and twin.verify()[1] == 0
    kc = {rid: cd.key[L] for L, (_, rid) in cd.ids.items()}
    kt = {rid: td.key[L] for L, (_, rid) in td.ids.items()}
    for a in AGENTS:
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert [kc[bytes(x)] for x in conv.list(a, which)] == [kt[bytes(x)] for x in twin.list(a, which)], (a, which)
    by_key = {td.key[L]: L for L in td.ids}
    assert sorted(cd.key.values(), key=str) == sorted(by_key, key=str)
    for L, k in cd.key.items():
        (a, rc), (_, rt) = cd.ids[L], td.ids[by_key[k]]
        jc, jt = conv.get_record_json(a, rc), twin.get_record_json(a, rt)
        if jc is not None and jt is not None:
            jc, jt = jc.replace(format_uuid(rc).encode(), b"ID"), jt.replace(format_uuid(rt).encode(), b"ID")
        assert jc == jt, k
        assert conv.get_response_body(a, rc) == twin.get_response_body(a, rt), k
    assert len(dispatch(conv)) == len(dispatch(twin))


@pytest.mark.parametrize("rows", ["same", "npot"])
@pytest.mark.parametrize("ids", sorted(IDS))
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_converted_engine_behaves_like_the_same_form_restore(to, ids, rows, tmp_path):
    sflags = P | IDS[ids] | R | SOURCE_V[to]
    tflags = sflags ^ V
    path, drv, used = source(tmp_path, sflags, seed=12)
    hd, _, _ = parse(read(path))
    S = {"same": RING_ROWS, "npot": 777}[rows]
    with A.Engine(restore_from=path, **kw(sflags)) as twin, A.Engine(restore_from=path, **kw(tflags, S, 2 * VSLAB, 2 * RESP)) as conv:
        same_engine(conv, twin, drv, used, int(hd["tail"]))
        cd, td = FormKeyDriver(drv), FormKeyDriver(drv)
        run_on([(conv, cd), (twin, td)], S // 120 + 2)          # more than one lap of the new ring
        assert conv.stats()["rows_used"] - used > S
        same_by_key(conv, cd, twin, td)


# ---- 3. agr_verify after the conversion
def test_verify_counts_exactly_the_rows_with_bytes_past_their_record(tmp_path):
    flags = P | M | R
    drv = FormDriver(flags, 21)
    with A.Engine(**kw(flags)) as eng:
        drv.build([eng], 2)
        recs = records_array(make_requests(99, 40, AGENTS))
        raw = recs.view(np.uint8).reshape(40, 512)
        planted = []
        for i in range(0, 40, 3):
            n = compact_len(raw[i])
            if n < 512:
                raw[i, n + (7 * i) % (512 - n)] = 0x5A
                planted.append(i)
        ids = np.zeros((40, 16), dtype=np.uint8)
        first = eng.ingest_ex(recs, np.zeros(40, dtype=A.verdict_dtype), ids)
        assert eng.verify()[1] == 0 and len(planted) > 5
        eng.snapshot(str(tmp_path / "src.snap"))
    hd, _, sec = parse(read(tmp_path / "src.snap"))
    assert bad_rows(hd, sec) == [first + i for i in planted]
    with A.Engine(restore_from=str(tmp_path / "src.snap"), **kw(flags | V)) as back:
        assert back.verify()[1] == len(planted)
        a = recs[planted[0]]["agent_id"].decode()
        got = back.get_record_var(a, bytes(ids[planted[0]]))   # the payload is the row's, cut at the compact length
        assert len(got) == compact_len(raw[planted[0]]) and got[96:].tobytes() == raw[planted[0], 96: len(got)].tobytes()


# ---- 4. a delta chain converts, and the converted engine starts a new one
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_delta_chain_converts(to, tmp_path):
    sflags = P | M | R | SOURCE_V[to]
    tflags = sflags ^ V
    drv = FormDriver(sflags, 16)
    with A.Engine(**kw(sflags | CHAIN)) as eng:
        drv.build([eng], 6)
        for k in range(3):
            if k:
                run_on([(eng, drv)], 1)
            eng.snapshot(str(tmp_path / f"c{k}.snap"))
        used = eng.stats()["rows_used"]
        assert [read(tmp_path / f"c{k}.snap")[:8] for k in range(3)] == [b"AGRSNAP3", b"AGRDELT1", b"AGRDELT1"]
        tail = int(parse_delta(read(tmp_path / "c2.snap"))["hd"]["tail"])
        with A.Engine(restore_from=str(tmp_path / "c2.snap"), **kw(tflags | CHAIN, 700, 2 * VSLAB, 2 * RESP)) as back:
            same_engine(back, eng, drv, used, tail)
            back.snapshot(str(tmp_path / "d0.snap"))
            assert read(tmp_path / "d0.snap")[:8] == b"AGRSNAP3"          # a new chain
            rnd = drv.round = drv.round + 1
            for e in (back, eng):
                e.expire(T0 + rnd * STEP, STEP + STEP // 2)
                e.reclaim()
            rows, now = drv.batch([back, eng], 120, rnd)
            drv.complete([back, eng], rows, now, 100)
            back.snapshot(str(tmp_path / "d1.snap"))
            d1 = parse_delta(read(tmp_path / "d1.snap"))
            assert d1["parent"] == str((tmp_path / "d0.snap").resolve())
            used = back.stats()["rows_used"]
            with A.Engine(restore_from=str(tmp_path / "d1.snap"), **kw(tflags, 700, 2 * VSLAB, 2 * RESP)) as again:
                assert again.verify()[1] == 0
                for L, (a, rid) in drv.ids.items():
                    if L < used:
                        assert again.get_record_json(a, rid) == back.get_record_json(a, rid) == eng.get_record_json(a, rid), L


# ---- 5. far along the arrival counter
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_far_along_the_arrival_counter(to, tmp_path):
    sflags = P | M | R | SOURCE_V[to]
    drv = FormDriver(sflags, 14)
    with A.Engine(**kw(sflags)) as eng:
        eng.skip_arrivals((1 << 40) + 3)
        drv.build([eng], 6)
        eng.snapshot(str(tmp_path / "far.snap"))
    hd, _, _ = parse(read(tmp_path / "far.snap"))
    tail = int(hd["tail"])
    assert tail > (1 << 40)
    with A.Engine(restore_from=str(tmp_path / "far.snap"), **kw(sflags ^ V, 300 + int(hd["rows_used"]) - tail)) as back:
        live = [L for L in sorted(drv.ids) if L >= tail]
        gone = [L for L in sorted(drv.ids) if L < tail]
        assert live and gone
        for L in gone[-20:]:
            assert back.get_record_json(*drv.ids[L]) is None
        got = [back.get_record_json(*drv.ids[L]) for L in live]
        assert sum(g is not None for g in got) > len(live) // 2
        pend = [L for L, g in zip(live, got) if g is not None and b'"status":"pending"' in g][:10]
        assert pend
        res = back.complete(outcomes([(drv.ids[L][1], drv.ids[L][0], K.AGR_OUT_RESPONSE, 200, T0 + 99 * STEP) for L in pend] +
                                     [(drv.ids[gone[-1]][1], drv.ids[gone[-1]][0], K.AGR_OUT_RESPONSE, 200, T0 + 99 * STEP)]))
        assert list(res) == [0] * len(pend) + [K.AGR_ENOTFOUND]


# ---- 6. hash-id mode: the dedupe index is rebuilt from the converted rows
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_hash_mode_dedupe_after_a_conversion(to, tmp_path):
    sflags = P | R | SOURCE_V[to]
    path, drv, used = source(tmp_path, sflags, seed=15)
    hd, _, _ = parse(read(path))
    with A.Engine(restore_from=path, **kw(sflags ^ V, 901)) as back:
        live = [L for L in sorted(drv.ids) if L >= int(hd["tail"]) and back.get_record_json(*drv.ids[L]) is not None]
        a, rid = drv.ids[live[-1]]
        reqs = make_requests(77, 2, [a])
        reqs[1].rid = rid                                          # a fresh record that reuses a live id
        if back.varlen:
            blob, offs = var_batch(reqs)
            blob[offs[0] + 72] |= K.AGR_F_REPLAY                    # (agr_record.flags)
            blob[offs[0] + 16: offs[0] + 32] = np.frombuffer(rid, dtype=np.uint8)
            out, _, _ = back.ingest_var(blob, offs)
        else:
            recs = records_array(reqs)
            recs[0]["flags"] |= K.AGR_F_REPLAY
            recs[0]["replay_of"] = np.frombuffer(rid, dtype=np.uint8)   # a replay naming a pre-restart id
            out = np.zeros(2, dtype=A.verdict_dtype)
            back.ingest_ex(recs, out, np.zeros((2, 16), dtype=np.uint8))
        assert out[0]["flags"] & K.AGR_VF_KNOWN
        assert out[1]["flags"] & K.AGR_VF_DUP_ID


# ---- 7. the single-request front end on the converted engine
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_single_request_front_end_after_a_conversion(to, tmp_path):
    sflags = P | M | R | SOURCE_V[to]
    path, drv, used = source(tmp_path, sflags, seed=17)
    hd, _, _ = parse(read(path))
    with A.Engine(restore_from=path, **kw((sflags ^ V) | K.AGR_CFG_COMBINE, 1000, 2 * VSLAB, 2 * RESP)) as conv, \
            A.Engine(restore_from=path, **kw(sflags, 1000, 2 * VSLAB, 2 * RESP)) as twin:
        reqs = make_requests(91, 8, AGENTS)
        recs = records_array(reqs)
        blob, offs = var_batch(reqs)
        for k in range(8):                                         # the twin one record per batch, as the tickets are
            if twin.varlen:
                twin.ingest_var(blob[offs[k]: offs[k + 1]], (offs[k: k + 2] - offs[k]).astype(np.uint32))
            else:
                twin.ingest(recs[k: k + 1])
        if conv.varlen:                                            # one variable-length record per ticket
            tickets = [conv.submit_ingest(blob[offs[k]: offs[k + 1]]) for k in range(8)]
        else:                                                      # one 512 B record per ticket
            tickets = [conv.submit_ingest(recs[k: k + 1]) for k in range(8)]
        assert [conv.wait(t) for t in tickets] == [0] * 8
        pend = [L for L in sorted(drv.ids) if L < used and twin.get_record_json(*drv.ids[L]) is not None][-6:]
        for L in pend:
            a, rid = drv.ids[L]
            o = outcomes([(rid, a, K.AGR_OUT_RESPONSE, 201, T0 + 50 * STEP)])
            assert conv.wait(conv.submit_complete_ex(o, b"X: y\n", b"body %d" % L)) == 0
            assert twin.complete_ex(o, [b"X: y\nbody %d" % L], np.array([5], dtype=np.uint32))[1][0] == 0
        same_engine(conv, twin, drv, used + 8, int(hd["tail"]))


# ---- 8. refusals
def _code(fn):
    try:
        fn()
        return 0, ""
    except A.AgrError as e:
        return e.code, str(e)


class BigDriver(Driver):
    """the variable-length records of Driver: bodies of up to 6000 B"""


def test_refusals_leave_nothing_held(tmp_path):
    vpath, _, vused = source(tmp_path, P | M | V | R, 18, "var.snap", driver=BigDriver)
    fpath, _, fused = source(tmp_path, P | M | R, 18, "fixed.snap")
    apath, _, aused = source(tmp_path, P | M, 18, "append.snap")
    hd, ag, sec = parse(read(vpath))
    with pytest.raises(NotRepresentable) as ref:
        convert(hd, ag, sec, P | M | R, RING_ROWS, 0, RESP)
    count, row, ln = re.search(r"(\d+) live records .*row (\d+), (\d+) B", str(ref.value)).groups()
    hdf, agf, secf = parse(read(fpath))
    need_v, _ = needs(hdf, agf, secf, P | M | V | R)
    cases = [(vpath, kw(P | M | R), K.AGR_EINVAL, [f"{count} live records", f"row {row}, {ln} B", "512 B"]),
             (fpath, kw(P | M | V | R, RING_ROWS, need_v - 1, RESP), K.AGR_ENOSPC, ["vslab_bytes", "by 1 B"]),
             (fpath, kw(P | M | V, 1 << 12, VSLAB, RESP), K.AGR_EINVAL, ["id mode"]),     # a ring into an append-only engine
             (apath, kw(P | M | V, 1 << 12, VSLAB, RESP), K.AGR_EINVAL, ["id mode"]),     # append-only into append-only
             (fpath, kw(P | V | R), K.AGR_EINVAL, ["id mode"]),                          # another id mode
             (fpath, dict(kw(P | M | V | R), id_secret=SECRET + 1), K.AGR_EINVAL, ["id_secret"])]
    own = {vpath: (P | M | V | R, vused), fpath: (P | M | R, fused), apath: (P | M, aused)}
    for p, cfg, code, words in cases:
        got = _code(lambda: A.Engine(restore_from=p, **cfg).close())
        assert got[0] == code and all(w in got[1] for w in words), (cfg, got)
        flags, used = own[p]
        with A.Engine(restore_from=p, **own_kw(flags)) as back:
            assert back.verify()[1] == 0 and back.stats()["rows_used"] == used
    with A.Engine(restore_from=fpath, **kw(P | M | V | R, RING_ROWS, need_v, RESP)) as exact:   # exactly what it needs
        assert exact.verify()[1] == 0


# ---- 9. at scale: many count and row tiles, byte-move CTAs across segment ends
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_conversion_at_scale(to, tmp_path):
    sflags = P | M | R | SOURCE_V[to]
    tflags = sflags ^ V
    window = (1 << 21) + 77
    rig, path, src, _ = scale_source(tmp_path, sflags, window, "wraps", seed=5)
    try:
        hd, ag, sec = src
        S_t = window + 12345
        want = convert(hd, ag, sec, tflags, S_t, 1 << 40, 1 << 40)
        vcap, rcap = (int(want[0]["vused"]) if tflags & V else 0), int(want[0]["resp_used"]) + 16
        want[0]["vcap"], want[0]["resp_cap"] = vcap, rcap
        bad = bad_rows(hd, sec) if to == "to_var" else []
        with A.Engine(restore_from=path, slab_rows=S_t, max_agents=16, id_secret=int(hd["id_secret"]), flags=tflags,
                      vslab_bytes=vcap, resp_bytes=rcap, max_batch=1 << 16) as back:
            assert back.verify()[1] == len(bad)
            back.snapshot(str(tmp_path / "after.snap"))
            assert_file(parse(read(tmp_path / "after.snap")), want, bool(tflags & V), to)
            same_reads(back, rig.eng, *rig.rows())
    finally:
        rig.close()


# ---- 10. timing
@pytest.mark.parametrize("to", sorted(SOURCE_V))
def test_conversion_time_is_reported(to, tmp_path):
    sflags = P | M | R | SOURCE_V[to]
    path, _, _ = source(tmp_path, sflags, seed=19)
    with A.Engine(restore_from=path, **kw((sflags ^ V) | K.AGR_CFG_TIMING)) as back:
        assert back.op_time(4) > 0
