"""agr_restore into other capacities: the relocated state against the plain reference (tests/resizeref.py), file for file,
and the relocated engine against a same-geometry restore of the same file, call for call, across the restart and on through
further laps of its new ring."""
import copy

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from jsoncase import make_requests, records_array
from oracle.gojson import format_uuid
from resizeref import relocate
from snapfile import HEADER, WORDS, parse, parse_delta, referenced
from test_snapshot_online_gpu import AGENTS, RESP, RING_ROWS, SECRET, STEP, T0, VSLAB, Driver, outcomes, assert_same_engine, submit_ingest

pytestmark = pytest.mark.gpu

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
MODES = {"hash_ring": P | R, "mint_ring": P | M | R, "var_mint_ring": P | V | M | R, "var_hash_ring": P | V | R}


def kw(flags, slab_rows=RING_ROWS, vslab=VSLAB, resp=RESP):
    return dict(slab_rows=slab_rows, max_agents=16, id_secret=SECRET, flags=flags, vslab_bytes=vslab if flags & V else 0, resp_bytes=resp)


def source(tmp_path, flags, seed=11, rounds=6):
    """A ring that went round several times (stored responses, error texts, expiry, release), its snapshot and driver."""
    drv = Driver(flags, seed)
    with A.Engine(**kw(flags)) as eng:
        drv.build([eng], rounds)
        path = str(tmp_path / "src.snap")
        eng.snapshot(path)
        used = eng.stats()["rows_used"]
    return path, drv, used


def needs(hd, sec):
    """Record bytes and response bytes the live rows of a file take once packed."""
    _, _, big = relocate(hd, b"", sec, int(hd["flags"]), 1 << 20, 1 << 40, 1 << 40)
    return (len(big["slab"]) if int(hd["flags"]) & V else 0), len(big["resp"])


def geometries(hd, sec):
    """(slab_rows, vslab_bytes, resp_bytes) of every case: more rows, fewer that still hold the window, a count that is no
    power of two, larger and smaller byte rings (the smaller ones just above what the live rows take)."""
    need_v, need_r = needs(hd, sec)
    window = int(hd["rows_used"]) - int(hd["tail"])
    return {"more_rows": (2 * RING_ROWS, VSLAB, RESP), "fewer_rows": (window + 3, VSLAB, RESP), "npot_rows": (777, VSLAB, RESP),
            "bigger_bytes": (RING_ROWS, 3 * VSLAB, 3 * RESP), "smaller_bytes": (RING_ROWS, max(need_v + 100, 1 << 14), need_r + 48)}


@pytest.mark.parametrize("geom", ["more_rows", "fewer_rows", "npot_rows", "bigger_bytes", "smaller_bytes"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_file_after_the_restore_is_the_reference(mode, geom, tmp_path):
    flags = MODES[mode]
    path, _, _ = source(tmp_path, flags)
    hd, ag, sec = parse(open(path, "rb").read())
    S, vcap, rcap = geometries(hd, sec)[geom]
    hd_w, ag_w, sec_w = relocate(hd, ag, sec, flags, S, vcap, rcap)
    with A.Engine(restore_from=path, **kw(flags, S, vcap, rcap)) as back:
        assert back.verify()[1] == 0
        out = str(tmp_path / "after.snap")
        back.snapshot(out)
    hd_g, ag_g, sec_g = parse(open(out, "rb").read())
    assert hd_g.tobytes() == np.array(hd_w, dtype=HEADER).tobytes(), (hd_g, hd_w)
    assert ag_g == ag_w
    for name in WORDS + ("completed_log", "failed_log"):
        assert np.array_equal(sec_g[name], sec_w[name]), name
    slab_m, resp_m, live = referenced(sec_w, hd_w, bool(flags & V))
    assert len(live) > 100 and resp_m.sum() > 1000
    assert np.array_equal(sec_g["slab"][slab_m], sec_w["slab"][slab_m])
    assert np.array_equal(sec_g["resp"][resp_m], sec_w["resp"][resp_m])


class KeyDriver(Driver):
    """The driver of one engine after the restart.  Rings of other sizes skip rows at other places at the end of a lap, so the
    same calls land on other row ids (and, minted, other ids): rows are compared by their arrival key instead — the row id
    itself for rows from before the restart, (round, index in the batch) for the ones after."""

    def __init__(self, drv):
        self.__dict__.update(copy.deepcopy(drv.__dict__))
        self.key = {L: L for L in self.ids}

    def batch(self, engines, n, rnd):
        rows, now = super().batch(engines, n, rnd)
        for k, L in enumerate(rows):
            self.key[L] = (rnd, k)
        return rows, now


def run_on(pairs, rounds):
    """The same rounds on every (engine, driver): expiry and release of what is older than the previous round, a batch,
    completions with bytes."""
    for _ in range(rounds):
        for eng, drv in pairs:
            rnd = drv.round = drv.round + 1
            eng.expire(T0 + rnd * STEP, STEP + STEP // 2)
            eng.reclaim()
            rows, now = drv.batch([eng], 120, rnd)
            drv.complete([eng], rows, now, 100)


def assert_same_by_key(back, bd, twin, td, var):
    """What assert_same_engine compares, with rows matched by arrival key and minted ids masked in the JSON."""
    assert back.verify()[1] == 0 and twin.verify()[1] == 0
    kb = {rid: bd.key[L] for L, (_, rid) in bd.ids.items()}
    kt = {rid: td.key[L] for L, (_, rid) in td.ids.items()}
    for a in AGENTS:
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            got, want = [kb[bytes(x)] for x in back.list(a, which)], [kt[bytes(x)] for x in twin.list(a, which)]
            assert got == want, (a, which)
    by_key = {td.key[L]: L for L in td.ids}
    assert sorted(bd.key.values(), key=str) == sorted(by_key, key=str)
    for L, k in bd.key.items():
        (a, rb), (_, rt) = bd.ids[L], td.ids[by_key[k]]
        jb, jt = back.get_record_json(a, rb), twin.get_record_json(a, rt)
        if jb is not None and jt is not None:
            jb, jt = jb.replace(format_uuid(rb).encode(), b"ID"), jt.replace(format_uuid(rt).encode(), b"ID")
        assert jb == jt, k
        assert back.get_response_body(a, rb) == twin.get_response_body(a, rt), k
    scan_b, scan_t = (back.replay_scan_var(), twin.replay_scan_var()) if var else (back.replay_scan(), twin.replay_scan())
    assert len(scan_b[0]) == len(scan_t[0])


@pytest.mark.parametrize("rows", ["more", "fewer", "npot"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_resized_engine_behaves_like_the_same_geometry_restore(mode, rows, tmp_path):
    flags = MODES[mode]
    var = bool(flags & V)
    path, drv, used = source(tmp_path, flags, seed=12)
    hd, _, _ = parse(open(path, "rb").read())
    S = {"more": 2048, "fewer": int(hd["rows_used"] - hd["tail"]) + 130, "npot": 777}[rows]
    with A.Engine(restore_from=path, **kw(flags)) as twin, A.Engine(restore_from=path, **kw(flags, S, 2 * VSLAB, 2 * RESP)) as back:
        assert_same_engine(back, twin, drv, used, var)          # the restart itself: row for row
        if not var:
            for a in AGENTS:
                assert back.pending_json(a) == twin.pending_json(a)
            n = min(used - int(hd["tail"]), 200)
            (jb, ob), (jt, ot) = back.rows_json(used - n, n, as_array=True), twin.rows_json(used - n, n, as_array=True)
            assert jb == jt and np.array_equal(ob, ot)
        bd, td = KeyDriver(drv), KeyDriver(drv)
        run_on([(back, bd), (twin, td)], S // 120 + 2)          # at least one more lap of the new ring
        assert back.stats()["rows_used"] - used > S
        assert_same_by_key(back, bd, twin, td, var)


def test_append_only_restored_as_a_ring(tmp_path):
    flags = P | M
    drv = Driver(flags, seed=13)
    with A.Engine(slab_rows=4096, max_agents=16, id_secret=SECRET, flags=flags, resp_bytes=4 << 20) as eng:
        drv.build([eng], 30)                                     # 3640 rows of 4096
        path = str(tmp_path / "append.snap")
        eng.snapshot(path)
        used = eng.stats()["rows_used"]
        with pytest.raises(A.AgrError) as e:                     # the whole slab is the window
            A.Engine(restore_from=path, **kw(P | M | R, used - 1, 0, 4 << 20))
        assert e.value.code == K.AGR_ENOSPC and "window" in str(e.value)
        ring = lambda S: A.Engine(restore_from=path, **kw(P | M | R, S, 0, 8 << 20))
        with ring(used) as exact, ring(5000) as roomy:
            assert_same_engine(exact, eng, drv, used, False)
            assert_same_engine(roomy, eng, drv, used, False)
            drv.ring = True
            de, dr = KeyDriver(drv), KeyDriver(drv)
            run_on([(exact, de), (roomy, dr)], 5000 // 120 + 2)  # a full lap of both rings, every row released on the way
            assert exact.stats()["rows_used"] > used + 5000
            assert_same_by_key(exact, de, roomy, dr, False)


@pytest.mark.parametrize("skip", [(1 << 32) + 5, (1 << 40) + 3])
def test_far_along_the_arrival_counter(skip, tmp_path):
    flags = P | M | R
    drv = Driver(flags, seed=14)
    with A.Engine(**kw(flags)) as eng:
        eng.skip_arrivals(skip)
        drv.build([eng], 6)
        path = str(tmp_path / "far.snap")
        eng.snapshot(path)
    hd, _, _ = parse(open(path, "rb").read())
    tail = int(hd["tail"])
    assert tail > skip
    with A.Engine(restore_from=path, **kw(flags, 300 + int(hd["rows_used"]) - tail)) as back:
        live = [L for L in sorted(drv.ids) if L >= tail]
        gone = [L for L in sorted(drv.ids) if L < tail]
        assert live and gone
        for L in gone[-20:]:
            a, rid = drv.ids[L]
            assert back.get_record_json(a, rid) is None
        got = [back.get_record_json(*drv.ids[L]) for L in live]
        assert sum(g is not None for g in got) > len(live) // 2
        pend = [L for L, g in zip(live, got) if g is not None and b'"status":"pending"' in g][:10]
        assert pend
        res = back.complete(outcomes([(drv.ids[L][1], drv.ids[L][0], K.AGR_OUT_RESPONSE, 200, T0 + 99 * STEP) for L in pend] +
                                     [(drv.ids[gone[-1]][1], drv.ids[gone[-1]][0], K.AGR_OUT_RESPONSE, 200, T0 + 99 * STEP)]))
        assert list(res) == [0] * len(pend) + [K.AGR_ENOTFOUND]


def test_hash_mode_dedupe_after_a_resize(tmp_path):
    flags = P | R
    path, drv, used = source(tmp_path, flags, seed=15)
    hd, _, sec = parse(open(path, "rb").read())
    with A.Engine(restore_from=path, **kw(flags, 901)) as back:
        live = [L for L in sorted(drv.ids) if L >= int(hd["tail"]) and back.get_record(*drv.ids[L]) is not None]
        a, rid = drv.ids[live[-1]]
        reqs = make_requests(77, 2, [a])
        reqs[1].rid = rid                                          # a fresh record that reuses a live id
        recs = records_array(reqs)
        recs[0]["flags"] |= K.AGR_F_REPLAY
        recs[0]["replay_of"] = np.frombuffer(rid, dtype=np.uint8)   # a replay naming a pre-restart id
        out = np.zeros(2, dtype=A.verdict_dtype)
        back.ingest_ex(recs, out, np.zeros((2, 16), dtype=np.uint8))
        assert out[0]["flags"] & K.AGR_VF_KNOWN
        assert out[1]["flags"] & K.AGR_VF_DUP_ID


def test_delta_chain_into_other_capacities(tmp_path):
    flags = P | M | R | K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT
    drv = Driver(P | M | R, seed=16)
    with A.Engine(**kw(flags)) as eng:
        drv.build([eng], 6)
        for k in range(3):
            if k:
                run_on([(eng, drv)], 1)
            eng.snapshot(str(tmp_path / f"c{k}.snap"))
        used = eng.stats()["rows_used"]
        assert open(tmp_path / "c2.snap", "rb").read(8) == b"AGRDELT1"
        with A.Engine(restore_from=str(tmp_path / "c2.snap"), **kw(flags, 700, 0, 2 * RESP)) as back:
            assert_same_engine(back, eng, drv, used, False)
            back.snapshot(str(tmp_path / "d0.snap"))
            assert open(tmp_path / "d0.snap", "rb").read(8) == b"AGRSNAP3"   # a new chain
            rnd = drv.round = drv.round + 1                      # one round on both, row for row (no lap end in either)
            for e in (back, eng):
                e.expire(T0 + rnd * STEP, STEP + STEP // 2)
                e.reclaim()
            rows, now = drv.batch([back, eng], 120, rnd)
            drv.complete([back, eng], rows, now, 100)
            back.snapshot(str(tmp_path / "d1.snap"))
            d1 = parse_delta(open(tmp_path / "d1.snap", "rb").read())
            assert d1["parent"] == str((tmp_path / "d0.snap").resolve())
            used = back.stats()["rows_used"]
            with A.Engine(restore_from=str(tmp_path / "d1.snap"), **kw(P | M | R, 700, 0, 2 * RESP)) as again:
                assert_same_engine(again, back, drv, used, False)
                assert_same_engine(again, eng, drv, used, False)


def test_single_request_front_end_after_a_resize(tmp_path):
    flags = P | M | R
    path, drv, used = source(tmp_path, flags, seed=17)
    with A.Engine(restore_from=path, **kw(flags | K.AGR_CFG_COMBINE, 1000, 0, 2 * RESP)) as back, \
            A.Engine(restore_from=path, **kw(flags)) as twin:
        recs = records_array(make_requests(91, 8, AGENTS))
        tickets = [submit_ingest(back, recs[k: k + 1]) for k in range(8)]
        assert [back.wait(t) for t in tickets] == [0] * 8
        twin.ingest(recs)
        pend = [L for L in sorted(drv.ids) if L < used and twin.get_record(*drv.ids[L]) is not None][-6:]
        for L in pend:
            a, rid = drv.ids[L]
            o = outcomes([(rid, a, K.AGR_OUT_RESPONSE, 201, T0 + 50 * STEP)])
            assert back.wait(back.submit_complete_ex(o, b"X: y\n", b"body %d" % L)) == 0
            assert twin.complete_ex(o, [b"X: y\nbody %d" % L], np.array([5], dtype=np.uint32))[0] == 0
        assert_same_engine(back, twin, drv, used, False)


def _code(fn):
    try:
        fn()
        return 0, ""
    except A.AgrError as e:
        return e.code, str(e)


def test_refusals_leave_nothing_held(tmp_path):
    flags = P | M | V | R
    path, drv, used = source(tmp_path, flags, seed=18)
    hd, _, sec = parse(open(path, "rb").read())
    need_v, need_r = needs(hd, sec)
    window = int(hd["rows_used"] - hd["tail"])
    cases = [(kw(flags, window - 1), K.AGR_ENOSPC, "slab_rows"),
             (kw(flags, RING_ROWS, need_v - 1, RESP), K.AGR_ENOSPC, "vslab_bytes"),
             (kw(flags, RING_ROWS, VSLAB, need_r - 16), K.AGR_ENOSPC, "resp_bytes"),
             (kw(P | M | V, 1 << 12, VSLAB, RESP), K.AGR_EINVAL, "id mode"),                 # a ring into an append-only engine
             (kw(P | V | R, 600), K.AGR_EINVAL, "id mode"),
             (dict(kw(flags, 600), id_secret=SECRET + 1), K.AGR_EINVAL, "id_secret")]
    for cfg, code, word in cases:
        got = _code(lambda: A.Engine(restore_from=path, **cfg).close())
        assert got[0] == code and word in got[1], (cfg, got)
        with A.Engine(restore_from=path, **kw(flags, 600, 2 * VSLAB, 2 * RESP)) as back:
            assert back.verify()[1] == 0 and back.stats()["rows_used"] == used


def test_relocation_time_is_reported(tmp_path):
    flags = P | M | R
    path, _, _ = source(tmp_path, flags, seed=19)
    with A.Engine(restore_from=path, **kw(flags | K.AGR_CFG_TIMING, 1000)) as back:
        assert back.op_time(4) > 0
    with A.Engine(restore_from=path, **kw(flags | K.AGR_CFG_TIMING)) as same:
        with pytest.raises(A.AgrError):
            same.op_time(4)
