"""AGR_CFG_DELTA_SNAPSHOT: agr_snapshot writes a delta (AGRDELT1) on the engine's previous snapshot whenever it can, and
agr_restore follows a delta's parents back to the full file.  A plain reader (snapfile.py) applies each delta to the parsed sections
of its parent; at every step the result must be what a twin engine without the flags writes as a full file at the same point,
and the chain must restore to the twin's state."""
import os
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from jsoncase import make_requests, records_array, var_batch
from snapfile import BLOCK_ROWS, WORDS, apply, expected_blocks, parse, parse_delta, referenced
from test_snapshot_online_gpu import (AGENTS, MODES, RESP, RING_ROWS, VSLAB, Driver, PipeSnapshot, SECRET, STEP, T0, M, P, R, V,
                                      assert_same_engine, engine_kw, outcomes, submit_ingest, while_writing)

pytestmark = pytest.mark.gpu

DELTA_FLAGS = K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT


def delta_kw(flags):
    kw = engine_kw(flags, True)
    kw["flags"] |= K.AGR_CFG_DELTA_SNAPSHOT
    return kw


def assert_same_sections(hd, agents, sec, hd_t, agents_t, sec_t, var):
    assert hd.tobytes() == hd_t.tobytes()
    assert agents == agents_t
    for name in WORDS + ("completed_log", "failed_log"):
        assert np.array_equal(sec[name], sec_t[name]), name
    slab_m, resp_m, live = referenced(sec_t, hd_t, var)
    assert np.array_equal(sec["slab"][slab_m], sec_t["slab"][slab_m])
    assert np.array_equal(sec["resp"][resp_m], sec_t["resp"][resp_m])


def traffic(drv, engines, step, combine, ttl=3 * STEP):
    """One round of calls, the same on every engine: a batch, completions with bytes, errors into the failed log, expiry
    (and in ring modes release), at step 2 a dropped and a new agent, and tickets with AGR_CFG_COMBINE."""
    rnd = drv.round + step
    now = T0 + rnd * STEP
    state = drv.rng.bit_generator.state
    for eng in engines:
        drv.rng.bit_generator.state = state
        rows, _ = drv.batch([eng], 20, rnd)
        drv.complete([eng], rows, now, 60)
        eng.expire(now, ttl)
        if drv.ring:
            eng.reclaim()
            eng.reclaim_async()
        if step == 2:
            eng.drop_agent(AGENTS[1])
            eng.set_agent_state("agent-new-%d" % step, "running")
        if combine:
            recs = records_array(make_requests(90 + step, 8, AGENTS))
            tickets = [submit_ingest(eng, recs[k: k + 1]) for k in range(8)]
            assert [eng.wait(t) for t in tickets] == [0] * 8


def read(p):
    with open(p, "rb") as f:
        return f.read()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_chain_equals_the_twin_and_restores_like_it(mode, tmp_path):
    flags = MODES[mode]
    var, ring, combine = bool(flags & V), bool(flags & R), bool(flags & K.AGR_CFG_COMBINE)
    drv = Driver(flags, seed=9)
    with A.Engine(**delta_kw(flags)) as eng, A.Engine(**engine_kw(flags, False)) as twin:
        drv.build([eng, twin], 6 if ring else 2)
        p0, t0 = str(tmp_path / "s0.snap"), str(tmp_path / "t0.snap")
        eng.snapshot(p0)
        twin.snapshot(t0)
        data = read(p0)
        assert data[:8] == b"AGRSNAP3"
        hd, agents, sec = parse(data)
        assert_same_sections(hd, agents, sec, *parse(read(t0)), var)
        prev_t = parse(read(t0))
        last = p0
        for step in (1, 2, 3):
            p, tp = str(tmp_path / ("s%d.snap" % step)), str(tmp_path / ("t%d.snap" % step))
            if step == 2:                                           # written into a pipe while traffic goes on
                traffic(drv, [eng, twin], step, combine)
                twin.snapshot(tp)
                snap = PipeSnapshot(eng, tmp_path)
                rng = drv.rng.bit_generator.state                   # the twin gets the same calls once the file is written
                # (a TTL that keeps the rows of steps 1 and 2: they stay live in the parent files of the last delta)
                while_writing(snap, lambda: traffic(drv, [eng], 10, combine, 12 * STEP))
                blob = snap.drain()
                with open(p, "wb") as f:
                    f.write(blob)
                drv.rng.bit_generator.state = rng
                traffic(drv, [twin], 10, combine, 12 * STEP)
                # the pipe's name is the parent of the next delta: put the bytes there
                os.replace(p, snap.path)
                p = snap.path
            else:
                traffic(drv, [eng, twin], step, combine)
                eng.snapshot(p)
                twin.snapshot(tp)
            d = parse_delta(read(p))
            assert d["parent"] == os.path.realpath(last)
            hd_t, agents_t, sec_t = parse(read(tp))
            sec = apply(sec, d)
            assert_same_sections(d["hd"], d["agents"], sec, hd_t, agents_t, sec_t, var)
            wl, ll = expected_blocks(prev_t[2], prev_t[0], sec_t, hd_t)
            assert d["wl"].tolist() == wl, step
            assert [x.tolist() for x in d["ll"]] == ll, step
            assert len(wl) < (len(sec_t["state"]) + BLOCK_ROWS - 1) // BLOCK_ROWS or len(sec_t["state"]) <= 2 * BLOCK_ROWS
            prev_t, last = (hd_t, agents_t, sec_t), p
        used = int(prev_t[0]["rows_used"])
        kw = engine_kw(flags, False)
        with A.Engine(restore_from=last, **kw) as back, A.Engine(restore_from=tp, **kw) as want:
            assert_same_engine(back, want, drv, used, var)
            if not (flags & M):                                     # hash ids: a replay of an id stored before the last delta
                parent_used = int(parse_delta(read(last))["dh"]["rows_lo"])
                L = min(L for L, (a, rid) in drv.ids.items() if L < parent_used and back.get_record_json(a, rid) is not None)
                a, rid = drv.ids[L]
                r = make_requests(77, 1, [a])[0]
                r.rid, r.now = rid, T0 + (drv.round + 20) * STEP
                got = []
                for e in (back, want):
                    v = np.zeros(1, dtype=A.verdict_dtype)
                    e.ingest_ex(records_array([r]), v, np.zeros((1, 16), dtype=np.uint8))
                    got.append(int(v[0]["flags"]))
                assert got[0] == got[1] and got[0] & K.AGR_VF_DUP_ID and not got[0] & K.AGR_VF_STORED, got


# ---- the policy: a delta when it pays, a full file otherwise
def _small_engine(extra=0):
    eng = A.Engine(slab_rows=1 << 12, max_agents=16, id_secret=SECRET, flags=P | M | DELTA_FLAGS | extra)
    for a in AGENTS:
        eng.set_agent_state(a, "running")
    return eng


def _ingest(eng, seed, n, now=T0):
    reqs = make_requests(seed, n, AGENTS)
    for r in reqs:
        r.now = now
    ids = np.zeros((n, 16), dtype=np.uint8)
    first = eng.ingest_ex(records_array(reqs), np.zeros(n, dtype=A.verdict_dtype), ids)
    return first, reqs, ids


def test_policy(tmp_path):
    with _small_engine() as eng:
        _ingest(eng, 1, 300)
        a = str(tmp_path / "a.snap")
        eng.snapshot(a)
        assert read(a)[:8] == b"AGRSNAP3"                        # nothing to build on
        _ingest(eng, 2, 10)
        b = str(tmp_path / "b.snap")
        eng.snapshot(b)
        assert read(b)[:8] == b"AGRDELT1"                        # a small change
        assert len(read(b)) < len(read(a)) // 10
        _ingest(eng, 3, 10)
        other = os.path.join(str(tmp_path), ".", "sub", "..", "b.snap")
        os.mkdir(os.path.join(str(tmp_path), "sub"))
        assert other != b and os.path.realpath(other) == os.path.realpath(b)
        eng.snapshot(other)                                      # a file of the chain, under another spelling
        assert read(b)[:8] == b"AGRSNAP3"
        _ingest(eng, 4, 10)
        c = str(tmp_path / "c.snap")
        eng.snapshot(c)
        assert read(c)[:8] == b"AGRDELT1" and parse_delta(read(c))["parent"] == os.path.realpath(b)
        # traffic that rewrites every row's words each time: the deltas add up to a full file within ~10 snapshots
        _, reqs, ids = _ingest(eng, 10, 800, T0 + STEP)
        kinds = []
        for k in range(12):
            ops = [(bytes(ids[i]), reqs[i].agent_id, K.AGR_OUT_RESPONSE, 200, T0 + (k + 2) * STEP) for i in range(800)]
            eng.complete_ex(outcomes(ops), [b""] * 800)
            p = str(tmp_path / ("big%d.snap" % k))
            eng.snapshot(p)
            kinds.append(read(p)[:8])
            if kinds[-1] == b"AGRSNAP3":
                break
        assert kinds[0] == b"AGRDELT1" and kinds[-1] == b"AGRSNAP3", kinds
        with A.Engine(restore_from=p, slab_rows=1 << 12, max_agents=16, flags=P | M) as back:
            assert back.verify()[1] == 0 and back.stats()["rows_used"] == eng.stats()["rows_used"]


def test_failed_write_gives_a_full_file_and_leaves_no_pin(tmp_path):
    with A.Engine(slab_rows=512, max_agents=16, resp_bytes=16 << 10, id_secret=SECRET, flags=P | M | R | DELTA_FLAGS) as eng:
        for a in AGENTS:
            eng.set_agent_state(a, "running")
        _ingest(eng, 1, 200)
        eng.snapshot(str(tmp_path / "a.snap"))
        _ingest(eng, 2, 200)                                     # a delta larger than the pipe holds
        fifo = str(tmp_path / "dead.fifo")
        os.mkfifo(fifo)
        err = {}

        def run():
            try:
                eng.snapshot(fifo)
            except A.AgrError as e:
                err["e"] = e
        t = threading.Thread(target=run, daemon=True)
        t.start()
        f = open(fifo, "rb", buffering=0)
        f.read(8)
        f.close()                                                # the reader goes away: the write fails
        t.join(120)
        assert not t.is_alive() and "e" in err
        # no pin is left: the whole ring can be released and refilled
        eng.expire(T0 + 100 * STEP, STEP)
        eng.reclaim()
        for k in range(3):
            _ingest(eng, 20 + k, 200, T0 + 200 * STEP)
            eng.expire(T0 + 300 * STEP, STEP)
            eng.reclaim()
        p = str(tmp_path / "after.snap")
        eng.snapshot(p)
        assert read(p)[:8] == b"AGRSNAP3"


# ---- refusals
def test_refusals(tmp_path):
    with pytest.raises(A.AgrError) as e:
        A.Engine(slab_rows=1 << 12, flags=P | M | K.AGR_CFG_DELTA_SNAPSHOT)
    assert e.value.code == K.AGR_EINVAL and "ONLINE" in str(e.value)
    kw = dict(slab_rows=1 << 12, max_agents=16, flags=P | M)
    with _small_engine() as eng:
        _ingest(eng, 1, 300)
        a, b, c = (str(tmp_path / n) for n in ("a.snap", "b.snap", "c.snap"))
        eng.snapshot(a)
        _ingest(eng, 2, 30)
        eng.snapshot(b)
        _ingest(eng, 3, 30)
        eng.snapshot(c)
        assert read(c)[:8] == b"AGRDELT1"
        with A.Engine(restore_from=c, **kw) as back:
            assert back.verify()[1] == 0
        full_a = read(a)
        # truncated delta
        data = read(c)
        with open(c, "wb") as f:
            f.write(data[:-5])
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=c, **kw)
        assert e.value.code == K.AGR_EINVAL and "truncated" in str(e.value)
        with open(c, "wb") as f:
            f.write(data)
        # a parent replaced by another snapshot of the same engine
        with _small_engine() as other:
            _ingest(other, 1, 300)
            _ingest(other, 9, 5)
            other.snapshot(a)
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=c, **kw)
        assert e.value.code == K.AGR_EINVAL and "digest" in str(e.value)
        # a missing parent
        os.remove(a)
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=c, **kw)
        assert e.value.code == K.AGR_EINVAL and "parent" in str(e.value) and "a.snap" in str(e.value)
        with open(a, "wb") as f:
            f.write(full_a)
        # another id mode / record form
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=c, slab_rows=1 << 12, max_agents=16, flags=P)
        assert e.value.code == K.AGR_EINVAL
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=c, slab_rows=1 << 12, max_agents=16, flags=P | M | V)
        assert e.value.code == K.AGR_EINVAL
        with A.Engine(restore_from=c, **kw) as back:              # and the chain still restores
            assert back.verify()[1] == 0


# ---- a restored engine continues its chain
@pytest.mark.parametrize("mode", sorted(MODES))
def test_restart_continues_the_chain(mode, tmp_path):
    flags = MODES[mode]
    var, combine = bool(flags & V), bool(flags & K.AGR_CFG_COMBINE)
    drv = Driver(flags, seed=11)
    kw = engine_kw(flags, False)
    with A.Engine(**kw) as twin:
        with A.Engine(**delta_kw(flags)) as eng:
            drv.build([eng, twin], 4 if drv.ring else 2)
            a, b = str(tmp_path / "a.snap"), str(tmp_path / "b.snap")
            eng.snapshot(a)
            traffic(drv, [eng, twin], 1, combine)
            eng.snapshot(b)
            assert read(b)[:8] == b"AGRDELT1"
        with A.Engine(restore_from=b, **delta_kw(flags)) as eng:
            traffic(drv, [eng, twin], 2, combine)
            c = str(tmp_path / "c.snap")
            eng.snapshot(c)
        d = parse_delta(read(c))
        assert d["parent"] == os.path.realpath(b)
        t = str(tmp_path / "t.snap")
        twin.snapshot(t)
        hd_t = parse(read(t))[0]
        assert d["hd"].tobytes() == hd_t.tobytes()
        with A.Engine(restore_from=c, **kw) as back, A.Engine(restore_from=t, **kw) as want:
            assert_same_engine(back, want, drv, int(hd_t["rows_used"]), var)


# ---- rows reserved before a cut and ingested after it (agr_reserve_rows / agr_fill_rows take fixed-size records)
@pytest.mark.parametrize("mode", ["hash", "mint", "ring", "ring_combine"])
def test_rows_reserved_across_a_cut(mode, tmp_path):
    flags = MODES[mode]
    ring = bool(flags & R)
    with A.Engine(**delta_kw(flags)) as eng:
        for a in AGENTS:
            eng.set_agent_state(a, "running")
        _ingest(eng, 1, 100)
        first = eng.reserve_rows(16)
        eng.snapshot(str(tmp_path / "a.snap"))
        reqs = make_requests(5, 16, AGENTS)
        for k, r in enumerate(reqs):                             # the first 8 are old enough to expire below
            r.now = T0 if k < 8 else T0 + 10 * STEP
        eng.fill_rows(first, records_array(reqs))
        eng.ingest_rows(first, 16)
        if ring:                                                 # the tail moves past the parent's ingested bound
            eng.expire(T0 + 10 * STEP, 5 * STEP)
            eng.reclaim()
            assert eng.stats()["rows_tail"] == first + 8
        _ingest(eng, 2, 10, T0 + 10 * STEP)
        p = str(tmp_path / "b.snap")
        eng.snapshot(p)
        d = parse_delta(read(p))
        lo = first + 8 if ring else first
        assert int(d["dh"]["rows_lo"]) == lo
        kw = engine_kw(flags, False)
        with A.Engine(restore_from=p, **kw) as back:
            assert back.verify()[1] == 0
            got, want = back.rows_json(lo, first + 16 - lo), eng.rows_json(lo, first + 16 - lo)
            assert got[0] == want[0] and len(got[0]) > (first + 16 - lo) * 100


# ---- the three rings wrap inside one delta
class Twins:
    """The delta engine and a twin without the flags, driven by the same calls; ids[logical row] = (agent, Request.ID)."""

    def __init__(self, flags):
        self.flags, self.var = flags, bool(flags & V)
        self.eng, self.twin = A.Engine(**delta_kw(flags)), A.Engine(**engine_kw(flags, False))
        self.both = (self.eng, self.twin)
        self.ids, self.seed, self.clock = {}, 100, T0
        for e in self.both:
            for a in AGENTS:
                e.set_agent_state(a, "running")

    def close(self):
        for e in self.both:
            e.close()

    def rows(self, n, body=300):
        self.seed += 1
        reqs = make_requests(self.seed, n, AGENTS)
        for r in reqs:
            r.now = self.clock
            if self.var:
                r.path, r.headers, r.body = b"/x", {}, bytes(body)
        got = []
        for e in self.both:
            if self.var:
                _, ids, first = e.ingest_var(*var_batch(reqs))
            else:
                ids = np.zeros((n, 16), dtype=np.uint8)
                first = e.ingest_ex(records_array(reqs), np.zeros(n, dtype=A.verdict_dtype), ids)
            got.append((first, ids.tobytes()))
        assert got[0] == got[1]
        first, ids = got[0][0], np.frombuffer(got[0][1], dtype=np.uint8).reshape(n, 16)
        for k, r in enumerate(reqs):
            self.ids[first + k] = (r.agent_id, bytes(ids[k]))
        return first

    def resp(self, n):
        L = self.rows(1, 100)
        a, rid = self.ids[L]
        for e in self.both:
            assert e.store_response(a, rid, b"", bytes((L + k) & 255 for k in range(n)))

    def release(self):
        self.clock += 100 * STEP
        for e in self.both:
            e.expire(self.clock, STEP)
            e.reclaim()

    def cursors(self, tmp_path):
        """(rows_used, vused, resp_used) of the twin: the header of a blocking snapshot."""
        p = str(tmp_path / "probe.snap")
        self.twin.snapshot(p)
        hd = parse(read(p))[0]
        return int(hd["rows_used"]), int(hd["vused"]), int(hd["resp_used"])


def _bring(t, tmp_path, which, cap, lo, hi, step):
    """Releases everything and appends (rows, record bytes or response bytes) until the cursor's place in its lap is in
    [lo, hi); a piece that does not fit before the end of the lap wraps to its start."""
    for _ in range(200):
        t.release()
        pos = t.cursors(tmp_path)[which] % cap
        if lo <= pos < hi:
            return
        n = min(step, (lo - pos) if pos < lo else (cap - pos))
        if which == 0:
            t.rows(max(1, n))
        elif which == 1:
            t.rows(1, max(0, min(n, 8000) - 120))
        else:
            t.resp(max(16, n - 32))
    pytest.fail("cursor %d did not reach [%d, %d)" % (which, lo, hi))


@pytest.mark.parametrize("mode", ["ring", "var_ring", "ring_combine"])
def test_rings_wrap_inside_one_delta(mode, tmp_path):
    flags = MODES[mode]
    t = Twins(flags)
    try:
        S, VC, RC = RING_ROWS, VSLAB, RESP
        if t.var:
            _bring(t, tmp_path, 1, VC, VC - 24000, VC - 12000, 8000)
        else:
            _bring(t, tmp_path, 0, S, S - 90, S - 60, 100)
        _bring(t, tmp_path, 2, RC, RC - 6000, RC - 3000, 8000)
        t.release()
        p0, p1, t1 = (str(tmp_path / n) for n in ("s0.snap", "s1.snap", "t1.snap"))
        t.eng.snapshot(p0)
        assert read(p0)[:8] == b"AGRSNAP3"
        # past the end of every ring, nothing released in between
        if t.var:
            for _ in range(4):
                t.rows(1, 7800)
        else:
            t.rows(100)
        t.resp(4000)
        t.resp(4000)
        t.eng.snapshot(p1)
        t.twin.snapshot(t1)
        d = parse_delta(read(p1))
        assert len(d["rows"]) == 2 and len(d["resp"]) == 2, (d["rows"], d["resp"])
        assert d["rows"][1][0] == 0 and d["resp"][1][0] == 0
        hd0, agents0, sec0 = parse(read(p0))
        hd_t, agents_t, sec_t = parse(read(t1))
        sec = apply(sec0, d)
        assert_same_sections(d["hd"], d["agents"], sec, hd_t, agents_t, sec_t, t.var)
        slab_m, resp_m, live = referenced(sec_t, hd_t, t.var)
        assert slab_m[: 512].any() and resp_m[: 512].any()             # live bytes at the start of both rings
        kw = engine_kw(flags, False)
        with A.Engine(restore_from=p1, **kw) as back:
            assert back.verify()[1] == 0
            used = int(hd_t["rows_used"])
            for L, (a, rid) in t.ids.items():
                if L < used:
                    assert back.get_record_json(a, rid) == t.twin.get_record_json(a, rid), L
                    assert back.get_response_body(a, rid) == t.twin.get_response_body(a, rid), L
    finally:
        t.close()
