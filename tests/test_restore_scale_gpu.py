"""Snapshot and restore at scale against plain references: the relocation of a restore into other capacities across its
tiles and its scan's rounds (resizeref.relocate), the delta files' block lists, digests and staging chunks (snapfile), and
the dedupe index a restore rebuilds in hash-id mode (k1ref.Ref.restore).  Engines are filled on the device in bulk; each
restore is snapshotted again and the file is compared with the reference section by section."""
import copy

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from k1ref import Ref, hash_id
from resizeref import relocate
from snapfile import HEADER, LOGS, WORDS, apply, digest, expected_blocks, parse, parse_delta, referenced, sections

pytestmark = pytest.mark.gpu

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
ONLINE_DELTA = K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT
SECRET = 0x5EED_1234_ABCD_0019
SEC = 1_000_000_000
T0, STEP = 1_700_000_000 * SEC, 3600 * SEC
AGENTS = ["agent-scale-0", "agent-scale-1", "agent-scale-2", "agent-scale-3", "agent-scale-drop"]
NOBODY = len(AGENTS)                                  # an agent index that names no agent: the row is not found (state 0)
NAMES = np.array([a.encode() for a in AGENTS] + [b"agent-nobody"], dtype="S32")
TILE = 2048                                           # RL_TILE: rows per CTA of the relocation's row kernels
CARRY = TILE * 256                                    # k_rl_scan carries its totals into a second round past this many rows
SEGS = np.array([0, 1, 15, 16, 17, 511, 4097])       # response / error lengths; RL_CHUNK (16 KiB) boundaries fall inside them
BLOCK = 256


def r16(x):
    return (np.asarray(x, dtype=np.int64) + 15) & ~15


def read(p):
    with open(p, "rb") as f:
        return f.read()


class Rig:
    """One engine, filled in bulk: logical row -> (agent index, Request.ID) in arrays."""

    def __init__(self, flags, slab_rows, *, vcap=0, resp=8 << 20, max_batch=0, restore_from=None, seed=0):
        self.flags, self.var, self.mint = flags, bool(flags & V), bool(flags & M)
        self.kw = dict(slab_rows=slab_rows, max_agents=16, id_secret=SECRET, flags=flags, vslab_bytes=vcap if flags & V else 0,
                       resp_bytes=resp, max_batch=max_batch or min(slab_rows, 1 << 16))
        self.eng = A.Engine(restore_from=restore_from, **self.kw)
        self.batch = max(1, min(self.eng.max_batch, slab_rows // 4))
        self.slab_rows, self.next = slab_rows, 0                    # next: the row the next batch starts at
        self.rng = np.random.default_rng(seed)
        self.first, self.agent, self.ids = [], [], []
        if restore_from is None:
            for a in AGENTS:
                self.eng.set_agent_state(a, "running")

    def close(self):
        self.eng.close()

    def rows(self):
        """(logical rows, agent index, ids) of every row added, in arrival order"""
        L = np.concatenate([f + np.arange(len(a)) for f, a in zip(self.first, self.agent)]) if self.first else np.zeros(0, np.int64)
        return L, np.concatenate(self.agent), np.concatenate(self.ids)

    def records(self, agent, ids, seq, plen):
        n = len(agent)
        recs = np.zeros(n, dtype=A.record_dtype)
        recs["request_id"] = ids
        recs["agent_id"] = NAMES[agent]
        recs["seq"] = seq
        recs["flags"] = 2 << K.AGR_F_METHOD_SHIFT
        recs["path_len"], recs["hdr_len"], recs["body_len"] = 2, 0, plen - 2
        recs["status"], recs["max_retries"] = K.AGR_ST_PENDING, 3
        recs["payload"] = np.frombuffer(self.rng.bytes(n * 416), dtype=np.uint8).reshape(n, 416)
        recs["payload"][:, :2] = np.frombuffer(b"/x", dtype=np.uint8)
        return recs

    def ingest(self, recs, plen):
        """one batch of records (fixed stride: reserve, fill, K1 over the rows; variable length: agr_ingest_var of the records'
        first 96 + plen bytes); returns (first row, verdicts, ids)"""
        n = len(recs)
        if self.var:
            size = 96 + r16(plen)
            offs = np.zeros(n + 1, dtype=np.uint32)
            offs[1:] = np.cumsum(size)
            blob = np.zeros(int(offs[-1]), dtype=np.uint8)
            raw = recs.view(np.uint8).reshape(n, 512)
            width = int(size.max())
            at = offs[:-1, None].astype(np.int64) + np.arange(width)
            keep = np.arange(width) < size[:, None]
            blob[at[keep]] = raw[:, :width][keep]
            out, ids, first = self.eng.ingest_var(blob, offs)
        else:
            first = self.eng.reserve_rows(n)
            self.eng.fill_rows(first, recs)
            out = self.eng.ingest_rows(first, n)
            ids = self.eng.mint_ids(first, n) if self.mint else recs["request_id"].copy()
        return first, out, ids

    def add(self, agent, ids=None, seq=T0, plen=None):
        """rows for agent indices `agent` (caller ids `ids` unless minted), in batches; returns (first row, verdicts)"""
        n = len(agent)
        agent = np.asarray(agent, dtype=np.int64)
        ids = np.zeros((n, 16), np.uint8) if ids is None else np.asarray(ids, dtype=np.uint8)
        seq = np.broadcast_to(np.asarray(seq, dtype=np.uint64), (n,))
        plen = self.rng.integers(2, 60, n) if plen is None else np.broadcast_to(plen, (n,))
        first0, verdicts = None, []
        k = 0
        while k < n:
            # a ring hands a batch out in one physical run: batches end at the ring's end, so that no row is skipped there
            m = min(n - k, self.batch, self.slab_rows - self.next % self.slab_rows if self.flags & R else n)
            j = slice(k, k + m)
            k += m
            first, out, got = self.ingest(self.records(agent[j], ids[j], seq[j], plen[j]), plen[j])
            self.next = first + m
            first0 = first if first0 is None else first0
            self.first.append(first); self.agent.append(agent[j]); self.ids.append(np.asarray(got, dtype=np.uint8))
            verdicts.append(out)
        return first0, np.concatenate(verdicts)

    def outcomes(self, agent, ids, kind, t):
        outs = np.zeros(len(agent), dtype=A.outcome_dtype)
        outs["request_id"], outs["agent_id"] = ids, NAMES[agent]
        outs["kind"], outs["http_status"], outs["seq"] = kind, 200 if kind == K.AGR_OUT_RESPONSE else 0, t
        return outs

    def complete(self, agent, ids, kind, lens, t):
        """completions of these rows in batches, each with a segment of lens[k] random bytes (a response's first bytes are its
        header when it has more than 8)"""
        lens = np.broadcast_to(np.asarray(lens, dtype=np.int64), (len(agent),))
        for k in range(0, len(agent), self.batch):
            j = slice(k, k + self.batch)
            ln = lens[j]
            offs = np.zeros(len(ln) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum(ln)
            blob = np.frombuffer(self.rng.bytes(max(int(offs[-1]), 1)), dtype=np.uint8).copy()
            hl = np.where(ln > 8, 5, 0).astype(np.uint32) if kind == K.AGR_OUT_RESPONSE else None
            rc, res = self.eng.complete_ex(self.outcomes(agent[j], ids[j], kind, t), (blob, offs), hl)
            assert rc == 0 and (res == 0).all(), (rc, np.unique(res))

    def snapshot(self, path):
        self.eng.snapshot(str(path))
        return str(path)


def assert_file(got, want, var, what=""):
    """a parsed full file against the reference one: header, agent table, every per-row word and log, the referenced bytes"""
    (hd_g, ag_g, sec_g), (hd_w, ag_w, sec_w) = got, want
    assert hd_g.tobytes() == np.array(hd_w, dtype=HEADER).tobytes(), (what, hd_g, hd_w)
    assert ag_g == ag_w, what
    for name in WORDS + LOGS:
        a, b = sec_g[name], sec_w[name]
        if not np.array_equal(a, b):
            bad = np.nonzero(a != b)[0] if len(a) == len(b) else None
            pytest.fail("%s %s: %s" % (what, name, "length %d != %d" % (len(a), len(b)) if bad is None else
                                       "%d rows differ, first %s: %s != %s" % (len(bad), bad[:4], a[bad[:4]], b[bad[:4]])))
    slab_m, resp_m, _ = referenced(sec_w, hd_w, var)
    assert np.array_equal(sec_g["slab"][slab_m], sec_w["slab"][slab_m]), what
    assert np.array_equal(sec_g["resp"][resp_m], sec_w["resp"][resp_m]), what


def snap_of(eng, path):
    eng.snapshot(str(path))
    return parse(read(path))


def same_reads(back, src, L, agent, ids, k=300, seed=0):
    """get_record_json / get_response_body of a sample of rows (first, last and random ones) on both engines"""
    rng = np.random.default_rng(seed)
    pick = np.unique(np.concatenate([[0, len(L) - 1], rng.integers(0, len(L), k)])) if len(L) else []
    for i in pick:
        a = AGENTS[agent[i]] if agent[i] < NOBODY else "agent-nobody"
        rid = bytes(ids[i])
        assert back.get_record_json(a, rid) == src.get_record_json(a, rid), int(L[i])
        assert back.get_response_body(a, rid) == src.get_response_body(a, rid), int(L[i])


# ------------------------------------------------------------------------------------------------ relocation
def fill_window(rig, window, seed):
    """window rows: every 7th not found, some of a fourth agent that is dropped at the end; completions with responses and
    errors of SEGS lengths spread over the whole window (and every row of the first tiles), a few hundred rows failed for
    good; the completed log then holds AGR_RID_NONE entries of the dropped agent"""
    rng = np.random.default_rng(seed)
    agent = rng.integers(0, 4, window)
    agent[np.arange(window) % 7 == 3] = NOBODY
    agent[np.arange(window) % 11 == 5] = 4
    ids = None if rig.mint else np.frombuffer(rng.bytes(16 * window), dtype=np.uint8).reshape(window, 16)
    first, v = rig.add(agent, ids, seq=T0)
    L, ag, rid = rig.rows()
    found = ag < NOBODY
    near = np.zeros(window, dtype=bool)
    near[: 3 * TILE] = True
    near[rng.integers(0, window, 2500)] = True
    near &= found
    sel = np.nonzero(near)[0]
    err = sel[rng.random(len(sel)) < 0.4]
    rig.complete(ag[err], rid[err], K.AGR_OUT_ERROR, SEGS[rng.integers(0, len(SEGS), len(err))], T0 + STEP)
    resp = sel[rng.random(len(sel)) < 0.6]
    rig.complete(ag[resp], rid[resp], K.AGR_OUT_RESPONSE, SEGS[rng.integers(0, len(SEGS), len(resp))], T0 + 2 * STEP)
    gone = np.setdiff1d(sel, resp)[:400]
    for k in range(3):                                              # three errors: out of retries, into the failed log
        rig.complete(ag[gone], rid[gone], K.AGR_OUT_ERROR, 17 + k, T0 + (3 + k) * STEP)
    rig.eng.drop_agent(AGENTS[4])
    return first


def geometry(window, where):
    """(source slab_rows, first row id) of a window whose tail lies at physical row 0, in the middle of the ring, or so that
    the window wraps the ring's end"""
    S = window + window // 2 + 1000 + (window & 1)
    start = {"at_0": 3 * S, "middle": 2 * S + (S - window) // 2, "wraps": 2 * S - window // 2 - 1}[where]
    return S, start


def source(tmp_path, flags, window, where, seed):
    S, start = geometry(window, where)
    var = bool(flags & V)
    rig = Rig(flags, S, vcap=(S + 16) * 192, resp=64 << 20, seed=seed)
    rig.eng.skip_arrivals(start)
    rig.next = start
    fill_window(rig, window, seed)
    path = rig.snapshot(tmp_path / "src.snap")
    hd, ag, sec = parse(read(path))
    assert int(hd["tail"]) == start and int(hd["rows_used"]) == start + window
    if where == "wraps" and window > 1:
        assert start % S + window > S
    elif where == "at_0":
        assert start % S == 0
    _, _, packed = relocate(hd, ag, sec, flags, window, 1 << 40, 1 << 40)
    need = (len(packed["slab"]) if var else 0, len(packed["resp"]))
    return rig, path, (hd, ag, sec), need


def check_relocation(rig, path, src, need, tmp_path, S_t, spare, tag):
    flags, var = rig.flags, rig.var
    hd, ag, sec = src
    vcap, rcap = need[0] + spare, need[1] + spare
    want = relocate(hd, ag, sec, flags, S_t, vcap, rcap)
    back = Rig(flags, S_t, vcap=vcap, resp=rcap, restore_from=path)
    try:
        assert back.eng.verify()[1] == 0
        assert_file(snap_of(back.eng, tmp_path / ("after_%s.snap" % tag)), want, var, tag)
        same_reads(back.eng, rig.eng, *rig.rows())
    finally:
        back.close()


SMALL_WINDOWS = [1, TILE - 1, TILE, TILE + 1]


@pytest.mark.parametrize("where", ["at_0", "middle", "wraps"])
@pytest.mark.parametrize("window", SMALL_WINDOWS)
@pytest.mark.parametrize("mode", ["fixed_mint", "fixed_hash", "var_mint", "var_hash"])
def test_relocation_tile_edges(mode, window, where, tmp_path):
    flags = P | R | (V if mode.startswith("var") else 0) | (M if mode.endswith("mint") else 0)
    rig, path, src, need = source(tmp_path, flags, window, where, seed=window + len(where))
    try:
        S = int(src[0]["slab_rows"])
        for S_t, tag in ((2 * S + 5, "bigger"), (window + 3, "smaller"), (window + 1001, "npot")):
            check_relocation(rig, path, src, need, tmp_path, S_t, 48, tag)
    finally:
        rig.close()


def assert_refusals(path, flags, window, need):
    """AGR_ENOSPC one row and one byte under what the live window takes, and a restore at exactly that size"""
    var = bool(flags & V)
    cases = [(window - 1, need[0] + 16, need[1] + 16, "slab_rows"), (window, need[0] + 16, need[1] - 1, "resp_bytes")]
    if var:
        cases.append((window, need[0] - 1, need[1] + 16, "vslab_bytes"))
    for S_t, vc, rc, word in cases:
        with pytest.raises(A.AgrError) as e:
            A.Engine(restore_from=path, slab_rows=S_t, max_agents=16, id_secret=SECRET, flags=flags,
                     vslab_bytes=vc if var else 0, resp_bytes=rc)
        assert e.value.code == K.AGR_ENOSPC and word in str(e.value), (word, str(e.value))


@pytest.mark.parametrize("window", [CARRY - 1, CARRY, CARRY + 1])
@pytest.mark.parametrize("mode", ["var_hash", "fixed_mint"])
def test_relocation_scan_carry(mode, window, tmp_path):
    """windows around 256 tiles, the first that k_rl_scan takes in two rounds; the fixed-stride form runs the carry itself
    (2^19 + 1 rows) only, the variable-length form all three"""
    if mode == "fixed_mint" and window != CARRY + 1:
        pytest.skip("the fixed-stride form runs the carry case only")
    flags = P | R | (V | 0 if mode == "var_hash" else M)
    rig, path, src, need = source(tmp_path, flags, window, "wraps", seed=window % 97)
    try:
        assert need[1] > 4 * 16384
        check_relocation(rig, path, src, need, tmp_path, window + 12345, 0, "npot")   # byte rings exactly full
        if window == CARRY + 1:
            assert_refusals(path, flags, window, need)
    finally:
        rig.close()


# ------------------------------------------------------------------------------------------------ delta files
def per_chunk(max_batch, var):
    """word blocks per staging chunk of a delta's writer and of its restore: snap_stage_bytes / rec_bytes"""
    stage = max(min(max_batch * 512, 32 << 20), 1 << 20)
    return stage // (BLOCK * (64 + (12 if var else 0)))


class DeltaPair:
    """An engine that writes delta files and a twin without the flags, driven by the same calls; the twin's full file at
    each cut is what the chain must hold."""

    def __init__(self, flags, slab_rows, tmp_path):
        var = bool(flags & V)
        kw = dict(vcap=slab_rows * 192, resp=16 << 20, max_batch=2048)
        self.d, self.t = Rig(flags | ONLINE_DELTA, slab_rows, seed=1, **kw), Rig(flags, slab_rows, seed=1, **kw)
        self.flags, self.var, self.tmp, self.k = flags, var, tmp_path, 0
        self.files, self.fulls, self.digests = [], [], []

    def both(self, fn):
        st = [r.rng.bit_generator.state for r in (self.d, self.t)]
        assert st[0] == st[1]
        for r in (self.d, self.t):
            fn(r)

    def cut(self):
        """a snapshot of both; checks the delta against the twin's consecutive full files and digests"""
        p, tp = self.tmp / ("d%d.snap" % self.k), self.tmp / ("t%d.snap" % self.k)
        self.k += 1
        self.d.snapshot(p)
        self.t.snapshot(tp)
        full = parse(read(tp))
        dg = digest(full[0], full[2], SECRET)
        data = read(p)
        if self.files:
            assert data[:8] == b"AGRDELT1"
            d = parse_delta(data)
            assert tuple(int(x) for x in d["dh"]["digest"]) == dg
            assert tuple(int(x) for x in d["dh"]["parent_digest"]) == self.digests[-1]
            prev = self.fulls[-1]
            wl, ll = expected_blocks(prev[2], prev[0], full[2], full[0])
            got = (d["wl"].tolist(), [x.tolist() for x in d["ll"]])
            assert got == (wl, ll), (self.k, got, (wl, ll))
            sec = apply(self.chain, d)
            assert_file((d["hd"], d["agents"], sec), full, self.var, "delta %d" % self.k)
            self.chain = sec
        else:
            assert data[:8] == b"AGRSNAP3"
            self.chain = parse(data)[2]
            wl, ll = None, None
        self.files.append(str(p)); self.fulls.append(full); self.digests.append(dg)
        return wl, ll


@pytest.mark.parametrize("mode", ["ring", "var_ring", "append", "var_append"])
def test_delta_blocks_digests_and_chunks(mode, tmp_path):
    ring, var = "ring" in mode, mode.startswith("var")
    flags = P | M | (R if ring else 0) | (V if var else 0)
    n = (1 << 18) + 3                                               # R mod 4 = 3: every section ends in a short piece
    pair = DeltaPair(flags, n + (1 << 14) if ring else n + 4096, tmp_path)
    try:
        rng = np.random.default_rng(3)
        agent = rng.integers(0, 4, n)
        agent[:40] = 4                                              # the dropped agent's rows: early in the completed log
        pair.both(lambda r: r.add(agent, seq=T0 + 5 * STEP * (np.arange(n) >= 2048)))
        L, ag, ids = pair.d.rows()
        assert np.array_equal(ids, pair.t.rows()[2])
        rows = lambda r, idx: (ag[idx], ids[idx])
        done = np.nonzero(ag < 4)[0][:1500]                         # completions: the logs span two blocks and more
        pair.both(lambda r: r.complete(*rows(r, np.concatenate([np.arange(40), done])), K.AGR_OUT_RESPONSE, 5, T0 + STEP))
        assert len(pair.fulls) == 0
        pair.cut()
        nb = (n + BLOCK - 1) // BLOCK
        one = lambda i, kind=K.AGR_OUT_RESPONSE, ln=3: pair.both(lambda r: r.complete(*rows(r, np.array([i])), kind, ln, T0 + 2 * STEP))
        steps = [("first row of a block", lambda: one(700 * BLOCK), [700]),
                 ("last row of a block", lambda: one(900 * BLOCK + BLOCK - 1), [900]),
                 ("a completed row's times", lambda: one(done[-1], K.AGR_OUT_RESPONSE, 5), [int(done[-1]) // BLOCK]),
                 ("the short last piece", lambda: one(n - 1), [nb - 1]),
                 ("a dropped agent's log entries", lambda: pair.both(lambda r: r.eng.drop_agent(AGENTS[4])), None)]
        for what, fn, want in steps:
            fn()
            wl, ll = pair.cut()
            assert want is None or set(want) <= set(wl), (what, wl)
            a, b = pair.fulls[-2][2], pair.fulls[-1][2]
            changed = [w for w in WORDS if not np.array_equal(a[w], b[w])]
            if what.startswith("a completed"):                    # a second StoreResponse of the same length: 8-byte words only
                assert set(changed) <= {"resp_off", "ptime", "mtime"} and "mtime" in changed, changed
            if what.startswith("a dropped"):
                assert 0 in ll[0], (what, ll)                      # the entries rewritten lie in the log's first block
        # a block list longer than one staging chunk of the writer and of the restore, its short last block right after the
        # chunk boundary
        per = per_chunk(2048, var)
        blocks = np.arange(1, per + 1) * 3
        idx = np.concatenate([blocks * BLOCK + 7, [n - 2]])
        idx = idx[ag[idx] < 4]
        assert len(idx) == per + 1
        pair.both(lambda r: r.complete(*rows(r, idx), K.AGR_OUT_ERROR, 16, T0 + 3 * STEP))
        wl, _ = pair.cut()
        assert wl == sorted((idx // BLOCK).tolist()) and len(wl) == per + 1 and wl[-1] == nb - 1
        if ring:                                                   # a release compacts the logs; then they grow past the old length
            old = [len(pair.fulls[-1][2][x]) for x in LOGS]
            pair.both(lambda r: (r.eng.expire(T0 + 10 * STEP, 8 * STEP + STEP // 2), r.eng.reclaim()))
            pair.cut()
            assert len(pair.fulls[-1][2]["completed_log"]) < old[0] and int(pair.fulls[-1][0]["tail"]) > 0
            more = np.nonzero(ag < 4)[0][3000: 3000 + old[0] + 1200]
            pair.both(lambda r: r.complete(*rows(r, more), K.AGR_OUT_RESPONSE, 1, T0 + 11 * STEP))
            pair.cut()
            assert len(pair.fulls[-1][2]["completed_log"]) > old[0]
        last, full = pair.files[-1], pair.fulls[-1]
        S = int(full[0]["slab_rows"])
        for mb in (2048, 0):                                        # the restore's staging chunks: as small as the writer's, and large
            back = Rig(flags, S, vcap=S * 192, resp=16 << 20, max_batch=mb, restore_from=last)
            try:
                assert back.eng.verify()[1] == 0
                assert_file(snap_of(back.eng, tmp_path / "in_place.snap"), full, var, "in place %d" % mb)
            finally:
                back.close()
        hd_f, ag_f, sec_f = full
        want = relocate(hd_f, ag_f, sec_f, flags | R, S + 777, S * 192, 16 << 20)
        back = Rig(flags | R, S + 777, vcap=S * 192, resp=16 << 20, restore_from=last)
        try:
            assert_file(snap_of(back.eng, tmp_path / "moved.snap"), want, var, "relocated")
            same_reads(back.eng, pair.t.eng, L, ag, ids)
        finally:
            back.close()
    finally:
        pair.d.close(); pair.t.close()


def test_digest_refuses_a_parent_changed_in_its_short_last_piece(tmp_path):
    """a full file of 2^18 + 3 rows whose state and mtime sections end in short pieces: a byte flipped in either, and the
    delta written on it is refused with the digest message; put back, the chain restores"""
    flags = P | M
    n = (1 << 18) + 3
    d = Rig(flags | ONLINE_DELTA, n + 64, seed=4)
    try:
        agent = np.random.default_rng(4).integers(0, 4, n)
        d.add(agent, seq=T0)
        p0 = d.snapshot(tmp_path / "a.snap")
        L, ag, ids = d.rows()
        d.complete(ag[:3], ids[:3], K.AGR_OUT_RESPONSE, 4, T0 + STEP)
        p1 = d.snapshot(tmp_path / "b.snap")
        assert read(p1)[:8] == b"AGRDELT1"
        hd, _, sec = parse(read(p0))
        assert tuple(int(x) for x in parse_delta(read(p1))["dh"]["parent_digest"]) == digest(hd, sec, SECRET)
        names = [s[0] for s in sections(hd)]
        end = HEADER.itemsize + 33 * int(hd["n_agents"]) + sum(sec[x].nbytes for x in names[: names.index("route")])
        for name in ("state", "mtime"):                              # the last byte of each: inside a 12 and an 8 byte piece
            data = bytearray(read(p0))
            at = (end if name == "state" else len(data)) - 1
            data[at] ^= 0x01
            with open(tmp_path / "a.snap", "wb") as f:
                f.write(bytes(data))
            with pytest.raises(A.AgrError) as e:
                A.Engine(restore_from=p1, slab_rows=n + 64, max_agents=16, id_secret=SECRET, flags=flags)
            assert e.value.code == K.AGR_EINVAL and "digest" in str(e.value), name
            data[at] ^= 0x01
            with open(tmp_path / "a.snap", "wb") as f:
                f.write(bytes(data))
        with A.Engine(restore_from=p1, slab_rows=n + 64, max_agents=16, id_secret=SECRET, flags=flags) as back:
            assert back.verify()[1] == 0
    finally:
        d.close()


# ------------------------------------------------------------------------------------------------ hash-id index after a restore
def colliding_ids(n, table_slots, rng):
    """n distinct ids whose home slots (k1ref.hash_id & mask) crowd the last n / 2 slots of the table, so that probe chains
    collide and many wrap past its end"""
    out = []
    mask = np.uint64(table_slots - 1)
    lo = table_slots - max(n // 2, 64)
    while sum(len(x) for x in out) < n:
        c = np.frombuffer(rng.bytes(16 << 20), dtype=np.uint8).reshape(-1, 16)
        out.append(c[(hash_id(c) & mask) >= lo])
    ids = np.concatenate(out)[:n]
    assert len(np.unique(ids.view("V16"))) == n
    return ids


def index_case(flags, slab_rows, seed):
    """The A / P / Z / C sequence many times over in one hash-id engine, with its plain reference (k1ref.Ref):
      Z  rows at the tail that expire (and not-found rows between them);
      P  a stored row that a StoreResponse keeps from expiring, so the release stops there;
      A  stored rows behind P that expire before the release (ids X);
      L  rows that stay stored, and L1 rows among them that expire after the release;
      C  later rows that carry X again (stored in a ring: the release took X out of the index), the ids of L rows
         (duplicates), and ids of other A rows twice in one batch (the second a duplicate).
    A fifth of the A and L ids have home slots crowded at the end of the table.  Returns (rig, ref, the window's distinct
    ids)."""
    ring = bool(flags & R)
    rng = np.random.default_rng(seed)
    rig = Rig(flags, slab_rows, resp=32 << 20, seed=seed)
    ref = Ref({a: (rig.eng.agent_slot(a), K.AGR_AGENT_RUNNING) for a in AGENTS}, mint=False)
    table = 1 << int(np.ceil(np.log2(2 * slab_rows)))
    nz, na, nl1, nl = 3000, 1 << 17, 1 << 16, (1 << 18) + (1 << 16)
    coll = colliding_ids(60000, table, rng)
    ids = np.frombuffer(rng.bytes(16 * (nz + 1 + na + nl)), dtype=np.uint8).reshape(-1, 16).copy()
    a0, l0 = nz + 1, nz + 1 + na
    ids[a0: a0 + 25000] = coll[:25000]
    ids[l0: l0 + 15000] = coll[25000: 40000]                         # L1 rows
    ids[l0 + nl1: l0 + nl1 + 20000] = coll[40000:]                   # L2 rows
    kind = np.array(["Z"] * nz + ["P"] + ["A"] * na + ["L1"] * nl1 + ["L2"] * (nl - nl1))
    order = np.concatenate([np.arange(a0), a0 + rng.permutation(na + nl)])   # A and L interleaved behind P
    kind, ids = kind[order], ids[order]
    agent = rng.integers(0, 4, len(kind))
    agent[(kind == "Z") & (np.arange(len(kind)) % 5 == 0)] = NOBODY
    seq = np.select([kind == "L1", kind == "L2"], [T0 + 8 * STEP, T0 + 12 * STEP], T0).astype(np.uint64)
    first, v = rig.add(agent, ids, seq=seq)
    ref.ingest(rig.records(agent, ids, seq, np.full(len(agent), 30)), first)
    assert np.array_equal(v["flags"], ref.route[first: first + len(agent)] >> 26)
    rig.complete(agent[nz: nz + 1], ids[nz: nz + 1], K.AGR_OUT_RESPONSE, 40, T0 + 9 * STEP)
    ref.touch([first + nz], T0 + 9 * STEP)
    for now in (T0 + 10 * STEP, ):
        assert rig.eng.expire(now, 5 * STEP) == ref.expire(now, 5 * STEP) > na
    if ring:
        assert rig.eng.reclaim() == ref.reclaim() == nz
    a_rows, l_rows = np.nonzero(kind == "A")[0], np.nonzero(kind != "A")[0][nz + 1:]
    again = a_rows[rng.random(len(a_rows)) < 0.5]
    twice = a_rows[:500]
    c_src = np.concatenate([again, l_rows[:3000], twice, twice])
    c_ids, c_agent = ids[c_src], rng.integers(0, 4, len(c_src))
    c_seq = np.full(len(c_src), T0 + 10 * STEP, dtype=np.uint64)
    first_c, vc = rig.add(c_agent, c_ids, seq=c_seq)
    ref.ingest(rig.records(c_agent, c_ids, c_seq, np.full(len(c_src), 30)), first_c)
    assert np.array_equal(vc["flags"], ref.route[first_c: first_c + len(c_src)] >> 26)
    stored = int(((vc["flags"] & K.AGR_VF_STORED) != 0).sum())
    assert (stored > 60000) if ring else stored == 0
    now = T0 + 13 * STEP + STEP // 2                                  # L1 expires; nothing is released after it
    assert rig.eng.expire(now, 5 * STEP) == ref.expire(now, 5 * STEP) == nl1
    assert len(ref.stored_rows()) >= 1 << 18
    return rig, ref, np.unique(np.concatenate([ids, c_ids]).view("V16")).view(np.uint8).reshape(-1, 16)


def verdicts(eng, ref, ids, owner_agent):
    """a replay naming every id (by the agent of the row that carries it), then a fresh record carrying every id: the
    engine's verdict flags and the reference's (ref is changed)"""
    n = len(ids)
    recs = np.zeros(n, dtype=A.record_dtype)
    recs["agent_id"] = NAMES[owner_agent]
    recs["flags"] = (2 << K.AGR_F_METHOD_SHIFT) | K.AGR_F_REPLAY
    recs["replay_of"] = ids
    recs["request_id"] = np.frombuffer(np.random.default_rng(n).bytes(16 * n), dtype=np.uint8).reshape(n, 16)
    recs["path_len"], recs["body_len"], recs["max_retries"], recs["status"] = 2, 10, 3, K.AGR_ST_PENDING
    recs["seq"] = T0 + 20 * STEP
    fresh = recs.copy()
    fresh["flags"] = 2 << K.AGR_F_METHOD_SHIFT
    fresh["replay_of"] = 0
    fresh["request_id"] = ids
    got, want = [], []
    for batch in (recs, fresh):
        for k in range(0, n, eng.max_batch):
            b = np.ascontiguousarray(batch[k: k + eng.max_batch])
            out = np.zeros(len(b), dtype=A.verdict_dtype)
            first = eng.ingest_ex(b, out, np.zeros((len(b), 16), dtype=np.uint8))
            got.append(out["flags"])
            want.append(ref.ingest(b, first)["verdict"]["flags"])
    return np.concatenate(got), np.concatenate(want)


@pytest.mark.parametrize("ring", [True, False])
def test_hash_index_after_a_restore(ring, tmp_path):
    """Restored in place from a delta chain, relocated, and in place from a full file: the file after the restore is the one
    before it (no row demoted), the index holds what Ref.restore() says, and every id's replay and fresh record get the
    verdicts the reference predicts; they are the never-restarted engine's too, except (ring) for the ids of rows that
    expired since the last release, which the restored engine accepts again.  Append-only: nothing changes at all."""
    base = P | (R if ring else 0)
    S = 1 << 21
    rig, ref, ids = index_case(base | ONLINE_DELTA, S, seed=21 if ring else 22)
    try:
        L, ag, _ = rig.rows()
        row_agent = dict(zip(L.tolist(), ag.tolist()))
        oa = np.array([row_agent.get(ref.owner.get(x.tobytes()), 0) for x in ids])
        p0 = rig.snapshot(tmp_path / "s0.snap")
        live = ref.stored_rows()[-200:]                            # a delta on it: completions of a few live rows
        rig.complete(np.array([row_agent[x] for x in live]), ref.idb[live], K.AGR_OUT_RESPONSE, 9, T0 + 11 * STEP)
        p1 = rig.snapshot(tmp_path / "s1.snap")
        d1 = parse_delta(read(p1))
        before = (d1["hd"], d1["agents"], apply(parse(read(p0))[2], d1))
        kw = dict(slab_rows=S, max_agents=16, id_secret=SECRET, flags=base, resp_bytes=32 << 20)
        moved = dict(kw, slab_rows=S + 4097, flags=base | R)
        cases = [("chain", p1, kw, before), ("moved", p1, moved, relocate(*before, base | R, S + 4097, 0, 32 << 20)),
                 ("full", str(tmp_path / "after_chain.snap"), kw, before)]
        got = {}
        for what, path, cfg, want in cases:
            r = copy.deepcopy(ref)
            r.restore(bool(cfg["flags"] & R))
            with A.Engine(restore_from=path, **cfg) as back:
                assert back.verify()[1] == 0
                assert_file(snap_of(back, tmp_path / ("after_%s.snap" % what)), want, False, what)
                used = int(back.debug_read("index_used", 0, 1)[0])
                assert used == r.index_used(), (what, used, r.index_used())
                g, w = verdicts(back, r, ids, oa)
                bad = np.nonzero(g != w)[0]
                assert len(bad) == 0, (what, len(bad), g[bad[:5]], w[bad[:5]])
                got[what] = g
        g_twin, w_twin = verdicts(rig.eng, copy.deepcopy(ref), ids, oa)
        assert np.array_equal(g_twin, w_twin)
        same = g_twin == got["chain"]
        if ring:
            assert (~same).sum() >= 1 << 16 and (g_twin[~same] & K.AGR_VF_DUP_ID).all()
            assert not (got["chain"][~same] & K.AGR_VF_DUP_ID).any()
        else:
            assert same.all()
    finally:
        rig.close()
