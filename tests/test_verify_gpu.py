"""The integrity sweep (agr_verify, k_verify) against tests/verifyref.py on every path that writes a record and its checksum:
K1 (agr_ingest, agr_ingest_ex, reserved rows filled from the host or on the device), the service kernel in both record forms,
the exchange's holes and received rows, K1v at every stored length up to 8 KiB, the 512-byte slots of variable-length
reservations, and restores in place, relocated, converted into the other record form and from a delta chain.

Every case first checks the checksum words against the reference checksum of the bytes the test sent (which also catches a
wrong copy into the slab) and that the sweep reports (rows checked, 0).  Then it plants corruption in HBM at chunk edges, at
the checksum's blind spots, past a record's length, in expired and released rows and at the grid's edges, and the sweep
must report exactly the number of bad rows the reference finds in the engine's own per-row words and bytes, so that a miss
and a false positive fail alike."""
import ctypes as C
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1ref
import k1vref
import verifyref as VR
from agentainer_lab_b200 import constants as K
from snapfile import parse

pytestmark = pytest.mark.gpu

P, M, V, R, CB = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING, K.AGR_CFG_COMBINE
SECRET = 0x5EED_7E51_F1ED_0001
AGENTS = [A.synth_agent_id(k) for k in range(4)]
STATUS = ["running", "stopped", "running", "stopped"]
REC = 512
_rt = C.CDLL("libcudart.so")


def dev_read(ptr, n):
    out = np.zeros(max(n, 1), dtype=np.uint8)
    assert _rt.cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(n), 2) == 0
    return out[:n]


def dev_write(ptr, b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    assert _rt.cudaMemcpy(C.c_void_p(ptr), C.c_void_p(b.ctypes.data), C.c_size_t(len(b)), 1) == 0


def flip(ptr, mask=0x5A):
    dev_write(ptr, dev_read(ptr, 1) ^ np.uint8(mask))


def engine(flags, **kw):
    kw.setdefault("slab_rows", 1 << 12)
    kw.setdefault("max_agents", 64)
    kw.setdefault("id_secret", SECRET)
    if flags & V:
        kw.setdefault("vslab_bytes", 8 << 20)
    e = A.Engine(flags=flags, **kw)
    e.ring = bool(flags & R)
    for a, s in zip(AGENTS, STATUS):
        e.set_agent_state(a, s)
    return e


def fixed_records(n, first_index, seed, seq0=1, strangers=True):
    """n synthetic 512-byte records of AGENTS, seq = seq0 + i; every 17th names an unregistered agent (NOT_FOUND, not stored)"""
    r = A.synth_fill_host(first_index, n, seed=seed, n_agents=len(AGENTS))
    r["seq"] = seq0 + np.arange(n, dtype=np.uint64)
    if strangers:
        r["agent_id"][::17] = b"agent-nobody"
    return r


def var_batch(lens, rng, seq0=1):
    h = k1vref.headers(len(lens), AGENTS, rng, seq0=seq0)
    k1vref.fit_lens(h, lens, rng)
    return k1vref.blob_from(h, lens, rng)


class Dev:
    """the engine's per-row words by physical row and its slab, as the sweep sees them"""

    def __init__(self, eng, tmp_path=None, resv=()):
        s = eng.stats()
        self.used, self.tail = s["rows_used"], s["rows_tail"]
        self.S = s["rows_cap"]
        self.ring, self.var = eng.ring, eng.varlen
        self.span = min(self.used, self.S) if self.ring else self.used
        self.resv = resv
        if self.var:                                          # voff / vlen only travel in a snapshot file
            p = str(tmp_path / "view.snap")
            eng.snapshot(p)
            with open(p, "rb") as f:
                hd, _, sec = parse(f.read())
            self.state, self.cksum, self.voff, self.vlen = sec["state"], sec["cksum"], sec["voff"], sec["vlen"]
            self.slab = np.asarray(sec["slab"])
        else:
            lo = self.used - self.span
            ph = self.phys(np.arange(lo, self.used))
            self.state = np.zeros(self.span, np.uint32)
            self.cksum = np.zeros(self.span, np.uint64)
            if self.span:
                self.state[ph] = eng.debug_read("state", lo, self.span)
                self.cksum[ph] = eng.debug_read("cksum", lo, self.span)
            self.voff = self.vlen = None
            self.slab = dev_read(slab_base(eng), self.span * REC) if self.span else np.zeros(0, np.uint8)
        self.base = slab_base(eng)

    def phys(self, rid):
        return np.asarray(rid, dtype=np.int64) % self.S if self.ring else np.asarray(rid, dtype=np.int64)

    def sweep(self):
        return VR.sweep(self.state, self.cksum, self.slab, span=self.span, ring=self.ring, resv=self.resv, slab_rows=self.S,
                        voff=self.voff, vlen=self.vlen)

    def at(self, rid, off):
        """device address of byte `off` of logical row rid's record"""
        p = int(self.phys(rid))
        return self.base + (int(self.voff[p]) if self.var else p * REC) + off


def slab_base(eng):
    s = eng.stats()
    rid = s["rows_tail"]
    ptr = eng.slab_ptr(rid)
    assert ptr, "empty window"
    ph = rid % s["rows_cap"] if eng.ring else rid
    return ptr - ph * REC


def agree(eng, tmp_path=None, resv=(), bad=None):
    """agr_verify equals the reference sweep over the engine's words and bytes; returns the reference"""
    ref = Dev(eng, tmp_path, resv).sweep()
    got = eng.verify()
    assert got == (ref.checked, len(ref.bad)), (got, ref.checked, ref.bad.tolist()[:20])
    if bad is not None:
        assert len(ref.bad) == bad, (ref.bad.tolist()[:20], bad)
    return ref


# ---------------------------------------------------------------------------------------------- the reservation case
@pytest.mark.parametrize("fill", ["host", "device"])
@pytest.mark.parametrize("mint", [False, True])
def test_undecided_reservation_is_not_counted(mint, fill):
    """append-only, fixed stride: rows reserved and filled but not yet decided hold bytes and a zero checksum; the sweep
    skips them and checks the decided rows after them, and after agr_ingest_rows checks everything"""
    with engine(P | (M if mint else 0)) as eng:
        a = fixed_records(300, 0, seed=3)
        eng.ingest(a)
        f = eng.reserve_rows(100)
        if fill == "host":
            mid = fixed_records(100, 300, seed=4)
            eng.fill_rows(f, mid)
        else:
            eng.synth_fill_rows(300, f, 100, seed=4, n_agents=len(AGENTS))
        b = fixed_records(200, 400, seed=5)
        _, f2 = eng.ingest(b)
        assert f2 == f + 100
        assert eng.verify() == (500, 0)
        agree(eng, resv=[(f, f + 100)], bad=0)
        d = Dev(eng, resv=[(f, f + 100)])
        flip(d.at(f2 + 7, 200))                                        # a decided row after the reservation is swept
        flip(d.at(f + 3, 200))                                         # a reserved row is not
        assert eng.verify() == (500, 1)
        agree(eng, resv=[(f, f + 100)], bad=1)
        flip(d.at(f2 + 7, 200))
        flip(d.at(f + 3, 200))
        eng.ingest_rows(f, 100)
        assert eng.verify() == (600, 0)
        agree(eng, bad=0)


# ---------------------------------------------------------------------------------------------- fixed stride
FIXED_PATHS = ["ingest", "ingest_ex", "fill_rows", "synth_fill_rows", "submit_ingest"]


def feed(eng, path, recs, first_index=0, seed=0):
    """the records through one path; returns the first row.  synth_fill_rows: the device writes the records that
    synth_fill_host(first_index, n, seed) gives on the host"""
    n = len(recs)
    if path == "ingest":
        return eng.ingest(recs)[1]
    if path == "ingest_ex":
        return eng.ingest_ex(recs, np.zeros(n, A.verdict_dtype), np.zeros((n, 16), np.uint8))
    if path in ("fill_rows", "synth_fill_rows"):
        f = eng.reserve_rows(n)
        if path == "fill_rows":
            eng.fill_rows(f, recs)
        else:
            eng.synth_fill_rows(first_index, f, n, seed=seed, n_agents=len(AGENTS))
        eng.ingest_rows(f, n)
        return f
    rids = [eng.poll(eng.submit_ingest(recs[i]))["rid"] for i in range(n)]
    assert rids == list(range(rids[0], rids[0] + n))
    return rids[0]


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("mint", [False, True])
@pytest.mark.parametrize("path", FIXED_PATHS)
def test_fixed_stride_paths(path, mint, ring):
    flags = P | (M if mint else 0) | (R if ring else 0) | (CB if path == "submit_ingest" else 0)
    n = 40 if path == "submit_ingest" else 300
    blind = path != "synth_fill_rows"
    with engine(flags) as eng:
        if blind:
            recs = fixed_records(n, 0, seed=9)
            # payload words that let a swap and a double bit-31 flip pass unseen: 0 and 0x80000000 two words apart
            w = recs.view(np.uint8).reshape(n, REC).view("<u4")
            w[1, 40], w[1, 42] = 0, 0x80000000
        else:
            recs = A.synth_fill_host(0, n, seed=9, n_agents=len(AGENTS))
        f = feed(eng, path, recs, 0, 9)
        assert (eng.debug_read("cksum", f, n) == k1ref.cksum(recs)).all()
        ref = agree(eng, bad=0)
        assert ref.checked == n
        d = Dev(eng)
        stored = (d.state[d.phys(np.arange(f, f + n))] & VR.ST_STORED) != 0
        srows = [f + i for i in range(n) if stored[i] and i != 1]
        # one byte in chunks 0, 5 (bytes 80..95) and 31, each in its own row; two bytes in one more row (counts once)
        for k, c in enumerate((0, 5, 31)):
            flip(d.at(srows[k], 16 * c + 9))
        flip(d.at(srows[3], 100)); flip(d.at(srows[3], 400))
        # a swap of two unequal chunks, in another row
        a0, a1 = d.at(srows[4], 128), d.at(srows[4], 256)
        c0, c1 = dev_read(a0, 16), dev_read(a1, 16)
        assert (c0 != c1).any()
        dev_write(a0, c1); dev_write(a1, c0)
        # a row that K1 did not store: counted on an append-only engine, not on a ring
        strangers = [f + i for i in range(n) if not stored[i]]
        if strangers:
            flip(d.at(strangers[0], 300))
        if blind:
            # what the checksum cannot see, in row 1: words 40 and 42 (0, 0x80000000) swapped; bit 31 of words 60 and 62
            dev_write(d.at(f + 1, 160), np.array([0x80000000], "<u4").view(np.uint8))
            dev_write(d.at(f + 1, 168), np.zeros(4, np.uint8))
            flip(d.at(f + 1, 243), 0x80); flip(d.at(f + 1, 251), 0x80)
        agree(eng, bad=5 + (1 if strangers and not ring else 0))


@pytest.mark.parametrize("G", [2, 3])
@pytest.mark.parametrize("mint", [False, True])
def test_exchange_holes_and_received_rows(G, mint):
    """each rank of a simulated world: a batch whose peers' records leave holes, then the records its peers sent it"""
    from agentainer_lab_b200.sharding import make_rank_batch, owned_agents
    own = owned_agents(G, 6)
    flags = P | (M if mint else 0)
    engs = [A.Engine(slab_rows=1 << 13, max_agents=256, max_batch=4096, flags=flags, id_secret=SECRET) for _ in range(G)]
    try:
        for r, e in enumerate(engs):
            e.ring = False
            e.debug_world(r, G)
            for a in own[r]:
                e.set_agent_state(a, "running" if int(a[-1]) % 2 else "stopped")
        firsts, segs, infos = [], [], []
        for r, e in enumerate(engs):
            b = make_rank_batch(r, G, own, 500, seed=7 + r, p_cross_replay=0.05, p_missteer=0.08, first_index=r * 1000)
            f = e.reserve_rows(len(b))
            e.fill_rows(f, b)
            send, info = e.debug_exchange_begin(f, len(b))
            firsts.append((f, len(b))); infos.append(info)
            o, seg = 0, {}
            for q in range(G):
                if q != r and info.sent_to[q]:
                    seg[q] = send[o: o + info.sent_to[q]]; o += info.sent_to[q]
            segs.append(seg)
        recv, back = [], [dict() for _ in range(G)]
        for o, e in enumerate(engs):                                  # the owner's merge order: sources by rank
            srcs = [s for s in range(G) if s != o and o in segs[s]]
            inc = np.ascontiguousarray(np.concatenate([segs[s][o] for s in srcs])) if srcs else np.zeros(0, A.record_dtype)
            recv.append(None)
            if len(inc):
                f2 = e.reserve_rows(len(inc))
                e.fill_rows(f2, inc)
                v = e.ingest_rows(f2, len(inc))
                assert (e.debug_read("cksum", f2, len(inc)) == k1ref.cksum(inc)).all()
                recv[o] = (f2, len(inc))
                k = 0
                for s in srcs:
                    back[s][o] = v[k: k + len(segs[s][o])]
                    k += len(segs[s][o])
        for r, e in enumerate(engs):
            parts = [back[r][q] for q in range(G) if q in back[r]]
            e.debug_exchange_end(np.concatenate(parts) if parts else np.zeros(0, A.verdict_dtype), firsts[r][1])
        for r, e in enumerate(engs):
            ref = agree(e, bad=0)
            assert ref.checked == e.stats()["rows_used"]
            d = Dev(e)
            f, n = firsts[r]
            flip(d.at(f, 3)); flip(d.at(f + n - 1, 500))               # first and last row of the exchanged batch
            if recv[r]:
                flip(d.at(recv[r][0] + recv[r][1] - 1, 88))           # a received row
            agree(e, bad=2 + (1 if recv[r] else 0))
    finally:
        for e in engs:
            e.close()


# ---------------------------------------------------------------------------------------------- variable length
VAR_LENS = [96, 112, 512, 528, 1024, 4096, 8176, 8192, 8192, 8192, 8192, 8192, 8192, 8192, 8192, 8192, 496, 8192, 96]
EDGE_CHUNKS = [0, 5, 31, 32, 33, 63, 64, 511]


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("mint", [False, True])
def test_varlen_ingest_every_length(mint, ring, tmp_path):
    rng = np.random.default_rng(21 + 2 * mint + ring)
    with engine(P | V | (M if mint else 0) | (R if ring else 0)) as eng:
        blob, offs = var_batch(VAR_LENS, rng)
        _, _, f = eng.ingest_var(blob, offs)
        n = len(VAR_LENS)
        assert (eng.debug_read("cksum", f, n) == k1vref.cksum(blob, offs)).all()
        ref = agree(eng, tmp_path, bad=0)
        assert ref.checked == n
        d = Dev(eng, tmp_path)
        assert (d.vlen[d.phys(np.arange(f, f + n))] == np.diff(offs)).all()
        stored = (d.state[d.phys(np.arange(f, f + n))] & VR.ST_STORED) != 0
        big = [f + i for i in range(n) if VAR_LENS[i] == 8192 and stored[i]]
        assert len(big) >= 5, "the agents' statuses store every record"
        for k, c in enumerate(EDGE_CHUNKS[: len(big)]):               # one chunk edge per 8 KiB record, last chunk included
            flip(d.at(big[k], 16 * c + 15))
        flip(d.at(f + n - 1, VAR_LENS[-1]))                           # one byte past the last record's vlen
        flip(d.at(f + 1, 16 * 6 + 2))                                 # the 112-byte record's last chunk
        agree(eng, tmp_path, bad=min(len(big), len(EDGE_CHUNKS)) + 1)


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("mint", [False, True])
def test_varlen_reserved_slots(mint, ring, tmp_path):
    with engine(P | V | (M if mint else 0) | (R if ring else 0)) as eng:
        recs = fixed_records(200, 0, seed=13)
        f = eng.reserve_rows(200)
        eng.fill_rows(f, recs)
        assert eng.verify() == (0, 0)                                 # nothing decided yet
        eng.ingest_rows(f, 200)
        assert (eng.debug_read("cksum", f, 200) == k1ref.cksum(recs)).all()
        ref = agree(eng, tmp_path, bad=0)
        assert ref.checked == 200
        d = Dev(eng, tmp_path)
        assert (d.vlen[d.phys(np.arange(f, f + 200))] == 512).all()
        assert (d.state[d.phys([f + 2, f + 199])] & VR.ST_STORED).all()
        flip(d.at(f + 2, 0)); flip(d.at(f + 199, 511))               # the first and the last chunk of a slot
        agree(eng, tmp_path, bad=2)


@pytest.mark.parametrize("ring", [False, True])
@pytest.mark.parametrize("mint", [False, True])
def test_varlen_tickets_span_slots(mint, ring, tmp_path):
    """records of 1, 2, 15 and 16 request-ring slots through the service kernel (k_svc_var)"""
    lens = [96, 512, 528, 1024, 7680, 7696, 8176, 8192, 8192]
    rng = np.random.default_rng(5 + mint + 2 * ring)
    with engine(P | V | CB | (M if mint else 0) | (R if ring else 0)) as eng:
        blob, offs = var_batch(lens, rng)
        rids = [eng.poll(eng.submit_ingest(blob[offs[i]: offs[i + 1]]))["rid"] for i in range(len(lens))]
        assert rids == list(range(rids[0], rids[0] + len(lens)))
        f = rids[0]
        assert (eng.debug_read("cksum", f, len(lens)) == k1vref.cksum(blob, offs)).all()
        ref = agree(eng, tmp_path, bad=0)
        assert ref.checked == len(lens)
        d = Dev(eng, tmp_path)
        assert (d.state[d.phys([f + 1, f + 4, f + 7])] & VR.ST_STORED).all()
        flip(d.at(f + 1, 511)); flip(d.at(f + 4, 16 * 479)); flip(d.at(f + 7, 16 * 511 + 8))     # each record's last chunk
        agree(eng, tmp_path, bad=3)


# ---------------------------------------------------------------------------------------------- after a restore
def zero_tails(recs):
    """zeros past path + headers + body, as the layout requires: the compact form of the row then has the row's checksum"""
    pl = (recs["path_len"].astype(np.int64) + recs["hdr_len"] + recs["body_len"])[:, None]
    b = recs.view(np.uint8).reshape(len(recs), REC)
    b[:, 96:][np.arange(REC - 96)[None, :] >= pl] = 0
    return recs


@pytest.mark.parametrize("kind", ["in_place", "relocated", "fixed_to_var", "var_to_fixed", "delta"])
def test_after_restore(kind, tmp_path):
    rng = np.random.default_rng(77)
    src_flags = P | M | R | (V if kind == "var_to_fixed" else 0) | (K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT if kind == "delta" else 0)
    dst = {"in_place": (src_flags, 1 << 12), "relocated": (src_flags, 3000), "fixed_to_var": (P | M | R | V, 2048),
           "var_to_fixed": (P | M | R, 2048), "delta": (src_flags, 1 << 12)}[kind]
    path = str(tmp_path / "a.snap")
    with engine(src_flags) as eng:
        if src_flags & V:
            lens = rng.choice([96, 112, 256, 496, 512], 700)
            blob, offs = var_batch(lens, rng)
            eng.ingest_var(blob, offs)
        else:
            eng.ingest(zero_tails(fixed_records(700, 0, seed=31, strangers=False)))
        eng.snapshot(path)
        if kind == "delta":
            eng.ingest(fixed_records(300, 700, seed=32, strangers=False))
            path = str(tmp_path / "b.snap")
            eng.snapshot(path)
        want = eng.debug_read("cksum", 0, eng.stats()["rows_used"])
    flags, S = dst
    with A.Engine(flags=flags, slab_rows=S, max_agents=64, id_secret=SECRET, vslab_bytes=(8 << 20) if flags & V else 0,
                  restore_from=path) as e2:
        e2.ring = True
        used = e2.stats()["rows_used"]
        assert (e2.debug_read("cksum", 0, used) == want).all()        # checksums move unchanged
        ref = agree(e2, tmp_path, bad=0)
        assert ref.checked == min(used, S)
        d = Dev(e2, tmp_path)
        live = [r for r in range(used) if d.state[d.phys(r)] & VR.ST_STORED]
        flip(d.at(live[0], 1)); flip(d.at(live[-1], 95)); flip(d.at(live[len(live) // 2], 16 * 5))
        agree(e2, tmp_path, bad=3)


# ---------------------------------------------------------------------------------------------- grid edges
@pytest.mark.parametrize("n", [1, 7, 8, 9])
def test_rows_span_at_the_block_edges(n):
    """eight warps per block: one row, a block short of one row, a full block, a full block and one row"""
    with engine(P) as eng:
        recs = fixed_records(n, 0, seed=41, strangers=False)
        eng.ingest(recs)
        assert (eng.debug_read("cksum", 0, n) == k1ref.cksum(recs)).all()
        agree(eng, bad=0)
        d = Dev(eng)
        flip(d.at(n - 1, 17))
        if n > 1:
            flip(d.at(0, 480))
        agree(eng, bad=1 if n == 1 else 2)


@pytest.mark.parametrize("mint", [False, True])
def test_ring_window_wraps(mint):
    """rows_used > slab_rows: the first and last physical rows hold records; an expired row and released rows do not count"""
    S = 64
    with engine(P | R | (M if mint else 0), slab_rows=S, max_batch=64) as eng:
        a = fixed_records(32, 0, seed=51, seq0=100, strangers=False)
        b = fixed_records(32, 32, seed=52, seq0=10_000_000, strangers=False)
        eng.ingest(a); eng.ingest(b)
        eng.expire(1_000_000, 500_000)
        eng.reclaim()
        c = fixed_records(16, 64, seed=53, seq0=10_000_000, strangers=False)
        c["seq"][5] = 200                                            # expires below, but stays behind live rows
        _, f = eng.ingest(c)
        assert f == 64 and eng.stats()["rows_used"] == 80
        assert eng.expire(1_000_000, 500_000) == 1
        assert (eng.debug_read("cksum", 32, 48) == k1ref.cksum(np.concatenate([b, c]))).all()
        ref = agree(eng, bad=0)
        assert ref.checked == S
        d = Dev(eng)
        assert d.state[0] & VR.ST_STORED and d.state[S - 1] & VR.ST_STORED
        flip(d.base + 0 * REC + 7); flip(d.base + (S - 1) * REC + 505)     # first and last physical rows
        flip(d.base + 5 * REC + 200)                                       # the expired row
        flip(d.base + 20 * REC + 200)                                      # a released row
        agree(eng, bad=2)


def test_ring_of_2_to_the_22_plus_3_rows():
    S = (1 << 22) + 3
    with engine(P | M | R, slab_rows=S, max_batch=1 << 20) as eng:
        recs = fixed_records(1 << 20, 0, seed=61, strangers=False)
        ck = k1ref.cksum(recs)
        for k in range(4):
            eng.ingest(recs)
        eng.ingest(recs[:3])
        assert eng.stats()["rows_used"] == S
        got = eng.debug_read("cksum", 0, S)
        assert (got[: 4 << 20].reshape(4, -1) == ck).all() and (got[4 << 20:] == ck[:3]).all()
        assert eng.verify() == (S, 0)
        base = slab_base(eng)
        for p in (0, (1 << 22) - 1, 1 << 22, S - 1):
            flip(base + p * REC + 300)
        # every row is stored (registered agents, minted ids) and one changed byte is always seen (tests/test_verify_ref.py)
        assert (eng.debug_read("state", 0, S) & VR.ST_STORED != 0).all()
        assert eng.verify() == (S, 4)


# ---------------------------------------------------------------------------------------------- byte ring laps
def test_lapped_varlen_byte_ring(tmp_path):
    """a variable-length ring whose rows and bytes have gone round: released rows' old bytes now hold newer records"""
    rng = np.random.default_rng(91)
    with engine(P | V | M | R, slab_rows=128, vslab_bytes=256 << 10) as eng:
        for step in range(12):
            seq0 = 1 + 1000 * step
            eng.expire(seq0, 1)                                      # everything older than this batch
            eng.reclaim()
            lens = rng.choice([96, 512, 1024, 4096], 20)
            blob, offs = var_batch(lens, rng, seq0=seq0)
            _, _, f = eng.ingest_var(blob, offs)
            assert (eng.debug_read("cksum", f, 20) == k1vref.cksum(blob, offs)).all()
        assert eng.stats()["rows_used"] > 128
        ref = agree(eng, tmp_path, bad=0)
        assert ref.checked == 128 and len(ref.examined) == 20
        d = Dev(eng, tmp_path)
        flip(d.at(f + 19, int(lens[-1]) - 1))
        agree(eng, tmp_path, bad=1)


# ---------------------------------------------------------------------------------------------- live callers
def test_verify_while_ticket_callers_submit():
    with engine(P | M | CB, slab_rows=1 << 13) as eng:
        recs = fixed_records(4 * 300, 0, seed=71)
        stop_err = []

        def caller(t):
            try:
                for i in range(t * 300, (t + 1) * 300):
                    eng.poll(eng.submit_ingest(recs[i]))
            except Exception as ex:
                stop_err.append(ex)
        th = [threading.Thread(target=caller, args=(t,)) for t in range(4)]
        for t in th:
            t.start()
        try:
            seen = [eng.verify()[1] for _ in range(5)]
        finally:
            for t in th:                                             # the callers finish before the engine may close
                t.join()
        assert not stop_err
        assert seen == [0] * 5
        assert eng.verify() == (1200, 0)
        agree(eng, bad=0)
