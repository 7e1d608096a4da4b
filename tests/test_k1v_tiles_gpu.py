"""The variable-length ingest (K1v, csrc/agr_k1_var.cu) in both its forms — staged (1-D bulk TMA into a per-warp stage,
k1_variant 0) and LSU (k1_variant 0x20) — against the plain reference of tests/k1vref.py, at the tile shapes where the
two forms change code path, and with many tiles per warp.

Every case is a list of batches built from record lengths and headers.  For each form and id mode it checks:
  - verdicts, ids, the state / route words and the agr_stats counters against a fixed-stride twin engine fed
    k1vref.twin_records() of the same batches (the fixed-stride K1 is pinned to the oracle by test_parity_gpu.py);
  - plain predictions: stored / too long / duplicate id / dedupe hits of hand-placed replays, the stored rows' state words;
  - debug_read("cksum") of every record against k1vref.cksum();
  - voff / vlen of every row and the slab bytes, from a snapshot file (tests/snapfile.py);
  - every stored record's bytes through one replay_scan_var, a sample through get_record_var (before and after
    completions), against k1vref.readback(); the pending lists; verify();
and that the two forms agree byte for byte."""
import hashlib
import os
import tempfile
from dataclasses import dataclass, field
from functools import lru_cache

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1vref as kr
import snapfile
from agentainer_lab_b200 import constants as K

pytestmark = pytest.mark.gpu

FORMS = {"staged": 0, "lsu": 0x20}
MODES = {"hash": 0, "mint": K.AGR_CFG_MINT_IDS}
BASE = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_VARLEN
SECRET = 0x5eed1234
COUNTERS = ("ingested", "stored", "replay_flagged", "dedupe_hits", "forwarded", "queued", "unavailable", "not_found", "dup_ids",
            "malformed")
AGENTS = {"agent-run": "running", "agent-run2": "running", "agent-stop": "stopped", "agent-drop": "running"}
FOUND = ("agent-run", "agent-run2", "agent-stop")
RUNNING = ("agent-run", "agent-run2")
NAMES = ["agent-run", "agent-run2", "agent-stop", "agent-nobody", "agent-drop"]   # agent-nobody is never registered
ST_STORED = 0x20


@lru_cache(maxsize=None)
def sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def mint(first, n):
    with A.Engine(slab_rows=64, max_agents=4, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS, id_secret=SECRET) as e:
        return e.mint_ids(first, n)


@dataclass
class Batch:
    h: np.ndarray                      # headers as fed
    lens: np.ndarray
    blob: np.ndarray = None
    offs: np.ndarray = None
    known: dict = field(default_factory=dict)       # record -> predicted AGR_VF_KNOWN of a hand-placed replay
    dup_losers: list = field(default_factory=list)  # hash mode: records whose caller id an earlier record of the batch carries


@dataclass
class Case:
    steps: list                        # Batch, or "expire" (expire everything + reclaim)
    rows: int
    vslab: int
    flags: int = 0


def _agents(rng, n, p=(0.4, 0.25, 0.25, 0.05, 0.05)):
    return rng.choice(len(NAMES), n, p=p)


def _mixed_lens(rng, n):
    """log-uniform 96 B .. 8 KiB"""
    return np.minimum(kr.MAXREC, np.exp(rng.uniform(np.log(96), np.log(kr.MAXREC), n)).astype(np.int64) // 16 * 16)


def _batch(lens, rng, seq0, mode, agent_of=None) -> Batch:
    lens = np.asarray(lens, dtype=np.int64)
    h = kr.headers(len(lens), NAMES, rng, seq0=seq0, agent_of=_agents(rng, len(lens)) if agent_of is None else agent_of)
    kr.fit_lens(h, lens, rng)
    return Batch(h, lens)


def _finish(b: Batch, rng):
    b.blob, b.offs = kr.blob_from(b.h, b.lens, rng)
    return b


# ------------------------------------------------------------------------------------------------------- families
def _make_bad(h, lens, idx, kind):
    """records idx claim one byte more than their stored payload (kind 0), or the largest lengths the fields hold (kind 1)"""
    pay = lens[idx] - kr.HDR
    if kind == 0:
        h["body_len"][idx] = pay + 1 - h["path_len"][idx].astype(np.int64) - h["hdr_len"][idx]
    else:
        h["path_len"][idx], h["hdr_len"][idx], h["body_len"][idx] = 0xFFFF, 0xFFFF, 0xFFFFFFFF


def fam_most_per_tile(mode):
    """every record 96 B (header only): 86 starts in tile 0, 5-6 starts in every sweep row; more tiles than staged warps, so
    warps whose next tile holds >= 64 records use the third offset register"""
    rng = np.random.default_rng(101)
    ntiles = 16 * sms() + 64
    n = -(-ntiles * kr.TILE // 96)
    return Case([_finish(_batch(np.full(n, 96), rng, 1, mode), rng)], rows=1 << (n + 1024).bit_length(), vslab=n * 96 + (1 << 20))


def fam_one_per_tile(mode):
    rng = np.random.default_rng(102)
    b = _batch(np.full(300, 8192), rng, 1, mode)
    return Case([_finish(b, rng)], rows=1 << 12, vslab=8 << 20)


STAGE_SPEC = [("rec", 6400), ("rec", 6400),                                   # tile 0: ends exactly at so[0] + 12800
              ("to", 2 * kr.TILE), ("rec", 6400), ("rec", 6416),              # tile 2: one chunk past the stage
              ("to", 4 * kr.TILE), ("rec", 4000), ("rec", 4176), ("rec", 8192),   # tile 4: last start 16 B before tile 5, 8 KiB long
              ("to", 7 * kr.TILE), ("rec", 4000), ("rec", 8192),              # tile 7: a long last record inside the stage
              ("to", 9 * kr.TILE - 96 * 40)] + [("rec", 96)] * 100 + [("rec", 8192), ("rec", 8192), ("rec", 96)]


def fam_stage_edges(mode):
    rng = np.random.default_rng(103)
    lens = kr.layout(STAGE_SPEC)
    lens2 = kr.layout([("rec", 496)] + STAGE_SPEC)                           # tile 0 now runs past its stage
    return Case([_finish(_batch(lens, rng, 1, mode), rng), _finish(_batch(lens2, rng, 10001, mode), rng)], rows=1 << 12, vslab=8 << 20)


ROW_SPEC = [("rec", 496),                        # next start at chunk 31
            ("rec", 528),                        # starts at chunk 31, its successor at chunk 64 = row 2, chunk 0
            ("rec", 3008)] + [("rec", 96)] * 42 + [  # chunks 64 .. 252: rows 3 .. 6 hold no start; then rows of 5-6 starts
            ("rec", 112), ("rec", 8192),         # last start 16 B before tile 1, 8 KiB long: a 1023-chunk sweep from the base
            ("rec", 96),                         # tile 1: one record, one row
            ("to", 3 * kr.TILE - 16), ("rec", 7776)] + [("rec", 96)] * 5 + [   # tile 3: starts late, five starts in one row
            ("to", 5 * kr.TILE), ("rec", 4000), ("rec", 8192), ("rec", 96)]


def fam_row_edges(mode):
    rng = np.random.default_rng(104)
    lens = kr.layout(ROW_SPEC)
    lens2 = kr.layout([("rec", 2000)] + ROW_SPEC)
    return Case([_finish(_batch(lens, rng, 1, mode), rng), _finish(_batch(lens2, rng, 10001, mode), rng)], rows=1 << 12, vslab=8 << 20)


def fam_tiny(mode):
    rng = np.random.default_rng(105)
    steps = []
    for k, lens in enumerate(([96, 8192], [8192], [96], [5008], [96, 8192, 8192, 96])):
        steps.append(_finish(_batch(lens, rng, 1 + 100 * k, mode, agent_of=np.zeros(len(lens), dtype=np.int64)), rng))
    return Case(steps, rows=1 << 10, vslab=1 << 20)


def _many_spec(rng, target):
    """mixed lengths with runs of 96 B records between long ones, and now and then a run of 86 starting at a tile base"""
    spec, at = [], 0
    while at < target:
        u = rng.random()
        if u < 0.08:
            nxt = (at // kr.TILE + 1) * kr.TILE
            if nxt - at >= 96 or nxt == at:
                spec.append(("to", nxt)); at = nxt
            spec += [("rec", 96)] * 86; at += 86 * 96
        elif u < 0.3:
            k = int(rng.choice([1, 2, 3, 7, 20, 40]))
            spec += [("rec", 96)] * k; at += 96 * k
        elif u < 0.4:
            spec.append(("rec", 8192)); at += 8192
        else:
            v = int(_mixed_lens(rng, 1)[0]); spec.append(("rec", v)); at += v
    if at % kr.TILE == 0:
        spec.append(("rec", 96))                 # the next batch then starts at an offset that is not 8 KiB aligned
    return spec


def _place(b: Batch, first: int, ids_of, mode, rng, earlier=None):
    """Duplicate caller ids across CTAs (hash mode decides them; in mint mode they are ignored) and replay-flagged records
    naming targets in every relation K1v's batch-wide resolution must handle.  b.known gets the plain prediction."""
    h, lens = b.h, b.lens
    o = np.concatenate([[0], np.cumsum(lens)])
    t = kr.tile_owners(o)
    ag = np.array([NAMES.index(a.decode()) for a in h["agent_id"]])
    found = ag < 3
    fresh = found & kr.fits(h, lens)               # would be stored
    replay = np.zeros(len(h), dtype=bool)
    taken = np.zeros(len(h), dtype=bool)
    S = sms()
    cta = lambda i, lsu: int(kr.cta_of(t.tile[i], t.ntiles, S, lsu))

    def other_cta(i, j):
        return cta(i, False) != cta(j, False) and cta(i, True) != cta(j, True)

    cand = np.nonzero(fresh)[0]
    # duplicate ids: the earliest row must win, whichever CTA gets there first
    for _ in range(24):
        j, i = sorted(rng.choice(cand, 2, replace=False))
        if taken[i] or taken[j] or not other_cta(i, j):
            continue
        h["request_id"][i] = h["request_id"][j]
        taken[i] = taken[j] = True
        if mode == "hash":
            b.dup_losers.append(int(i)); fresh[i] = False

    def replay_of(i, j, agent=None):
        h["flags"][i] |= K.AGR_F_REPLAY
        h["replay_of"][i] = ids_of(j)
        h["agent_id"][i] = h["agent_id"][j] if agent is None else agent
        replay[i] = taken[i] = True

    too_long = found & ~kr.fits(h, lens)
    n, F = len(h), t.first

    def pick(cands, pred, tries=20000):
        """a record i not used yet and a target j among cands(i) with pred(i, j)"""
        for _ in range(tries):
            i = int(rng.integers(0, n))
            if taken[i]:
                continue
            c = cands(i)
            if len(c) == 0:
                continue
            j = int(rng.choice(c))
            if pred(i, j):
                return i, j
        raise AssertionError("no such pair in the batch")

    k_ = lambda i: int(t.tile[i])
    usable = lambda j: fresh[j] and not replay[j]
    cats = {
        "same tile":           (lambda i: np.arange(F[k_(i)], i), lambda i, j: usable(j)),
        "other warp same CTA": (lambda i: np.arange(F[k_(i) - 1], F[k_(i)]) if k_(i) % 8 else [], lambda i, j: usable(j)),
        "other CTA":           (lambda i: np.arange(0, F[k_(i) - 15]) if k_(i) >= 16 else [], lambda i, j: usable(j) and other_cta(i, j)),
        "later row":           (lambda i: np.arange(F[k_(i) + 1], n) if k_(i) + 1 < t.ntiles else [], lambda i, j: usable(j)),
        "target is a replay":  (lambda i: np.nonzero(replay[:i])[0], lambda i, j: True),
        "target too long":     (lambda i: np.nonzero(too_long[:i] & ~replay[:i])[0], lambda i, j: True),
        "other agent":         (lambda i: np.arange(0, i), lambda i, j: usable(j) and ag[j] != 0),
    }
    for name, (cands, pred) in cats.items():
        for _ in range(6):
            i, j = pick(cands, pred)
            hit = name in ("same tile", "other warp same CTA", "other CTA")
            replay_of(i, j, agent=b"agent-run" if name == "other agent" else None)
            b.known[i] = hit                       # a hit's target is stored, so its agent (now also i's) is found
    for _ in range(4):                             # a replay of an unknown agent: not found, never a hit
        i, j = pick(*cats["same tile"])
        replay_of(i, j, agent=b"agent-nobody"); b.known[i] = False
    if earlier is not None:                        # targets of the previous batch
        eb, efirst = earlier
        ef = np.nonzero(np.array([a.decode() in FOUND for a in eb.h["agent_id"]]) & kr.fits(eb.h, eb.lens)
                        & ((eb.h["flags"] & K.AGR_F_REPLAY) == 0))[0]
        ef = np.setdiff1d(ef, eb.dup_losers)
        for j in rng.choice(ef, 12, replace=False):
            i = int(rng.choice(np.nonzero(~taken)[0]))
            h["flags"][i] |= K.AGR_F_REPLAY
            h["replay_of"][i] = ids_of(-1 - int(j))
            h["agent_id"][i] = eb.h["agent_id"][j]
            taken[i] = True
            b.known[i] = True


def fam_many_tiles(mode):
    """one batch of at least 3 tiles per staged warp and 2 per LSU warp, then a second at an offset that is not 8 KiB aligned;
    replays and duplicate ids spread over warps and CTAs"""
    rng = np.random.default_rng(106)
    S = sms()
    target = max(3 * 16 * S, 2 * 5 * 8 * S) * kr.TILE + kr.TILE
    l1 = kr.layout(_many_spec(rng, target))
    b1 = _batch(l1, rng, 1, mode)
    l2 = kr.layout(_many_spec(rng, 150 * kr.TILE))
    b2 = _batch(l2, rng, 1 + len(l1), mode)
    for b in (b1, b2):                              # records that claim more than they store
        bad = rng.choice(len(b.lens), len(b.lens) // 100, replace=False)
        _make_bad(b.h, b.lens, bad[: len(bad) // 2], 0)
        _make_bad(b.h, b.lens, bad[len(bad) // 2:], 1)
    n1, n2 = len(l1), len(l2)
    ids = mint(0, n1 + n2) if mode == "mint" else None

    def ids_of(b, first):
        def f(j):
            if j < 0:                               # record -1 - j of batch 1
                return ids[-1 - j] if ids is not None else b1.h["request_id"][-1 - j]
            return ids[first + j] if ids is not None else b.h["request_id"][j]
        return f
    _place(b1, 0, ids_of(b1, 0), mode, rng)
    _place(b2, n1, ids_of(b2, n1), mode, rng, earlier=(b1, 0))
    _finish(b1, rng); _finish(b2, rng)
    assert b1.offs[-1] % kr.TILE != 0
    rows = 1 << (n1 + n2 + 1024).bit_length()
    return Case([b1, b2], rows=rows, vslab=int(b1.offs[-1]) + int(b2.offs[-1]) + (1 << 20))


def fam_length_rule(mode):
    """path + headers + body equal to the stored payload (stored), one byte more (AGR_VF_BAD_LEN), and the largest values
    the fields hold (0xFFFF + 0xFFFF + 0xFFFFFFFF must not wrap); 96 B records that claim one body byte"""
    rng = np.random.default_rng(108)
    lens = np.concatenate([_mixed_lens(rng, 600), np.full(40, 96)])
    b = _batch(lens, rng, 1, mode, agent_of=rng.choice(3, len(lens)))
    pay = lens - kr.HDR
    kind = rng.integers(0, 4, len(lens))
    exact = kind == 1
    b.h["body_len"][exact] = pay[exact] - b.h["path_len"][exact].astype(np.int64) - b.h["hdr_len"][exact]
    _make_bad(b.h, lens, np.nonzero((kind == 2) & (lens > 96))[0], 0)
    _make_bad(b.h, lens, np.nonzero(kind == 3)[0], 1)
    one = np.nonzero((kind == 2) & (lens == 96))[0]
    b.h["path_len"][one], b.h["hdr_len"][one], b.h["body_len"][one] = 0, 0, 1
    return Case([_finish(b, rng)], rows=1 << 11, vslab=8 << 20)


def fam_ring(mode):
    """AGR_CFG_RING with a 1 MiB byte slab and 1024 rows: batches of about 330 KB; the fourth and the seventh do not fit the
    rest of the lap and are placed at physical offset 0 (rows skip to the next lap too); expire + reclaim between laps"""
    rng = np.random.default_rng(109)
    steps, seq = [], 1
    for k in range(7):
        if k in (3, 5):
            steps.append("expire")
        spec, at = [], 0
        while at < 310000:
            v = int(_mixed_lens(rng, 1)[0]); spec.append(("rec", v)); at += v
        lens = kr.layout(spec + [("to", 330000 + 16 * k)] + [("rec", 96)] * (k + 1))
        steps.append(_finish(_batch(lens, rng, seq, mode), rng))
        seq += len(lens)
        assert len(lens) <= 512
    return Case(steps, rows=1024, vslab=1 << 20, flags=K.AGR_CFG_RING)


FAMILIES = {"most_per_tile": fam_most_per_tile, "one_per_tile": fam_one_per_tile, "stage_edges": fam_stage_edges,
            "row_edges": fam_row_edges, "tiny": fam_tiny, "many_tiles": fam_many_tiles, "length_rule": fam_length_rule,
            "ring": fam_ring}


@lru_cache(maxsize=None)
def case(name, mode) -> Case:
    return FAMILIES[name](mode)


# ------------------------------------------------------------------------------------------------------- engines
def engine(c: Case, mode, form=None):
    """form None: the fixed-stride twin"""
    flags = BASE | MODES[mode] | c.flags
    kw = dict(slab_rows=c.rows, max_agents=64, id_secret=SECRET)
    if form is None:
        flags &= ~K.AGR_CFG_VARLEN
    else:
        kw.update(vslab_bytes=c.vslab, k1_variant=FORMS[form])
    e = A.Engine(flags=flags, **kw)
    for a, s in AGENTS.items():
        e.set_agent_state(a, s)
    e.drop_agent("agent-drop")
    return e


def expire_all(e):
    e.expire(1 << 60, 1)
    e.reclaim()


@lru_cache(maxsize=None)
def twin(name, mode):
    c = case(name, mode)
    out = []
    with engine(c, mode) as e:
        for b in c.steps:
            if isinstance(b, str):
                expire_all(e)
                continue
            n = len(b.lens)
            v, ids = np.zeros(n, dtype=A.verdict_dtype), np.zeros((n, 16), dtype=np.uint8)
            first = e.ingest_ex(kr.twin_records(b.blob, b.offs), v, ids)
            out.append(dict(first=first, v=v, ids=ids, state=e.debug_read("state", first, n), route=e.debug_read("route", first, n)))
        return out, e.stats()


def _diff(a, b, what):
    bad = np.nonzero(a != b)[0]
    return f"{what}: {len(bad)} rows differ, first {bad[:8].tolist()}"


def plain_checks(b: Batch, v, state, mode):
    h, lens = b.h, b.lens
    names = [a.decode() for a in h["agent_id"]]
    found = np.array([a in FOUND for a in names])
    running = np.array([a in RUNNING for a in names])
    replay = (h["flags"] & K.AGR_F_REPLAY) != 0
    fl = v["flags"].astype(np.int64)
    bad = found & ~replay & ~kr.fits(h, lens)
    stored = found & ~replay & ~bad
    if mode == "hash":
        stored[b.dup_losers] = False
        assert (fl[b.dup_losers] & K.AGR_VF_DUP_ID).all()
    assert (((fl & K.AGR_VF_STORED) != 0) == stored).all(), _diff((fl & K.AGR_VF_STORED) != 0, stored, "stored")
    assert (((fl & K.AGR_VF_BAD_LEN) != 0) == bad).all(), _diff((fl & K.AGR_VF_BAD_LEN) != 0, bad, "bad length")
    assert (v["code"][~found] == K.AGR_V_NOT_FOUND).all()
    assert (state[stored] == kr.stored_state(h[stored], running[stored])).all() and (state[~stored] == 0).all()
    for i, k in b.known.items():
        assert bool(fl[i] & K.AGR_VF_KNOWN) == k, (i, k, int(fl[i]))
    return int(bad.sum())


def full_check(e, c: Case, mode, live, dig, tmp, final):
    """snapshot words and bytes, read-backs, pending lists and verify() over the batches ingested since the last expire"""
    ring = bool(c.flags & K.AGR_CFG_RING)
    path = os.path.join(tmp, "k1v.snap")
    e.snapshot(path)
    with open(path, "rb") as f:
        _, _, sec = snapfile.parse(f.read())
    os.remove(path)
    blobs, offs, rows, logical, state, aux, ids, hs = [], [0], [], [], [], [], [], []
    for b, first, base in live:
        n = len(b.lens)
        lg = first + np.arange(n, dtype=np.int64)
        ph = lg % c.rows if ring else lg
        assert (sec["voff"][ph] == base + b.offs[:-1].astype(np.uint64)).all(), _diff(sec["voff"][ph], base + b.offs[:-1], "voff")
        assert (sec["vlen"][ph] == np.diff(b.offs)).all(), "vlen"
        assert sec["slab"][base: base + len(b.blob)].tobytes() == b.blob.tobytes(), "slab bytes"
        dig.update(sec["voff"][ph].tobytes()); dig.update(sec["vlen"][ph].tobytes())
        blobs.append(b.blob); offs += (b.offs[1:].astype(np.int64) + offs[-1]).tolist()
        rows.append(ph); logical.append(lg); hs.append(b.h)
        state.append(e.debug_read("state", first, n)); aux.append(e.debug_read("aux", first, n))
        ids.append(e.mint_ids(first, n) if mode == "mint" else b.h["request_id"])
    blob, offs = np.concatenate(blobs), np.array(offs, dtype=np.int64)
    rows, logical, state, aux, ids, h = (np.concatenate(x) for x in (rows, logical, state, aux, ids, hs))
    exp = kr.readback(blob, offs, state, aux, ids if mode == "mint" else None)
    stored = (state & ST_STORED) != 0
    slots = {a.encode(): e.agent_slot(a) for a in FOUND}
    slot = np.array([slots.get(a, -1) for a in h["agent_id"].tolist()])
    # every stored record through one replay scan: agents by slot, FIFO inside
    e.set_agent_state("agent-stop", "running")
    disp, vb, vo = e.replay_scan_var()
    e.set_agent_state("agent-stop", "stopped")
    sel = np.nonzero(stored)[0]
    sel = sel[np.lexsort((logical[sel], slot[sel]))]
    assert len(disp) == len(sel) and (disp["rid"].astype(np.int64) == logical[sel]).all(), "dispatch order"
    want, wo = kr.gather(exp, offs, sel)
    assert (vo == wo).all(), "scan offsets"
    if vb.tobytes() != want.tobytes():
        d = np.nonzero(vb != want)[0]
        j = np.searchsorted(wo, d[0], side="right") - 1
        raise AssertionError(f"scan bytes: {len(d)} differ, first in record {sel[j]} at byte {d[0] - wo[j]}")
    dig.update(disp.tobytes()); dig.update(vb.tobytes())
    # a sample by id, too long records included (they miss), and after completions
    rng = np.random.default_rng(len(offs))
    bad = np.nonzero((kr.fits(h, np.diff(offs)) == False) & (slot >= 0) & ((h["flags"] & 1) == 0))[0]   # noqa: E712
    sample = np.concatenate([rng.choice(sel, min(48, len(sel)), replace=False), bad[:16]]).astype(np.int64)

    def by_id(k):
        return e.get_record_var(h["agent_id"][k].decode(), bytes(ids[k]))
    for k in sample:
        got = by_id(k)
        if not stored[k]:
            assert got is None, k
            continue
        assert got is not None and got.tobytes() == exp[offs[k]: offs[k + 1]].tobytes(), k
        dig.update(got.tobytes())
    if not ring:                                     # pending lists: the stored records of each agent in row order
        for a in FOUND:
            got = e.list(a, K.AGR_LIST_PENDING)
            mine = np.nonzero(stored & (h["agent_id"] == a.encode()))[0]
            assert got.tobytes() == np.ascontiguousarray(ids[mine]).tobytes(), a
    if final and len(sel):
        done = rng.choice(sel, min(24, len(sel)), replace=False)
        outs = np.zeros(len(done), dtype=A.outcome_dtype)
        outs["request_id"] = ids[done]
        outs["agent_id"] = h["agent_id"][done]
        outs["kind"] = np.where(np.arange(len(done)) % 3 == 2, K.AGR_OUT_ERROR, K.AGR_OUT_RESPONSE)
        outs["http_status"] = 200 + np.arange(len(done)) * 7
        assert (e.complete(outs) == 0).all()
        for k in done:
            lg = int(logical[k])
            st, ax = e.debug_read("state", lg, 1), e.debug_read("aux", lg, 1)
            assert st[0] != state[k]
            one = kr.readback(blob[offs[k]: offs[k + 1]], [0, offs[k + 1] - offs[k]], st, ax, ids[k:k + 1] if mode == "mint" else None)
            got = by_id(k)
            assert got is not None and got.tobytes() == one.tobytes(), k
            dig.update(got.tobytes())
    rows_checked, mismatched = e.verify()
    assert mismatched == 0 and rows_checked >= int(stored.sum())


RESULTS = {}


def run(name, mode, form):
    """K1v over the case, every check; returns a digest of everything K1v produced (for the forms' comparison)"""
    key = (name, mode, form)
    if key in RESULTS:
        return RESULTS[key]
    c = case(name, mode)
    tw, tstats = twin(name, mode)
    dig = hashlib.sha256()
    ring = bool(c.flags & K.AGR_CFG_RING)
    malformed = 0
    with engine(c, mode, form) as e, tempfile.TemporaryDirectory() as tmp:
        live, vused, bi = [], 0, 0
        for b in c.steps:
            if isinstance(b, str):
                full_check(e, c, mode, live, dig, tmp, False)
                expire_all(e)
                live = []
                continue
            n, nbytes = len(b.lens), int(b.offs[-1])
            if ring and vused % c.vslab + nbytes > c.vslab:
                vused += c.vslab - vused % c.vslab            # a blob never wraps: it starts the next lap
            base = vused % c.vslab if ring else vused
            vused += nbytes
            v, ids, first = e.ingest_var(b.blob, b.offs)
            t = tw[bi]; bi += 1
            assert first == t["first"]
            assert v.tobytes() == t["v"].tobytes(), _diff(v.view("<u8"), t["v"].view("<u8"), "verdicts")
            assert ids.tobytes() == t["ids"].tobytes(), "ids"
            state, route = e.debug_read("state", first, n), e.debug_read("route", first, n)
            assert (state == t["state"]).all(), _diff(state, t["state"], "state")
            assert (route == t["route"]).all(), _diff(route, t["route"], "route")
            ck = e.debug_read("cksum", first, n)
            assert (ck == kr.cksum(b.blob, b.offs)).all(), _diff(ck, kr.cksum(b.blob, b.offs), "cksum")
            malformed += plain_checks(b, v, state, mode)
            for x in (v, ids, state, route, ck):
                dig.update(x.tobytes())
            live.append((b, first, base))
        full_check(e, c, mode, live, dig, tmp, True)
        s = e.stats()
        for k in COUNTERS:
            assert s[k] == tstats[k], (k, s[k], tstats[k])
        assert s["malformed"] == malformed
        dig.update(repr([s[k] for k in COUNTERS]).encode())
    RESULTS[key] = dig.hexdigest()
    return RESULTS[key]


# ------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_most_records_per_tile(form, mode):
    t = kr.tile_owners(case("most_per_tile", mode).steps[0].offs)
    assert t.cnt[0] == kr.MAXCNT - 1 and t.cnt.max() == kr.MAXCNT - 1
    assert t.ntiles > 16 * sms() and (t.cnt[16 * sms():] >= 64).any()     # some staged warp's NEXT tile holds >= 64
    spr = t.starts_per_row()
    assert spr[:, 2].max() == 6 and (spr[:, 2] >= 5).mean() > 0.99
    run("most_per_tile", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_one_record_per_tile(form, mode):
    o = case("one_per_tile", mode).steps[0].offs
    t = kr.tile_owners(o)
    assert (t.cnt == 1).all() and (o % kr.TILE == 0).all()
    run("one_per_tile", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_stage_edges(form, mode):
    steps = case("stage_edges", mode).steps
    t, o = kr.tile_owners(steps[0].offs), steps[0].offs
    has = t.cnt > 0
    assert ((t.span == kr.STAGE) & (t.nglobal == 0)).any() and ((t.span == kr.STAGE + 16) & (t.nglobal == 1)).any()
    last = t.first[1:][has] - 1                                                     # each tile's last record
    assert (((o[last] % kr.TILE) == kr.TILE - 16) & (np.diff(o)[last] == 8192) & t.global_read[last]).any()
    assert (o[t.first[:-1][has]] % kr.TILE != 0).any()                             # a tile whose first start is late
    nglobal = sum(int(kr.tile_owners(b.offs).nglobal.sum()) for b in steps)
    assert nglobal >= 4
    print(f"stage edges: {nglobal} records summed through global loads")
    run("stage_edges", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_row_edges(form, mode):
    t = kr.tile_owners(case("row_edges", mode).steps[0].offs)
    same = t.tile[1:] == t.tile[:-1]
    assert (t.chunk % 32 == 31).any()
    assert (same & (t.chunk[1:] % 32 == 0) & (t.row[1:] > t.row[:-1])).any()
    empty = np.where(same, t.row[1:] - t.row[:-1] - 1, 0)                          # rows between two starts that hold none
    assert empty.max() >= 3
    assert ((t.sweep <= 32) & (t.cnt >= 5)).any() and ((t.sweep <= 32) & (t.cnt == 1)).any()
    assert t.sweep.max() == 1023 and t.chunk[0] == 0
    run("row_edges", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_trailing_tile_and_tiny_batches(form, mode):
    steps = case("tiny", mode).steps
    assert kr.tile_owners(steps[0].offs).cnt.tolist() == [2, 0] and [len(b.lens) for b in steps[1:4]] == [1, 1, 1]
    assert steps[2].lens.tolist() == [96]
    run("tiny", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_many_tiles_per_warp(form, mode):
    c = case("many_tiles", mode)
    t = kr.tile_owners(c.steps[0].offs)
    S = sms()
    staged, lsu = kr.tiles_per_warp(t.ntiles, S, False), kr.tiles_per_warp(t.ntiles, S, True)
    assert staged >= 3 and lsu >= 2
    assert (t.cnt == 0).any() and (t.cnt == 1).any() and (t.cnt == kr.MAXCNT - 1).any() and len(np.unique(t.cnt)) > 40
    print(f"many tiles: {t.ntiles} tiles, {staged:.2f} per staged warp, {lsu:.2f} per LSU warp ({S} SMs), "
          f"{int(c.steps[0].offs[-1]) >> 20} MiB; second batch at slab offset {int(c.steps[0].offs[-1])}")
    run("many_tiles", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_length_rule(form, mode):
    b = case("length_rule", mode).steps[0]
    s = b.h["path_len"].astype(np.int64) + b.h["hdr_len"] + b.h["body_len"].astype(np.int64)
    assert (s == b.lens - 96).any() and (s == b.lens - 95).any() and (s == 0xFFFF + 0xFFFF + 0xFFFFFFFF).any()
    run("length_rule", mode, form)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_byte_ring(form, mode):
    c, vused, laps = case("ring", mode), 0, 0
    for b in c.steps:
        if not isinstance(b, str):
            if vused % c.vslab + int(b.offs[-1]) > c.vslab:
                vused += c.vslab - vused % c.vslab; laps += 1
            vused += int(b.offs[-1])
    assert laps == 2
    run("ring", mode, form)


OA = ["agent-runa", "agent-runb", "agent-stop", "agent-none", "agent-drop"]   # one length: a replay's path keeps its size


def oracle_events(mode):
    """a batch of 320 requests over several CTAs of both forms, with replays naming an earlier row of the same tile, of the
    tile before (another warp of the same CTA), of a tile 16 before (another CTA), a later row, a replay, another agent's
    record; then a batch of 80 with replays of the first; then a replay tick.  Ids: the engine's minted ids (predicted from
    the row) or the scenario's."""
    import dataclasses
    from scenario import Req, make_var_batch, rid_of
    rng = np.random.default_rng(110)
    n1, n2 = 320, 80
    ids = mint(0, n1 + n2) if mode == "mint" else None
    rid = (lambda k: bytes(ids[k])) if ids is not None else (lambda k: rid_of(k + 1))
    ag = _agents(rng, n1 + n2)
    sizes = np.exp(rng.uniform(np.log(16), np.log(5000), n1 + n2)).astype(int)
    reqs = [Req(OA[ag[k]], rid(k), k + 1, body=rng.integers(32, 127, sizes[k], dtype=np.uint8).tobytes()) for k in range(n1 + n2)]
    _, o1 = make_var_batch(reqs[:n1])
    t = kr.tile_owners(o1)
    F = t.first
    assert t.ntiles >= 24
    found = lambda j: ag[j] < 3 and not reqs[j].replay

    def rep(i, j, agent=None):
        if reqs[i].replay or not 0 <= j < n1 + n2:
            return
        reqs[i] = dataclasses.replace(reqs[i], replay=True, replay_of=reqs[j].rid, agent_id=agent or reqs[j].agent_id)
    for k in range(t.ntiles):
        if t.cnt[k] >= 2 and found(F[k]):
            rep(F[k + 1] - 1, F[k])                                       # same tile
        if k % 8 and t.cnt[k] and t.cnt[k - 1] and found(F[k - 1]):
            rep(F[k], F[k - 1])                                           # another warp of the same CTA
        if k >= 16 and t.cnt[k] >= 3 and t.cnt[k - 16] and found(F[k - 16]):
            rep(F[k] + 1, F[k - 16])                                      # another CTA
        if k + 2 < t.ntiles and t.cnt[k] >= 4 and t.cnt[k + 2] and ag[F[k + 2]] == 2:
            rep(F[k] + 2, F[k + 2])                                       # a later row (of a stopped agent: the replay is queued,
                                                                          # so no outcome of it meets the later record)
        if k >= 2 and t.cnt[k] >= 5 and reqs[F[k - 2]].replay:
            rep(F[k] + 3, F[k - 2])                                       # the target is a replay
        if k % 5 == 0 and t.cnt[k] >= 6:
            rep(F[k] + 4, F[k] + 1, agent="agent-runa" if ag[F[k] + 1] != 0 else "agent-runb")   # another agent's record
    for k in range(n1, n1 + n2, 3):
        rep(k, int(rng.integers(0, n1)))                                  # the previous batch
    assert sum(r.replay for r in reqs) > 40
    backends = [("response", 200), ("dial",), ("error",), ("response", 500)]
    ev = [("agent", "agent-runa", "running"), ("agent", "agent-runb", "running"), ("agent", "agent-stop", "stopped"),
          ("agent", "agent-drop", "running"), ("remove", "agent-drop")]
    ev += [("req", r, backends[k % 4]) for k, r in enumerate(reqs[:n1])]
    ev += [("agent", "agent-stop", "stopped")]
    ev += [("req", r, backends[k % 3]) for k, r in enumerate(reqs[n1:])]
    ev += [("tick", {}, None)]
    return ev


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", FORMS)
def test_decisions_against_oracle(form, mode):
    from scenario import assert_same, run_engine, run_oracle
    ev = oracle_events(mode)
    with A.Engine(flags=BASE | MODES[mode], slab_rows=1 << 12, max_agents=64, vslab_bytes=64 << 20, k1_variant=FORMS[form],
                  id_secret=SECRET) as eng:
        got = run_engine(eng, ev)
        hits = eng.stats()["dedupe_hits"]
    assert_same(run_oracle(ev), got)
    assert hits > 20


@pytest.mark.parametrize("name", FAMILIES)
@pytest.mark.parametrize("mode", MODES)
def test_forms_agree(name, mode):
    assert run(name, mode, "staged") == run(name, mode, "lsu")
