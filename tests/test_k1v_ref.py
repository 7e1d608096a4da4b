"""The plain K1v reference (tests/k1vref.py) on hand-worked cases: tile ownership at tile boundaries, a trailing tile that owns
nothing, the most starts one tile can hold, the stage and sweep facts the GPU tests rely on, the checksum against the
record-at-a-time loop, the fixed-stride twin's length split at its exact boundary, and the read-back bytes.  CPU only."""
import numpy as np

import k1vref as kr
from agentainer_lab_b200 import constants as K


def tile_first_loop(offsets):
    """k1v_tile_index, one record at a time: record i is the first record of every tile boundary in (start(i-1), start(i)]."""
    o = [int(x) for x in offsets]
    n, ntiles = len(o) - 1, (o[-1] + kr.TILE - 1) // kr.TILE
    tf = [None] * (ntiles + 1)
    for i in range(n + 1):
        lo = 0 if i == 0 else o[i - 1] // kr.TILE + 1
        hi = ntiles if i == n else o[i] // kr.TILE
        for t in range(lo, hi + 1):
            tf[t] = i
    return tf


def offs_of(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)


def test_record_on_a_tile_boundary():
    o = offs_of([8192, 96, 8096, 96])              # records 1 and 3 start exactly at 8192 and 16384
    t = kr.tile_owners(o)
    assert t.first.tolist() == [0, 1, 3, 4] == tile_first_loop(o)
    assert t.cnt.tolist() == [1, 2, 1] and t.tile.tolist() == [0, 1, 1, 2]
    assert t.span.tolist() == [8192, 8192, 96] and not t.over.any()


def test_trailing_tile_owns_nothing():
    o = offs_of([96, 8192, 8192])                  # starts 0, 96, 8288; the blob reaches into tile 2, where nothing starts
    t = kr.tile_owners(o)
    assert t.ntiles == 3 and t.first.tolist() == [0, 2, 3, 3] == tile_first_loop(o)
    assert t.cnt.tolist() == [2, 1, 0] and t.span.tolist() == [8288, 8192, 0]
    assert t.over.tolist() == [False, False, False]
    assert t.sweep.tolist() == [518, 512, 0]
    o = offs_of([8192 - 16, 8192, 96])             # starts 0, 8176 (16 B before tile 1), 16368 (16 B before tile 2)
    t = kr.tile_owners(o)
    assert t.first.tolist() == [0, 2, 3, 3] == tile_first_loop(o)
    assert t.span[0] == 8176 + 8192 and t.over[0] and t.nglobal[0] == 1 and t.global_read.tolist() == [False, True, False]
    assert t.sweep[0] == 1023                      # the longest sweep the LSU form can meet
    assert t.chunk[2] == 0 and t.span[1] == 96     # tile 1's first start is 16368, not its base


def test_most_starts_in_one_tile():
    o = offs_of([96] * 200)
    t = kr.tile_owners(o)
    assert t.cnt[0] == 86 == kr.MAXCNT - 1 and t.first.tolist() == tile_first_loop(o)
    spr = t.starts_per_row()
    assert spr[0].tolist() == [0, 0, 6]            # chunks 0, 6, 12, 18, 24, 30
    r0 = spr[spr[:, 0] == 0]                       # 86 records x 6 chunks: rows 0..15 hold 5 or 6 starts each
    assert len(r0) == 16 and set(r0[:, 2].tolist()) == {5, 6} and r0[:, 2].sum() == 86


def test_stage_edges():
    t = kr.tile_owners(offs_of([6400, 6400, 96]))
    assert t.span[0] == kr.STAGE and not t.over[0] and t.nglobal[0] == 0
    t = kr.tile_owners(offs_of([6400, 6416, 96]))
    assert t.span[0] == kr.STAGE + 16 and t.over[0] and t.global_read.tolist() == [False, True, False]
    lens = kr.layout([("rec", 496), ("rec", 528), ("to", 8192 * 3 - 16), ("rec", 7776)])
    o = offs_of(lens)
    assert o[2] == 1024 and (o[-2], o[-1]) == (8192 * 3 - 16, 8192 * 4 - 432) and (np.diff(o) >= 96).all()
    t = kr.tile_owners(o)
    assert t.chunk[1] == 31 and t.chunk[2] == 64 and t.row[2] == 2


def test_grid():
    assert kr.grid(10, 132, False) == (1, 16) and kr.grid(10, 132, True) == (2, 8)
    assert kr.grid(100000, 132, False) == (132, 16) and kr.grid(100000, 132, True) == (660, 8)
    assert kr.cta_of(np.array([0, 15, 16, 2112, 2128]), 100000, 132, False).tolist() == [0, 0, 1, 0, 1]


def test_cksum_matches_the_loop():
    rng = np.random.default_rng(5)
    lens = np.array([96, 112, 8192, 4000, 96, 5008, 8192, 96] * 5, dtype=np.int64)
    blob = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8)
    blob[96:96 + 4 * 28] = 0xFF                     # words near 2^32: the sums wrap
    offs = offs_of(lens)
    ck = kr.cksum(blob, offs)
    for i in range(len(lens)):
        w = blob[offs[i]: offs[i + 1]].view(np.uint32).astype(np.uint64)
        c0 = int(w.sum()) & 0xFFFFFFFF
        c1 = int((w * np.arange(1, len(w) + 1, dtype=np.uint64)).sum()) & 0xFFFFFFFF
        assert int(ck[i]) == (c1 << 32) | c0, i


def _batch(lens, sums):
    rng = np.random.default_rng(7)
    h = kr.headers(len(lens), ["agent-a"], rng)
    h["path_len"], h["hdr_len"] = 10, 20
    h["body_len"] = np.asarray(sums) - 30
    return h, kr.blob_from(h, lens, rng)


def test_twin_keeps_the_fits_split_at_the_boundary():
    lens = [256, 256, 96, 8192, 8192, 512]
    h, (blob, offs) = _batch(lens, [160, 161, 30, 8096, 8097, 416])
    h[2]["body_len"] = 1                           # 96 B record: no payload, one body byte claimed
    h[5]["path_len"], h[5]["hdr_len"], h[5]["body_len"] = 0xFFFF, 0xFFFF, 0xFFFFFFFF
    blob, offs = kr.blob_from(h, lens, np.random.default_rng(7))
    fit = kr.fits(h, lens)
    assert fit.tolist() == [True, False, False, True, False, False]
    t = kr.twin_records(blob, offs)
    s = t["path_len"].astype(np.int64) + t["hdr_len"] + t["body_len"].astype(np.int64)
    assert ((s <= 416) == fit).all() and s[1] > 416 and s[2] > 416 and s[4] > 416
    assert s[5] == 0xFFFF + 0xFFFF + 0xFFFFFFFF    # not wrapped
    assert s[0] == 160 and s[3] <= 416
    raw = t.view(np.uint8).reshape(len(t), 512)
    hb = kr.header_of(blob, offs).view(np.uint8).reshape(len(t), 96)
    for f in ("request_id", "replay_of", "agent_id", "seq", "flags", "status", "retry_count", "max_retries", "error_code", "resp_status"):
        assert (t[f] == h[f]).all(), f
    assert (raw[:, :72] == hb[:, :72]).all() and (raw[:, 84:96] == hb[:, 84:96]).all()


def test_readback_of_a_record_with_max_retries_0():
    rng = np.random.default_rng(9)
    lens = [160, 96]
    h = kr.headers(2, ["agent-a"], rng)
    kr.fit_lens(h, lens, rng)
    h["max_retries"] = [0, 5]
    blob, offs = kr.blob_from(h, lens, rng)
    state = kr.stored_state(h, [True, False])
    assert state.tolist() == [1 | 8 | 0x10 | 0x20 | 3 << 16, 1 | 8 | 0x20 | 5 << 16]
    aux = np.array([0, 503 | 4 << 16], dtype=np.uint32)
    ids = np.arange(32, dtype=np.uint8).reshape(2, 16)
    out = kr.readback(blob, offs, state, aux, ids)
    assert out[84:90].tolist() == [1, 0, 3, 0, 0, 0]         # pending, retry 0, max 3, no error, no response
    assert out[160 + 84: 160 + 90].tolist() == [1, 0, 5, 4, 503 & 255, 503 >> 8]
    assert out[:16].tolist() == list(range(16)) and out[160:176].tolist() == list(range(16, 32))
    keep = np.ones(len(blob), dtype=bool)
    for o in (0, 160):
        keep[o: o + 16] = False; keep[o + 84: o + 90] = False
    assert (out[keep] == blob[keep]).all()
    plain = kr.readback(blob, offs, state, aux)                # hash mode: the caller's id stays
    assert (plain[:16] == blob[:16]).all()
    sel, go = kr.gather(out, offs, [1, 0])
    assert go.tolist() == [0, 96, 256] and (sel[:96] == out[160:]).all() and (sel[96:] == out[:160]).all()


def test_layout_and_fit_lens_follow_the_wire_contract():
    rng = np.random.default_rng(11)
    lens = kr.layout([("rec", 96), ("to", 20000), ("rec", 8192), ("to", 40960 - 16), ("rec", 112)])
    o = offs_of(lens)
    assert 20000 in o.tolist() and 40944 in o.tolist() and o[-1] == 40944 + 112
    h = kr.headers(len(lens), ["a", "b"], rng)
    kr.fit_lens(h, lens, rng)
    s = h["path_len"].astype(np.int64) + h["hdr_len"] + h["body_len"]
    assert (96 + (s + 15) // 16 * 16 == lens).all() and kr.fits(h, lens).all()
    assert h["agent_id"].tolist()[:2] == [b"a", b"b"] and (h["request_id"][:, 0] & 1).all()
    assert int(K.AGR_VAR_MAX_RECORD) == kr.MAXREC
