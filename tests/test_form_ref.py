"""The plain reference of a restore that converts the record form (tests/formref.py) on small handmade snapshots.  Needs no
GPU."""
import numpy as np
import pytest

from agentainer_lab_b200 import constants as K
from formref import NoSpace, NotRepresentable, bad_rows, compact_len, convert, convert_loop
from resizeref import content, log_rows, relocate
from snapfile import HEADER, WORDS
from test_resize_ref import make

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
NONE = 0xFFFFFFFF
LIVE = set(range(30, 61)) - {33, 40, 41}
RESP = {L: (L * 13) % 70 for L in LIVE}
ERR = {L: (L * 7) % 20 for L in LIVE if L % 3 == 0}
LOGS = ([31, 44, 59, 35], [36, None, 60])


def records(sec, hd, seed=0, dirty=()):
    """Every live 512 B row of a fixed-stride file gets a record with valid lengths (path + headers + body from 0 to 416 B)
    and zeros past them, except the row ids in dirty, which get a non-zero byte past their compact length."""
    rng = np.random.default_rng(seed)
    rows = sec["slab"].reshape(-1, 512)
    S, ring = int(hd["slab_rows"]), bool(int(hd["flags"]) & R)
    for L in range(int(hd["tail"]), int(hd["rows_used"])):
        p = L % S if ring else L
        if sec["state"][p] == 0:
            continue
        total = 100 + L % 50 if L in dirty else int(rng.integers(0, 417)) if L % 4 else 416 - (L % 3)
        path = int(rng.integers(0, min(total, 60) + 1))
        hdr = int(rng.integers(0, total - path + 1))
        rows[p] = 0
        rows[p, :76] = rng.integers(0, 256, 76, dtype=np.uint8)
        rows[p, 76:84] = np.frombuffer(np.array([path, hdr], "<u2").tobytes() + np.array([total - path - hdr], "<u4").tobytes(), np.uint8)
        rows[p, 84:96] = rng.integers(0, 256, 12, dtype=np.uint8)
        rows[p, 96: 96 + total] = rng.integers(1, 256, total, dtype=np.uint8)
        if L in dirty:
            rows[p, compact_len(rows[p]) + int(rng.integers(0, 512 - compact_len(rows[p])))] = 7
    return hd, sec


def fixed(flags, slab_rows=40, tail=30, used=61, seed=0, dirty=()):
    hd, ag, sec = make(flags & ~V, slab_rows, tail, used, LIVE, resp=RESP, err=ERR, logs=LOGS, seed=seed)
    sec = {k: np.array(v) for k, v in sec.items()}
    records(sec, hd, seed, dirty)
    return hd, ag, sec


def variable(flags, slab_rows=40, tail=30, used=61, seed=0):
    hd, ag, sec = make(flags | V, slab_rows, tail, used, LIVE, resp=RESP, err=ERR, logs=LOGS, seed=seed)
    return hd, ag, {k: np.array(v) for k, v in sec.items()}


def same(a, b):
    (hd_a, ag_a, sec_a), (hd_b, ag_b, sec_b) = a, b
    assert np.array(hd_a, dtype=HEADER).tobytes() == np.array(hd_b, dtype=HEADER).tobytes(), (hd_a, hd_b)
    assert ag_a == ag_b
    assert sorted(sec_a) == sorted(sec_b)
    for name in sec_a:
        assert sec_a[name].dtype == sec_b[name].dtype and np.array_equal(sec_a[name], sec_b[name]), name


SOURCES = {"fixed_ring": (fixed, P | M | R), "fixed_append": (fixed, P | M), "var_ring": (variable, P | R), "var_append": (variable, P | M)}


@pytest.mark.parametrize("geom", [(40, 16000), (33, 16000), (77, 20000), (31, 15000)])
@pytest.mark.parametrize("src", sorted(SOURCES))
def test_loop_form_is_the_array_form(src, geom):
    build, flags = SOURCES[src]
    hd, ag, sec = build(flags)
    target = (int(hd["flags"]) ^ V) | R
    S, cap = geom
    a = convert(hd, ag, sec, target, S, cap, cap)
    same(a, convert_loop(hd, ag, sec, target, S, cap, cap))
    assert log_rows(a[0], a[2]) == log_rows(hd, sec)
    got, want = content(a[0], a[2]), content(hd, sec)
    assert sorted(got) == sorted(want) == sorted(LIVE)
    for L, (words, rec, segs) in got.items():
        w_words, w_rec, w_segs = want[L]
        assert words[:4] == w_words[:4] and words[-5:] == w_words[-5:] and segs == w_segs, L   # (vlen is the form's own)
        if target & V:                                  # the row's first compact-length bytes
            assert rec == w_rec[: compact_len(np.frombuffer(w_rec, np.uint8))], L
        else:                                           # the record, then zeros
            assert rec == w_rec + bytes(512 - len(w_rec)), L


@pytest.mark.parametrize("flags", [P | M | R, P | R, P | M])
def test_fixed_to_variable_and_back_is_a_relocation(flags):
    """On zero-padded records the round trip is what a relocation of the original into the last geometry gives."""
    hd, ag, sec = fixed(flags)
    mid = convert(hd, ag, sec, (flags | V) | R, 37, 16000, 3000)
    assert int(mid[0]["vused"]) == sum(compact_len(sec["slab"][(L % 40 if flags & R else L) * 512:][:512]) for L in LIVE)
    assert bad_rows(hd, sec) == []
    back = convert(*mid, flags | R, 50, 0, 2900)
    same(back, relocate(hd, ag, sec, flags | R, 50, 0, 2900))


def test_bad_rows_are_the_dirty_ones():
    dirty = {31, 44, 52, 59}
    hd, ag, sec = fixed(P | M | R, dirty=dirty)
    assert bad_rows(hd, sec) == sorted(dirty)
    mid = convert(hd, ag, sec, P | M | V | R, 40, 16000, 3000)
    back = convert(*mid, P | M | R, 40, 0, 3000)           # the bytes past the compact length do not come back
    for L in LIVE:
        p = L % 40
        a, b = back[2]["slab"][p * 512: (p + 1) * 512], sec["slab"][p * 512: (p + 1) * 512]
        assert np.array_equal(a, b) == (L not in dirty), L


def test_oversized_records_are_refused():
    hd, ag, sec = variable(P | R)
    L, dead = 45, 40
    sec["vlen"][L % 40] = 528
    sec["vlen"][dead % 40] = 4096                          # a row that holds no record does not count
    with pytest.raises(NotRepresentable, match=r"1 live records .* row 45, 528 B"):
        convert(hd, ag, sec, P | R, 40, 0, 3000)
    sec["vlen"][50 % 40] = 513
    with pytest.raises(NotRepresentable, match=r"2 live records .* row 45, 528 B"):
        convert(hd, ag, sec, P | R, 40, 0, 3000)
    with pytest.raises(NoSpace, match="window"):             # the window is refused first
        convert(hd, ag, sec, P | R, 30, 0, 3000)
    sec["vlen"][45 % 40] = sec["vlen"][50 % 40] = 512
    convert(hd, ag, sec, P | R, 40, 0, 3000)


def test_byte_rings_too_small():
    hd, ag, sec = fixed(P | M | R)
    need = int(convert(hd, ag, sec, P | M | V | R, 40, 1 << 20, 1 << 20)[0]["vused"])
    rsp = int(convert(hd, ag, sec, P | M | V | R, 40, 1 << 20, 1 << 20)[0]["resp_used"])
    with pytest.raises(NoSpace, match="vslab_bytes"):
        convert(hd, ag, sec, P | M | V | R, 40, need - 1, 1 << 20)
    with pytest.raises(NoSpace, match="resp_bytes"):
        convert(hd, ag, sec, P | M | V | R, 40, need, rsp - 1)
    assert int(convert(hd, ag, sec, P | M | V | R, 40, need, rsp)[0]["vused"]) == need


def test_empty_window():
    hd, ag, sec = make(P | M | R, 16, 20, 20, set())
    sec = {k: np.array(v) for k, v in sec.items()}
    out = convert(hd, ag, sec, P | M | V | R, 8, 64, 64)
    same(out, convert_loop(hd, ag, sec, P | M | V | R, 8, 64, 64))
    assert int(out[0]["vused"]) == 0 and all(not len(out[2][w]) or not out[2][w].any() for w in WORDS)
