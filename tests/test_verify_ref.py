"""CPU checks of tests/verifyref.py, the plain reference of the integrity sweep (agr_verify): hand-worked checksums with what
the checksum does and does not detect, and the sweep's rules for rows past vlen, non-stored rows, reservations and rows with
more than one change.  No GPU."""
import numpy as np
import pytest

import k1ref
import k1vref
import verifyref as V
from agentainer_lab_b200 import binding as B

M32 = (1 << 32) - 1


def ck(words):
    """the checksum by hand: c1 << 32 | c0, c0 = sum w_k, c1 = sum (k + 1) w_k, mod 2^32"""
    c0 = sum(int(w) for w in words) & M32
    c1 = sum((k + 1) * int(w) for k, w in enumerate(words)) & M32
    return (c1 << 32) | c0


def rows_of(words_per_row):
    """fixed-stride slab from rows of 128 u32 words"""
    return np.asarray(words_per_row, dtype="<u4").reshape(-1, 128).view(np.uint8).reshape(-1)


def fixed(words, *, ring=False, state=None, resv=(), slab_rows=None, cksum=None):
    """sweep a fixed-stride slab whose checksum words are the hand checksums of `cksum` (default: of `words`)"""
    words = np.asarray(words, dtype=np.uint32).reshape(-1, 128)
    n = len(words)
    ref = words if cksum is None else np.asarray(cksum, dtype=np.uint32).reshape(-1, 128)
    ck_words = np.array([ck(r) for r in ref], dtype=np.uint64)
    st = np.full(n, V.ST_STORED, np.uint32) if state is None else np.asarray(state, np.uint32)
    return V.sweep(st, ck_words, rows_of(words), span=n, ring=ring, resv=resv, slab_rows=slab_rows)


RNG = np.random.default_rng(20261018)
ROW = RNG.integers(0, 1 << 32, 128, dtype=np.uint64).astype(np.uint32)


def test_hand_checksum_matches_both_restatements():
    rows = RNG.integers(0, 1 << 32, (9, 128), dtype=np.uint64).astype(np.uint32)
    rows[0] = 0
    rows[1] = M32
    hand = np.array([ck(r) for r in rows], dtype=np.uint64)
    slab = rows_of(rows)
    assert (k1ref.cksum(slab.view(B.record_dtype)) == hand).all()
    assert (k1vref.cksum(slab, np.arange(10, dtype=np.uint32) * 512) == hand).all()
    assert (V.record_cksums(np.arange(9), slab) == hand).all()
    assert (V.record_cksums(np.arange(9), slab, voff=np.arange(9) * 512, vlen=np.full(9, 512)) == hand).all()


def test_k1ref_and_k1vref_agree_on_512_byte_records():
    recs = B.synth_fill_host(0, 300, seed=5, n_agents=7)
    blob = np.ascontiguousarray(recs).view(np.uint8).reshape(-1)
    assert (k1ref.cksum(recs) == k1vref.cksum(blob, np.arange(301, dtype=np.uint32) * 512)).all()


@pytest.mark.parametrize("k", range(128))
def test_every_word_of_a_512_byte_row_is_covered(k):
    for delta in (1, 0x80000000, int(RNG.integers(1, 1 << 32))):
        bad = ROW.copy()
        bad[k] = (int(bad[k]) + delta) & M32
        s = fixed(bad, cksum=ROW)
        assert s.checked == 1 and s.bad.tolist() == [0], (k, delta)
    assert fixed(ROW).bad.tolist() == []


@pytest.mark.parametrize("k", [0, 1024, 2047])
def test_first_middle_and_last_word_of_an_8_kib_record(k):
    w = RNG.integers(0, 1 << 32, 2048, dtype=np.uint64).astype(np.uint32)
    slab = np.concatenate([np.zeros(32, np.uint8), w.view(np.uint8)])
    state = np.array([V.ST_STORED], np.uint32)
    good = np.array([ck(w)], np.uint64)
    s = V.sweep(state, good, slab, span=1, ring=False, voff=np.array([32]), vlen=np.array([8192]))
    assert s.checked == 1 and s.bad.tolist() == []
    for delta in (1, 0x80000000, 0xFFFFFFFF):
        b = w.copy()
        b[k] = (int(b[k]) + delta) & M32
        sb = np.concatenate([np.zeros(32, np.uint8), b.view(np.uint8)])
        assert V.sweep(state, good, sb, span=1, ring=False, voff=np.array([32]), vlen=np.array([8192])).bad.tolist() == [0]


@pytest.mark.parametrize("a,b,d", [(0, 1, 1), (5, 6, 2), (0, 0x80000000, 1), (0, 0x80000000, 3), (0, 0x40000000, 2),
                                   (7, 0xFFFFFFFF, 127), (1, 2, 64)])
def test_swaps_of_unequal_words_that_are_detected(a, b, d):
    assert (d * (b - a)) % (1 << 32) != 0
    j = 127 - d
    row = ROW.copy()
    row[j], row[j + d] = a, b
    sw = row.copy()
    sw[j], sw[j + d] = b, a
    assert fixed(sw, cksum=row).bad.tolist() == [0]


def test_what_the_checksum_cannot_see():
    # a swap of words holding 0 and 0x80000000 two apart: c1 moves by 2 * 0x80000000 = 0 mod 2^32
    row = ROW.copy()
    row[4], row[6] = 0, 0x80000000
    sw = row.copy()
    sw[4], sw[6] = 0x80000000, 0
    assert ck(sw) == ck(row)
    assert fixed(sw, cksum=row).bad.tolist() == []
    # bit 31 flipped in words k and k + 2, at every k
    for k in range(126):
        fl = ROW.copy()
        fl[k] ^= 0x80000000
        fl[k + 2] ^= 0x80000000
        assert ck(fl) == ck(ROW), k
        assert fixed(fl, cksum=ROW).bad.tolist() == [], k
    # the same flip one word apart is seen
    fl = ROW.copy()
    fl[3] ^= 0x80000000
    fl[4] ^= 0x80000000
    assert fixed(fl, cksum=ROW).bad.tolist() == [0]


def test_a_change_past_vlen_is_not_counted():
    w = RNG.integers(0, 1 << 32, 64, dtype=np.uint64).astype(np.uint32)
    slab = w.view(np.uint8).copy()
    st = np.full(2, V.ST_STORED, np.uint32)
    ck2 = np.array([ck(w[:24]), ck(w[24:48])], np.uint64)           # two records of 96 B, then 64 B that no row holds
    kw = dict(span=2, ring=False, voff=np.array([0, 96]), vlen=np.array([96, 96]))
    assert V.sweep(st, ck2, slab, **kw).bad.tolist() == []
    slab[192] ^= 0xFF
    assert V.sweep(st, ck2, slab, **kw).bad.tolist() == []
    slab[191] ^= 0xFF
    assert V.sweep(st, ck2, slab, **kw).bad.tolist() == [1]


def test_vlen_zero_has_no_bytes_and_checksum_zero():
    slab = np.full(512, 0xAB, np.uint8)
    st = np.full(2, V.ST_STORED, np.uint32)
    kw = dict(span=2, ring=False, voff=np.array([0, 0]), vlen=np.array([0, 0]))
    s = V.sweep(st, np.array([0, 5], np.uint64), slab, **kw)
    assert s.checked == 2 and s.bad.tolist() == [1]


def test_two_changes_in_one_row_count_once():
    rows = np.tile(ROW, (3, 1))
    bad = rows.copy()
    bad[1, 0] ^= 1
    bad[1, 100] ^= 1 << 7
    s = fixed(bad, cksum=rows)
    assert s.checked == 3 and s.bad.tolist() == [1]


def test_non_stored_rows_skipped_on_a_ring_and_counted_append_only():
    rows = np.tile(ROW, (4, 1))
    bad = rows.copy()
    bad[:, 9] ^= 0x100                                               # every row changed
    state = np.array([V.ST_STORED, 0, V.ST_STORED | 0x7, 0x7], np.uint32)
    ring = fixed(bad, cksum=rows, ring=True, state=state, slab_rows=4)
    assert ring.checked == 4 and ring.bad.tolist() == [0, 2] and ring.examined.tolist() == [0, 2]
    flat = fixed(bad, cksum=rows, ring=False, state=state)
    assert flat.checked == 4 and flat.bad.tolist() == [0, 1, 2, 3]


def test_undecided_reservations_are_skipped():
    rows = np.tile(ROW, (10, 1))
    zero = np.zeros(10, np.uint64)
    slab = rows_of(rows)
    st = np.full(10, V.ST_STORED, np.uint32)
    # append-only: rows 3..5 reserved and filled, their checksum still 0
    s = V.sweep(st, zero, slab, span=10, ring=False, resv=[(3, 6)])
    assert s.checked == 7 and s.bad.tolist() == [0, 1, 2, 6, 7, 8, 9]
    # a ring of 10 rows whose reservation (logical 18..22) wraps: physical 8, 9, 0, 1
    s = V.sweep(st, zero, slab, span=10, ring=True, resv=[(18, 22)], slab_rows=10)
    assert s.checked == 6 and s.bad.tolist() == [2, 3, 4, 5, 6, 7]
    # rows past rows_span are not swept at all
    s = V.sweep(st, zero, slab, span=4, ring=False, resv=[(2, 3)])
    assert s.checked == 3 and s.bad.tolist() == [0, 1, 3]
