"""The plain restatement of the compare cut's keyed digest (snapfile.digest) against a one-piece-at-a-time loop, on small
files with every kind of short last piece.  Needs no GPU; tests/test_restore_scale_gpu.py holds the engine's digests to it."""
import numpy as np
import pytest

from agentainer_lab_b200 import constants as K
from snapfile import HEADER, WORDS, digest, digest_sections, sections

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
MASK = (1 << 64) - 1


def fmix(k):
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & MASK
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & MASK
    return k ^ (k >> 33)


def digest_loop(hd, sec, key):
    """k_snap_cmp's sum, piece by piece, in Python integers"""
    h0 = h1 = 0
    for s, b in digest_sections(hd, sec):
        skey = fmix((key ^ ((s + 1) << 56)) & MASK)
        for i in range(0, len(b), 16):
            piece = b[i: i + 16].ljust(16, b"\0")
            a, c = int.from_bytes(piece[:8], "little"), int.from_bytes(piece[8:], "little")
            t = fmix((skey + (i // 16) * 0x9E3779B97F4A7C15) & MASK)
            h0 = (h0 + fmix(fmix(t ^ a) ^ c)) & MASK
            h1 = (h1 + fmix(fmix(((t + 0x632BE59BD9B4E019) & MASK) ^ c) ^ a)) & MASK
    return h0, h1


def small(flags, rows, logs, seed=0):
    rng = np.random.default_rng(seed)
    hd = np.zeros(1, dtype=HEADER)[0]
    hd["magic"], hd["flags"], hd["rows_used"], hd["slab_rows"] = b"AGRSNAP3", flags, rows, max(rows, 1)
    hd["log_len"] = logs
    hd["vused"], hd["vcap"], hd["resp_used"], hd["resp_cap"] = 64, 64, 48, 48
    sec = {name: rng.integers(0, 1 << 63, count, dtype=np.uint64).astype(dt) for name, dt, count in sections(hd)}
    return hd, sec


# rows 1..3: 4 B words leave a last piece of 4, 8 or 12 bytes; logs of 1..3 entries the same
@pytest.mark.parametrize("rows", [0, 1, 2, 3, 4, 5, 7, 9])
@pytest.mark.parametrize("flags", [P | M, P | M | V | R, P | R])
def test_digest_is_the_piece_loop(flags, rows):
    for logs in ((0, 0), (1, 2), (3, 4), (5, 0)):
        hd, sec = small(flags, rows, logs, seed=rows)
        key = 0x5EED_1234_ABCD_0002 + rows
        assert digest(hd, sec, key) == digest_loop(hd, sec, key), logs


def test_which_sections_and_ids():
    hd, sec = small(P | M, 3, (2, 1))
    ids = [s for s, _ in digest_sections(hd, sec)]
    assert ids == [1, 2, 3, 4, 10, 11, 12, 13, 14, 15, 16, 7, 8]          # no slab, voff / vlen (empty), resp; the logs last
    hd, sec = small(P | M | V, 3, (2, 1))
    assert [s for s, _ in digest_sections(hd, sec)] == [1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 14, 15, 16, 7, 8]
    assert sum(len(b) for _, b in digest_sections(hd, sec)) == 3 * sum(np.dtype(dt).itemsize for n, dt, _ in sections(hd) if n in WORDS) + 12


def test_every_byte_and_place_counts():
    """a change anywhere in a summed section, the same bytes in another section, and the key all change the digest; the slab
    and the response bytes do not enter it"""
    hd, sec = small(P | M | V | R, 7, (3, 2), seed=4)
    key = 99
    base = digest(hd, sec, key)
    assert digest(hd, sec, key + 1) != base
    for name in WORDS + ("completed_log", "failed_log"):
        s2 = {k: v.copy() for k, v in sec.items()}
        s2[name].view(np.uint8)[-1] ^= 1
        assert digest(hd, s2, key) != base, name
    s2 = {k: v.copy() for k, v in sec.items()}
    s2["state"], s2["route"] = sec["route"].copy(), sec["state"].copy()   # the same bytes in the other section
    assert digest(hd, s2, key) != base
    s2 = {k: v.copy() for k, v in sec.items()}
    s2["slab"][:] ^= 0xFF
    s2["resp"][:] ^= 0xFF
    assert digest(hd, s2, key) == base
