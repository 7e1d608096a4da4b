"""The plain reference of a relocating restore (tests/resizeref.py) on small handmade snapshots.  Needs no GPU."""
import numpy as np
import pytest

from agentainer_lab_b200 import constants as K
from resizeref import NoSpace, content, log_rows, relocate
from snapfile import HEADER, WORDS, sections

P, M, V, R = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_VARLEN, K.AGR_CFG_RING
NONE = 0xFFFFFFFF


def make(flags, slab_rows, tail, used, live, resp=None, err=None, logs=((), ()), vcap=4096, resp_cap=4096, seed=0):
    """A full file's parsed form: rows [tail, used) of a ring (or an append-only slab), the row ids in live stored, each with
    a record of 40 + 7 * (L % 5) bytes (AGR_CFG_VARLEN) and the given response / error lengths, laid out the way an engine
    lays them: in arrival order from the window's first byte, wrapping at the capacity, responses on 16 B boundaries."""
    rng = np.random.default_rng(seed)
    resp, err = resp or {}, err or {}
    hd = np.zeros(1, dtype=HEADER)[0]
    hd["magic"], hd["flags"], hd["n_agents"], hd["shard"], hd["gen"] = b"AGRSNAP3", flags, 0, 3, 1
    hd["tail"], hd["rows_used"], hd["released_total"], hd["scan_lo"] = tail, used, tail, tail
    hd["slab_rows"], hd["vcap"], hd["resp_cap"], hd["id_secret"] = slab_rows, vcap if flags & V else 0, resp_cap, 77
    hd["log_len"] = [len(logs[0]), len(logs[1])]
    ring = bool(flags & R)
    vat, rat = 1000, 2000                                # where the window's bytes start (logical)
    hd["vtail"], hd["resp_tail"] = vat, rat
    phys = {L: (L % slab_rows if ring else L) for L in range(tail, used)}
    vbytes, rbytes, words = {}, {}, {}
    for L in range(tail, used):
        if L not in live:
            continue
        n = 40 + 7 * (L % 5)
        vbytes[L] = (vat, rng.integers(0, 256, n, dtype=np.uint8)); vat += n
        for kind, lens in (("resp", resp), ("err", err)):
            n = lens.get(L, 0)
            if n:
                rbytes[(L, kind)] = (rat, rng.integers(0, 256, n, dtype=np.uint8)); rat += (n + 15) & ~15
        words[L] = {w: int(rng.integers(1, 1 << 31)) for w in WORDS}
    hd["vused"] = vat if flags & V else 0
    hd["resp_used"] = rat
    sec = {name: np.zeros(count, dtype=dt) for name, dt, count in sections(hd)}
    for L, p in phys.items():
        if L not in live:
            continue
        for w in WORDS:
            if len(sec[w]):
                sec[w][p] = words[L][w]
        sec["state"][p] = 0x20 | (L & 7)
        if flags & V:
            o, b = vbytes[L]
            o = o % vcap if ring else o
            sec["voff"][p], sec["vlen"][p] = o, len(b)
            sec["slab"][o: o + len(b)] = b
        else:
            sec["slab"][p * 512: (p + 1) * 512] = rng.integers(0, 256, 512, dtype=np.uint8)
        sec["resp_len"][p] = sec["err_len"][p] = 0
        for kind, off, ln in (("resp", "resp_off", "resp_len"), ("err", "err_off", "err_len")):
            if (L, kind) in rbytes:
                o, b = rbytes[(L, kind)]
                o = o % resp_cap if ring else o
                sec[off][p], sec[ln][p] = o, len(b)
                sec["resp"][o: o + len(b)] = b
    for name, entries in zip(("completed_log", "failed_log"), logs):
        sec[name][:] = [NONE if L is None else phys[L] for L in entries]
    return hd, b"", sec


def test_identity_on_an_unchanged_ring():
    live = {20, 21, 23, 24, 26, 27}
    hd, ag, sec = make(P | M | V | R, 16, 18, 28, live, resp={21: 33, 24: 5}, err={21: 2, 26: 60}, logs=([21, 24], [26, None]))
    hd2, _, sec2 = relocate(hd, ag, sec, P | M | V | R, 16, 4096, 4096)
    assert content(hd2, sec2) == content(hd, sec)
    assert log_rows(hd2, sec2) == log_rows(hd, sec)
    for name in ("completed_log", "failed_log"):
        assert np.array_equal(sec2[name], sec[name])
    keep = [w for w in WORDS if w not in ("voff", "resp_off", "err_off")]
    for w in keep:
        assert np.array_equal(sec2[w], sec[w]), w
    for f in ("tail", "rows_used", "scan_lo", "released_total", "shard", "gen", "id_secret", "slab_rows"):
        assert hd2[f] == hd[f], f
    assert (int(hd2["vtail"]), int(hd2["resp_tail"])) == (0, 0)


@pytest.mark.parametrize("flags", [P | M | R, P | V | R, P | M | V | R])
def test_there_and_back(flags):
    live = set(range(30, 61)) - {33, 40, 41}
    resp = {L: (L * 13) % 70 for L in live}
    err = {L: (L * 7) % 20 for L in live if L % 3 == 0}
    hd, ag, sec = make(flags, 40, 30, 61, live, resp=resp, err=err, logs=([31, 44, 59, 35], [36, None, 60]))
    hd_b, _, sec_b = relocate(hd, ag, sec, flags, 33, 3000, 3000)
    hd_c, _, sec_c = relocate(hd_b, ag, sec_b, flags, 40, 4096, 4096)
    assert content(hd_b, sec_b) == content(hd_c, sec_c) == content(hd, sec)
    assert log_rows(hd_c, sec_c) == log_rows(hd_b, sec_b) == log_rows(hd, sec)


def test_logs_follow_their_rows_across_the_wrap():
    live = set(range(6, 12))
    hd, ag, sec = make(P | M | R, 8, 6, 12, live, logs=([7, 8, None, 11], [6]))
    assert list(sec["completed_log"]) == [7, 0, NONE, 3]
    _, _, big = relocate(hd, ag, sec, P | M | R, 16, 0, 4096)
    assert list(big["completed_log"]) == [7, 8, NONE, 11] and list(big["failed_log"]) == [6]
    _, _, small = relocate(hd, ag, sec, P | M | R, 6, 0, 4096)
    assert list(small["completed_log"]) == [1, 2, NONE, 5] and list(small["failed_log"]) == [0]


def test_append_only_into_a_ring():
    live = set(range(0, 9)) - {4}
    hd, ag, sec = make(P | M | V, 64, 0, 9, live, resp={2: 17}, logs=([2, 8], []))
    hd, ag, sec = make(P | M | V, 64, 0, 9, live - {0, 1, 2, 3}, resp={5: 17}, logs=([5, 8], []))
    hd2, _, sec2 = relocate(hd, ag, sec, P | M | V | R, 9, 4096, 4096)
    assert len(sec2["state"]) == 9 and content(hd2, sec2) == content(hd, sec)
    hd, ag, sec = make(P | M | V, 64, 0, 9, live, resp={2: 17}, logs=([2, 8], []))
    hd2, _, sec2 = relocate(hd, ag, sec, P | M | V | R, 12, 4096, 4096)
    assert int(hd2["flags"]) & R and content(hd2, sec2) == content(hd, sec)
    assert list(sec2["completed_log"]) == [2, 8]
    with pytest.raises(NoSpace):
        relocate(hd, ag, sec, P | M | V | R, 8, 4096, 4096)          # 9 rows of window


def test_packing_order_and_alignment():
    live = {10, 11, 12, 14}
    hd, ag, sec = make(P | M | V | R, 8, 9, 15, live, resp={10: 17, 12: 16, 14: 1}, err={10: 3, 11: 40, 14: 0})
    hd2, _, sec2 = relocate(hd, ag, sec, P | M | V | R, 16, 4096, 4096)
    p = {L: L % 16 for L in live}
    vl = {L: 40 + 7 * (L % 5) for L in live}
    assert [int(sec2["voff"][p[L]]) for L in (10, 11, 12, 14)] == [0, vl[10], vl[10] + vl[11], vl[10] + vl[11] + vl[12]]
    assert int(hd2["vused"]) == sum(vl.values())
    # responses then errors, row by row, each from a 16 B boundary; empty segments take no bytes and read offset 0
    assert (int(sec2["resp_off"][p[10]]), int(sec2["err_off"][p[10]])) == (0, 32)
    assert (int(sec2["resp_off"][p[11]]), int(sec2["err_off"][p[11]])) == (0, 48)
    assert (int(sec2["resp_off"][p[12]]), int(sec2["err_off"][p[12]])) == (96, 0)
    assert (int(sec2["resp_off"][p[14]]), int(sec2["err_off"][p[14]])) == (112, 0)
    assert int(hd2["resp_used"]) == 128 and int(hd2["resp_tail"]) == 0
    assert all(int(sec2[o][q]) % 16 == 0 for o in ("resp_off", "err_off") for q in p.values())
    # a row that holds no record (row 13, skipped or released) keeps its words but no bytes
    assert int(sec2["state"][13]) == 0 and int(sec2["voff"][13]) == 0


def test_the_three_refusals():
    live = set(range(100, 120))
    hd, ag, sec = make(P | M | V | R, 32, 100, 120, live, resp={L: 30 for L in live})
    need_v = sum(40 + 7 * (L % 5) for L in live)
    relocate(hd, ag, sec, P | M | V | R, 20, need_v, 20 * 32)          # exactly full: fits
    with pytest.raises(NoSpace, match="window"):
        relocate(hd, ag, sec, P | M | V | R, 19, 4096, 4096)
    with pytest.raises(NoSpace, match="vslab"):
        relocate(hd, ag, sec, P | M | V | R, 20, need_v - 1, 4096)
    with pytest.raises(NoSpace, match="resp"):
        relocate(hd, ag, sec, P | M | V | R, 20, 4096, 20 * 32 - 1)
