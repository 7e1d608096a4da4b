"""The plain reference of a relocating restore (tests/resizeref.py) on small handmade snapshots.  Needs no GPU."""
import numpy as np
import pytest

from agentainer_lab_b200 import constants as K
from resizeref import NoSpace, content, log_rows, relocate, relocate_loop
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


def random_file(seed, flags, S, tail, window, vcap=1 << 14, resp_cap=1 << 14):
    """A parsed full file with random words on every row of the window: about a third of the rows dead (state 0) but keeping
    their lengths and offsets, response / error lengths from 0 up (many 0), the live rows' bytes laid out from a random point
    of each byte ring (wrapping), logs of random window rows and 0xFFFFFFFF entries."""
    rng = np.random.default_rng(seed)
    ring, var = bool(flags & R), bool(flags & V)
    used = tail + window
    hd = np.zeros(1, dtype=HEADER)[0]
    hd["magic"], hd["flags"], hd["shard"], hd["gen"], hd["id_secret"] = b"AGRSNAP3", flags, 1, 1, 5
    hd["tail"], hd["rows_used"], hd["released_total"], hd["scan_lo"] = tail, used, tail, tail
    hd["slab_rows"], hd["vcap"], hd["resp_cap"] = S if ring else used, vcap if var else 0, resp_cap
    nlog = [int(rng.integers(0, 300)), int(rng.integers(0, 40))]
    hd["log_len"] = nlog
    hd["vused"], hd["resp_used"] = (vcap + 77 if ring else vcap) if var else 0, resp_cap + 33 if ring else resp_cap
    sec = {name: rng.integers(0, 1 << 31, count).astype(dt) if name in WORDS else np.zeros(count, dtype=dt)
           for name, dt, count in sections(hd)}
    sec["slab"][:] = rng.integers(0, 256, len(sec["slab"]), dtype=np.uint8)
    sec["resp"][:] = rng.integers(0, 256, len(sec["resp"]), dtype=np.uint8)
    cap = int(hd["slab_rows"])
    phys = [(L % cap) if ring else L for L in range(tail, used)]
    vat, rat = int(rng.integers(0, vcap)), int(rng.integers(0, resp_cap)) & ~15
    for p in phys:
        live = rng.random() > 0.35
        sec["state"][p] = (0x20 | 1) if live else 0
        for ln in ("resp_len", "err_len"):
            sec[ln][p] = rng.choice([0, 0, 1, 15, 16, 17, 40])
        if var:
            sec["vlen"][p] = int(rng.integers(1, 30))
        if not live:
            continue
        if var:
            n = int(sec["vlen"][p])
            if not ring and vat + n > vcap:
                vat = 0
            sec["voff"][p] = vat % vcap if ring else vat
            if ring and vat % vcap + n > vcap:                # a record never straddles the ring's end
                vat += vcap - vat % vcap
                sec["voff"][p] = 0
            vat += n
        for off, ln in (("resp_off", "resp_len"), ("err_off", "err_len")):
            n = int(sec[ln][p])
            if ring and rat % resp_cap + n > resp_cap:
                rat += resp_cap - rat % resp_cap
            if not ring and rat + n > resp_cap:
                rat = 0
            sec[off][p] = rat % resp_cap
            rat += (n + 15) & ~15
    for j, name in enumerate(("completed_log", "failed_log")):
        e = rng.choice(phys, nlog[j]).astype(np.uint32) if phys else np.zeros(nlog[j], dtype=np.uint32)
        e[rng.random(nlog[j]) < 0.2] = NONE
        sec[name][:] = e
    return hd, b"ag", sec


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("case", ["ring_mid", "ring_wraps", "ring_at_0", "append"])
@pytest.mark.parametrize("flags", [P | M | R, P | V | R, P | M | V | R])
def test_vector_form_is_the_loop(flags, case, seed):
    S = 97
    tail, window, src_flags = {"ring_mid": (2 * S + 10, 60, flags), "ring_wraps": (3 * S + 70, S - 3, flags),
                               "ring_at_0": (5 * S, S, flags), "append": (0, 120, flags & ~R)}[case]
    hd, ag, sec = random_file(seed, src_flags, S, tail, window)
    for slab_rows in (window, window + 1, 64 + seed, 256, 1000):
        try:
            want = relocate_loop(hd, ag, sec, flags, slab_rows, 1 << 14, 1 << 14)
        except NoSpace as e:
            with pytest.raises(NoSpace, match=str(e)):
                relocate(hd, ag, sec, flags, slab_rows, 1 << 14, 1 << 14)
            continue
        got = relocate(hd, ag, sec, flags, slab_rows, 1 << 14, 1 << 14)
        assert got[0].tobytes() == want[0].tobytes() and got[1] == want[1]
        for name in want[2]:
            assert np.array_equal(got[2][name], want[2][name]), (slab_rows, name)
    if window:
        assert (sec["state"] == 0).any() and (sec["resp_len"][sec["state"] == 0] > 0).any()
        assert (sec["completed_log"] == NONE).any() or len(sec["completed_log"]) < 5


@pytest.mark.parametrize("flags", [P | M | R, P | M | V | R])
def test_vector_form_refuses_like_the_loop(flags):
    hd, ag, sec = random_file(3, flags, 64, 200, 50)
    _, _, packed = relocate_loop(hd, ag, sec, flags, 64, 1 << 20, 1 << 20)
    need_v, need_r = (len(packed["slab"]) if flags & V else 0), len(packed["resp"])
    for args, word in (((49, 1 << 20, 1 << 20), "window"), ((64, 1 << 20, need_r - 1), "resp"), ((64, 1 << 20, need_r), None)) + \
            ((((64, need_v - 1, 1 << 20), "vslab"), ((64, need_v, 1 << 20), None)) if flags & V else ()):
        for fn in (relocate, relocate_loop):
            if word is None:
                fn(hd, ag, sec, flags, *args)
            else:
                with pytest.raises(NoSpace, match=word):
                    fn(hd, ag, sec, flags, *args)
