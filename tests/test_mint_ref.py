"""Engine-minted request ids far along the arrival counter, on the CPU: the functions of csrc/agr_common.h (what the kernels and
the host ship, compiled into tests/mint_harness.cpp) against the plain restatement in tests/mintref.py.

A ring counts arrivals in 64 bits, and an id holds 40 bits of its row.  These tests pin down what happens at and past 2^40:
ids stay distinct (the 2^40-row period is folded into the generation field), and a lookup places an id in the live window, so
it resolves exactly the rows of the window and nothing else."""
import json
import os
import random
import subprocess

import pytest

from mintref import M40, ROW_LIMIT, decode, mint, split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECRETS = [0x1234567890ABCDEF, 0x9E3779B97F4A7C15, 1, 0xFFFFFFFFFFFFFFFF]
EDGES = [0, 2**32, 2**40, 2**41, 2**48, ROW_LIMIT - 3000]
SPAN = 3000


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("mint") / "mint_harness")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "mint_harness.cpp")],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr

    def run(cmds):
        out = subprocess.run([exe], input="\n".join(cmds) + "\n", capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        return out.stdout.split("\n")[:-1]
    return run


def harness_mint(run, secret, shard, gen, first, n):
    return [tuple(int(w, 16) for w in l.split()) for l in run([f"m {secret} {shard} {gen} {first} {n}"])]


def harness_decode(run, secret, shard, gen, tail, head, ids):
    out = run([f"d {secret} {shard} {gen} {tail} {head} {lo} {hi}" for lo, hi in ids])
    return [None if l == "none" else int(l) for l in out]


def window(edge):
    lo = max(0, edge - SPAN)
    return lo, min(edge + SPAN, ROW_LIMIT) - lo


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("shard", [0, 255])
def test_header_mints_what_the_reference_mints(harness, edge, shard):
    first, n = window(edge)
    for secret in SECRETS:
        got = harness_mint(harness, secret, shard, 1, first, n)
        assert got == [mint(first + i, secret, shard) for i in range(n)], (hex(secret), first)


def test_ids_below_2_40_are_the_ones_minted_before():
    """Ids recorded from the engine before the 2^40-row period entered the generation field: rows below 2^40 keep them, so
    existing snapshots and callers stay valid."""
    cases = json.load(open(os.path.join(ROOT, "tests", "golden", "mint_ids_below_2_40.json")))
    assert cases and all(c["row"] < 2**40 for c in cases)
    for c in cases:
        assert mint(c["row"], c["secret"], c["shard"], c["gen"]) == (int(c["lo"], 16), int(c["hi"], 16)), c


@pytest.mark.parametrize("edge", EDGES)
def test_uuid_bits_and_distinct_ids_across_each_edge(edge):
    first, n = window(edge)
    for secret in SECRETS[:2]:
        for shard in (0, 255):
            ids = [mint(first + i, secret, shard) for i in range(n)]
            for lo, hi in ids:
                assert (lo >> 52) & 0xF == 0x4                       # UUID version 4 (byte 6's high nibble)
                assert (hi >> 6) & 0x3 == 0x2                        # RFC 4122 variant (byte 8's top bits 10)
            assert len(set(ids)) == n


def test_rows_one_period_apart_get_different_ids():
    rng = random.Random(7)
    rows = [0, 5, 2**32 + 5, M40 - 36, M40] + [rng.randrange(0, 2**40) for _ in range(200)]
    for secret in SECRETS:
        for a in rows:
            ids = {mint(a + k * 2**40, secret) for k in range(0, 4096, 37)} | {mint(a + k * 2**40, secret) for k in (1, 2, 3, 4095)}
            assert len(ids) == len(set(range(0, 4096, 37)) | {1, 2, 3, 4095})
            assert mint(a + 2**40, secret)[0] != mint(a, secret)[0]      # the low word alone already tells the periods apart


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("slab_rows", [4097, 2**20])
def test_window_decode_accepts_exactly_the_window(harness, edge, slab_rows):
    """A window of slab_rows rows that straddles the edge (where the edge allows): every row's id decodes to that row, and ids
    minted outside the window (just outside, one or more 2^40 periods away, another shard or generation, one bit flipped)
    decode to nothing."""
    secret, shard, gen = 0x1234567890ABCDEF, 3, 1
    tail = max(0, min(edge - slab_rows // 3, ROW_LIMIT - slab_rows))
    head = tail + slab_rows
    rng = random.Random(edge ^ slab_rows)
    inside = sorted({tail, head - 1, edge if tail <= edge < head else tail + 1} | {rng.randrange(tail, head) for _ in range(1500)})
    ids = [mint(a, secret, shard, gen) for a in inside]
    assert harness_decode(harness, secret, shard, gen, tail, head, ids) == inside
    assert [decode(lo, hi, secret, shard, gen, tail, head) for lo, hi in ids] == inside
    outside = [a for a in range(max(0, tail - 300), tail)] + list(range(head, head + 300))
    outside += [a + k * 2**40 for a in inside[:200] for k in (-3, -1, 1, 2, 4095) if 0 <= a + k * 2**40]
    bad = [mint(a, secret, shard, gen) for a in outside]
    bad += [mint(a, secret, shard ^ 1, gen) for a in inside[:100]] + [mint(a, secret, shard, gen + 1) for a in inside[:100]]
    bad += [mint(a, secret ^ 0x10, shard, gen) for a in inside[:100]]
    for lo, hi in ids[:40]:
        bad += [(lo ^ (1 << b), hi) for b in range(64)] + [(lo, hi ^ (1 << b)) for b in range(64)]
    got = harness_decode(harness, secret, shard, gen, tail, head, bad)
    assert got == [None] * len(bad), [(i, g) for i, g in enumerate(got) if g is not None][:5]
    assert all(decode(lo, hi, secret, shard, gen, tail, head) is None for lo, hi in bad[:2000])


def test_decode_is_relative_to_the_window_not_to_2_40():
    """The same low 40 bits name different rows in different windows; only the row in the window is accepted."""
    secret = SECRETS[0]
    for a in (5, 2**40 + 5, 2**41 + 5, 2**48 + 5):
        lo, hi = mint(a, secret)
        for tail in (a - 10, a, a - 4096 + 1):
            assert decode(lo, hi, secret, 0, 1, max(0, tail), max(0, tail) + 4096) == a
        assert decode(lo, hi, secret, 0, 1, a + 1, a + 4097) is None
        assert split(lo.to_bytes(8, "little") + hi.to_bytes(8, "little")) == (lo, hi)
