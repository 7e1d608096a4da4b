"""The plain K4 reference (tests/k4ref.py) on the CPU: the published FNV-1a 64 vectors, agreement with the library's host shard
hash, and partitions worked out by hand.  tests/test_k4_exchange_gpu.py holds the kernels to this reference."""
import numpy as np
import pytest

import agentainer_lab_b200 as A
from k4ref import expected, fnv1a64, owners, partition, unpermute


def test_fnv1a64_published_vectors():
    assert fnv1a64(b"") == 0xCBF29CE484222325
    assert fnv1a64(b"a") == 0xAF63DC4C8601EC8C
    assert fnv1a64(b"foobar") == 0x85944171F73967E8
    assert fnv1a64(b"foobar\0junk") == fnv1a64(b"foobar")          # the id ends at its first NUL


@pytest.mark.parametrize("G", [1, 2, 3, 5, 8, 17, 31, 32])
def test_reference_owner_matches_host_agent_shard(G):
    rng = np.random.default_rng(G)
    ids = ["agent-1700000000000000000", "a", "x" * 31] + [
        "".join(chr(c) for c in rng.integers(0x21, 0x7F, rng.integers(1, 32))) for _ in range(60)]
    raw = np.zeros((len(ids), 32), np.uint8)
    for i, a in enumerate(ids):
        raw[i, : len(a)] = np.frombuffer(a.encode(), np.uint8)
        assert fnv1a64(a.encode()) == A.agent_hash(a)
    assert [int(o) for o in owners(raw, 0, G)] == [A.agent_shard(a, G) for a in ids]


def test_high_bytes_hash_unsigned():
    b = bytes([0x80, 0xFF, 0x41, 0xC3])
    h = FNV = 0xCBF29CE484222325
    for c in b:
        h = ((h ^ c) * 0x100000001B3) & ((1 << 64) - 1)
    assert fnv1a64(b) == h and h != FNV


# G = 3, seven items with owners 2 0 1 2 0 2 1: totals 2 2 3, offsets 0 2 4 7
OWN = [2, 0, 1, 2, 0, 2, 1]


def test_hand_partition_outcome_form():
    p = partition(OWN, 3, 1, inplace=False)
    assert list(p["gtotal"]) == [2, 2, 3] and list(p["goff"]) == [0, 2, 4, 7]
    assert list(p["perm"]) == [4, 0, 2, 5, 1, 6, 3]


@pytest.mark.parametrize("me,perm,send_order", [
    (0, [2, 0, 0, 3, 1, 4, 1], [2, 6, 0, 3, 5]),       # owner 0's items stay; everything above moves down by 2
    (1, [2, 0, 2, 3, 1, 4, 3], [1, 4, 0, 3, 5]),
    (2, [4, 0, 2, 5, 1, 6, 3], [1, 4, 2, 6]),          # no owner above the last rank: nothing moves
])
def test_hand_partition_in_place(me, perm, send_order):
    p = partition(OWN, 3, me, inplace=True)
    got = [int(x) for i, x in enumerate(p["perm"]) if OWN[i] != me]
    assert got == [x for i, x in enumerate(perm) if OWN[i] != me]
    # the send buffer, as item indices, and the rows left as holes
    raw = np.zeros((7, 48), np.uint8)
    raw[:, 0] = np.arange(7) + 1
    names = {0: b"", 1: b"", 2: b""}
    for g in range(3):                    # an agent id per owner, found by search
        k = 0
        while fnv1a64(f"ag{k}".encode()) % 3 != g:
            k += 1
        names[g] = f"ag{k}".encode()
    for i, o in enumerate(OWN):
        raw[i, 16: 16 + len(names[o])] = np.frombuffer(names[o], np.uint8)
    e = expected(raw, 16, 3, me, inplace=True)
    assert list(e["owner"]) == OWN
    assert [int(x) - 1 for x in e["send"][: len(send_order), 0]] == send_order
    assert not e["send"][len(send_order):].any() and not e["local"].any()
    assert list(e["holes"]) == [o != me for o in OWN]
    assert np.array_equal(e["items"], raw)


def test_hand_unpermute():
    p = partition(OWN, 3, 1, inplace=True)
    loc = np.arange(100, 107, dtype=np.uint32)
    rem = np.arange(200, 207, dtype=np.uint32)
    out = unpermute(OWN, p["perm"], p["goff"], 1, True, loc, rem)
    assert list(out) == [202, 200, 102, 203, 201, 204, 106]
    p = partition(OWN, 3, 1, inplace=False)
    out = unpermute(OWN, p["perm"], p["goff"], 1, False, loc.astype(np.uint64), rem.astype(np.uint64))
    assert list(out) == [204, 200, 100, 205, 201, 206, 101]
