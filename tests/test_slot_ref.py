"""The plain slot-layout reference (tests/slotref.py) on hand-worked cases and on random sequences."""
import numpy as np

from slotref import SLOT, slot_layout

CAP = 128 * SLOT                     # 128 slots


def test_append_only_fills_then_refuses():
    assert slot_layout(CAP, False, [("reserve", 100), ("reserve", 28), ("reserve", 1)]) == [0, 100 * SLOT, "ENOSPC"]
    # a release does not give an append-only slab its bytes back
    assert slot_layout(CAP, False, [("reserve", 128), ("release_all",), ("reserve", 1)]) == [0, None, "ENOSPC"]


def test_ring_skips_to_the_start_instead_of_wrapping():
    ops = [("reserve", 40), ("reserve", 40), ("reserve", 40), ("release_all",), ("reserve", 40)]
    assert slot_layout(CAP, True, ops) == [0, 40 * SLOT, 80 * SLOT, None, 0]       # 8 slots at the end are skipped


def test_ring_refusals():
    assert slot_layout(CAP, True, [("reserve", 65)]) == ["EINVAL"]                  # more than half the ring
    assert slot_layout(CAP, True, [("reserve", 64), ("reserve", 64), ("reserve", 1)]) == [0, 64 * SLOT, "ENOSPC"]
    # the skip counts: 40 + 40 + (8 skipped) + 60 > 128 with the tail at 0
    assert slot_layout(CAP, True, [("reserve", 40), ("reserve", 40), ("reserve", 60)]) == [0, 40 * SLOT, "ENOSPC"]
    # a refusal changes nothing
    assert slot_layout(CAP, True, [("reserve", 64), ("reserve", 65), ("reserve", 64)]) == [0, "EINVAL", 64 * SLOT]


def test_random_sequences_never_wrap_or_overlap_live_slots():
    rng = np.random.default_rng(3)
    for ring in (False, True):
        for _ in range(200):
            ops = [("release_all",) if rng.random() < 0.2 else ("reserve", int(rng.integers(1, 80))) for _ in range(30)]
            got = slot_layout(CAP, ring, ops)
            live = []                                                   # [start, end) of the slots since the last release
            for op, g in zip(ops, got):
                if op[0] == "release_all":
                    live = []
                    continue
                if isinstance(g, str):
                    assert g in ("ENOSPC", "EINVAL")
                    continue
                a, b = g, g + op[1] * SLOT
                assert 0 <= a and b <= CAP                              # never wraps
                assert all(b <= x or a >= y for x, y in live)           # never on a slot still in use
                live.append((a, b))
