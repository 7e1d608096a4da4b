"""tests/agentslotref.py, the plain model of agent slot reuse, on hand-worked cases (the GPU tests check the engine against it)."""
from agentslotref import ENOSPC, AgentTable, held_slots, next_slot

FORWARD, QUEUED, NOT_FOUND = 1, 2, 4


def route(slot, code, flags=0):
    return (flags << 26) | (code << 23) | slot


def test_held_slots_counts_decided_rows_only():
    words = [
        route(3, FORWARD),
        route(5, QUEUED, flags=0x3),
        route(0x7FFFFF, NOT_FOUND),              # a request for an unknown or removed agent carries no slot
        0,                                        # hole, skipped row, released row or reserved row not decided yet
        route(7, 0),                             # no verdict: holds nothing whatever its slot bits say
    ]
    assert held_slots(words) == {3, 5}


def test_never_used_slots_come_first():
    assert next_slot(2, 4, removed={0, 1}, held=set()) == 2          # exactly as before the table filled
    assert next_slot(4, 4, removed=set(), held=set()) == ENOSPC


def test_lowest_unheld_removed_slot():
    assert next_slot(4, 4, removed={1, 2, 3}, held={1}) == 2
    assert next_slot(4, 4, removed={3, 1}, held=set()) == 1
    assert next_slot(4, 4, removed={1, 2}, held={1, 2}) == ENOSPC
    assert next_slot(64, 64, removed={31, 32, 63}, held={31}) == 32
    assert next_slot(64, 64, removed={63}, held=set()) == 63


def test_table_reuses_and_forgets():
    t = AgentTable(2)
    assert t.register("a", set()) == 0 and t.register("b", set()) == 1
    assert t.register("c", set()) == ENOSPC                         # nothing removed
    t.drop("a")
    assert t.register("c", {0}) == ENOSPC                            # a's rows still hold slot 0
    assert t.register("a", {0}) == 0                                 # revived on its own slot
    t.drop("a")
    assert t.register("c", set()) == 0                               # a's rows are gone: c takes its slot
    assert t.slot("a") is None and t.slot("c") == 0
    t.drop("b")
    assert t.register("a", set()) == 1                               # "a" again is a new agent, on b's slot
    assert t.names == ["c", "a"]
