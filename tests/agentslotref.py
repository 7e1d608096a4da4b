"""Plain restatement of the engine's agent slot allocator (DESIGN.md section 3, "Agent slots"): which slot a new agent id takes.

A slot is held while a row of the live window [rows_tail, rows_used) records a decision for it: its route word has a verdict code
other than 0 and carries the slot.  AGR_V_NOT_FOUND rows carry RT_SLOT_NONE; holes, skipped rows, released rows and reserved rows
not decided yet have route word 0.  A new id takes the next never-used slot while one remains, else the lowest slot that is removed
and not held, else the call fails with AGR_ENOSPC."""
ENOSPC = -4
SLOT_MASK = 0x7FFFFF
SLOT_NONE = 0x7FFFFF
CODE_SHIFT = 23


def held_slots(routes):
    """Slots that the route words of the live window hold."""
    out = set()
    for r in routes:
        r = int(r)
        if (r >> CODE_SHIFT) & 7 and (r & SLOT_MASK) != SLOT_NONE:
            out.add(r & SLOT_MASK)
    return out


def next_slot(handed_out, max_agents, removed, held):
    """The slot of the next new agent id: handed_out slots exist (0 .. handed_out - 1), removed = slots whose agent was removed,
    held = held_slots of the window.  Returns the slot or ENOSPC."""
    if handed_out < max_agents:
        return handed_out
    free = sorted(set(removed) - set(held))
    return free[0] if free else ENOSPC


class AgentTable:
    """The agent table as the engine keeps it: names by slot, statuses, and the slots handed out so far."""

    def __init__(self, max_agents):
        self.max_agents = max_agents
        self.names = []                          # slot -> name
        self.removed = set()

    def slot(self, name):
        return self.names.index(name) if name in self.names else None

    def register(self, name, held):
        """agr_set_agent_state of a name: its slot (revived if removed), a new slot by the rule, or ENOSPC."""
        s = self.slot(name)
        if s is not None:
            self.removed.discard(s)
            return s
        s = next_slot(len(self.names), self.max_agents, self.removed, held)
        if s == ENOSPC:
            return s
        if s == len(self.names):
            self.names.append(name)
        else:
            self.names[s] = name                 # the old name is forgotten
            self.removed.discard(s)
        return s

    def drop(self, name):
        s = self.slot(name)
        if s is not None:
            self.removed.add(s)
        return s
