"""The test rig of the K3 and TTL-sweep tests: one engine, the plain restatement (tests/k3ref.py) of what it must return, and
the records a test ingested (for the byte-for-byte compare)."""
import numpy as np

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from k3ref import K3Ref, OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR

AGENT_NANOS0 = 1_700_000_000_000_000_000


def agent_names(n):
    return [f"agent-{AGENT_NANOS0 + 1000003 * k}" for k in range(n)]


class Rig:
    """One engine, the restatement, and the records the test ingested (for the byte-for-byte compare)."""

    def __init__(self, *, slab_rows, max_agents, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS, keep_records=True, base=0,
                 mint_ids=None, **kw):
        self.eng = A.Engine(device=0, slab_rows=slab_rows, max_agents=max_agents, flags=flags, **kw)
        # base: the engine's arrival counter when the rig starts (agr_debug_skip_arrivals); the restatement and the kept records
        # count rows from there.  mint_ids(first, n): where the ids of minted rows come from (default: the engine's agr_mint_ids)
        self.base = base
        if base:
            self.eng.skip_arrivals(base)
        self.mint_ids = mint_ids or self.eng.mint_ids
        self.ref = K3Ref()
        self.mint = bool(flags & K.AGR_CFG_MINT_IDS)
        self.names = []
        self.keep = keep_records
        self.recs = np.zeros(0, dtype=A.record_dtype)       # by logical row (zeros: no record)
        self.rng = np.random.default_rng(slab_rows * 7 + max_agents)
        self.seq = 0

    def close(self):
        self.eng.close()

    def register(self, n, p_running=0.6):
        names = agent_names(len(self.names) + n)[len(self.names):]
        st = np.where(self.rng.random(n) < p_running, K.AGR_AGENT_RUNNING, K.AGR_AGENT_STOPPED)
        slots = self.eng.set_agent_states(names, st)
        assert list(slots) == list(range(len(self.names), len(self.names) + n))
        self.names += names
        self.ref.set_agents(slots, st)

    def set_status(self, slot, status):
        self.eng.set_agent_state(self.names[slot], status)
        self.ref.set_agents([slot], [status])

    def drop(self, slot):
        self.eng.drop_agent(self.names[slot])
        self.ref.drop_agent(slot)

    def records(self, slots):
        n = len(slots)
        recs = np.zeros(n, dtype=A.record_dtype)
        nm = np.array([s.encode() for s in self.names] + [b"agent-unknown"], dtype="S32")
        recs["agent_id"] = nm[np.where(np.asarray(slots) >= 0, slots, len(self.names))]
        recs["request_id"] = self.rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
        recs["request_id"][:, 6] = (recs["request_id"][:, 6] & 0x0F) | 0x40
        recs["seq"] = self.seq + 1 + np.arange(n)
        self.seq += n
        recs["flags"] = K.METHOD_CODES["POST"] << K.AGR_F_METHOD_SHIFT
        recs["path_len"], recs["hdr_len"], recs["body_len"] = 5, 0, 2
        recs["payload"][:, :7] = np.frombuffer(b"/chat{}", dtype=np.uint8)
        recs["payload"][:, 7:11] = self.rng.integers(0, 256, size=(n, 4), dtype=np.uint8)   # bytes past body_len ride along
        recs["status"], recs["max_retries"] = K.AGR_ST_PENDING, 3
        return recs

    def ingest(self, slots):
        """One agr_ingest call; returns its first row (counted from base)."""
        slots = np.asarray(slots, dtype=np.int64)
        recs = self.records(slots)
        _, first = self.eng.ingest(recs, want_verdicts=False)
        ids = self.mint_ids(first, len(recs)) if self.mint else recs["request_id"]
        first -= self.base
        self.ref.add_rows(first, slots, ids)
        self.keep_rows(first, recs)
        return first

    def keep_rows(self, first, recs):
        if not self.keep:
            return
        end = first + len(recs)
        if end > len(self.recs):
            grown = np.zeros(max(end, 2 * len(self.recs)), dtype=A.record_dtype)
            grown[: len(self.recs)] = self.recs
            self.recs = grown
        self.recs[first:end] = recs

    def complete(self, rows, kinds, https=None, chunk=1 << 16):
        """One agr_complete per chunk, in call order; returns the outcomes (for other implementations to apply)."""
        rows = np.asarray(rows, dtype=np.int64)
        kinds = np.asarray(kinds)
        https = np.zeros(len(rows), np.int64) if https is None else np.asarray(https)
        outs = np.zeros(len(rows), dtype=A.outcome_dtype)
        outs["request_id"] = self.ref.ids[rows]
        nm = np.array([s.encode() for s in self.names], dtype="S32")
        outs["agent_id"] = nm[np.maximum(self.ref.slot[rows], 0)]
        outs["kind"], outs["http_status"] = kinds, https
        outs["seq"] = self.recs["seq"][rows] if self.keep else 0     # a completion's time = its record's: expiry follows the record
        for a in range(0, len(rows), min(chunk, self.eng.max_batch)):
            self.eng.complete(np.ascontiguousarray(outs[a: a + min(chunk, self.eng.max_batch)]), want_results=False)
        self.ref.complete(rows, kinds, https)
        return outs

    def random_outcomes(self, frac=0.4):
        """Complete, fail or retry a random share of the pending rows (a few rows get several outcomes in one call)."""
        lo, hi = self.ref.tail, self.ref.bound()
        rows = np.flatnonzero(self.ref.inq[lo:hi] & self.ref.stored[lo:hi]) + lo
        pick = rows[self.rng.random(len(rows)) < frac]
        pick = np.concatenate([pick, pick[: len(pick) // 8]])
        self.rng.shuffle(pick)
        kinds = self.rng.choice([OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR], size=len(pick), p=[0.6, 0.3, 0.1])
        return self.complete(pick, kinds, self.rng.choice([200, 404, 500], size=len(pick)))

    # ---- the comparisons
    def expected_records(self, rows):
        exp = self.recs[rows].copy()
        exp["request_id"] = self.ref.ids[rows]
        for f, v in self.ref.header_fields(rows).items():
            exp[f] = v
        return exp

    def check_tick(self, with_records=None):
        with_records = self.keep if with_records is None else with_records
        disp, recs = self.eng.replay_scan(with_records=with_records)
        rows, slots = self.ref.tick()
        assert len(disp) == len(rows), f"dispatched {len(disp)} rows, the reference {len(rows)}"
        assert np.array_equal(disp["rid"].astype(np.int64) - self.base, rows), "dispatch rows / order differ"
        assert np.array_equal(disp["agent_slot"].astype(np.int64), slots)
        assert np.array_equal(disp["request_id"], self.ref.ids[rows])
        if with_records:
            exp = self.expected_records(rows)
            assert recs.tobytes() == exp.tobytes(), _first_field_diff(recs, exp)
        return len(rows)

    def check_agent(self, slot, with_records=None):
        with_records = self.keep if with_records is None else with_records
        name = self.names[slot]
        got = self.eng.pending(name)
        rows = self.ref.pending(slot)
        assert len(got) == len(rows), f"agent slot {slot}: pending {len(got)} != {len(rows)}"
        assert np.array_equal(got["request_id"], self.ref.ids[rows])
        if with_records:
            exp = self.expected_records(rows)
            assert got.tobytes() == exp.tobytes(), _first_field_diff(got, exp)
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            ids = self.eng.list(name, which)
            lrows = self.ref.list(slot, which)
            assert len(ids) == len(lrows), f"agent slot {slot} list {which}: {len(ids)} != {len(lrows)}"
            assert np.array_equal(ids, self.ref.ids[lrows]), f"agent slot {slot} list {which} differs"

    def check(self, sample=8):
        n = self.check_tick()
        slots = list(range(len(self.names)))
        if len(slots) > sample:
            slots = sorted(set(self.rng.choice(len(slots), sample, replace=False).tolist()) | {0, len(slots) - 1})
        for s in slots:
            self.check_agent(s)
        return n


def _first_field_diff(got, exp):
    for i in range(min(len(got), len(exp))):
        if got[i].tobytes() != exp[i].tobytes():
            bad = [f for f in A.record_dtype.names if got[i][f].tobytes() != exp[i][f].tobytes()]
            return f"record {i}: fields {bad} differ"
    return "record count differs"


def layout(kind, n_rows, n_agents, rng, first_row=0):
    """Agent slot of each row.  same32 / distinct32 are the two adversarial layouts of the __match_any_sync ranking."""
    live = np.flatnonzero(rng.random(n_agents) >= 0.1)          # about a tenth of the agents get no rows
    if len(live) == 0:
        live = np.arange(n_agents)
    r = np.arange(first_row, first_row + n_rows)
    if kind == "uniform":
        return live[rng.integers(0, len(live), n_rows)]
    if kind == "zipf":
        w = 1.0 / np.arange(1, len(live) + 1) ** 1.2
        return live[rng.choice(len(live), n_rows, p=w / w.sum())]
    if kind == "same32":                                          # all 32 rows of a 32-row step: one agent
        return live[(r // 32) * 7 % len(live)]
    if kind == "distinct32":                                      # the 32 rows of a step: 32 different agents (when there are)
        return live[(r % 32 + r // 32) % len(live)]
    raise ValueError(kind)
