"""The K3 restatement (tests/k3ref.py) against the literal reference (oracle/model.py), on the scenario streams of
tests/scenario.py: every tick's dispatch order (process_agents), the LRANGE of all three lists, and the (status, retry_count,
response status) of every stored record.  CPU only: this keeps the restatement the GPU K3 tests compare with honest."""
import numpy as np
import pytest

from k3ref import K3Ref, OUT_RESPONSE, OUT_DIAL_ERR, OUT_ERROR, LIST_PENDING, LIST_COMPLETED, LIST_FAILED
from scenario import ZERO16, all_agents, all_fresh, random_scenario, run_oracle

STATUS = {"created": 0, "running": 1, "stopped": 2, "paused": 3, "failed": 4}
NAMES = {1: "pending", 2: "processing", 3: "completed", 4: "failed"}


def run_k3ref(events):
    """What the Go glue does with the C-ABI (scenario.run_engine), with K1's verdict and K2's outcome lookup restated:
    only the K3 views come out of the restatement under test."""
    ref = K3Ref()
    slot_of, status = {}, {}
    row_of = {}                                             # (agent, id) -> row of the stored record
    ticks = []

    def outcome(rows, kinds, https, agent, rid, kind, http=0):
        rows.append(row_of.get((agent, rid), -1)); kinds.append(kind); https.append(http)

    for e in events:
        if e[0] == "agent":
            if e[1] not in slot_of:
                slot_of[e[1]] = len(slot_of)
            status[e[1]] = e[2]
            ref.set_agents([slot_of[e[1]]], [STATUS[e[2]]])
        elif e[0] == "req":
            r, backend = e[1], e[2]
            known = r.agent_id in status
            rows, kinds, https = [], [], []
            if known and not r.replay:                          # StoreRequest
                row = ref.n
                ref.add_rows(row, [slot_of[r.agent_id]], np.frombuffer(r.rid, np.uint8)[None])
                row_of[(r.agent_id, r.rid)] = row
            tracked = r.rid if not r.replay else (r.replay_of if r.replay_of != ZERO16 else None)
            if known and status[r.agent_id] == "running" and tracked is not None:   # forwarded, interceptTransport
                kind = {"response": OUT_RESPONSE, "dial": OUT_DIAL_ERR, "error": OUT_ERROR}[backend[0]]
                outcome(rows, kinds, https, r.agent_id, tracked, kind, backend[1] if backend[0] == "response" else 0)
            ref.complete(rows, kinds, https)
        elif e[0] == "tick":
            assert e[2] is None
            backends = e[1]
            disp_rows, disp_slots = ref.tick()
            name = {s: a for a, s in slot_of.items()}
            order = [(name[int(s)], bytes(ref.ids[r]).hex()) for r, s in zip(disp_rows, disp_slots)]
            ticks.append(order)
            rows, kinds, https = [], [], []
            for agent, hx in order:                             # replayRequest through the proxy (the agent is running)
                rid = bytes.fromhex(hx)
                b = backends.get(hx, ("response", 200))
                if b[0] == "response":
                    outcome(rows, kinds, https, agent, rid, OUT_RESPONSE, b[1]); outcome(rows, kinds, https, agent, rid, OUT_RESPONSE, b[1])
                elif b[0] == "dial":
                    outcome(rows, kinds, https, agent, rid, OUT_DIAL_ERR); outcome(rows, kinds, https, agent, rid, OUT_RESPONSE, 502)
                elif b[0] == "error":
                    outcome(rows, kinds, https, agent, rid, OUT_ERROR); outcome(rows, kinds, https, agent, rid, OUT_RESPONSE, 502)
                else:
                    outcome(rows, kinds, https, agent, rid, OUT_ERROR)
            ref.complete(rows, kinds, https)
        else:
            raise ValueError(e[0])
    lists = {}
    for a in all_agents(events):
        if a not in slot_of:
            lists[a] = {"pending": [], "completed": [], "failed": []}
            continue
        lists[a] = {q: [bytes(ref.ids[r]).hex() for r in ref.list(slot_of[a], w)]
                    for q, w in (("pending", LIST_PENDING), ("completed", LIST_COMPLETED), ("failed", LIST_FAILED))}
    records = {}
    for a, rid in all_fresh(events):
        row = row_of.get((a, rid))
        if row is not None:
            f = ref.header_fields([row])
            records[(a, rid.hex())] = (NAMES[int(f["status"][0])], int(f["retry_count"][0]), int(f["resp_status"][0]))
    # agr_pending of every agent: the stored members of its pending list, oldest first
    pend = {a: [bytes(ref.ids[r]).hex() for r in ref.pending(s)] for a, s in slot_of.items()}
    return ticks, lists, records, pend


@pytest.mark.parametrize("seed", range(12))
def test_k3ref_equals_oracle(seed):
    n_agents = [1, 2, 3, 5, 8, 13][seed % 6]
    events = random_scenario(100 + seed, n_events=400, n_agents=n_agents, p_replay=0.15)
    o = run_oracle(events)
    ticks, lists, records, pend = run_k3ref(events)
    assert ticks == o.ticks
    assert lists == o.lists
    assert records == o.records
    # GetPendingRequests (requests.go:197-225): the pending list's stored records; nothing expires in these streams
    for a, p in pend.items():
        assert p == o.lists[a]["pending"]
    assert sum(len(t) for t in ticks) > 0


U64 = (1 << 64) - 1


@pytest.mark.parametrize("seed", range(6))
def test_k3ref_sweep_equals_the_model_clock(seed):
    """K3Ref.sweep against MiniRedis's key expiry (SET ... EX at the SET's clock, GET at the sweep's clock): random records and
    outcomes whose times run backwards (clock skew), sweeps at exactly t + ttl and t + ttl - 1 of some live row, sweeps behind
    every time, time 0 and times up to UINT64_MAX.  After every sweep the set of stored rows is the set of live keys."""
    from oracle.model import MiniRedis, RedisNil
    rng = np.random.default_rng(900 + seed)
    ttl = [1, 1000, 10**9, 1 << 40, 7, 12345][seed]
    redis = MiniRedis()
    redis.ticks_per_second = ttl                        # SET ... EX 1 = ttl of the stream's unit
    ref = K3Ref()
    ref.set_agents([0], [1])

    def some_time(base):
        c = rng.random()
        if c < 0.05:
            return 0
        if c < 0.10:
            return U64 - int(rng.integers(0, 3))
        return max(0, min(U64, base + int(rng.integers(-3 * ttl, 3 * ttl + 1))))

    base = int(rng.choice([0, 5 * ttl, U64 - 50 * ttl if ttl < 1 << 40 else 1 << 60]))
    swept = 0
    for step in range(60):
        base = max(0, min(U64, base + int(rng.integers(0, 2 * ttl + 1))))
        n = int(rng.integers(1, 20))
        times = [some_time(base) for _ in range(n)]
        first = ref.n
        ref.add_rows(first, np.zeros(n, np.int64), np.zeros((n, 16), np.uint8), created=times)
        for r, t in zip(range(first, first + n), times):
            redis.now = t
            redis.set(f"k{r}", r, ttl_s=1)
        rows = rng.integers(0, ref.n, size=int(rng.integers(0, 12)))
        kinds = rng.choice([OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR], size=len(rows))
        otimes = [some_time(base) for _ in rows]
        for r, k, t in zip(rows.tolist(), kinds.tolist(), otimes):
            if ref.stored[r] and k != OUT_DIAL_ERR:     # a SET of a key that exists (not swept yet)
                assert f"k{r}" in redis.strings
                redis.now = t
                redis.set(f"k{r}", r, ttl_s=1)
        ref.complete(rows, kinds, np.zeros(len(rows), np.int64), times=otimes)
        live = np.flatnonzero(ref.stored[: ref.n])
        c = rng.random()
        if c < 0.6 and len(live):                       # exactly at a live row's expiry, or 1 ns before it
            t = int(ref.mtime[int(rng.choice(live))])
            now = t + ttl - int(rng.integers(0, 2))
        elif c < 0.8:
            now = max(0, base - int(rng.integers(0, 4 * ttl)))   # the clock behind most times
        else:
            now = int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2))
        now = min(now, U64)
        before = set(live.tolist())
        swept += ref.sweep(now, ttl)
        redis.now = now
        alive = set()
        for r in before:
            try:
                redis.get(f"k{r}")
                alive.add(r)
            except RedisNil:
                pass
        assert alive == set(np.flatnonzero(ref.stored[: ref.n]).tolist()), f"step {step}: now {now}"
    assert swept > 0
