"""Agent slot reuse: once every slot has been handed out, a new agent id takes the lowest slot whose agent was removed and that no
row of the live window still carries (tests/agentslotref.py is the plain statement of the rule).  An engine with a small agent
table runs many agent lifetimes — register, ingest with replays and duplicates, complete with bytes, drop, expire, reclaim — next
to a twin engine whose table never fills.  Everything but the slot numbers must read the same on both, the slots must follow the
rule, and the old name of a reused slot must be forgotten everywhere."""
import threading

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentslotref import ENOSPC, AgentTable, held_slots
from jsoncase import make_requests, records_array, var_batch

pytestmark = pytest.mark.gpu
SEC = 1_000_000_000
HOUR = 3600 * SEC
T0 = 1_700_000_000 * SEC
TTL = 2 * HOUR
SECRET = 0x5EC0_1234_ABCD_0001
P, M, R, V = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_MINT_IDS, K.AGR_CFG_RING, K.AGR_CFG_VARLEN


def window_routes(eng):
    st = eng.stats()
    n = st["rows_used"] - st["rows_tail"]
    return eng.debug_read("route", st["rows_tail"], n) if n else np.zeros(0, dtype=np.uint32)


def outcomes(rows):
    outs = np.zeros(len(rows), dtype=A.outcome_dtype)
    for j, (rid, agent, kind, http, seq) in enumerate(rows):
        outs[j]["request_id"] = np.frombuffer(rid, dtype=np.uint8)
        outs[j]["agent_id"] = agent.encode()
        outs[j]["kind"], outs[j]["http_status"], outs[j]["seq"] = kind, http, seq
    return outs


class Churn:
    """An engine with max_agents slots and its twin without a limit, driven through the same calls."""

    def __init__(self, flags, max_agents, lifetimes, slab_rows=512, **kw):
        self.flags, self.var, self.mint = flags, bool(flags & V), bool(flags & M)
        self.kw = dict(slab_rows=slab_rows, flags=flags, id_secret=SECRET, vslab_bytes=(slab_rows * 1024) if flags & V else 0,
                       resp_bytes=64 << 10, **kw)
        self.eng = A.Engine(max_agents=max_agents, **self.kw)
        self.twin = A.Engine(max_agents=lifetimes + 16, **self.kw)
        self.table = AgentTable(max_agents)
        self.live, self.gone, self.ids = [], [], {}         # agents registered and not dropped / forgotten names / agent -> ids
        self.reused = self.refused = 0
        self.rng = np.random.default_rng(max_agents * 31 + flags)
        self.same_counters = True                            # (a restored engine's counters start from zero)
        self.seed = 0

    def close(self):
        self.eng.close(); self.twin.close()

    def register(self, name, status):
        new_name, handed_out = self.table.slot(name) is None, len(self.table.names)
        want = self.table.register(name, held_slots(window_routes(self.eng)))
        try:
            got = self.eng.set_agent_state(name, status)
        except A.AgrError as e:
            got = e.code
            assert "still held by live rows" in str(e)
        assert got == want, (name, got, want)
        if got == ENOSPC:
            self.refused += 1
            return None
        self.reused += new_name and got < handed_out                         # a slot taken from a forgotten agent
        self.twin.set_agent_state(name, status)
        self.live.append(name)
        return got

    def ingest(self, reqs, replays=()):
        """fresh requests, then (in a second batch) replay-flagged copies naming earlier ids and, with caller ids, duplicates"""
        out = []
        for batch in (reqs, list(replays)):
            if not batch:
                continue
            recs = records_array(batch)
            for i, r in enumerate(batch):
                if getattr(r, "replay_target", None) is not None:
                    recs[i]["flags"] |= K.AGR_F_REPLAY
                    recs[i]["replay_of"] = np.frombuffer(r.replay_target, dtype=np.uint8)
            res = []
            for e in (self.eng, self.twin):
                if self.var:
                    blob, offs = var_batch(batch)
                    if any(getattr(r, "replay_target", None) is not None for r in batch):
                        # the replay header fields live in the 96-byte header of each variable-length record
                        hdr = np.frombuffer(blob, dtype=np.uint8).copy()
                        for i, r in enumerate(batch):
                            h = hdr[offs[i]:offs[i] + 96].view(A.header_dtype)
                            h["flags"] = recs[i]["flags"]; h["replay_of"] = recs[i]["replay_of"]
                        blob = hdr
                    v, ids, first = e.ingest_var(blob, offs)
                else:
                    v = np.zeros(len(batch), dtype=A.verdict_dtype); ids = np.zeros((len(batch), 16), dtype=np.uint8)
                    first = e.ingest_ex(recs, v, ids)
                res.append((v, ids, first))
            (v, ids, first), (tv, tids, tfirst) = res
            assert first == tfirst and (ids == tids).all()
            assert (v["code"] == tv["code"]).all() and (v["flags"] == tv["flags"]).all() and (v["http_status"] == tv["http_status"]).all()
            for i, r in enumerate(batch):
                slot = self.table.slot(r.agent_id)
                if v[i]["code"] == K.AGR_V_NOT_FOUND:
                    assert slot is None or slot in self.table.removed
                else:
                    assert int(v[i]["agent_slot"]) == slot
                if self.mint or not (v[i]["flags"] & K.AGR_VF_DUP_ID):
                    r.rid = bytes(ids[i])
            out.append(v)
        return out

    def step(self, k, now):
        """one lifetime: a new agent, traffic for every live agent, a few completions, the oldest dropped, TTL + reclaim"""
        name = f"agent-{1700000000000000000 + k}"
        self.register(name, "running" if k % 3 else "stopped")
        agents = self.live + ([self.gone[-1]] if self.gone else [])            # plus a forgotten or removed name
        self.seed += 1
        reqs = make_requests(self.seed, 3 * len(agents), agents, max_payload=416)
        for i, r in enumerate(reqs):
            r.now = now + i
            if not self.mint:
                r.rid = bytes(self.rng.integers(0, 256, 16, dtype=np.uint8))
        replays = []
        for a in agents:
            for old in self.ids.get(a, [])[-1:]:
                q = make_requests(self.seed + 7919, 1, [a])[0]; q.now = now + 100; q.replay_target = old
                replays.append(q)
        if not self.mint and reqs:
            d = make_requests(self.seed + 104729, 1, [reqs[0].agent_id])[0]; d.now = now + 101; d.rid = reqs[0].rid
            replays.append(d)                                                  # a duplicate caller id
        v = self.ingest(reqs, replays)[0]
        for r, vv in zip(reqs, v):
            if vv["flags"] & K.AGR_VF_STORED:
                self.ids.setdefault(r.agent_id, []).append(r.rid)
        # the running agents answer their forwarded requests; some answers carry bytes
        ops = [(r.rid, r.agent_id, K.AGR_OUT_RESPONSE if j % 2 else K.AGR_OUT_ERROR, 200, now + SEC)
               for j, (r, vv) in enumerate(zip(reqs, v)) if vv["code"] == K.AGR_V_FORWARD]
        if ops:
            for e in (self.eng, self.twin):
                assert (e.complete(outcomes(ops)) == 0).all()
                for rid, a, kind, _, _ in ops[:2]:
                    if kind == K.AGR_OUT_RESPONSE:
                        assert e.store_response(a, rid, b"Server: x\n", b"body-" + rid[:4])
        self.check(agents)
        if len(self.live) >= self.table.max_agents or (self.live and k % 4 == 0):
            a = self.live.pop(0)
            for e in (self.eng, self.twin):
                e.drop_agent(a)
            self.table.drop(a)
            self.gone.append(a)
        for e in (self.eng, self.twin):
            e.expire(now, TTL)
            e.reclaim()

    def check(self, agents):
        for a in agents:
            assert self.eng.pending_json(a) == self.twin.pending_json(a), a
            for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
                assert (self.eng.list(a, which) == self.twin.list(a, which)).all(), (a, which)
            for rid in self.ids.get(a, [])[-4:]:
                assert self.eng.get_record_json(a, rid) == self.twin.get_record_json(a, rid)
                assert self.eng.get_response_body(a, rid) == self.twin.get_response_body(a, rid)
        # names whose slot went to another agent are forgotten everywhere
        for a in self.gone[-6:]:
            if self.table.slot(a) is not None:
                continue
            for fn in (self.eng.agent_slot, self.eng.drop_agent):
                with pytest.raises(A.AgrError) as e:
                    fn(a)
                assert e.value.code == K.AGR_ENOTFOUND
            assert self.eng.pending_json(a)[1] == 0 and len(self.eng.list(a, K.AGR_LIST_COMPLETED)) == 0
            for rid in self.ids.get(a, [])[-3:]:
                assert self.eng.get_record_json(a, rid) is None and self.eng.get_record(a, rid) is None
        # the replay scan: the same requests (the engine groups them by slot, and the slots differ between the two)
        d1 = self.eng.replay_scan(with_records=False)[0]
        d2 = self.twin.replay_scan(with_records=False)[0]
        d1, d2 = np.sort(d1, order="rid"), np.sort(d2, order="rid")
        assert (d1["rid"] == d2["rid"]).all() and (d1["request_id"] == d2["request_id"]).all()
        s1, s2 = self.eng.stats(), self.twin.stats()
        assert s1["rows_used"] == s2["rows_used"] and s1["rows_tail"] == s2["rows_tail"]
        if not self.same_counters:
            return
        for key in ("rows_used", "rows_tail", "stored", "dedupe_hits", "forwarded", "queued", "not_found", "dup_ids",
                    "completions", "completion_misses", "failures", "completed_log_len", "failed_log_len"):
            assert s1[key] == s2[key], key


@pytest.mark.parametrize("max_agents", [1, 8])
@pytest.mark.parametrize("mode", ["mint", "hash", "mint-var"])
def test_churn_matches_an_engine_without_a_limit(mode, max_agents):
    flags = P | R | (M if mode.startswith("mint") else 0) | (V if mode.endswith("var") else 0)
    lifetimes = 3000 if max_agents == 1 else 2000
    c = Churn(flags, max_agents, lifetimes)
    try:
        for k in range(lifetimes):
            c.step(k, T0 + k * HOUR)
        assert c.reused >= lifetimes // 20 and c.refused > 0
        assert c.eng.stats()["agents"] == max_agents
        st = c.eng.stats()
        assert st["rows_used"] > 2 * 512                  # the ring lapped: windows crossed its end
        assert c.eng.verify()[1] == 0
    finally:
        c.close()


def numpy_held(routes):
    """held_slots of tests/agentslotref.py, vectorised for windows of tens of millions of rows"""
    code, slot = (routes >> 23) & 7, routes & 0x7FFFFF
    return set(np.unique(slot[(code != 0) & (slot != 0x7FFFFF)]).tolist())


def test_held_slots_at_a_large_wrapped_window():
    """A 2^26-row ring whose window wraps: removed agents with exactly one decided row each — at the window's first row, past the
    first grid-stride pass of k_slot_refs, at the first physical row after the wrap, far into the wrapped range and at the
    window's last row — keep their slots; removed agents with no rows or only AGR_V_NOT_FOUND rows give theirs back, lowest first.
    The engine's choices are checked against a numpy scan of the window's route words."""
    ROWS, B, NS = 1 << 26, 1 << 20, 64
    with A.Engine(slab_rows=ROWS, max_agents=NS, max_batch=B, flags=P | M | R, id_secret=SECRET, log_entries=1 << 20,
                  resp_bytes=1 << 20) as eng:
        special = {"first": 63, "pass2": 31, "wrap": 32, "far": 7, "last": 0, "norows": 5, "notfound": 40}
        names = [None] * NS
        for role, s in special.items():
            names[s] = f"special-{role}"
        filler = iter([A.synth_agent_id(k) for k in range(16)] + [f"spare-{k}" for k in range(NS)])
        names = [n if n is not None else next(filler) for n in names]
        for s, a in enumerate(names):
            assert eng.set_agent_state(a, "stopped") == s
        by_role = {role: names[s] for role, s in special.items()}
        eng.drop_agent(by_role["notfound"])

        def fill(n):
            while n:
                k = min(n, B)
                first = eng.reserve_rows(k)
                eng.synth_fill_rows(first, first, k, n_agents=16)
                eng.ingest_rows(first, k, want_verdicts=False)
                n -= k

        def one(role):
            out = np.zeros(1, dtype=A.verdict_dtype); ids = np.zeros((1, 16), dtype=np.uint8)
            row = eng.ingest_ex(records_array(make_requests(len(role), 1, [by_role[role]])), out, ids)
            assert int(out[0]["code"]) == (K.AGR_V_NOT_FOUND if role == "notfound" else K.AGR_V_QUEUED)
            return row

        tail = ROWS - 3 * B - 5                                   # physical tail 3 (mod 4): the scan's first load is masked
        eng.skip_arrivals(tail)
        rows = {"first": one("first")}
        fill(1_500_000)                                        # past what one pass of the largest grid covers (~1.08 M rows)
        rows["pass2"] = one("pass2")
        fill(ROWS - (tail + 1_500_002) % ROWS)                       # up to the physical end of the ring
        rows["wrap"] = one("wrap")
        fill(20_000_000)
        rows["notfound"] = one("notfound")
        rows["far"] = one("far")
        st = eng.stats()
        fill(ROWS - 1 - (st["rows_used"] - st["rows_tail"]))
        rows["last"] = one("last")
        st = eng.stats()
        assert st["rows_tail"] == tail and st["rows_used"] - tail == ROWS
        assert rows["first"] == tail and rows["wrap"] % ROWS == 0 and rows["last"] == tail + ROWS - 1
        for role in ("first", "pass2", "wrap", "far", "last", "norows"):
            eng.drop_agent(by_role[role])
        routes = eng.debug_read("route", tail, ROWS)
        for role, row in rows.items():
            want = 0x7FFFFF if role == "notfound" else special[role]
            assert int(routes[row - tail]) & 0x7FFFFF == want, role
        removed = {special[r] for r in ("first", "pass2", "wrap", "far", "last", "norows", "notfound")}
        held = numpy_held(routes) & removed
        assert held == {special[r] for r in ("first", "pass2", "wrap", "far", "last")}
        got = []
        for k in range(NS):
            try:
                got.append(eng.set_agent_state(f"fresh-{k}", "running"))
            except A.AgrError as e:
                assert e.code == K.AGR_ENOSPC and f"({len(held)} removed" in str(e)
                break
        assert got == sorted(removed - held) == [special["norows"], special["notfound"]]


def test_held_slots_with_the_candidate_bitmap_in_l2():
    """More than 2^18 slots: the candidate bitmap does not fit shared memory and k_slot_refs reads it through L2."""
    NS = (1 << 18) + 64
    with A.Engine(slab_rows=1 << 12, max_agents=NS, flags=P | M, id_secret=SECRET) as eng:
        names = [f"a-{k}" for k in range(NS)]
        assert (eng.set_agent_states(names, ["stopped"] * NS) == np.arange(NS)).all()
        with_rows = [3, (1 << 18) - 1, (1 << 18) + 10, NS - 1]
        out = np.zeros(len(with_rows), dtype=A.verdict_dtype); ids = np.zeros((len(with_rows), 16), dtype=np.uint8)
        eng.ingest_ex(records_array([make_requests(s, 1, [names[s]])[0] for s in with_rows]), out, ids)
        assert (out["code"] == K.AGR_V_QUEUED).all()
        no_rows = [(1 << 18) - 2, (1 << 18) + 20]
        for s in with_rows + no_rows:
            eng.drop_agent(names[s])
        assert numpy_held(eng.debug_read("route", 0, len(with_rows))) == set(with_rows)
        assert [eng.set_agent_state(f"fresh-{k}", "running") for k in range(2)] == no_rows
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("fresh-2", "running")
        assert e.value.code == K.AGR_ENOSPC and f"({len(with_rows)} removed" in str(e.value)


def test_a_slot_freed_below_the_free_list_is_taken_first():
    """The lowest removed, unheld slot is taken even when an earlier scan left higher slots on its list."""
    with A.Engine(slab_rows=1 << 10, max_agents=3, flags=P | M | R, id_secret=SECRET) as eng:
        for a in ("A", "B", "C"):
            eng.set_agent_state(a, "running")
        eng.drop_agent("B"); eng.drop_agent("C")
        assert eng.set_agent_state("D", "running") == 1        # the scan lists slots 1 and 2
        eng.drop_agent("A")
        assert eng.set_agent_state("E", "running") == 0        # slot 0 is lower than the list's 2
        assert eng.set_agent_state("F", "running") == 2
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("G", "running")
        assert e.value.code == K.AGR_ENOSPC and "(0 removed" in str(e.value)
        # a held slot below the list does not hide the list: slot 0's agent has a row, slot 1's none
        out = np.zeros(1, dtype=A.verdict_dtype); ids = np.zeros((1, 16), dtype=np.uint8)
        eng.ingest_ex(records_array(make_requests(1, 1, ["E"])), out, ids)
        eng.drop_agent("E"); eng.drop_agent("D")
        assert eng.set_agent_state("H", "running") == 1
        eng.drop_agent("F")
        assert eng.set_agent_state("I", "running") == 2
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("J", "running")
        assert e.value.code == K.AGR_ENOSPC and "(1 removed" in str(e.value)


def test_undecided_rows_hold_nothing_and_resolve_names_when_decided():
    """Reserved rows not decided yet hold no slot; when decided after the reuse they resolve each name as it is then."""
    with A.Engine(slab_rows=4096, max_agents=2, flags=P | M | R, id_secret=SECRET) as eng:
        assert eng.set_agent_state("agent-a", "running") == 0 and eng.set_agent_state("agent-b", "running") == 1
        first = eng.reserve_rows(8)
        reqs = [r for pair in zip(make_requests(3, 4, ["agent-a"]), make_requests(4, 4, ["agent-c"])) for r in pair]
        eng.fill_rows(first, records_array(reqs))
        eng.drop_agent("agent-a")
        assert eng.set_agent_state("agent-c", "stopped") == 0        # agent-a's reserved rows hold nothing
        v = eng.ingest_rows(first, 8)
        for r, vv in zip(reqs, v):
            if r.agent_id == "agent-a":
                assert int(vv["code"]) == K.AGR_V_NOT_FOUND            # decided now: agent-a is forgotten
            else:
                assert int(vv["code"]) == K.AGR_V_QUEUED and int(vv["agent_slot"]) == 0
        assert eng.pending_json("agent-c")[1] == sum(r.agent_id == "agent-c" for r in reqs)


def test_exchange_holes_hold_nothing():
    """Rows the exchange shipped to their owner shard are holes of this shard's window: the shipped agent's slot is free."""
    names = [f"agent-{k}" for k in range(200)]
    away = next(a for a in names if A.agent_shard(a, 2) == 1)
    with A.Engine(slab_rows=4096, max_agents=1, flags=P | M | R, id_secret=SECRET) as eng:
        eng.debug_world(0, 2)
        assert eng.set_agent_state(away, "stopped") == 0
        reqs = make_requests(4, 64, [away])
        first = eng.reserve_rows(64)
        eng.fill_rows(first, records_array(reqs))
        send, info = eng.debug_exchange_begin(first, 64)
        assert len(send) == 64                                           # every row went to shard 1
        eng.debug_exchange_end(np.zeros(len(send), dtype=A.verdict_dtype), 64)
        assert held_slots(eng.debug_read("route", first, 64)) == set()
        eng.drop_agent(away)
        assert eng.set_agent_state("agent-next", "running") == 0


def test_non_ring_engine_reuses_only_agents_without_decided_rows():
    with A.Engine(slab_rows=1 << 12, max_agents=3, flags=P | M, id_secret=SECRET) as eng:
        for a in ("agent-a", "agent-b", "agent-c"):
            eng.set_agent_state(a, "stopped")
        out = np.zeros(2, dtype=A.verdict_dtype); ids = np.zeros((2, 16), dtype=np.uint8)
        eng.ingest_ex(records_array(make_requests(5, 2, ["agent-b"])), out, ids)
        for a in ("agent-a", "agent-b", "agent-c"):
            eng.drop_agent(a)
        assert eng.set_agent_state("agent-d", "running") == 0
        assert eng.set_agent_state("agent-e", "running") == 2
        with pytest.raises(A.AgrError) as e:
            eng.set_agent_state("agent-f", "running")
        assert e.value.code == K.AGR_ENOSPC and "(1 removed" in str(e.value)
        assert eng.set_agent_state("agent-b", "running") == 1         # b was never forgotten: revived on its slot


def test_bulk_feed_with_reuse_equals_single_calls():
    kw = dict(slab_rows=1 << 12, max_agents=24, flags=P | M | R, id_secret=SECRET)
    with A.Engine(**kw) as one, A.Engine(**kw) as bulk:
        first = [f"agent-{k}" for k in range(24)]
        for e in (one, bulk):
            e.set_agent_states(first, ["running"] * 24)
            out = np.zeros(4, dtype=A.verdict_dtype); ids = np.zeros((4, 16), dtype=np.uint8)
            e.ingest_ex(records_array(make_requests(9, 4, first[:2])), out, ids)   # agents 0 and 1 hold their slots
            for a in first[:20]:
                e.drop_agent(a)
        names = [f"agent-{k}" for k in range(24, 44)] + first[:3] + [f"agent-{k}" for k in range(44, 50)]
        sts = ["running", "stopped"] * (len(names) // 2) + ["running"] * (len(names) % 2)
        want = []
        for a, s in zip(names, sts):
            try:
                want.append(one.set_agent_state(a, s))
            except A.AgrError as e:
                want.append(e.code)
        with pytest.raises(A.AgrError) as e:
            bulk.set_agent_states(names, sts)                          # some entries are refused: the call reports the first
        assert e.value.code == K.AGR_ENOSPC and ENOSPC in want
        for a, w in zip(names, want):
            if w >= 0 and one.agent_slot(a) == w:
                assert bulk.agent_slot(a) == w, a
            elif w == ENOSPC:
                with pytest.raises(A.AgrError):
                    bulk.agent_slot(a)
        for e in (one, bulk):
            out = np.zeros(8, dtype=A.verdict_dtype); ids = np.zeros((8, 16), dtype=np.uint8)
            e.ingest_ex(records_array(make_requests(11, 8, names[:4] + first[:2])), out, ids)
            if e is one:
                v1 = out.copy()
            else:
                assert (out == v1).all()


@pytest.mark.parametrize("kind", ["blocking", "online", "delta"])
def test_snapshots_across_a_reuse(kind, tmp_path):
    extra = {"blocking": 0, "online": K.AGR_CFG_ONLINE_SNAPSHOT, "delta": K.AGR_CFG_ONLINE_SNAPSHOT | K.AGR_CFG_DELTA_SNAPSHOT}[kind]
    c = Churn(P | M | R | extra, 4, 120)
    try:
        paths = []
        for k in range(60):
            c.step(k, T0 + k * HOUR)
            if k % 12 == 11:
                paths.append(str(tmp_path / f"s{k}.snap"))
                c.eng.snapshot(paths[-1])
        assert c.reused > 5
        back = [A.Engine(max_agents=4, restore_from=paths[-1], **c.kw)]
        kw2 = dict(c.kw, slab_rows=4096)
        back.append(A.Engine(max_agents=4, restore_from=paths[-1], **kw2))          # relocated into another capacity
        try:
            for b in back:
                for a in c.live:
                    assert b.agent_slot(a) == c.eng.agent_slot(a)
                for a in c.live + c.gone[-4:]:
                    assert b.pending_json(a) == c.eng.pending_json(a)
                    for rid in c.ids.get(a, [])[-3:]:
                        assert b.get_record_json(a, rid) == c.eng.get_record_json(a, rid)
            # the engine restored in place continues the churn exactly as the engine it was cut from
            twin_eng, c.eng = c.eng, back[0]
            c.twin.close()
            c.twin = twin_eng
            c.same_counters = False
            for k in range(60, 96):
                c.step(k, T0 + k * HOUR)
        finally:
            for b in back[1:]:
                b.close()
    finally:
        c.close()


def test_front_end_answers_stay_correct_while_agents_churn():
    flags = P | M | R | K.AGR_CFG_COMBINE
    with A.Engine(slab_rows=1 << 14, max_agents=4, flags=flags, id_secret=SECRET) as eng:
        eng.set_agent_state("agent-live", "running")
        stop = threading.Event()
        errors = []

        def caller(seed):
            reqs = make_requests(seed, 200, ["agent-live"])
            for r in reqs:
                r.now = T0
            recs = records_array(reqs)
            for i in range(len(reqs)):
                if stop.is_set():
                    break
                ans = eng.poll(eng.submit_ingest(recs[i]))
                v = ans["verdict"][0]
                if int(v["code"]) != K.AGR_V_FORWARD or int(v["agent_slot"]) != 0:
                    errors.append((seed, i, int(v["code"]), int(v["agent_slot"])))
        threads = [threading.Thread(target=caller, args=(s,)) for s in (1, 2, 3)]
        for t in threads:
            t.start()
        reused = 0
        for k in range(60):
            a = f"agent-{k}"
            try:
                eng.set_agent_state(a, "stopped")
            except A.AgrError as e:
                assert e.code == K.AGR_ENOSPC
                continue
            reqs = make_requests(50 + k, 2, [a])
            for r in reqs:
                r.now = T0
            out = np.zeros(2, dtype=A.verdict_dtype); ids = np.zeros((2, 16), dtype=np.uint8)
            eng.ingest_ex(records_array(reqs), out, ids)
            assert (out["code"] == K.AGR_V_QUEUED).all()
            eng.drop_agent(a)
            eng.expire(T0 + 10 * HOUR, TTL)                                    # every row so far expires and is released
            eng.reclaim()
            reused += 1
        stop.set()
        for t in threads:
            t.join()
        assert not errors, errors[:5]
        assert reused > 10 and eng.agent_slot("agent-live") == 0
