"""Parity of the CUDA path (through the C-ABI) against the oracle and the golden KATs.  GPU only.
Integer / byte work: the bar is bit-exact on verdicts, per-record (status, retry, response), per-agent
pending / completed / failed id sequences (with the Q7 duplicates) and per-tick replay dispatch order."""
import os

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from kats import SCENARIOS, load_golden
from scenario import run_oracle, run_engine, assert_same, random_scenario, Req, rid_of, make_records

pytestmark = pytest.mark.gpu
GOLD, _ = load_golden()


def engine(**kw):
    kw.setdefault("slab_rows", 1 << 15)
    kw.setdefault("max_agents", 256)
    return A.Engine(**kw)


MINT = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS


@pytest.mark.parametrize("kat", sorted(SCENARIOS))
def test_kats_with_engine_minted_ids(kat):
    """AGR_CFG_MINT_IDS: the engine mints Request.ID (as StoreRequest does, requests.go:87); every KAT still holds."""
    with engine(flags=MINT) as eng:
        got = run_engine(eng, SCENARIOS[kat])
    exp = GOLD[kat]
    assert got.verdicts == exp["verdicts"] and got.ticks == exp["ticks"] and got.records == exp["records"]
    for a, qs in exp["lists"].items():
        assert got.lists[a] == qs, (kat, a)


@pytest.mark.parametrize("seed", range(8))
def test_random_streams_with_engine_minted_ids(seed):
    ev = random_scenario(200 + seed, n_events=400, n_agents=2 + seed % 6, p_replay=0.2)
    ref = run_oracle(ev)
    with engine(flags=MINT) as eng:
        assert_same(ref, run_engine(eng, ev))
    with engine(flags=MINT) as eng:                                   # the same stream in random-size batches
        assert_same(ref, run_engine(eng, ev, rng=np.random.default_rng(seed)))


def test_minted_ids_are_uuid4_unique_and_verified_exactly():
    with engine(flags=MINT, id_secret=0xfeedface12345678) as eng:
        eng.set_agent_state("agent-1", "stopped")
        reqs = [Req("agent-1", rid_of(i), i) for i in range(1, 2001)]
        v, first = eng.ingest(make_records(reqs))
        ids = eng.mint_ids(first, 2000)
        assert len({bytes(x) for x in ids}) == 2000
        assert (ids[:, 6] >> 4 == 4).all() and (ids[:, 8] >> 6 == 2).all()
        assert [bytes(x) for x in eng.list("agent-1", 0)] == [bytes(x) for x in ids]          # pending list speaks minted ids
        rec = eng.get_record("agent-1", bytes(ids[7]))
        assert bytes(rec["request_id"]) == bytes(ids[7]) and int(rec["seq"]) == 8
        # one flipped bit anywhere in the id is a miss (exact 128-bit check, not a tag compare)
        for bit in (0, 37, 63, 64, 100, 127):
            bad = bytearray(bytes(ids[7])); bad[bit // 8] ^= 1 << (bit % 8)
            assert eng.get_record("agent-1", bytes(bad)) is None
        assert eng.get_record("agent-1", rid_of(8)) is None                                  # the caller's own id is not a key
        outs = np.zeros(2, dtype=A.outcome_dtype)
        outs["agent_id"] = b"agent-1"; outs["kind"] = K.AGR_OUT_RESPONSE; outs["http_status"] = 200
        outs[0]["request_id"] = ids[3]; outs[1]["request_id"] = np.frombuffer(rid_of(4), dtype=np.uint8)
        assert list(eng.complete(outs)) == [0, K.AGR_ENOTFOUND]



@pytest.mark.parametrize("kat", sorted(SCENARIOS))
def test_kat_against_golden_and_oracle(kat):
    with engine() as eng:
        got = run_engine(eng, SCENARIOS[kat])
    exp = GOLD[kat]
    assert got.verdicts == exp["verdicts"]
    assert got.ticks == exp["ticks"]
    for a, qs in exp["lists"].items():
        assert got.lists[a] == qs, (kat, a)
    assert got.records == exp["records"]
    assert_same(run_oracle(SCENARIOS[kat]), got)


@pytest.mark.parametrize("seed", range(12))
def test_random_streams_match_oracle(seed):
    ev = random_scenario(seed, n_events=400, n_agents=2 + seed % 6)
    with engine() as eng:
        assert_same(run_oracle(ev), run_engine(eng, ev))


@pytest.mark.parametrize("seed", range(6))
def test_result_does_not_depend_on_batching(seed):
    """Same stream, requests batched 1-by-1, in random-size batches, or all at once: identical observables."""
    ev = random_scenario(100 + seed, n_events=250, n_agents=4, p_replay=0.25)
    ref = run_oracle(ev)
    with engine() as eng:
        assert_same(ref, run_engine(eng, ev, max_batch=1))
    with engine() as eng:
        assert_same(ref, run_engine(eng, ev, rng=np.random.default_rng(seed)))


def test_ragged_batches_match_c_port():
    """Batch sizes around the 32-record tile and a batch that is not at row 0 (the TMA kernel's partial tiles and its tile
    schedule): every verdict, every per-agent list and the counters against the C restatement of the reference, and
    AGR_VF_KNOWN / dedupe_hits against the plain reference of the dedupe-hit rule."""
    import k1ref
    from oracle.cpu_ref import CRef
    for seed in (3, 8):
        ev = random_scenario(seed, n_events=400, n_agents=5)
        with engine() as eng:
            assert_same(run_oracle(ev), run_engine(eng, ev))
    sizes = (1, 31, 32, 33, 63, 64, 65, 1000, 2049, 700)
    recs = A.synth_fill_host(0, sum(sizes), seed=9, n_agents=8, dup_permille=100)
    agents = [A.synth_agent_id(k) for k in range(8)]
    with engine() as eng, CRef() as ref:
        for e in (eng, ref):
            for k, a in enumerate(agents):
                e.set_agent_state(a, "running" if k % 3 else "stopped")
        v0, v1, off = [], [], 0
        for n in sizes:
            chunk = np.ascontiguousarray(recs[off:off + n]); off += n
            v0.append(eng.ingest(chunk)[0]); v1.append(ref.ingest(chunk)[0])
        v0, v1 = np.concatenate(v0), np.concatenate(v1)
        assert (v0["code"] == v1["code"]).all() and ((v0["flags"] & 0x7) == (v1["flags"] & 0x7)).all()
        assert (v0["agent_slot"] == v1["agent_slot"]).all()
        for a in agents:
            for w in (0, 1, 2):
                assert eng.list(a, w).tobytes() == ref.list(a, w).tobytes(), (a, w)
        known, _ = k1ref.dedupe_hits(recs, recs["request_id"], agents)
        assert (((v0["flags"] & K.AGR_VF_KNOWN) != 0) == known).all()
        s, fl = eng.stats(), v1["flags"]
        code = lambda c: int((v1["code"] == c).sum())
        exp = dict(ingested=len(recs), stored=int(((fl & K.AGR_VF_STORED) != 0).sum()), replay_flagged=int(((fl & K.AGR_VF_REPLAY) != 0).sum()),
                   dedupe_hits=int(known.sum()), forwarded=code(K.AGR_V_FORWARD), queued=code(K.AGR_V_QUEUED),
                   unavailable=code(K.AGR_V_UNAVAILABLE), not_found=code(K.AGR_V_NOT_FOUND), dup_ids=0)
        assert {k: s[k] for k in exp} == exp
        assert exp["dedupe_hits"] > 100 and exp["queued"] > 0


@pytest.mark.parametrize("mode", ["hash", "mint"])
def test_checksum_matches_numpy(mode):
    """cksum[rid] = (sum (k+1) w_k) << 32 | sum w_k over the 128 LE words — checked through a device read-back, in both
    instantiations of the K1 kernel (caller ids / engine-minted ids)."""
    import ctypes as C
    n = 777
    recs = A.synth_fill_host(0, n, seed=4, n_agents=4)
    w = recs.view(np.uint32).reshape(n, 128).astype(np.uint64)
    c0 = w.sum(axis=1) & 0xFFFFFFFF
    c1 = (w * np.arange(1, 129, dtype=np.uint64)).sum(axis=1) & 0xFFFFFFFF
    with engine(flags=MINT if mode == "mint" else K.AGR_CFG_PERSISTENCE) as eng:
        for k in range(4):
            eng.set_agent_state(A.synth_agent_id(k), "running")
        eng.ingest(recs)
        got = eng.debug_read("cksum", 0, n)
    assert (got == ((c1 << np.uint64(32)) | c0)).all()


def test_chunked_pipelined_ingest_equals_one_launch():
    """agr_ingest pipelines H2D chunks (128 Ki records) against K1 on a second stream: same verdicts, state and lists as
    ONE K1 launch over the same rows, from pageable and from pinned host memory."""
    n, na = 300_000, 32
    recs = A.synth_fill_host(0, n, seed=31, n_agents=na, dup_permille=100)

    def setup(e):
        for k in range(na):
            e.set_agent_state(A.synth_agent_id(k), "running" if k % 4 else "stopped")
    with engine(slab_rows=n, max_batch=n) as e0, engine(slab_rows=n, max_batch=n) as e1, engine(slab_rows=n, max_batch=n) as e2:
        for e in (e0, e1, e2):
            setup(e)
        first = e0.reserve_rows(n)
        e0.synth_fill_rows(0, first, n, seed=31, n_agents=na, dup_permille=100)
        v0 = e0.ingest_rows(first, n)
        v1, _ = e1.ingest(recs)                                    # pageable -> bounce buffers, 3 chunks
        pin, pv = e2.pinned(n), e2.pinned(n, A.verdict_dtype)
        pin.array[:] = recs
        v2, _ = e2.ingest(pin.array, out=pv.array)                 # pinned in, pinned out
        assert v0.tobytes() == v1.tobytes() == v2[:n].tobytes()
        assert e0.debug_read("verdict", first, n).tobytes() == v0.tobytes()       # the read-back bench.py --dump-outputs uses
        for k in ("state", "route", "cksum"):
            assert e0.debug_read(k, 0, n).tobytes() == e1.debug_read(k, 0, n).tobytes() == e2.debug_read(k, 0, n).tobytes()
        s0, s1, s2 = e0.stats(), e1.stats(), e2.stats()
        for k in ("stored", "replay_flagged", "dedupe_hits", "forwarded", "queued", "unavailable", "dup_ids"):
            assert s0[k] == s1[k] == s2[k], k
        del v2
        pin.free(); pv.free()


def test_config1_stream_on_gpu():
    """BASELINE config 1 (10 k records / 16 agents / stop-start / one tick) through the CUDA path == Python oracle."""
    from scenario import config1_events
    ev, _ = config1_events()
    with engine() as eng:
        assert_same(run_oracle(ev), run_engine(eng, ev, max_batch=4096))


@pytest.mark.parametrize("mode", ["hash", "mint"])
def test_config3_shape_against_c_port(mode):
    """BASELINE config 3's shape (Zipf s = 1.2 over 256 ids, 10 % replay-flagged duplicates) at 200 k records, with a
    mixed agent population, completions, a stop/start and a tick: CUDA path == C restatement on every verdict, every
    per-agent list and the replay dispatch order."""
    from oracle.cpu_ref import CRef
    n, na = 200_000, 256
    agents = [A.synth_agent_id(k) for k in range(na)]
    outs = np.zeros(n, dtype=A.outcome_dtype)
    flags = MINT if mode == "mint" else 0
    with A.Engine(slab_rows=1 << 19, max_agents=512, max_batch=1 << 18, flags=flags) as eng, CRef() as ref:
        if mode == "mint":
            # the stream's duplicates name engine-minted ids; the checker is given the same ids the engine will mint
            recs = A.synth_fill_host(0, n, seed=3, n_agents=na, zipf_milli=1200, dup_permille=100, mint=(eng, 0))
            recs["request_id"] = eng.mint_ids(0, n)
        else:
            recs = A.synth_fill_host(0, n, seed=3, n_agents=na, zipf_milli=1200, dup_permille=100)
        for e in (eng, ref):
            for k, a in enumerate(agents):
                e.set_agent_state(a, "stopped" if k % 5 == 1 else "running")      # incl. the rank-1 hot agent
        results = []
        for e in (eng, ref):
            v, _ = e.ingest(recs)
            fwd = (v["code"] == K.AGR_V_FORWARD) & ((v["flags"] & K.AGR_VF_TRACKED) != 0)
            m = int(fwd.sum())
            outs[:m]["request_id"] = np.where(((recs["flags"][fwd] & 1) != 0)[:, None], recs["replay_of"][fwd], recs["request_id"][fwd])
            outs[:m]["agent_id"] = recs["agent_id"][fwd]
            kinds = np.array([K.AGR_OUT_RESPONSE, K.AGR_OUT_RESPONSE, K.AGR_OUT_RESPONSE, K.AGR_OUT_ERROR, K.AGR_OUT_DIAL_ERR], dtype=np.uint8)
            outs[:m]["kind"] = kinds[np.arange(m) % 5]
            outs[:m]["http_status"] = 200
            res = e.complete(np.ascontiguousarray(outs[:m]))
            for k, a in enumerate(agents):
                if k % 5 == 1:
                    e.set_agent_state(a, "running")
            disp, _ = e.replay_scan(with_records=False) if e is eng else e.replay_scan()
            results.append((v, res, disp))
        (v0, r0, d0), (v1, r1, d1) = results
        assert (v0["code"] == v1["code"]).all() and ((v0["flags"] & 0x7) == (v1["flags"] & 0x7)).all()
        assert (v0["agent_slot"] == v1["agent_slot"]).all()
        assert (r0 == r1).all()
        assert len(d0) == len(d1) > 10_000
        assert (d0["agent_slot"] == d1["agent_slot"]).all() and d0["request_id"].tobytes() == d1["request_id"].tobytes()
        for a in agents[:12] + agents[100:104]:
            for w in (0, 1, 2):
                assert eng.list(a, w, cap=1 << 16).tobytes() == ref.list(a, w, cap=1 << 16).tobytes(), (a, w)
        assert eng.stats()["dedupe_hits"] > 10_000            # the duplicates really resolved to earlier stored rows


@pytest.mark.parametrize("mode", ["hash", "mint"])
def test_config5_crash_replay_cycles_against_c_port(mode):
    """BASELINE config 5's event shape on fixed 512 B records: a sustained stream in batches; every few batches 1 % of
    the agents 'crash' — status still running, forwards end in dial errors, so their records stay pending with retry
    untouched (Q12) — then they come back and ONE tick replays each crashed agent's whole pending queue in FIFO order
    (Q14), each replay completing twice (Q7).  CUDA path == C restatement on verdicts, dispatch order and lists."""
    from oracle.cpu_ref import CRef
    na, B, nb = 200, 20_000, 10
    agents = [A.synth_agent_id(k) for k in range(na)]
    flags = MINT if mode == "mint" else 0
    rng = np.random.default_rng(5)
    with A.Engine(slab_rows=1 << 19, max_agents=512, max_batch=1 << 17, flags=flags) as eng, CRef() as ref:
        for e in (eng, ref):
            for a in agents:
                e.set_agent_state(a, "running")
        crashed = np.zeros(na, dtype=bool)
        total_replayed = 0
        for b in range(nb):
            recs = A.synth_fill_host(b * B, B, seed=9, n_agents=na, zipf_milli=1200)
            if mode == "mint":
                recs["request_id"] = eng.mint_ids(eng.stats()["rows_used"], B)
            if b % 3 == 1:
                crashed[rng.choice(na, size=max(1, na // 100 * 2), replace=False)] = True     # ~1-2 % of the agents
            idx = (np.array([int(x[6:]) for x in recs["agent_id"]]) - 1700000000000000000) // 1000003
            outs = np.zeros(B, dtype=A.outcome_dtype)
            outs["request_id"], outs["agent_id"], outs["http_status"] = recs["request_id"], recs["agent_id"], 200
            outs["kind"] = np.where(crashed[idx], K.AGR_OUT_DIAL_ERR, K.AGR_OUT_RESPONSE)
            got = []
            for e in (eng, ref):
                v, _ = e.ingest(recs)
                r = e.complete(outs)
                got.append((v["code"].copy(), r.copy()))
            assert (got[0][0] == got[1][0]).all() and (got[0][1] == got[1][1]).all()
            if b % 3 == 2:                      # the crashed agents restart; one tick replays their queues
                crashed[:] = False
                d0, r0 = eng.replay_scan(with_records=True)
                d1, r1 = ref.replay_scan()
                assert len(d0) == len(d1) and (d0["agent_slot"] == d1["agent_slot"]).all()
                assert d0["request_id"].tobytes() == d1["request_id"].tobytes()
                assert r0["payload"].tobytes() == r1["payload"].tobytes()          # the gathered records are the stored ones
                total_replayed += len(d0)
                rep = np.zeros(2 * len(d0), dtype=A.outcome_dtype)                  # server-side + worker-side completion (Q7)
                rep["request_id"] = np.repeat(d0["request_id"], 2, axis=0)
                rep["agent_id"] = np.repeat(r0["agent_id"], 2)
                rep["kind"], rep["http_status"] = K.AGR_OUT_RESPONSE, 200
                for e in (eng, ref):
                    e.complete(rep)
        assert total_replayed > 1000
        for a in agents[:8] + [agents[k] for k in (50, 120, 199)]:
            for w in (0, 1, 2):
                assert eng.list(a, w, cap=1 << 16).tobytes() == ref.list(a, w, cap=1 << 16).tobytes(), (a, w)
        assert sum(len(eng.list(a, 0)) for a in agents) == 0


def test_ingest_ex_returns_the_ids_the_engine_knows():
    recs = A.synth_fill_host(0, 3000, seed=5, n_agents=4)
    for flags in (0, MINT):
        with engine(flags=flags) as eng:
            for k in range(4):
                eng.set_agent_state(A.synth_agent_id(k), "running")
            eng.ingest(recs[:1000])
            out, ids = np.zeros(2000, dtype=A.verdict_dtype), np.zeros((2000, 16), dtype=np.uint8)
            first = eng.ingest_ex(np.ascontiguousarray(recs[1000:]), out, ids)
            assert first == 1000 and (out["code"] == K.AGR_V_FORWARD).all()
            exp = eng.mint_ids(first, 2000) if flags else recs["request_id"][1000:]
            assert (ids == exp).all()


def test_persistence_disabled():
    ev = [("agent", "agent-1", "running"), ("agent", "agent-2", "stopped"),
          ("req", Req("agent-1", rid_of(1), 1), ("response", 200)), ("req", Req("agent-2", rid_of(2), 2), ("response", 200))]
    with engine(flags=0x80000000) as eng:      # any non-zero flags word without AGR_CFG_PERSISTENCE
        got = run_engine(eng, ev)
    assert_same(run_oracle(ev, persistence=False), got)
    assert got.verdicts == [(1, 0, False, False), (3, 503, False, False)]


def test_duplicate_fresh_id_is_a_persistence_failure():
    """ABI contract (not reachable in the reference, whose ids come from uuid.New): a fresh record whose id is already
    stored — in an earlier batch or EARLIER IN THE SAME BATCH — is not stored and goes on untracked."""
    with engine() as eng:
        eng.set_agent_state("agent-1", "running")
        eng.set_agent_state("agent-2", "stopped")
        reqs = [Req("agent-1", rid_of(1), 1), Req("agent-2", rid_of(2), 2), Req("agent-1", rid_of(1), 3),
                Req("agent-2", rid_of(2), 4), Req("agent-2", rid_of(1), 5)]
        v, _ = eng.ingest(make_records(reqs))
        assert [int(x) for x in v["code"]] == [1, 2, 1, 3, 3]
        assert [int(x) & K.AGR_VF_STORED for x in v["flags"]] == [1, 1, 0, 0, 0]
        assert [bool(int(x) & K.AGR_VF_DUP_ID) for x in v["flags"]] == [False, False, True, True, True]
        v2, _ = eng.ingest(make_records([Req("agent-1", rid_of(2), 6), Req("agent-1", rid_of(7), 7)]))
        assert [bool(int(x) & K.AGR_VF_DUP_ID) for x in v2["flags"]] == [True, False]
        assert [bytes(x).hex() for x in eng.list("agent-2", 0)] == [rid_of(2).hex()]
        s = eng.stats()
        assert s["dup_ids"] == 4 and s["stored"] == 3


def test_large_batch_duplicate_race_is_resolved_by_arrival_order():
    """Many duplicates inside one big batch: whichever thread wins the insert race, the LOWEST row keeps the id."""
    n = 1 << 14
    reqs = A.synth_fill_host(0, n, seed=21, n_agents=8)
    reqs2 = reqs.copy()
    dup_src = np.arange(0, n // 2, 7)
    dup_dst = n - 1 - np.arange(len(dup_src))
    reqs2["request_id"][dup_dst] = reqs2["request_id"][dup_src]
    with engine(slab_rows=1 << 16) as eng:
        for k in range(8):
            eng.set_agent_state(A.synth_agent_id(k), "running" if k % 2 else "stopped")
        v, _ = eng.ingest(reqs2)
        dup = (v["flags"] & K.AGR_VF_DUP_ID) != 0
        assert set(np.nonzero(dup)[0]) == set(dup_dst)
        assert ((v["flags"][~dup] & K.AGR_VF_STORED) != 0).all()
        assert set(v["code"][dup]) <= {K.AGR_V_FORWARD, K.AGR_V_UNAVAILABLE}
        assert set(v["code"][~dup]) <= {K.AGR_V_FORWARD, K.AGR_V_QUEUED}
        s = eng.stats()
        assert s["stored"] == n - len(dup_dst) and s["dup_ids"] == len(dup_dst)
        assert s["queued"] == int((v["code"] == K.AGR_V_QUEUED).sum()) and s["unavailable"] == int((v["code"] == K.AGR_V_UNAVAILABLE).sum())


def test_known_flag_means_stored_earlier():
    with engine() as eng:
        eng.set_agent_state("agent-1", "running")
        reqs = [Req("agent-1", rid_of(1), 1, replay=True, replay_of=rid_of(2)),   # names a LATER row of the same batch
                Req("agent-1", rid_of(2), 2),
                Req("agent-1", rid_of(3), 3, replay=True, replay_of=rid_of(2))]
        v, _ = eng.ingest(make_records(reqs))
        assert [bool(int(x) & K.AGR_VF_KNOWN) for x in v["flags"]] == [False, False, True]
        assert eng.stats()["dedupe_hits"] == 1


def test_pending_and_get_record_views():
    ev = [("agent", "agent-1", "stopped")] + [("req", Req("agent-1", rid_of(i), i, body=b"x" * i), ("response", 200)) for i in range(1, 40)]
    with engine() as eng:
        run_engine(eng, ev)
        pend = eng.pending("agent-1")
        assert [bytes(r["request_id"]) for r in pend] == [rid_of(i) for i in range(1, 40)]
        assert (pend["status"] == K.AGR_ST_PENDING).all() and (pend["body_len"] == np.arange(1, 40)).all()
        rec = eng.get_record("agent-1", rid_of(7))
        assert int(rec["seq"]) == 7 and bytes(rec["payload"][rec["path_len"] + rec["hdr_len"]:][:7]) == b"x" * 7
        assert eng.get_record("agent-1", rid_of(99)) is None
        assert eng.get_record("agent-2", rid_of(7)) is None


def test_full_size_properties_1m():
    """BASELINE config 2 at full size (1 M records, 256 agents, all running): size-independent properties."""
    n, na = 1 << 20, 256
    with A.Engine(slab_rows=n, max_agents=512, max_batch=n) as eng:
        for k in range(na):
            eng.set_agent_state(A.synth_agent_id(k), "running")
        first = eng.reserve_rows(n)
        eng.synth_fill_rows(0, first, n, seed=2, n_agents=na)
        v = eng.ingest_rows(first, n)
        assert (v["code"] == K.AGR_V_FORWARD).all() and ((v["flags"] & K.AGR_VF_STORED) != 0).all()
        s = eng.stats()
        assert s["ingested"] == n and s["stored"] == n and s["forwarded"] == n and s["dup_ids"] == 0
        host = A.synth_fill_host(0, 4096, seed=2, n_agents=na)
        slots = {A.synth_agent_id(k).encode(): k for k in range(na)}
        assert [slots[x] for x in host["agent_id"]] == list(v["agent_slot"][:4096])
        # every record pending, per-agent FIFO == arrival order
        a0 = A.synth_agent_id(3)
        ids = eng.list(a0, K.AGR_LIST_PENDING, cap=1 << 14)
        mask = host["agent_id"] == a0.encode()
        assert [bytes(x) for x in ids[: mask.sum()]] == [bytes(x) for x in host["request_id"][mask]]
        assert sum(len(eng.list(A.synth_agent_id(k), 0, cap=1 << 14)) for k in range(0, na, 37)) > 0


def test_flat_combining_of_concurrent_single_request_calls():
    """AGR_CFG_COMBINE: many threads calling agr_ingest_ex / agr_complete with ONE request each get the same answers as a
    serial run, in far fewer K1 launches; the ring order is the event order (per-agent FIFO = order of the row ids)."""
    import threading
    nt, per = 16, 60
    agents = ["agent-%d" % k for k in range(4)]
    with engine(flags=MINT | K.AGR_CFG_COMBINE, slab_rows=1 << 14) as eng:
        for k, a in enumerate(agents):
            eng.set_agent_state(a, "stopped" if k % 2 else "running")
        results = [[] for _ in range(nt)]

        def worker(t):
            for i in range(per):
                a = agents[(t + i) % 4]
                rec = make_records([Req(a, rid_of(1 + t * per + i), 1 + t * per + i)])
                out, ids = np.zeros(1, dtype=A.verdict_dtype), np.zeros((1, 16), dtype=np.uint8)
                first = eng.ingest_ex(rec, out, ids)
                results[t].append((a, int(out[0]["code"]), first, bytes(ids[0])))
                if int(out[0]["code"]) == K.AGR_V_FORWARD:
                    o = np.zeros(1, dtype=A.outcome_dtype)
                    o["request_id"], o["agent_id"], o["kind"], o["http_status"] = ids[0], a.encode(), K.AGR_OUT_RESPONSE, 200
                    assert list(eng.complete(o)) == [0]

        ths = [threading.Thread(target=worker, args=(t,)) for t in range(nt)]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
        flat = [x for r in results for x in r]
        assert len({x[2] for x in flat}) == nt * per                       # every request got its own row
        assert all((code == K.AGR_V_QUEUED) == (agents.index(a) % 2 == 1) for a, code, _, _ in flat)
        assert all(bytes(eng.mint_ids(first, 1)[0]) == rid for _, _, first, rid in flat)
        for k, a in enumerate(agents):
            mine = sorted((first, rid) for aa, _, first, rid in flat if aa == a)
            pend = [bytes(x) for x in eng.list(a, K.AGR_LIST_PENDING)]
            comp = [bytes(x) for x in eng.list(a, K.AGR_LIST_COMPLETED)]
            if k % 2:
                assert pend == [rid for _, rid in mine] and comp == []     # FIFO == row order == ring order
            else:
                assert pend == [] and sorted(comp) == sorted(rid for _, rid in mine)
        s = eng.stats()
        assert s["stored"] == nt * per and s["k1_launches"] < 2 * nt * per


@pytest.mark.parametrize("cfg", ["c2", "c3"])
def test_full_size_configs_against_c_port(cfg):
    """BASELINE configs[1] (1 M records, 256 agent ids, uniform) and configs[2] (10 M records, Zipf s = 1.2, 10 % replay-flagged
    duplicates) at their FULL size, engine-minted ids, in 1 M-record batches: every verdict of every record, the result code of
    every outcome (every forwarded request is answered in arrival order, one in 5003 fails), the replay tick's dispatch list after
    a stop / start of a fifth of the agents, and whole per-agent lists — CUDA path == C restatement of the reference, bit for bit.
    (Answering in arrival order keeps the reference's LREM at the head of its list: its O(queue) scan would otherwise make the
    checker quadratic — ten minutes for this test.)"""
    from oracle.cpu_ref import CRef
    B, na = 1 << 20, 256
    # the C port really marshals / unmarshals JSON like the Go code: ~9 s per million requests on the GPU boxes' hosts, so C3 at its
    # AGR_QUICK_PARITY=1 cuts the 10 M stream to 2 M
    nb = 1 if cfg == "c2" else (2 if os.environ.get("AGR_QUICK_PARITY") else 10)
    zipf, dup = (0, 0) if cfg == "c2" else (1200, 100)
    agents = [A.synth_agent_id(k) for k in range(na)]
    with A.Engine(slab_rows=nb * B + 1024, max_agents=512, max_batch=B, flags=MINT) as eng, CRef() as ref:
        for e in (eng, ref):
            for k, a in enumerate(agents):
                e.set_agent_state(a, "stopped" if k % 5 == 1 else "running")          # incl. the rank-1 hot agent
        hits = 0
        SUB = 1 << 15          # answered every 32 Ki requests: the C port keeps a list as an array, so removing the head of a long
                               # pending list is a memmove — long queues of RUNNING agents would make the checker quadratic
        for b in range(nb):
            big = A.synth_fill_host(b * B, B, seed=3, n_agents=na, zipf_milli=zipf, dup_permille=dup, mint=(eng, 0))
            big["request_id"] = eng.mint_ids(b * B, B)                                # the checker gets the ids the engine mints
            for c in range(0, B, SUB):
                recs = np.ascontiguousarray(big[c:c + SUB])
                v0, first = eng.ingest(recs)
                v1, _ = ref.ingest(recs)
                assert first == b * B + c
                assert (v0["code"] == v1["code"]).all() and ((v0["flags"] & 0x7) == (v1["flags"] & 0x7)).all(), (b, c)   # (KNOWN is the engine's own annotation)
                assert (v0["agent_slot"] == v1["agent_slot"]).all()
                hits += int(((v0["flags"] & K.AGR_VF_KNOWN) != 0).sum())
                fwd = np.nonzero((v0["code"] == K.AGR_V_FORWARD) & ((v0["flags"] & K.AGR_VF_TRACKED) != 0) & ((recs["flags"] & 1) == 0))[0]
                outs = np.zeros(len(fwd), dtype=A.outcome_dtype)
                outs["request_id"], outs["agent_id"] = recs["request_id"][fwd], recs["agent_id"][fwd]
                outs["kind"] = np.where(np.arange(len(fwd)) % 5003 == 3, K.AGR_OUT_ERROR, K.AGR_OUT_RESPONSE)
                outs["http_status"], outs["seq"] = 200, b * B + c + SUB
                assert (eng.complete(outs) == ref.complete(outs)).all(), (b, c)
        if dup:
            assert hits > nb * B // 20                                                 # the duplicates really resolved
        for e in (eng, ref):
            for k, a in enumerate(agents):
                if k % 5 == 1:
                    e.set_agent_state(a, "running")
        d0, _ = eng.replay_scan(with_records=False, cap=nb * B)
        d1, _ = ref.replay_scan()
        assert len(d0) == len(d1) > nb * B // 20
        assert (d0["agent_slot"] == d1["agent_slot"]).all() and d0["request_id"].tobytes() == d1["request_id"].tobytes()
        for a in agents[:4] + agents[100:102]:
            for w in (0, 1, 2):
                assert eng.list(a, w, cap=1 << 22).tobytes() == ref.list(a, w, cap=1 << 22).tobytes(), (a, w)
        s = eng.stats()
        assert s["ingested"] == nb * B
