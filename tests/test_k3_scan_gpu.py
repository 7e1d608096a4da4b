"""K3 (the replay tick agr_replay_scan / agr_replay_scan_var, agr_pending and agr_list) against the plain restatement in
tests/k3ref.py, at the shapes where select_locked / agr_launch_k3_select change code path:

  1. more than K3_SMEM_GROUPS = 512 registered agents: global-memory counters, k3_mark<false> / k3_place<false>;
  2. more than 1024 agents: k3_scan_total loops with a carry;
  3. exactly 512 agents: k3_place<true> at 32 KiB dynamic + 16 KiB static shared memory;
  4. the scalar row path of k3_mark (rings whose slab_rows % 4 != 0);
  5. warps that own more than 1024 rows (k3_place loops over several selection blocks);
  6. cap < total (AGR_ECAP with the true count);
  7. scan windows that start off a multiple of 4 (p.lo = lo & ~3, p.lo_real = lo).

Every dispatch entry (rid, agent slot, request id), every record agr_replay_scan gathers (byte for byte, with the live state
patched in) and every pending / list view of a sample of agents is compared with the restatement."""
import ctypes as C

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from k3ref import OUT_RESPONSE, OUT_ERROR
from k3rig import AGENT_NANOS0, Rig, layout

pytestmark = pytest.mark.gpu

AGENT_COUNTS = [1, 2, 31, 32, 33, 511, 512, 513, 1024, 1025, 4096]


@pytest.mark.parametrize("n_agents", AGENT_COUNTS)
def test_k3_agent_counts(n_agents):
    """Paths 1-3: <= 512 groups (shared-memory counters; at exactly 512 k3_place<true> sits at the 48 KiB launch limit),
    > 512 (k3_mark<false> / k3_place<false> with the matrix in global memory), > 1024 (k3_scan_total's carry loop).  Mint mode
    at every count, hash-id mode at 33, 513 and 1025; uniform, Zipf 1.2 and the two adversarial 32-row layouts; running and
    stopped agents, dropped agents and agents without rows."""
    modes = [K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS] + ([K.AGR_CFG_PERSISTENCE] if n_agents in (33, 513, 1025) else [])
    for flags in modes:
        for kind in ("uniform", "zipf", "same32", "distinct32"):
            rig = Rig(slab_rows=1 << 16, max_agents=max(n_agents, 64), flags=flags)
            try:
                rig.register(n_agents)
                rows = int(min(40_000, 6 * n_agents + 3000))
                slots = layout(kind, rows, n_agents, rig.rng)
                for a in range(0, rows, 9973):
                    rig.ingest(slots[a: a + 9973])
                if n_agents > 2:
                    for s in rig.rng.choice(n_agents, max(1, n_agents // 20), replace=False):
                        rig.drop(int(s))                          # slots are never reused
                rig.random_outcomes(0.3)
                assert rig.check() > 0 or n_agents <= 2
                rig.random_outcomes(0.3)
                rig.check()
            finally:
                rig.close()


def test_k3_window_shapes():
    """Path 7: windows [lo, hi) with hi - lo in {1, 3, 4, 5, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025} and lo at each
    residue mod 4, reached by completing a head prefix, ticking (the mark moves), ingesting more and ticking again; rows below
    the mark never come back and every pending row above it does.  Reserved-but-unfilled rows bound hi."""
    widths = [1, 3, 4, 5, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025]
    rig = Rig(slab_rows=1 << 17, max_agents=64)
    try:
        rig.register(40)
        for s in range(0, 40, 3):
            rig.set_status(s, K.AGR_AGENT_RUNNING)
        seen = set()
        for res in range(4):
            for w in widths:
                # move the mark to the top with lo % 4 == res: filler rows, completed at once
                pad = (res - rig.ref.n) % 4 + 4
                first = rig.ingest(layout("uniform", pad, 40, rig.rng))
                rig.complete(np.arange(first, first + pad), np.full(pad, OUT_RESPONSE), np.full(pad, 200))
                lo = rig.ref.n
                rig.check_tick()
                assert lo % 4 == res
                rig.ingest(layout("zipf", w, 40, rig.rng))
                n = rig.check_tick()
                assert n <= w
                # complete a head prefix: the mark moves to the first row still pending, at whatever residue
                k = max(1, w // 3)
                rig.complete(np.arange(lo, lo + k), np.full(k, OUT_RESPONSE), np.full(k, 200))
                rig.check_tick()
                seen.add((lo + k) % 4)
                for s in (0, 3, 7):
                    rig.check_agent(s)
                rig.random_outcomes(0.5)
                rig.check_tick()
                rest = np.flatnonzero(rig.ref.inq[lo: rig.ref.n]) + lo      # clear the window for the next shape
                rig.complete(rest, np.full(len(rest), OUT_RESPONSE), np.full(len(rest), 200))
        assert seen == {0, 1, 2, 3}
        # reserved rows that K1 has not filled bound every scan; rows ingested after them stay invisible until they are filled
        first_r = rig.eng.reserve_rows(37)
        rig.ref.reserve(first_r, 37)
        rig.ingest(layout("uniform", 100, 40, rig.rng))
        rig.check()
        recs = rig.records(layout("uniform", 37, 40, rig.rng))
        rig.eng.fill_rows(first_r, recs)
        rig.eng.ingest_rows(first_r, 37, want_verdicts=False)
        rig.ref.add_rows(first_r, [rig.names.index(a.decode()) for a in recs["agent_id"]],
                         rig.eng.mint_ids(first_r, 37))
        rig.keep_rows(first_r, recs)
        rig.check()
    finally:
        rig.close()


def ring_laps(R, n_laps, rig, patterns):
    """Fill the ring lap after lap with batches of the given sizes, complete / expire / reclaim, compare after every step."""
    mb = rig.eng.max_batch
    exact = padded = 0
    for lap in range(n_laps):
        sizes = [max(1, min(mb, s)) for s in patterns[lap % len(patterns)]]
        k = 0
        while True:
            b = sizes[k % len(sizes)]
            at = rig.ref.n % R
            pad = R - at if at + b > R else 0
            if rig.ref.n + pad + b - rig.ref.tail > R:
                break
            expect = rig.ref.n + pad                              # the engine skips the rows up to the end of the ring
            first = rig.ingest(layout("uniform", b, len(rig.names), rig.rng, rig.ref.n))
            assert first == expect
            padded += pad > 0
            exact += at + b == R
            k += 1
        rig.check()
        rig.random_outcomes(0.3)
        rig.check()
        # agr_expire: every record whose last write (= its own time here) is at or before the cutoff: the oldest 70 % of the window
        seqs = rig.recs["seq"][rig.ref.tail: rig.ref.n].astype(np.int64)
        live = seqs[seqs > 0]
        cut = int(live[int(len(live) * 0.7)])
        rows = np.flatnonzero((seqs > 0) & (seqs <= cut)) + rig.ref.tail
        assert rig.eng.expire(cut + 1, 1) == rig.ref.expire(rows)
        rig.check()
        assert rig.eng.reclaim() == rig.ref.reclaim()
        rig.check()
    return exact, padded


@pytest.mark.parametrize("R", [1001, 1002, 1003, 4097, 4099, 1004, 4100])
def test_k3_ring_not_multiple_of_4(R):
    """Path 4 (k3_mark's scalar row path: slab_rows % 4 != 0; 1004 and 4100 are the aligned controls) over several laps with
    expire and reclaim; laps end both exactly at the end of the ring and with the padding reserve_rows_locked inserts."""
    mb = R // 2                                                   # the most a ring takes in one batch
    rig = Rig(slab_rows=R, max_agents=64, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING, max_batch=mb)
    try:
        rig.register(24, p_running=0.7)
        with pytest.raises(A.AgrError):
            rig.eng.ingest(rig.records(np.zeros(mb + 1, np.int64)), want_verdicts=False)
        exact, padded = ring_laps(R, 6, rig, [[mb, mb, 1], [mb - 3, 7], [mb // 3 + 1], [mb, mb - 1, 2]])
        assert exact > 0 and padded > 0, "batches must end both exactly at the end of the ring and before padding"
    finally:
        rig.close()


def full_ring_1001(rig, ingest):
    """R = 1001: tail and scan mark at logical row 1002, then the ring full with 1001 pending rows of one running agent.  The
    window [1000, 2003) is one warp's run starting at physical row 1000; row 2002 must map to physical row 0."""
    R = 1001
    for b in (500, 500, 1):
        ingest(b)
    assert rig.ref.n == R
    rig.eng.expire(rig.seq + 1, 1); rig.ref.expire(np.arange(R))
    assert rig.eng.reclaim() == rig.ref.reclaim() == R
    ingest(1)
    rig.eng.expire(rig.seq + 1, 1); rig.ref.expire(np.arange(R, R + 1))
    assert rig.eng.reclaim() == rig.ref.reclaim() == 1
    assert rig.ref.tail == 1002
    for b in (500, 500, 1):
        ingest(b)
    assert rig.ref.n == 2003 and rig.ref.n - rig.ref.tail == R


def test_k3_full_ring_1001():
    """The newest row of a full ring whose size is not a multiple of 4, when one warp's run wraps twice."""
    rig = Rig(slab_rows=1001, max_agents=8, flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING)
    try:
        rig.register(1, p_running=1.0)
        full_ring_1001(rig, lambda b: rig.ingest(np.zeros(b, np.int64)))
        assert len(rig.ref.tick()[0]) == 1001
        assert rig.check() == 1001
        assert len(rig.eng.pending_json(rig.names[0])[0]) > 0 and rig.eng.pending_json(rig.names[0])[1] == 1001
    finally:
        rig.close()


def test_k3_full_ring_1001_varlen():
    """The same full ring through agr_replay_scan_var (AGR_CFG_VARLEN)."""
    from scenario import Req, make_var_batch
    rig = Rig(slab_rows=1001, max_agents=8, keep_records=False, vslab_bytes=1001 * 512,
              flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING | K.AGR_CFG_VARLEN)
    try:
        rig.register(1, p_running=1.0)
        name = rig.names[0]

        def ingest(b):
            reqs = [Req(name, bytes(16), rig.seq + 1 + i, body=b'{"m":%d}' % (rig.seq + i)) for i in range(b)]
            rig.seq += b
            blob, offs = make_var_batch(reqs)
            _, ids, first = rig.eng.ingest_var(blob, offs)
            rig.ref.add_rows(first, np.zeros(b, np.int64), ids)
        full_ring_1001(rig, ingest)
        disp, _, _ = rig.eng.replay_scan_var()
        rows, slots = rig.ref.tick()
        assert len(disp) == len(rows) == 1001
        assert np.array_equal(disp["rid"].astype(np.int64), rows) and np.array_equal(disp["request_id"], rig.ref.ids[rows])
    finally:
        rig.close()


def _call(fn, *args):
    n = C.c_uint32()
    rc = fn(*args, C.byref(n))
    return rc, int(n.value)


def test_k3_capacities():
    """Path 6: agr_replay_scan, agr_pending and agr_list called with cap = total - 1, total, total + 1.  On AGR_ECAP *n is the
    true total; the next call with room returns the same list; replay_dispatched counts only the calls that succeeded."""
    rig = Rig(slab_rows=1 << 15, max_agents=1100)
    try:
        rig.register(600, p_running=0.8)
        rig.ingest(layout("uniform", 20_000, 600, rig.rng))
        rig.random_outcomes(0.4)
        lib, h = rig.eng.lib, rig.eng.h
        rows, slots = rig.ref.tick()
        total = len(rows)
        before = rig.eng.stats()["replay_dispatched"]
        ok = 0
        for cap in (total - 1, total, total + 1):
            disp = np.zeros(cap, dtype=A.dispatch_dtype)
            rc, n = _call(lib.agr_replay_scan, h, disp.ctypes.data, None, cap)
            assert n == total
            if cap < total:
                assert rc == K.AGR_ECAP
            else:
                assert rc == 0 and np.array_equal(disp["rid"][:n].astype(np.int64), rows)
                assert np.array_equal(disp["request_id"][:n], rig.ref.ids[rows])
                ok += 1
        assert rig.eng.stats()["replay_dispatched"] - before == ok * total
        s = int(np.bincount(rig.ref.slot[rig.ref.tail: rig.ref.n][rig.ref.slot[rig.ref.tail: rig.ref.n] >= 0]).argmax())
        p3 = rig.ref.pending(s)[:5]
        rig.complete(np.repeat(p3, 3), np.full(15, OUT_ERROR))                 # three failures each: the failed list
        rig.complete(rig.ref.pending(s)[:4], np.full(4, OUT_RESPONSE), np.full(4, 200))
        name = rig.names[s].encode()
        prow = rig.ref.pending(s)
        for cap in (len(prow) - 1, len(prow), len(prow) + 1):
            out = np.zeros(max(cap, 1), dtype=A.record_dtype)
            rc, n = _call(lib.agr_pending, h, name, out.ctypes.data, cap)
            assert n == len(prow) and (rc == K.AGR_ECAP) == (cap < len(prow))
            if rc == 0:
                assert np.array_equal(out["request_id"][:n], rig.ref.ids[prow])
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            lrows = rig.ref.list(s, which)
            assert len(lrows) > 1
            for cap in (len(lrows) - 1, len(lrows), len(lrows) + 1):
                ids = np.zeros((cap, 16), dtype=np.uint8)
                rc, n = _call(lib.agr_list, h, name, which, ids.ctypes.data, cap)
                assert n == len(lrows) and (rc == K.AGR_ECAP) == (cap < len(lrows))
                if rc == 0:
                    assert np.array_equal(ids[:n], rig.ref.ids[lrows])
    finally:
        rig.close()


def cref_matches(cref, ref, names):
    """The C port's tick, pending and lists against the restatement (agent slot = registration index in both)."""
    disp, recs = cref.replay_scan(with_records=True)
    rows, slots = ref.tick()
    assert len(disp) == len(rows), f"C port dispatched {len(disp)} rows, the reference {len(rows)}"
    assert np.array_equal(disp["agent_slot"].astype(np.int64), slots)
    assert np.array_equal(disp["request_id"], ref.ids[rows])
    assert np.array_equal(recs["retry_count"], ref.header_fields(rows)["retry_count"])
    for s, name in enumerate(names):
        prow = ref.pending(s)
        got = cref.pending(name)
        assert np.array_equal(got["request_id"], ref.ids[prow]) and np.array_equal(got["retry_count"], ref.retry[prow]), name
        for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
            assert np.array_equal(cref.list(name, which), ref.ids[ref.list(s, which)]), f"{name} list {which}"
    return len(rows)


def test_k3_c_restatement_600_agents():
    """Past 512 agents (path 1) the engine, the restatement and the C port of the reference (oracle/cpu_ref.c) side by side:
    100 k rows over 600 agents (Zipf), running, stopped and dropped agents, two rounds of outcomes; the tick, agr_pending and
    the three lists of EVERY agent compared in both pairs.  Hash-id mode: the C port stores the caller's ids."""
    from oracle.cpu_ref import CRef
    rig = Rig(slab_rows=1 << 17, max_agents=1024, flags=K.AGR_CFG_PERSISTENCE)
    cref = CRef()
    try:
        rig.register(600, p_running=0.6)
        for s, name in enumerate(rig.names):
            cref.set_agent_state(name, rig.ref.agent_status[s])
        slots = layout("zipf", 100_000, 600, rig.rng)
        for a in range(0, len(slots), 10_000):
            first = rig.ingest(slots[a: a + 10_000])
            cref.ingest(np.ascontiguousarray(rig.recs[first: rig.ref.n]))
        for s in rig.rng.choice(600, 12, replace=False).tolist():
            rig.drop(s)
            cref.drop_agent(rig.names[s])
        for _ in range(2):
            outs = rig.random_outcomes(0.3)
            cref.complete(outs)
            n = rig.check_tick()
            assert n > 10_000 and cref_matches(cref, rig.ref, rig.names) == n
            for s in range(600):
                rig.check_agent(s, with_records=s % 50 == 0)
    finally:
        cref.close()
        rig.close()


def test_k3_log_mode_large():
    """K3_LOG_AGENT: completed and failed lists of more than 1 Mi entries for one hot agent among 1025, with Q7 duplicates (ids
    completed twice); the per-agent order is the call order."""
    n_hot = (1 << 20) + 5000
    rig = Rig(slab_rows=2 * n_hot + 8192, max_agents=1100, keep_records=False)
    try:
        rig.register(1025, p_running=0.5)
        hot = 700
        rows_all = []
        for a in range(0, 2 * n_hot + 6000, 1 << 19):
            b = min(1 << 19, 2 * n_hot + 6000 - a)
            slots = np.where(rig.rng.random(b) < 0.997, hot, rig.rng.integers(0, 1025, b))
            rows_all.append(np.arange(rig.ingest(slots), rig.ref.n))
        rows_all = np.concatenate(rows_all)
        rig.rng.shuffle(rows_all)
        half = len(rows_all) // 2
        done, fail = rows_all[:half], rows_all[half:]
        dup = done[rig.rng.random(len(done)) < 0.05]
        seq = np.concatenate([done, dup, fail, fail, fail])
        kinds = np.concatenate([np.full(len(done) + len(dup), OUT_RESPONSE), np.full(3 * len(fail), OUT_ERROR)])
        rig.complete(seq, kinds, np.full(len(seq), 200), chunk=1 << 19)
        for s in (hot, 0, 1024, 512):
            for which in (K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
                ids = rig.eng.list(rig.names[s], which)
                lrows = rig.ref.list(s, which)
                if s == hot:
                    assert len(lrows) > (1 << 20)
                assert len(ids) == len(lrows) and np.array_equal(ids, rig.ref.ids[lrows])
        rig.check_tick(with_records=False)
    finally:
        rig.close()


def _splitmix(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def synth_agents(seed, first_index, n, n_agents):
    """Agent index of synthetic records [first_index, +n) (agr_synth.h, uniform choice, no duplicates)."""
    i = np.arange(first_index, first_index + n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        u = _splitmix(np.uint64(seed) ^ _splitmix(i * np.uint64(64) + np.uint64(1)))
    return (u % np.uint64(n_agents)).astype(np.int64)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def synth_rig(n_rows, n_agents, seed):
    rig = Rig(slab_rows=n_rows + 4096, max_agents=n_agents, keep_records=False)
    try:
        rig.register(n_agents, p_running=0.5)
        # the synthetic stream names agent k "agent-<nanos0 + k * 1000003>": the rig registered them in that order
        assert A.synth_agent_id(n_agents - 1, agent_nanos0=AGENT_NANOS0) == rig.names[-1]
        host = A.synth_fill_host(0, 2000, seed=seed, n_agents=n_agents, agent_nanos0=AGENT_NANOS0)
        assert [rig.names.index(a.decode()) for a in host["agent_id"]] == synth_agents(seed, 0, 2000, n_agents).tolist()
        first = rig.eng.reserve_rows(n_rows)
        rig.eng.synth_fill_rows(0, first, n_rows, seed=seed, n_agents=n_agents, agent_nanos0=AGENT_NANOS0)
        for a in range(0, n_rows, rig.eng.max_batch):
            rig.eng.ingest_rows(first + a, min(rig.eng.max_batch, n_rows - a), want_verdicts=False)
        rig.ref.add_rows(first, synth_agents(seed, 0, n_rows, n_agents), rig.eng.mint_ids(first, n_rows))
    except BaseException:
        rig.close()
        raise
    return rig


def _check_big(rig, sample):
    rig.check_tick(with_records=False)
    for s in sample:
        rig.check_agent(s, with_records=False)


def test_k3_many_agents_per_warp_over_1024():
    """Path 5: 4096 agents x 2 Mi rows: max_warps = 4 Mi / 4096 binds, so a warp owns 2048 rows and k3_place runs two
    1024-item selection blocks per warp (and paths 1 and 2 at that size)."""
    rig = synth_rig(2 << 20, 4096, seed=11)
    try:
        k = rig.ref.n
        rig.complete(np.arange(0, k, 97), np.full(len(range(0, k, 97)), OUT_RESPONSE), np.full(len(range(0, k, 97)), 200))
        _check_big(rig, [0, 1, 2047, 4095])
    finally:
        rig.close()


def test_k3_window_beyond_grid():
    """Path 5 the other way: an append-only window of more than sm_count * 128 * 1024 rows (the warp count is capped at
    sm_count * 128), 256 agents."""
    n = sm_count() * 128 * 1024 + 4099
    rig = synth_rig(n, 256, seed=12)
    try:
        _check_big(rig, [0, 255])
    finally:
        rig.close()
