"""The kernels that decide which records the engine keeps — the TTL sweep (k_expire), the release of the ring's tail
(k_first_live, k_release_rows), the compaction of the completed / failed logs (k_log_count / k_log_scan / k_log_scatter) and
the tail of the response byte ring (k_bytes_span) — against the plain restatement in tests/k3ref.py (its sweep is checked
against oracle/model.py's clock by tests/test_k3_ref.py), over many 4096-row chunks.

After every engine call the test compares the expired and released counts, the STORED bit and the last-SET time of every row
of the live window, the replay tick and every agent's pending, completed and failed lists.  It also reads every chunk's time
bound (AGR_DBG_CMIN) and checks the invariant the sweep and k_first_live skip chunks on: the bound is 0 ("unknown") or at most
the earliest last-SET time of the chunk's stored rows, and ~0 ("no stored row") only when the chunk holds none.  Right after
agr_expire, every chunk the sweep had to visit (bound 0 or due, or reset by the host for append-only and variable-length
engines) holds the exact minimum.

One documented exception to the reference: a SET at time 0 counts as a SET at 1 ns (0 is "never SET" in the engine's mtime and
"unknown" in a bound), so the reference is given max(t, 1) for every time."""
import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from k3ref import OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR
from k3rig import Rig

pytestmark = pytest.mark.gpu

CH = 4096                        # AGR_CHUNK_ROWS
U64 = (1 << 64) - 1
ST_STORED = 0x20
TTL = 1_000_000
T0 = 10 ** 15
RING = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING
R_ODD = 5 * CH + 1234


def eff(t):
    """The engine's time of a SET: time 0 counts as 1 ns."""
    return np.maximum(np.asarray(t, dtype=np.uint64), np.uint64(1))


class TtlRig(Rig):
    def __init__(self, R, flags, **kw):
        kw.setdefault("max_batch", R // 2 if flags & K.AGR_CFG_RING else 0)
        super().__init__(slab_rows=R, max_agents=64, flags=flags, **kw)
        self.R = R
        self.flags = flags
        self.kw = dict(slab_rows=R, max_agents=64, flags=flags, **kw)
        self.ring = bool(flags & K.AGR_CFG_RING)
        self.host_bounds = not self.ring or bool(flags & K.AGR_CFG_VARLEN)   # agr_expire resets the bounds of new rows
        self.sweep_clean = 0
        self.lag = None                                  # agr_reclaim_async: what the previous call's scan found
        self.visits = self.exact = 0

    # ---- what the test does (engine and reference side by side)
    def phys(self, rows):
        rows = np.asarray(rows, dtype=np.int64)
        return rows % self.R if self.ring else rows

    def fits(self, b):
        if not self.ring:
            return self.ref.n + b <= self.R
        at = self.ref.n % self.R
        pad = self.R - at if at + b > self.R else 0
        return self.ref.n + pad + b - self.ref.tail <= self.R

    def ingest_t(self, slots, times, single=False):
        slots = np.asarray(slots, dtype=np.int64)
        recs = self.records(slots)
        recs["seq"] = np.asarray(times, dtype=np.uint64)
        if single:                                       # AGR_CFG_COMBINE: one record through the single-request ring
            out, ids = np.zeros(1, dtype=A.verdict_dtype), np.zeros((1, 16), dtype=np.uint8)
            first = self.eng.ingest_ex(recs, out, ids)
            if not self.mint:
                ids = recs["request_id"]
        else:
            _, first = self.eng.ingest(recs, want_verdicts=False)
            ids = self.eng.mint_ids(first, len(recs)) if self.mint else recs["request_id"]
        self.ref.add_rows(first, slots, ids, created=eff(times))
        self.keep_rows(first, recs)
        return first

    def outcomes(self, rows, kinds, times):
        outs = np.zeros(len(rows), dtype=A.outcome_dtype)
        outs["request_id"] = self.ref.ids[rows]
        nm = np.array([s.encode() for s in self.names], dtype="S32")
        outs["agent_id"] = nm[np.maximum(self.ref.slot[rows], 0)]
        outs["kind"], outs["http_status"], outs["seq"] = kinds, 200, np.asarray(times, dtype=np.uint64)
        return outs

    def complete_t(self, rows, kinds, times, tickets=0.0):
        rows = np.asarray(rows, dtype=np.int64)
        outs = self.outcomes(rows, kinds, times)
        single = self.rng.random(len(rows)) < tickets
        a = 0
        while a < len(rows):                             # call order kept: runs of batch outcomes, single tickets between
            if single[a]:
                self.eng.wait(self.eng.submit_complete(outs[a]))
                a += 1
                continue
            b = a
            while b < len(rows) and not single[b] and b - a < self.eng.max_batch:
                b += 1
            self.eng.complete(np.ascontiguousarray(outs[a:b]), want_results=False)
            a = b
        self.ref.complete(rows, kinds, np.full(len(rows), 200), times=eff(times))

    def cmin(self):
        return self.eng.debug_read("cmin", 0, (self.R + CH - 1) // CH)

    def chunk_min(self):
        """Per physical chunk: the earliest last-SET time of its stored rows (~0 - 1 for time ~0), ~0 if it holds none."""
        lo = self.ref.tail
        rows = np.flatnonzero(self.ref.stored[lo: self.ref.n]) + lo
        m = np.full((self.R + CH - 1) // CH, U64, dtype=np.uint64)
        np.minimum.at(m, self.phys(rows) // CH, np.minimum(self.ref.mtime[rows], np.uint64(U64 - 1)))
        return m

    def check_bounds(self, exact=None):
        b, m = self.cmin(), self.chunk_min()
        if self.host_bounds:                             # rows since the last sweep: their chunks are reset by the next one
            lo, hi = max(self.sweep_clean, self.ref.tail), self.ref.n
            if hi > lo:
                new = np.zeros(len(b), dtype=bool)
                new[np.unique(self.phys(np.arange(lo, hi)) // CH)] = True
                if self.ring and hi - lo >= self.R:
                    new[:] = True
                b = np.where(new, np.uint64(0), b)
        bad = np.flatnonzero((b != 0) & (b > m))
        assert len(bad) == 0, f"chunk {bad[0]}: bound {b[bad[0]]} above the earliest stored time {m[bad[0]]}"
        bad = np.flatnonzero((b == np.uint64(U64)) & (m != np.uint64(U64)))
        assert len(bad) == 0, f"chunk {bad[0]}: bound says 'no stored row' but it holds one at time {m[bad[0]]}"
        if exact is not None:
            bad = np.flatnonzero(exact & (b != m))
            assert len(bad) == 0, f"chunk {bad[0]} was swept: bound {b[bad[0]]}, exact minimum {m[bad[0]]}"
            self.visits += int(exact.sum())
            self.exact += int((exact & (m != np.uint64(U64))).sum())

    def check_rows(self, with_records=True, lists=True):
        lo, hi = self.ref.tail, self.ref.n
        assert self.eng.stats()["rows_tail"] == lo
        if hi > lo:
            st = (self.eng.debug_read("state", lo, hi - lo) & ST_STORED) != 0
            bad = np.flatnonzero(st != self.ref.stored[lo:hi])
            assert len(bad) == 0, f"row {lo + bad[0]}: STORED {st[bad[0]]}, reference {self.ref.stored[lo + bad[0]]}"
            mt = self.eng.debug_read("mtime", lo, hi - lo)
            t = eff(np.where(mt == 0, self.recs["seq"][lo:hi], mt))          # 0: the sweep takes created_at
            s = self.ref.stored[lo:hi]
            bad = np.flatnonzero(s & (t != self.ref.mtime[lo:hi]))
            assert len(bad) == 0, f"row {lo + bad[0]}: last-SET time {t[bad[0]]}, reference {self.ref.mtime[lo + bad[0]]}"
        if lists:
            self.check_tick(with_records=with_records)
            for s in range(len(self.names)):
                self.check_agent(s, with_records=with_records)

    def check_all(self, exact=None, **kw):
        self.check_bounds(exact)
        self.check_rows(**kw)

    def expire(self, now, ttl=TTL, want_count=True, **kw):
        b = self.cmin()
        n_ch = (min(self.ref.n, self.R) + CH - 1) // CH                    # the chunks the sweep's grid covers
        nu = np.uint64(now)
        visit = (b != np.uint64(U64)) & ((b == 0) | ((nu >= b) & (nu - b >= np.uint64(ttl))))
        if self.host_bounds:
            lo, hi = max(self.sweep_clean, self.ref.tail), self.ref.n
            if self.ring and hi - lo >= self.R:
                visit[:] = True
            elif hi > lo:
                visit[np.unique(self.phys(np.arange(lo, hi)) // CH)] = True
            self.sweep_clean = self.ref.bound()
        visit[n_ch:] = False
        got = self.eng.expire(now, ttl, want_count=want_count)
        exp = self.ref.sweep(now, ttl)
        if want_count:
            assert got == exp, f"agr_expire({now}, {ttl}) dropped {got} records, the reference {exp}"
        self.check_all(visit, **kw)
        return exp

    def dead_prefix(self):
        hi = self.ref.bound()
        live = np.flatnonzero(self.ref.stored[self.ref.tail: hi])
        return int(live[0]) if len(live) else hi - self.ref.tail

    def reclaim(self, use_async=False, **kw):
        if use_async:
            got = self.eng.reclaim_async()
            exp = self.ref.reclaim(self.lag) if self.lag is not None else 0
            self.lag = self.dead_prefix()
        else:
            got, exp = self.eng.reclaim(), self.ref.reclaim()
        assert got == exp, f"released {got} rows, the reference {exp}"
        self.check_all(**kw)
        return got

    def restart(self, path):
        self.eng.snapshot(path)
        self.eng.close()
        self.eng = A.Engine(restore_from=path, **self.kw)
        self.sweep_clean = 0
        self.lag = None                                  # the scan in flight went with the old handle
        assert (self.cmin() == 0).all(), "after a restore every bound is 'unknown'"
        self.check_all()


def now_at(rig, lo_q=0.2, hi_q=0.6):
    """A sweep time at exactly t + ttl, or 1 ns before it, for the last-SET time t of a stored row in the older part."""
    lo = rig.ref.tail
    rows = np.flatnonzero(rig.ref.stored[lo: rig.ref.n]) + lo
    if not len(rows):
        return None
    ts = np.sort(rig.ref.mtime[rows])
    t = int(ts[int(len(ts) * rig.rng.uniform(lo_q, hi_q))])
    return min(U64, t + TTL - int(rig.rng.integers(0, 2)))


def batch_times(rig, b, T, special=True):
    """created_at of a batch: rising from T, with one old record, one far in the future, time 0 or time ~0 among them."""
    t = T + np.arange(b, dtype=np.uint64) * np.uint64(3)
    if special and b > 4:
        r = rig.rng.random()
        i = int(rig.rng.integers(0, b))
        if r < 0.3:
            t[i] = T - 2 * TTL                                        # one old record in a chunk of new ones
        elif r < 0.45:
            t[i] = T + 4 * TTL
        elif r < 0.6:
            t[i] = 0
        elif r < 0.75:
            t[i] = U64
    return t


SIZES = [1237, 77, 3001, 509, 2053, 33, 1, 4099]


def drive_ring(rig, steps, *, tickets=0.0, single=0.0, use_async=False, want_count=True, restart_at=None, tmp_path=None):
    """Step after step: fill the ring up to about its size in odd-sized batches (their first rows are not multiples of 32, so K1
    tiles straddle chunk boundaries), answer part of the window with outcomes older and newer than the chunk bounds, sweep at
    t + ttl / t + ttl - 1 of a stored row (sometimes with the clock behind everything), release the tail."""
    T = T0
    k = 0
    forever = []
    for step in range(steps):
        T += TTL // 3
        added = 0
        while added < rig.R // 3:
            b = min(SIZES[k % len(SIZES)], rig.eng.max_batch)
            if not rig.fits(b):
                break
            k += 1
            t = batch_times(rig, b, T)
            if single and rig.rng.random() < single:
                for j in range(min(b, 5)):
                    if not rig.fits(1):
                        break
                    rig.ingest_t(rig.rng.integers(0, len(rig.names), 1), t[j: j + 1], single=True)
                b = min(b, 5)
            else:
                rig.ingest_t(rig.rng.integers(0, len(rig.names), b), t)
            added += b
        lo = rig.ref.tail
        live = np.flatnonzero(rig.ref.stored[lo: rig.ref.n]) + lo
        forever += live[rig.ref.mtime[live] == np.uint64(U64)].tolist()
        rig.check_all(with_records=step % 3 == 0)
        if len(live):
            pick = live[rig.rng.random(len(live)) < 0.3]
            pick = np.concatenate([pick, pick[: len(pick) // 8]])
            rig.rng.shuffle(pick)
            kinds = rig.rng.choice([OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR], size=len(pick), p=[0.5, 0.4, 0.1])
            c = rig.rng.random(len(pick))
            times = np.where(c < 0.3, T - TTL - rig.rng.integers(0, TTL, len(pick)),   # older than the bound: K2 lowers it
                             T + rig.rng.integers(0, TTL // 2, len(pick))).astype(np.uint64)   # newer: the TTL restarts
            times[c > 0.97] = 0
            times[(c > 0.95) & (c <= 0.97)] = U64
            rig.complete_t(pick, kinds, times, tickets=tickets)
            forever += pick[times == np.uint64(U64)].tolist()
            rig.check_all(with_records=False)
        # records and outcomes at ~0 never expire: answer them (the ring would stay blocked behind them)
        stuck = [r for r in set(forever) if r >= rig.ref.tail and rig.ref.stored[r] and rig.ref.mtime[r] == np.uint64(U64)]
        if stuck and step % 2 == 1:
            rig.complete_t(np.array(stuck), np.full(len(stuck), OUT_RESPONSE), np.full(len(stuck), T), tickets=tickets)
            forever = []
        if restart_at is not None and step == restart_at:
            rig.restart(str(tmp_path / "ttl.snap"))
        c = rig.rng.random()
        now = now_at(rig) if c < 0.75 else T - 3 * TTL if c < 0.85 else T + 2 * TTL
        if now is not None:
            rig.expire(now, want_count=want_count, with_records=False)
        if rig.ring:
            rig.reclaim(use_async=use_async, with_records=False)
    assert rig.visits > 0 and rig.exact > 0


def _rig(R, flags, names=12, **kw):
    rig = TtlRig(R, flags, **kw)
    rig.register(names, p_running=0.6)
    return rig


@pytest.mark.parametrize("R", [R_ODD, 8 * CH])
def test_ttl_ring_minted(R):
    """Fixed-stride ring, minted ids, TMA K1: 24 steps over 6 chunks (the last one partial when R = 5 * 4096 + 1234)."""
    rig = _rig(R, RING)
    try:
        drive_ring(rig, 24)
    finally:
        rig.close()


def test_ttl_ring_caller_ids():
    """Fixed-stride ring with the caller's ids: the dedupe index is rebuilt after every release."""
    rig = _rig(R_ODD, K.AGR_CFG_PERSISTENCE | K.AGR_CFG_RING)
    try:
        drive_ring(rig, 18)
    finally:
        rig.close()


def test_ttl_ring_tickets():
    """AGR_CFG_COMBINE: part of the records and outcomes go through the single-request ring (the service kernel's TTL
    bookkeeping), the rest through K1 / K2 batches."""
    rig = _rig(R_ODD, RING | K.AGR_CFG_COMBINE)
    try:
        drive_ring(rig, 12, tickets=0.05, single=0.3)
    finally:
        rig.close()


def test_ttl_ring_async_and_restore(tmp_path):
    """agr_expire without a count (asynchronous) and agr_reclaim_async one step behind; a snapshot and restore in the middle
    of the run (every bound becomes 'unknown' and the next sweep recomputes them)."""
    rig = _rig(R_ODD, RING)
    try:
        drive_ring(rig, 20, use_async=True, want_count=False, restart_at=9, tmp_path=tmp_path)
    finally:
        rig.close()


@pytest.mark.parametrize("flags", [K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS, K.AGR_CFG_PERSISTENCE])
def test_ttl_append_only(flags):
    """Append-only slab (minted and caller ids): K1 keeps no bounds, agr_expire resets the chunks filled since its last call.
    Sweeps are interleaved with ingests that land in a partly filled chunk, and a chunk emptied by one sweep (bound ~0) gets
    new rows before the next."""
    rig = _rig(9 * CH + 77, flags)
    try:
        T = T0
        for step in range(16):
            T += TTL // 3
            for b in (1237, 2053, 509):
                if rig.fits(b):
                    rig.ingest_t(rig.rng.integers(0, len(rig.names), b), batch_times(rig, b, T))
            rig.check_all(with_records=step % 4 == 0)
            lo = rig.ref.tail
            live = np.flatnonzero(rig.ref.stored[lo: rig.ref.n]) + lo
            pick = live[rig.rng.random(len(live)) < 0.25]
            times = np.where(rig.rng.random(len(pick)) < 0.3, T - TTL, T + 7).astype(np.uint64)
            rig.complete_t(pick, rig.rng.choice([OUT_RESPONSE, OUT_ERROR], size=len(pick)), times)
            now = now_at(rig, 0.3, 0.9) if step % 3 else T - 5 * TTL
            if now is not None:
                rig.expire(now, with_records=False)
        assert rig.exact > 0
    finally:
        rig.close()


def test_ttl_append_only_outcome_at_time_zero():
    """An outcome at time 0 on a record created later restarts the record's TTL at 0 (model.py: the key expires at 0 + ttl), not
    at created_at.  The engine counts the SET as one at 1 ns: the record is still there at exactly ttl and gone 1 ns later."""
    for flags in (K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS, RING):
        rig = _rig(2 * CH, flags, names=1)
        try:
            rig.set_status(0, K.AGR_AGENT_RUNNING)
            first = rig.ingest_t([0, 0], [5 * TTL, 5 * TTL])
            rig.complete_t(np.array([first]), [OUT_ERROR], [0])
            assert rig.expire(TTL) == 0                                # the documented 1 ns exception (the model drops it here)
            assert rig.expire(TTL + 1) == 1
            assert rig.ref.stored[first + 1] and not rig.ref.stored[first]
        finally:
            rig.close()


def test_ttl_max_time_is_not_no_stored_row():
    """A record created at UINT64_MAX, alone in its chunk once the rest of the chunk has expired, stays stored: the sweep's
    bound for it is ~0 - 1, not the "no stored row" value ~0, so k_first_live does not skip the chunk and agr_reclaim does not
    release it (or, with every other chunk empty too, the whole live window).  The same for an outcome at UINT64_MAX."""
    rig = _rig(3 * CH, RING, names=2)
    try:
        T = T0
        first = rig.ingest_t(np.zeros(CH, np.int64), batch_times(rig, CH, T, special=False))
        rig.ingest_t(np.zeros(CH, np.int64), batch_times(rig, CH, T + 10 * TTL, special=False))
        rig.complete_t(np.array([first + 100]), [OUT_ERROR], [U64])           # an outcome at ~0 in chunk 0
        rig.ingest_t(np.zeros(100, np.int64), np.full(100, U64, np.uint64))    # records at ~0 at the start of chunk 2
        rig.ingest_t(np.zeros(50, np.int64), batch_times(rig, 50, T, special=False))
        rig.check_all()
        rig.expire(T + 5 * TTL)                                               # chunk 0: only row 100 is left
        assert rig.reclaim() == 100
        rig.expire(T + 20 * TTL)                                              # everything but the ~0 rows
        assert rig.reclaim() == 0
        rig.complete_t(np.array([first + 100]), [OUT_RESPONSE], [T + 30 * TTL])
        rig.expire(T + 31 * TTL)
        assert rig.reclaim() == 2 * CH - 100
        assert int(rig.ref.stored[rig.ref.tail: rig.ref.n].sum()) == 100
        rig.complete_t(np.arange(2 * CH, 2 * CH + 100), np.full(100, OUT_RESPONSE), np.full(100, T))
        rig.expire(T + 2 * TTL)
        assert rig.reclaim() == 150
    finally:
        rig.close()


def test_ttl_varlen_ring():
    """Variable-length ring: K1 keeps no bounds, agr_expire resets the chunks filled since the last sweep; one gap of a ring's
    worth of rows between two sweeps takes the whole-ring reset."""
    from scenario import Req, make_var_batch
    R = 3 * CH + 999
    rig = _rig(R, RING | K.AGR_CFG_VARLEN, names=6, keep_records=False, vslab_bytes=R * 256)
    rig.recs = np.zeros(8 * R, dtype=A.record_dtype)                         # created_at by logical row
    try:
        T = T0

        def ingest(b, T):
            slots = rig.rng.integers(0, len(rig.names), b)
            t = batch_times(rig, b, T)
            reqs = [Req(rig.names[s], bytes(16), int(x), body=b'{"m":%d}' % i) for i, (s, x) in enumerate(zip(slots, t))]
            blob, offs = make_var_batch(reqs)
            _, ids, first = rig.eng.ingest_var(blob, offs)
            rig.ref.add_rows(first, slots, ids, created=eff(t))
            rig.recs["seq"][first: first + b] = t

        def lists():
            for s in range(len(rig.names)):
                for which in (K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED, K.AGR_LIST_PENDING):
                    assert np.array_equal(rig.eng.list(rig.names[s], which), rig.ref.ids[rig.ref.list(s, which)])
        for step in range(10):
            T += TTL // 3
            if step == 6:                                  # a ring's worth of rows between two sweeps: the whole-ring reset
                rig.expire(T + 100 * TTL, lists=False)
                rig.reclaim(lists=False)
                assert rig.ref.tail == rig.ref.n
                left = R                                   # exactly R rows, no padding: batches end at the end of the ring
                while left:
                    b = min(rig.eng.max_batch, left, R - rig.ref.n % R)
                    ingest(b, T)
                    left -= b
                assert rig.ref.n - rig.sweep_clean >= R
            for b in (1237, 509, 2053):
                if rig.fits(b):
                    ingest(b, T)
            lo = rig.ref.tail
            live = np.flatnonzero(rig.ref.stored[lo: rig.ref.n]) + lo
            pick = live[rig.rng.random(len(live)) < 0.3]
            rig.complete_t(pick, rig.rng.choice([OUT_RESPONSE, OUT_ERROR], size=len(pick)),
                           np.where(rig.rng.random(len(pick)) < 0.3, T - TTL, T + 5).astype(np.uint64))
            now = now_at(rig)
            if now is not None:
                rig.expire(now, lists=False)
            rig.reclaim(lists=False)
            lists()
        assert rig.exact > 0
    finally:
        rig.close()


def _ingest_plain(rig, b, t):
    slots = rig.rng.integers(0, len(rig.names), b)
    recs = rig.records(slots)
    recs["seq"] = t
    _, first = rig.eng.ingest(recs, want_verdicts=False)
    rig.ref.add_rows(first, slots, rig.eng.mint_ids(first, b), created=t)
    rig.recs["seq"][first: first + b] = t
    return np.arange(first, first + b)


def test_log_compaction_over_a_million_entries():
    """A ring whose completed log holds more than 1024 * 1024 entries (k_log_scan's carry loop), not a multiple of 1024 long:
    every row completed twice (a replay completes twice, Q7), agr_drop_agent tombstones in both logs, releases that end past
    the physical wrap; every agent's lists against the reference after every release."""
    R = 600_011
    rig = _rig(R, RING, names=9, keep_records=False)
    rig.recs = np.zeros(2 * R, dtype=A.record_dtype)
    try:
        T = T0
        rows = np.concatenate([_ingest_plain(rig, b, np.full(b, T, np.uint64)) for b in (R // 2, R // 2 - 40_000)])
        n = len(rows)
        rig.complete_t(np.concatenate([rows, rows[rig.rng.permutation(n)]]), np.full(2 * n, OUT_RESPONSE), np.full(2 * n, T + 10))
        f = rows[rig.rng.random(n) < 0.05]
        rig.complete_t(np.repeat(f, 3), np.full(3 * len(f), OUT_ERROR), np.full(3 * len(f), T + 10))
        assert len(rig.ref.logs[0]) > (1 << 20) and len(rig.ref.logs[0]) % 1024 != 0 and len(rig.ref.logs[1]) > 0
        rig.drop(3)                                        # tombstones (AGR_RID_NONE) in both logs
        newer = rows[int(n * 0.4):]                        # re-SET: the older 40 % of the window expires, the rest stays
        newer = newer[rig.ref.slot[newer] != 3]            # (a dropped agent's outcomes change nothing)
        rig.complete_t(newer, np.full(len(newer), OUT_RESPONSE), np.full(len(newer), T + 5 * TTL))
        rig.expire(T + 10 + TTL, with_records=False)
        assert rig.reclaim(with_records=False) >= int(n * 0.4)
        # across the physical wrap: rows up to the end of the ring, then a batch that starts at physical row 0
        _ingest_plain(rig, 40_000, np.full(40_000, T + 6 * TTL, np.uint64))
        pad = R - rig.ref.n
        b = _ingest_plain(rig, 200_000, np.full(200_000, T + 7 * TTL, np.uint64))
        assert b[0] == R and pad > 0
        rig.complete_t(b[::3], np.full(len(b[::3]), OUT_RESPONSE), np.full(len(b[::3]), T + 7 * TTL))
        rig.expire(T + 6 * TTL, with_records=False)
        rig.reclaim(with_records=False)
        assert rig.ref.tail == n
        rig.expire(T + 7 * TTL, with_records=False)
        assert rig.reclaim(with_records=False) == 40_000 + pad and rig.ref.tail == R
        rig.expire(T + 8 * TTL, with_records=False)
        assert rig.reclaim(with_records=False) == 200_000 and rig.ref.tail == R + 200_000
    finally:
        rig.close()


def test_response_byte_ring_exactly_full():
    """The response byte ring filled so that the oldest live blob starts exactly at the head (k_bytes_span: a distance of 0 is
    the whole ring), then the rows before it released: nothing more fits until that blob's rows go, then exactly the space
    they held; once with a batch region that skipped the end of the ring.  Every live blob reads back byte for byte."""
    cap = 4096
    rig = _rig(1024, RING, names=1, resp_bytes=cap)
    try:
        rig.set_status(0, K.AGR_AGENT_STOPPED)
        T = T0
        groups = {}
        for name, cnt, dt in (("P", 3, 0), ("A", 8, 1), ("B", 8, 2), ("C", 8, 3), ("D", 3, 4), ("E", 1, 5), ("F1", 2, 6),
                              ("F2", 1, 6), ("Z", 8, 100)):
            first = rig.ingest_t(np.zeros(cnt, np.int64), np.full(cnt, T + dt, np.uint64))
            groups[name] = (np.arange(first, first + cnt), T + dt)
        bodies = {}
        z = iter(groups["Z"][0].tolist())

        def store(name, size):
            rows, t = groups[name]
            segs = [bytes([(7 * r + j) & 0xff for j in range(size)]) for r in rows.tolist()]
            rc, _ = rig.eng.complete_ex(rig.outcomes(rows, np.full(len(rows), OUT_RESPONSE), np.full(len(rows), t)), segs)
            rig.ref.complete(rows, np.full(len(rows), OUT_RESPONSE), np.full(len(rows), 200), times=np.full(len(rows), t))
            if rc == 0:
                bodies.update(zip(rows.tolist(), segs))
            return rc

        def no_room(size=16):
            r = next(z)
            rc, _ = rig.eng.complete_ex(rig.outcomes(np.array([r]), [OUT_RESPONSE], [T + 100]), [b"x" * size])
            rig.ref.complete([r], [OUT_RESPONSE], [200], times=[T + 100])
            return rc == K.AGR_ENOSPC

        def read_back():
            live = [r for r in bodies if rig.ref.stored[r] and r >= rig.ref.tail]
            for r in live:
                assert rig.eng.get_response_body(rig.names[0], bytes(rig.ref.ids[r])) == bodies[r], f"row {r}"
            return len(live)

        def release(dt, count):
            rig.expire(T + dt + TTL)
            assert rig.reclaim() == count

        assert store("A", 256) == 0 and store("B", 256) == 0           # [0, 2048) and [2048, 4096): head = A's start
        release(0, 3)                                                 # the rows before A go; A's distance is 0 = the whole ring
        assert no_room() and read_back() == 16
        release(1, 8)                                                 # A goes: exactly its 2048 bytes come free
        assert store("C", 256) == 0 and no_room() and read_back() == 16
        release(2, 8)                                                 # B goes: [2048, 4096) free
        assert store("D", 512) == 0                                   # [2048, 3584)
        assert store("E", 1024) == K.AGR_ENOSPC                       # would skip [3584, 4096) and land on C
        del groups["E"]
        release(3, 8)                                                 # C goes
        groups["E"] = (np.array([next(z)]), T + 5)
        assert store("E", 1024) == 0                                  # skips the end of the ring: [0, 1024)
        release(4, 3)                                                 # D goes
        assert store("F1", 1024) == 0 and store("F2", 1024) == 0      # [1024, 3072), [3072, 4096): head = E's start again
        assert no_room() and read_back() == 4
    finally:
        rig.close()
