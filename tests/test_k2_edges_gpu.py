"""K2 (agr_complete, agr_complete_ex, and the outcome half of the service kernel) against the plain restatement of
tests/k2ref.py where the kernels change code path:
  * k2_append's decoupled look-back: batches on both sides of every K2_TILE (2048 ops) edge, up to 2^20 ops, with tiles that
    push nothing, only completed or only failed entries, and a last tile of 1 to 7 ops (the byte-wise tail of its 8-op loads);
  * k2_apply_one's chains: 1..12, 16, 40, 300 and 2049 ops of one row, at and past the K2_SORT_MAX = 8 register sort, placed
    ascending, descending, at random and across the first and the last tile, with retry saturating at 255;
  * the log clamp: the capacity inside a tile, at a tile edge, exactly at the end of a batch (not an overflow) and one past it;
  * misses: zero ids, unknown agents, the right id under the wrong agent, expired and released rows, dial errors;
  * bytes: every source residue mod 16, segment lengths around the 16-byte and 512-byte warp steps, winners in a tile
    other than their chain root's, and a byte region that does not fit;
  * the service kernel's own ordered append, clamp and copy (AGR_CFG_COMBINE), and its answer when a push is dropped.
After every call: each op's result and the call's return code, the counters, the log lengths, the three lists of every agent,
and the state / aux / last-SET words of every live row; byte cases also compare the wire form of every touched row and the
stored response bytes."""

import numpy as np
import pytest

import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.binding import _ptr
import k2ref as R
import k5ref

pytestmark = pytest.mark.gpu
MODES = ["hash", "mint"]
TILE = 2048
AGENT0 = 1_700_000_000_000_000_000
UNKNOWN = "agent-unknown"
STAT_KEYS = ["completions", "failures", "dead_lettered", "completion_misses", "dial_errors"]


def names(n):
    return [f"agent-{AGENT0 + 1000003 * k}" for k in range(n)]


class Rig:
    """One engine and the restatement of what it must hold."""

    def __init__(self, mode, *, slab_rows=1 << 14, n_agents=1, log_entries=0, max_batch=0, ring=False, combine=False,
                 skip_inflight=False, resp_bytes=0, wire=False, seed=1):
        flags = K.AGR_CFG_PERSISTENCE | (K.AGR_CFG_MINT_IDS if mode == "mint" else 0) | (K.AGR_CFG_RING if ring else 0)
        flags |= (K.AGR_CFG_COMBINE if combine else 0) | (K.AGR_CFG_SKIP_INFLIGHT if skip_inflight else 0)
        self.eng = A.Engine(device=0, slab_rows=slab_rows, max_agents=64, max_batch=max_batch, flags=flags, log_entries=log_entries,
                            resp_bytes=resp_bytes or 64 * slab_rows, id_secret=0x5eed)
        self.lib = self.eng.lib
        self.mint, self.ring, self.combine, self.wire = mode == "mint", ring, combine, wire
        self.ref = R.K2Ref(log_entries or 3 * slab_rows, skip_inflight=skip_inflight)
        self.names = names(n_agents)
        st = [K.AGR_AGENT_RUNNING if k % 3 != 1 else K.AGR_AGENT_STOPPED for k in range(n_agents)]
        assert list(self.eng.set_agent_states(self.names, st)) == list(range(n_agents))
        for a in self.names:
            self.ref.register(a)
        self.running = np.array([s == K.AGR_AGENT_RUNNING for s in st] + [False])
        self.rng = np.random.default_rng(seed)
        self.seq = 0

    def close(self):
        self.eng.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- what the test does
    def ingest(self, slots, max_retries=3):
        """Fresh records of these agent slots (-1: an unknown agent, not stored); returns their rows."""
        slots = np.asarray(slots, dtype=np.int64)
        chunk = min(1 << 16, self.eng.max_batch)
        rows = []
        nm = np.array([a.encode() for a in self.names] + [UNKNOWN.encode()], dtype="S32")
        mr = np.broadcast_to(np.asarray(max_retries), (len(slots),))
        for lo in range(0, len(slots), chunk):
            s, m = slots[lo:lo + chunk], mr[lo:lo + chunk]
            n = len(s)
            recs = np.zeros(n, dtype=A.record_dtype)
            recs["agent_id"] = nm[np.where(s >= 0, s, len(self.names))]
            recs["request_id"] = self.rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
            recs["request_id"][:, 6] = (recs["request_id"][:, 6] & 0x0F) | 0x40
            recs["seq"] = self.seq + 1 + np.arange(n)
            self.seq += n
            recs["flags"] = K.METHOD_CODES["POST"] << K.AGR_F_METHOD_SHIFT
            recs["path_len"], recs["body_len"] = 5, 2
            recs["payload"][:, :7] = np.frombuffer(b"/chat{}", dtype=np.uint8)
            recs["status"], recs["max_retries"] = K.AGR_ST_PENDING, m
            _, first = self.eng.ingest(recs, want_verdicts=False)
            ids = self.eng.mint_ids(first, n) if self.mint else recs["request_id"]
            wire = None
            if self.wire:
                wire = [k5ref.Rec(bytes(a), "POST", b"/chat", b"", b"{}", int(t), max_retries=int(x), rid=bytes(i))
                        for a, t, x, i in zip(recs["agent_id"], recs["seq"], m, ids)]
            self.ref.add_rows(first, s, ids, self.running[np.where(s >= 0, s, -1)], max_retries=m, created=recs["seq"],
                              ring=self.ring, recs=wire)
            rows.append(np.arange(first, first + n))
        return np.concatenate(rows)

    def outcomes(self, rows, kinds, agents=None, https=None, seqs=None, zero=None):
        """Outcomes naming these rows (agents: agent index per op, len(names) = unknown; default the row's own)."""
        rows = np.asarray(rows, dtype=np.int64)
        n = len(rows)
        ids = self.ref.ids[rows].copy()
        if zero is not None:
            ids[zero] = 0
        ag = np.maximum(self.ref.slot[rows], 0) if agents is None else np.asarray(agents)
        nm = np.array([a.encode() for a in self.names] + [UNKNOWN.encode()], dtype="S32")
        outs = np.zeros(n, dtype=A.outcome_dtype)
        outs["request_id"] = ids
        outs["agent_id"] = nm[ag]
        outs["kind"] = kinds
        outs["http_status"] = self.rng.integers(100, 600, size=n) if https is None else https
        outs["seq"] = self.rng.integers(0, 1 << 62, size=n, dtype=np.uint64) if seqs is None else seqs
        return outs

    def apply(self, outs, segs=None, hdr_lens=None, pad=0, check=True, bytes_fit=True):
        """One agr_complete (segs None) or agr_complete_ex call, on the engine and the restatement; then the comparisons."""
        n = len(outs)
        res = np.zeros(max(n, 1), dtype=np.int32)
        if segs is None:
            rc = self.lib.agr_complete(self.eng.h, _ptr(outs), n, _ptr(res))
        else:
            offs = np.zeros(n + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(s) for s in segs], dtype=np.uint64)
            offs += pad                                               # offsets[0] != 0: the batch starts inside the buffer
            blob = np.frombuffer(bytes(range(pad)) + b"".join(segs) + b"\0", dtype=np.uint8)
            hl = np.ascontiguousarray(hdr_lens if hdr_lens is not None else np.zeros(n), dtype=np.uint32)
            rc = self.lib.agr_complete_ex(self.eng.h, _ptr(outs), n, _ptr(blob), _ptr(offs), _ptr(hl), _ptr(res))
        err = (self.lib.agr_last_error() or b"").decode()
        want, want_rc = self.ref.complete(outs["request_id"], self._slots(outs), outs["kind"], outs["http_status"], outs["seq"],
                                          segs if (segs is not None and bytes_fit) else None, hdr_lens)
        assert rc in (0, K.AGR_ENOSPC), (rc, err)
        bytes_rc = 0 if (segs is None or bytes_fit) else K.AGR_ENOSPC
        assert rc == (want_rc or bytes_rc), (rc, want_rc, bytes_rc, err)
        if want_rc and not bytes_rc:
            assert "log full" in err and "byte slab" not in err, err
        if bytes_rc:
            assert "response byte slab" in err and (("log full" in err) == bool(want_rc)), err
        assert np.array_equal(res[:n], want), np.flatnonzero(res[:n] != want)[:10]
        if check:
            self.check()
        return rc, res[:n]

    def _slots(self, outs):
        lut = {a.encode(): s for a, s in self.ref.slots.items()}
        u, inv = np.unique(outs["agent_id"], return_inverse=True)
        return np.array([lut.get(x, -1) for x in u])[inv]

    # ---- the comparisons
    def check(self, lists=True):
        st = self.eng.stats()
        for k in STAT_KEYS:
            assert st[k] == self.ref.ctr[k], (k, st[k], self.ref.ctr[k])
        if self.combine:
            assert (st["log_overflow"] > 0) == (self.ref.ctr["log_overflow"] > 0)
        else:
            assert st["log_overflow"] == self.ref.ctr["log_overflow"]
        assert (st["completed_log_len"], st["failed_log_len"]) == self.ref.log_lens()
        lo, hi = self.ref.tail, self.ref.n
        rows = np.arange(lo, hi)
        got_st = self.eng.debug_read("state", lo, hi - lo)
        stored = self.ref.stored[lo:hi]
        assert np.array_equal((got_st & R.ST_STORED) != 0, stored)
        want = self.ref.state_words(rows)
        bad = np.flatnonzero(stored & (got_st != want))
        assert not len(bad), f"row {rows[bad[0]]}: state {got_st[bad[0]]:#x} != {want[bad[0]]:#x} ({len(bad)} rows)"
        aux = self.eng.debug_read("aux", lo, hi - lo)
        bad = np.flatnonzero(stored & (aux != self.ref.aux_words(rows)))
        assert not len(bad), f"row {rows[bad[0]]}: aux {aux[bad[0]]:#x} != {self.ref.aux_words(rows)[bad[0]]:#x}"
        mt = self.eng.debug_read("mtime", lo, hi - lo)
        bad = np.flatnonzero(stored & (mt != self.ref.mtime[lo:hi]))
        assert not len(bad), f"row {rows[bad[0]]}: mtime {mt[bad[0]]} != {self.ref.mtime[rows[bad[0]]]}"
        if lists:
            for s, a in enumerate(self.names):
                if s in self.ref.dropped:
                    continue
                for which in (K.AGR_LIST_PENDING, K.AGR_LIST_COMPLETED, K.AGR_LIST_FAILED):
                    got = self.eng.list(a, which, cap=1 << 16)
                    r = self.ref.list(s, which)
                    assert len(got) == len(r), (a, which, len(got), len(r))
                    assert np.array_equal(got, self.ref.ids[r]), (a, which, "order / entries differ")
        if self.wire:
            self.check_wire(lo, hi)

    def check_wire(self, lo, hi):
        recs = [self.ref.recs.get(r) or k5ref.Rec(b"", "", b"", b"", b"", 0, stored=False) for r in range(lo, hi)]
        got, offs = self.eng.rows_json(lo, hi - lo)
        want, woffs = k5ref.wire_rows(recs)
        if got != want:
            for i in range(hi - lo):
                g = got[int(offs[i]):int(offs[i + 1])]
                w = want[woffs[i]:woffs[i + 1]]
                assert g == w, f"row {lo + i}: {g[:200]!r} != {w[:200]!r}"
        for r in range(lo, hi):
            rec = self.ref.recs.get(r)
            if rec is not None and rec.stored:
                got = self.eng.get_response_body(rec.agent.decode(), rec.rid)
                assert got == (rec.resp_hdr + rec.resp_body if rec.responded else b""), r


def tile_kinds(n, rng):
    """Op kinds by tile: tile t % 4 == 0 mixed, 1 pushes nothing (dial errors), 2 only completed, 3 only failed."""
    t = np.arange(n) // TILE
    kinds = rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=n)
    kinds = np.where(t % 4 == 1, R.OUT_DIAL_ERR, kinds)
    kinds = np.where(t % 4 == 2, R.OUT_RESPONSE, kinds)
    return np.where(t % 4 == 3, R.OUT_ERROR, kinds)


SIZES = [1, 7, 8, 9, 2047, 2048, 2049, 4095, 4096, 4097, 8 * TILE - 3, 33 * TILE + 5, 1 << 20]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", SIZES)
def test_tile_edges_one_agent(mode, n):
    """One agent: the whole log order is the list order.  Every row takes one op (max_retries 1: every ERROR pushes), a
    second call on the same rows then mixes in misses and a few chains."""
    big = n > 1 << 17
    pad = 37
    with Rig(mode, slab_rows=1 << max(14, (n + pad + 1024).bit_length()), max_batch=max(n, 1 << 13), seed=n) as rig:
        rig.ingest(np.zeros(pad, dtype=np.int64), max_retries=1)      # rows before the batch's: start rows are not 0
        rows = rig.ingest(np.zeros(n, dtype=np.int64), max_retries=1)
        perm = rig.rng.permutation(rows)
        kinds = tile_kinds(n, rig.rng)
        if n >= 2 * TILE:
            assert {R.OUT_DIAL_ERR} == set(kinds[TILE:2 * TILE].tolist())
        rig.apply(rig.outcomes(perm, kinds), check=False)
        rig.check(lists=True)
        if big:
            return
        kinds = tile_kinds(n, rig.rng)[::-1].copy()
        agents = np.where(rig.rng.random(n) < 0.05, 1, 0)            # 1 = unknown agent: misses
        zero = rig.rng.random(n) < 0.03
        again = perm.copy()
        again[1::5] = again[::5][: len(again[1::5])]                  # two ops on some rows, in different tiles
        rig.apply(rig.outcomes(again, kinds, agents=agents, zero=zero))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [4097, 33 * TILE + 5])
def test_tile_edges_many_agents(mode, n):
    with Rig(mode, slab_rows=1 << 17, n_agents=40, max_batch=1 << 17, seed=7 + n) as rig:
        w = 1.0 / np.arange(1, 41) ** 1.2
        rows = rig.ingest(rig.rng.choice(40, size=n, p=w / w.sum()), max_retries=rig.rng.integers(0, 3, size=n))
        for _ in range(3):
            pick = rig.rng.choice(rows, size=n)                       # chains of every length the draw gives
            rig.apply(rig.outcomes(pick, tile_kinds(n, rig.rng)))


def chain_layout(L, place, n_fill, rng):
    """Positions of a chain of L ops among L + n_fill ops."""
    n = L + n_fill
    if place == "spread":                                            # first op at 0, last at the batch's end
        mid = np.sort(rng.choice(np.arange(1, n - 1), size=max(L - 2, 0), replace=False))
        return np.concatenate([[0], mid, [n - 1]])[:L] if L > 1 else np.array([0])
    if place == "block":
        s = int(rng.integers(0, n_fill + 1))
        return np.arange(s, s + L)
    return np.sort(rng.choice(n, size=L, replace=False))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("max_retries", [0, 1, 3, 255])
def test_chains(mode, max_retries):
    """One row with L ops in a call (ascending, descending: the chain walk is in link order, which the kernel sorts;
    random; first and last tile), single-op rows around it, then a second call on the same rows (head[] is clean)."""
    lengths = list(range(1, 13)) + [16, 40, 300, 2049]
    with Rig(mode, slab_rows=1 << 16, max_batch=1 << 14, seed=max_retries) as rig:
        for L in lengths:
            for place in ("block", "random", "spread"):
                n_fill = 2100 if (place == "spread" or L >= 300) else 40
                rows = rig.ingest(np.zeros(n_fill + 1, dtype=np.int64), max_retries=max_retries)
                pos = chain_layout(L, place, n_fill, rig.rng)
                ops = np.empty(L + n_fill, dtype=np.int64)
                mask = np.zeros(L + n_fill, dtype=bool)
                mask[pos] = True
                ops[mask] = rows[0]
                ops[~mask] = rig.rng.permutation(rows[1:])[:n_fill]
                p_err = 0.9 if L == 300 else 0.5                     # 300: retry runs into 255 with max_retries 255
                kinds = np.where(rig.rng.random(L + n_fill) < p_err, R.OUT_ERROR, R.OUT_RESPONSE)
                if place == "block" and L > 1:
                    kinds[pos] = kinds[pos][::-1]
                rig.apply(rig.outcomes(ops, kinds), check=False)
                rig.check(lists=False)
                rig.apply(rig.outcomes(ops[::-1].copy(), kinds), check=False)
                rig.check(lists=False)
        assert max_retries != 255 or rig.ref.retry.max() == 255
        rig.check()
        # many chained rows interleaved with single-op rows, across tiles
        rows = rig.ingest(np.zeros(600, dtype=np.int64), max_retries=max_retries)
        ops = np.concatenate([np.repeat(rows[:200], rig.rng.integers(2, 20, size=200)), rows[200:]])
        ops = rig.rng.permutation(ops)
        assert len(ops) > TILE
        for _ in range(2):
            rig.apply(rig.outcomes(ops, rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=len(ops))))


CAP_CASES = {                    # log_entries, completed pushes of the first call, dial errors spread among them (push nothing)
    "inside_tile": (3000, 5000, 300),
    "tile_edge": (4096, 6000, 0),   # the cap's entry is the first op of tile 2
    "batch_end": (4100, 4100, 300),
    "one_past": (4099, 4100, 300),
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", sorted(CAP_CASES))
def test_log_capacity(mode, case):
    cap, n, dial = CAP_CASES[case]
    with Rig(mode, slab_rows=1 << 14, log_entries=cap, max_batch=1 << 13, seed=cap) as rig:
        rows = rig.ingest(np.zeros(n + dial + 3000, dtype=np.int64), max_retries=1)
        kinds = np.full(n + dial, R.OUT_RESPONSE)
        kinds[rig.rng.choice(n + dial, size=dial, replace=False)] = R.OUT_DIAL_ERR
        rc, _ = rig.apply(rig.outcomes(rows[:n + dial], kinds))
        assert (rc == 0) == (case == "batch_end") and rig.ref.log_lens()[0] == cap
        rows = rows[dial:]
        # completed is full (or exactly full): failed still has room; then failed overflows while completed takes nothing
        m = 2000
        rc, _ = rig.apply(rig.outcomes(rows[n:n + m], np.full(m, R.OUT_ERROR)))
        assert rc == 0 and rig.ref.log_lens()[1] == m
        rc, _ = rig.apply(rig.outcomes(rows[n + m:n + 3000], np.full(1000, R.OUT_ERROR)))
        assert (rc != 0) == (m + 1000 > cap)
        # a batch after the log is full: transitions apply, nothing lands
        rc, _ = rig.apply(rig.outcomes(rig.rng.choice(rows, size=500), rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR], size=500)))
        assert rc == K.AGR_ENOSPC


@pytest.mark.parametrize("mode", MODES)
def test_log_capacity_after_reclaim(mode):
    """Ring: expire + agr_reclaim drop the released rows' log entries, and later pushes land after the survivors."""
    cap = 3000
    with Rig(mode, slab_rows=1 << 14, log_entries=cap, ring=True, max_batch=1 << 12, seed=5) as rig:
        old = rig.ingest(np.zeros(2000, dtype=np.int64), max_retries=1)
        rig.apply(rig.outcomes(old, np.full(2000, R.OUT_RESPONSE), seqs=np.full(2000, 10, dtype=np.uint64)))
        new = rig.ingest(np.zeros(3000, dtype=np.int64), max_retries=1)
        rig.apply(rig.outcomes(new[:1500], np.full(1500, R.OUT_RESPONSE), seqs=np.full(1500, 1 << 40, dtype=np.uint64)))
        assert rig.ref.log_lens()[0] == cap
        # the old rows' last SET is 10, the others' later: a sweep at now = 10 + ttl drops exactly the old rows
        ttl = 1 << 30
        n = rig.eng.expire(10 + ttl, ttl)
        due = np.flatnonzero(rig.ref.stored[:rig.ref.n] & (rig.ref.mtime[:rig.ref.n] <= 10))
        assert n == len(due)
        rig.ref.expire(due)
        live = np.flatnonzero(rig.ref.stored[rig.ref.tail:rig.ref.n])
        end = rig.ref.tail + (int(live[0]) if len(live) else rig.ref.n - rig.ref.tail)
        assert rig.eng.reclaim() == end - rig.ref.tail
        rig.ref.reclaim(end)
        rig.check()
        rc, _ = rig.apply(rig.outcomes(new[1500:], np.full(1500, R.OUT_RESPONSE), seqs=np.full(1500, 1 << 41, dtype=np.uint64)))
        assert rc == 0 and rig.ref.log_lens()[0] == 2500


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("skip_inflight", [False, True])
def test_misses_and_dial_errors(mode, skip_inflight):
    with Rig(mode, slab_rows=1 << 14, n_agents=4, ring=True, skip_inflight=skip_inflight, max_batch=1 << 13, seed=11) as rig:
        gone = rig.ingest(rig.rng.integers(0, 4, size=600))           # released below
        rows = rig.ingest(np.concatenate([rig.rng.integers(0, 4, size=5000), np.full(50, -1)]))
        # expire the first 600 rows (their last SET is their created_at, 1..600) and a stripe of the others, release the first
        ttl = 1 << 20
        touch = np.concatenate([rows[::7], rows[3::11]])            # rows[3::11] last SET at 5: expired by the sweep below
        rig.apply(rig.outcomes(touch, np.full(len(touch), R.OUT_RESPONSE),
                               seqs=np.where(np.arange(len(touch)) < len(rows[::7]), 1 << 30, 5).astype(np.uint64)))
        n = rig.eng.expire(600 + ttl, ttl)
        due = np.flatnonzero(rig.ref.stored[:rig.ref.n] & (rig.ref.mtime[:rig.ref.n] <= 600))
        assert n == len(due)
        rig.ref.expire(due)
        end = 600
        assert rig.eng.reclaim() == end
        rig.ref.reclaim(end)
        stale = rows[~rig.ref.stored[rows]][:80]                      # expired (and never stored), still in the window
        assert rig.ref.slot[stale].max() >= 0
        rig.eng.drop_agent(rig.names[3])
        rig.ref.drop(rig.names[3])
        rig.check()
        # a batch over two tiles of every kind of miss, mixed with hits and dial errors, and chains that hold misses
        n = 4500
        tgt = rig.rng.choice(np.concatenate([rows, gone, stale]), size=n)
        kinds = rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=n)
        own = np.where(rig.ref.slot[tgt] >= 0, rig.ref.slot[tgt], 0)
        x = rig.rng.random(n)
        agents = np.where(x < 0.1, 4, np.where(x < 0.2, (own + 1) % 4, own))     # 4: unknown agent; +1: the wrong agent
        gone_ids = np.isin(tgt, gone)
        outs = rig.outcomes(np.where(gone_ids, rows[0], tgt), kinds, agents=agents, zero=rig.rng.random(n) < 0.05)
        outs["request_id"][gone_ids] = rig.ref.ids[tgt[gone_ids]]
        rc, res = rig.apply(outs)
        assert (res == K.AGR_ENOTFOUND).sum() > 500
        chain = rig.rng.permutation(np.repeat(np.concatenate([rows[:30], stale[:10]]), 12))   # chains that hold misses
        own = np.maximum(rig.ref.slot[chain], 0)
        rig.apply(rig.outcomes(chain, rig.rng.choice([1, 2, 3], size=len(chain)),
                               agents=np.where(rig.rng.random(len(chain)) < 0.3, 4, own)))


def segments(rng, n, kinds, lens):
    """A segment per op: responses get "X-K: v" headers (hdr_len 0, in the middle, or the whole segment)."""
    segs, hls = [], []
    for k in range(n):
        L = int(lens[k % len(lens)])
        body = rng.integers(0, 256, size=L, dtype=np.uint8).tobytes()
        if kinds[k] == R.OUT_RESPONSE:
            h = k5ref.flat_headers([(b"X-K", b"v%d" % k)]) if k % 3 else b""
            if k % 3 == 2:
                body = b""
            segs.append(h + body)
            hls.append(len(h))
        elif kinds[k] == R.OUT_ERROR:
            segs.append(body)
            hls.append(0)
        else:
            segs.append(b"")
            hls.append(0)
    return segs, np.array(hls, dtype=np.uint32)


LENS = list(range(0, 49)) + [511, 512, 513, 1023, 1024, 1025, 4095, 4096, 4097]


@pytest.mark.parametrize("mode", MODES)
def test_bytes(mode):
    with Rig(mode, slab_rows=1 << 13, n_agents=2, max_batch=1 << 13, resp_bytes=256 << 20, wire=True, seed=13) as rig:
        rows = rig.ingest(rig.rng.integers(0, 2, size=1200), max_retries=3)
        for pad in (0, 5, 16, 23):
            n = 300
            tgt = rig.rng.choice(rows, size=n)
            kinds = rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=n, p=[0.5, 0.4, 0.1])
            segs, hls = segments(rig.rng, n, kinds, rig.rng.permutation(LENS))
            offs = np.cumsum([0] + [len(s) for s in segs])
            assert len(set((offs % 16).tolist())) == 16                # every source residue
            rig.apply(rig.outcomes(tgt, kinds), segs, hls, pad=pad)
        # winners in a tile other than the chain root's: a row's ops at the start, in the middle and at the end of 4500 ops
        n = 4500
        tgt = rig.rng.choice(rows[100:], size=n)
        for k, r in enumerate(rows[:20]):
            tgt[[k, TILE + 7 * k, n - 1 - k]] = r
        kinds = rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR], size=n)
        segs, hls = segments(rig.rng, n, kinds, [0, 1, 15, 17, 33, 100, 440])
        rig.apply(rig.outcomes(tgt, kinds), segs, hls, pad=9)
        # one 64 KiB + 1 error text
        segs = [rig.rng.integers(0, 256, size=(1 << 16) + 1, dtype=np.uint8).tobytes(), b"short"]
        rig.apply(rig.outcomes(rows[50:52], [R.OUT_ERROR, R.OUT_ERROR]), segs, np.zeros(2), pad=3)


@pytest.mark.parametrize("mode", MODES)
def test_bytes_that_do_not_fit(mode):
    """Ring byte slab: a batch whose region does not fit returns AGR_ENOSPC with the transitions applied and no byte stored;
    agr_last_error tells it from a full log, and names both when both happen."""
    with Rig(mode, slab_rows=1 << 12, log_entries=300, ring=True, resp_bytes=64 << 10, wire=True, seed=17) as rig:
        rows = rig.ingest(np.zeros(700, dtype=np.int64), max_retries=1)
        segs, hls = segments(rig.rng, 100, [R.OUT_RESPONSE] * 100, [40])
        rig.apply(rig.outcomes(rows[:100], np.full(100, R.OUT_RESPONSE)), segs, hls)
        segs, hls = segments(rig.rng, 100, [R.OUT_ERROR] * 100, [440])        # 44 800 B: more than half the ring
        rig.apply(rig.outcomes(rows[100:200], np.full(100, R.OUT_ERROR)), segs, hls, bytes_fit=False)
        segs, hls = segments(rig.rng, 300, [R.OUT_ERROR] * 300, [300])        # bytes and the failed log: both in agr_last_error
        rc, _ = rig.apply(rig.outcomes(rows[200:500], np.full(300, R.OUT_ERROR)), segs, hls, bytes_fit=False)
        assert rc == K.AGR_ENOSPC and rig.ref.log_lens() == (100, 300) and rig.ref.ctr["log_overflow"] == 1
        segs, hls = segments(rig.rng, 200, [R.OUT_RESPONSE] * 200, [400])      # bytes only: completed ends exactly at the cap
        rc, _ = rig.apply(rig.outcomes(rows[500:700], np.full(200, R.OUT_RESPONSE)), segs, hls, bytes_fit=False)
        assert rc == K.AGR_ENOSPC and rig.ref.log_lens() == (300, 300) and rig.ref.ctr["log_overflow"] == 1


# ------------------------------------------------------------------------------------------------ the service kernel
def submit(rig, outs, segs=None, hls=None):
    """Tickets for every outcome before any is collected; then every ticket collected, in order."""
    tickets = []
    for k in range(len(outs)):
        if segs is None:
            tickets.append(rig.eng.submit_complete(outs[k]))
        else:
            h = int(hls[k])
            tickets.append(rig.eng.submit_complete_ex(outs[k], segs[k][:h], segs[k][h:]))
    return np.array([rig.eng.wait(t) for t in tickets], dtype=np.int32)


@pytest.mark.parametrize("mode", MODES)
def test_service_kernel_tickets(mode):
    with Rig(mode, slab_rows=1 << 14, n_agents=3, combine=True, wire=True, seed=19) as rig:
        rows = rig.ingest(rig.rng.integers(0, 3, size=900), max_retries=rig.rng.integers(0, 4, size=900))
        for with_bytes in (False, True):
            n = 3000
            tgt = rig.rng.choice(rows, size=n)
            tgt[100:120] = rows[0]                                   # a chain longer than 8 inside one service batch
            tgt[500:540:2] = rows[1]
            kinds = rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR, R.OUT_DIAL_ERR], size=n, p=[0.5, 0.4, 0.1])
            agents = np.where(rig.rng.random(n) < 0.05, 3, np.maximum(rig.ref.slot[tgt], 0))
            outs = rig.outcomes(tgt, kinds, agents=agents)
            segs = hls = None
            if with_bytes:
                segs, hls = segments(rig.rng, n, kinds, [0, 1, 7, 15, 16, 17, 31, 200, 411, 425])
            got = submit(rig, outs, segs, hls)
            slots = rig._slots(outs)
            want, _ = rig.ref.complete(outs["request_id"], slots, outs["kind"], outs["http_status"], outs["seq"], segs, hls)
            assert np.array_equal(got, np.where(rig.ref.dropped_push, K.AGR_ENOSPC, want))
            rig.check()
        # agr_complete through the ring (n <= 32) and as a batch (n > 32), on the same rows, alternating
        for k in range(40):
            n = [1, 5, 32, 33, 200][k % 5]
            tgt = rig.rng.choice(rows[:60], size=n)
            rig.apply(rig.outcomes(tgt, rig.rng.choice([R.OUT_RESPONSE, R.OUT_ERROR], size=n)), check=(k % 5 == 4))
        rig.check()


@pytest.mark.parametrize("mode", MODES)
def test_service_kernel_log_capacity(mode):
    """Through the ring the caller learns of a dropped push as in a batch: AGR_ENOSPC from agr_complete / agr_complete_ex,
    a ticket result of AGR_ENOSPC; a call that ends exactly at the capacity returns 0."""
    cap = 40
    with Rig(mode, slab_rows=1 << 12, log_entries=cap, combine=True, resp_bytes=1 << 20, wire=True, seed=23) as rig:
        rows = rig.ingest(np.zeros(400, dtype=np.int64), max_retries=1)
        for lo in range(0, 40, 10):                                 # exactly to the cap: 0 every time
            rc, _ = rig.apply(rig.outcomes(rows[lo:lo + 10], np.full(10, R.OUT_RESPONSE)))
            assert rc == 0
        rc, _ = rig.apply(rig.outcomes(rows[40:41], [R.OUT_RESPONSE]))   # one past it
        assert rc == K.AGR_ENOSPC
        rc, _ = rig.apply(rig.outcomes(rows[41:71], np.full(30, R.OUT_ERROR)))      # failed: 30 of 40, room left
        assert rc == 0
        rc, _ = rig.apply(rig.outcomes(rows[71:91], np.full(20, R.OUT_ERROR)))      # failed overflows inside the call
        assert rc == K.AGR_ENOSPC
        rc, _ = rig.apply(rig.outcomes(rows[91:92], [R.OUT_DIAL_ERR]))            # pushes nothing: not an overflow
        assert rc == 0
        segs, hls = segments(rig.rng, 8, [R.OUT_RESPONSE] * 8, [0, 16, 100, 440])
        rc, _ = rig.apply(rig.outcomes(rows[92:100], np.full(8, R.OUT_RESPONSE)), segs, hls)
        assert rc == K.AGR_ENOSPC
        outs = rig.outcomes(rows[100:110], np.full(10, R.OUT_RESPONSE))
        got = submit(rig, outs)
        want, _ = rig.ref.complete(outs["request_id"], rig._slots(outs), outs["kind"], outs["http_status"], outs["seq"])
        assert (got == K.AGR_ENOSPC).all() and rig.ref.dropped_push.all()
        rig.check()
