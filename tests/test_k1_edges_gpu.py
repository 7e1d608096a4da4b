"""The fixed-stride ingest (K1: k1_ingest_tma, k1_post, and the record half of the service kernel k_svc) against the plain
reference of tests/k1ref.py, in both id modes, append-only and ring, at the edges where K1 changes code path:

  - the tile schedule: batches of 1, 31, 32, 33, 14 * 32 +- 1 records, and W - 1, W, W + 1, 2W + 1 and 3W tiles (W = 14 x SMs
    warps in the grid), and 2^20 records: a grid smaller than the SM count, warps of the last CTA with no tile, warps with one
    tile (the flush path only), warps with two or more (the cross-tile pipeline);
  - batch alignment (first row mod 32 of 0, 1, 31), tiles across a 4096-row chunk, slab ends that are not a multiple of 32 with a
    batch ending exactly there, ring laps with pad rows, batches at physical row 0 and arrival numbers unequal to the row;
  - random bytes in all 512 B of every record, lengths around the 416 B payload and at the u16 / u32 extremes, max_retries 0
    and 255, persistence off;
  - running, stopped, unknown, dropped and all-zero agents, a 32-byte name without NUL, names that collide in the agent table
    with a probe chain that wraps past its end;
  - caller ids that share a home slot of a small dedupe index (a chain across its end), duplicate ids in one tile, in two tiles
    of one warp, in two CTAs and across batches, zero ids, and the triples "rows A < B carry id X, a replay R > A names X";
  - replays of minted ids naming an earlier batch, an earlier tile, the same tile, a later row, the row itself, a released row
    and a row of the previous lap, with batches launched back to back;
  - the same batches through agr_ingest_rows_async, agr_ingest_rows, agr_ingest_ex and the chunked agr_ingest (every k1_post
    path), and through the service kernel (agr_ingest_ex with n <= 32, and tickets).

After every launch: every verdict, the route / state / checksum word of every row of the batch and of every row a replay names,
mtime of the stored rows and the chunk bounds of every chunk the batch touched (ring), all K1 counters, the pending list of
every agent, and (caller ids) how many ids the dedupe index holds."""
from functools import lru_cache

import numpy as np
import pytest

import agentainer_lab_b200 as A
import k1ref
from agentainer_lab_b200 import constants as K
from mintref import mint_bytes

pytestmark = pytest.mark.gpu

SECRET = 0x5eed1234
MODES = {"hash": 0, "mint": K.AGR_CFG_MINT_IDS}
MAX_AGENTS = 8                   # agent table of 16 entries: amask = 15
LONG = b"agent-with-a-name-of-32-bytes-xy"
assert len(LONG) == 32


def _colliding_names():
    """agent names whose home entry in a 16-entry agent table is the last one: their probe chain wraps to entry 0"""
    cand = [f"agent-c{k}".encode() for k in range(4000)]
    h = k1ref.hash_agent(cand) & np.uint64(15)
    return [cand[i] for i in np.nonzero(h == 15)[0][:5]]


COLL = _colliding_names()
# registration order: the four colliding names take entries 15, 0, 1, 2 (the fourth is dropped afterwards)
# LONG[:31] is registered; LONG itself (32 bytes, no NUL: not a name an agent can have) must not match it
AGENTS = [(COLL[0], "running"), (COLL[1], "stopped"), (COLL[2], "running"), (COLL[3], "running"), (b"agent-run", "running"),
          (b"agent-stop", "stopped"), (LONG[:31], "running")]
DROPPED = COLL[3]
NAMES = [a for a, _ in AGENTS] + [COLL[4], LONG, b""]   # COLL[4] collides but is never registered; b"": all-zero id
P_NAMES = np.array([0.17, 0.12, 0.12, 0.04, 0.2, 0.12, 0.13, 0.03, 0.04, 0.03])
FOUND = [a for a, _ in AGENTS if a != DROPPED]
RUNNING = [a for a, s in AGENTS if s == "running" and a != DROPPED]


@lru_cache(maxsize=None)
def sms() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def W() -> int:
    return k1ref.WARPS * sms()


# ------------------------------------------------------------------------------------------------------- engine + reference
class Rig:
    def __init__(self, mode, rows, *, ring=False, combine=False, persistence=True, table_slots=0, max_batch=0):
        # (flags 0 reads as the default configuration, persistence on: AGR_CFG_TIMING keeps a caller-id engine without it)
        flags = MODES[mode] | (K.AGR_CFG_PERSISTENCE if persistence else K.AGR_CFG_TIMING) | (K.AGR_CFG_RING if ring else 0) | \
            (K.AGR_CFG_COMBINE if combine else 0)
        self.mode, self.ring, self.rows = mode, ring, rows
        self.e = A.Engine(slab_rows=rows, max_agents=MAX_AGENTS, flags=flags, id_secret=SECRET, table_slots=table_slots,
                          max_batch=max_batch or min(rows, 1 << 20))
        for a, s in AGENTS:
            self.e.set_agent_state(a.decode(), s)
        self.slots = {a: self.e.agent_slot(a.decode()) for a, _ in AGENTS}
        self.e.drop_agent(DROPPED.decode())
        table = {a: (self.slots[a], K.AGENT_STATUS_CODES[s]) for a, s in AGENTS}
        table[DROPPED] = (table[DROPPED][0], "dropped")
        self.ref = k1ref.Ref(table, mint=mode == "mint", secret=SECRET, persistence=persistence)

    def close(self):
        self.e.close()

    def phys(self, L):
        return np.asarray(L) % self.rows if self.ring else np.asarray(L)

    # ---- checks
    def check_batch(self, out, recs, verdicts=None):
        e, first, n = self.e, out["first"], len(recs)
        exp_v = out["verdict"].view("<u8")
        for got in ([verdicts] if verdicts is not None else []) + [e.debug_read("verdict", first, n)]:
            _same(got.view("<u8"), exp_v, "verdict")
        _same(e.debug_read("route", first, n), out["route"], "route")
        _same(e.debug_read("state", first, n), out["state"], "state")
        _same(e.debug_read("cksum", first, n), out["cksum"], "checksum")
        if self.ring:
            st = out["stored"]
            _same(e.debug_read("mtime", first, n)[st], out["created"][st], "mtime of stored rows")
            self.check_cmin(first, n)
        # the rows the batch's replays name keep their words
        rep = np.nonzero((recs["flags"] & K.AGR_F_REPLAY) != 0)[0]
        tg = []
        for i in rep.tolist():
            t = self.ref._target(recs["replay_of"][i].tobytes(), first + n)
            if t is not None and t < first and t >= self.ref.tail:
                tg.append(t)
        if tg:
            tg = np.unique(tg)
            lo, hi = int(tg[0]), int(tg[-1]) + 1
            _same(e.debug_read("route", lo, hi - lo)[tg - lo], self.ref.route[tg], "route of replay targets")
            _same(e.debug_read("state", lo, hi - lo)[tg - lo], self.ref.state[tg], "state of replay targets")
        self.check_counters()

    def check_cmin(self, first, n):
        """every chunk the rows lie in: its bound is at most the earliest created_at of its stored rows (~0 only if it has none)"""
        ph = self.phys(first + np.arange(n))
        chunks = np.unique(ph // k1ref.CHUNK)
        cm = self.e.debug_read("cmin", 0, self.rows // k1ref.CHUNK + 1)
        live = self.ref.stored_rows()
        lph = self.phys(live)
        t = np.maximum(self.ref.created[live], 1)
        for c in chunks.tolist():
            m = (lph // k1ref.CHUNK) == c
            if m.any():
                lo = int(min(t[m].min(), (1 << 64) - 2))
                assert int(cm[c]) <= lo, f"chunk {c}: bound {int(cm[c])} above the earliest stored created_at {lo}"

    def check_counters(self):
        s = self.e.stats()
        got = {k: s[k] for k in k1ref.COUNTERS}
        assert got == self.ref.ctr, {k: (got[k], self.ref.ctr[k]) for k in got if got[k] != self.ref.ctr[k]}
        if self.mode == "hash":
            assert int(self.e.debug_read("index_used", 0, 1)[0]) == self.ref.index_used()

    def check_lists(self):
        lo, hi = self.ref.tail, self.ref.head
        if self.mode == "mint":
            ids = self.e.mint_ids(lo, hi - lo)
        else:
            ids = self.ref.idb[lo:hi]
        for a in FOUND:
            rows = np.array(self.ref.pending_rows(self.slots[a]), dtype=np.int64)
            got = self.e.list(a.decode(), K.AGR_LIST_PENDING)
            want = ids[rows - lo] if len(rows) else np.zeros((0, 16), dtype=np.uint8)
            assert got.shape == want.shape and got.tobytes() == want.tobytes(), (a, len(got), len(want))

    def check_window(self):
        """the route and state words of every live row"""
        lo, hi = self.ref.tail, self.ref.head
        for a in range(lo, hi, 1 << 20):
            b = min(hi, a + (1 << 20))
            _same(self.e.debug_read("route", a, b - a), self.ref.route[a:b], "route (window)")
            _same(self.e.debug_read("state", a, b - a), self.ref.state[a:b], "state (window)")


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape or (got != want).any():
        bad = np.nonzero(got != want)[0] if got.shape == want.shape else []
        k = bad[:6].tolist()
        raise AssertionError(f"{what}: {len(bad)} rows differ, first {k}: got {[hex(int(got[i])) for i in k]} "
                             f"want {[hex(int(want[i])) for i in k]}")


# ------------------------------------------------------------------------------------------------------- batches
def records(rng, n, *, agents=None, zero_ids=0.002):
    """n records of random bytes (all 512 B), with a random agent of NAMES, the replay bit clear, lengths that mostly fit and
    sometimes sit on or just past the 416 B payload or at the u16 / u32 extremes, max_retries anywhere in 0..255"""
    r = np.frombuffer(rng.integers(0, 256, n * 512, dtype=np.uint8).tobytes(), dtype=A.record_dtype).copy()
    r["agent_id"] = np.array(NAMES, dtype="S32")[rng.choice(len(NAMES), n, p=P_NAMES / P_NAMES.sum()) if agents is None else agents]
    r["flags"] &= ~np.uint32(K.AGR_F_REPLAY)
    u = rng.random(n)
    tot = rng.integers(0, 417, n)
    tot = np.where(u < 0.05, 416, np.where(u < 0.08, 417, tot))
    p = rng.integers(0, tot + 1)
    q = rng.integers(0, tot - p + 1)
    r["path_len"], r["hdr_len"], r["body_len"] = p, q, tot - p - q
    ext = np.nonzero((u > 0.08) & (u < 0.1))[0]
    r["path_len"][ext[0::3]], r["hdr_len"][ext[0::3]], r["body_len"][ext[0::3]] = 0xFFFF, 0xFFFF, 0xFFFFFFFF
    r["path_len"][ext[1::3]], r["hdr_len"][ext[1::3]], r["body_len"][ext[1::3]] = 0, 0, 0xFFFFFFFF
    r["path_len"][ext[2::3]], r["hdr_len"][ext[2::3]], r["body_len"][ext[2::3]] = 0xFFFF, 0, 0
    r["max_retries"] = np.where(u > 0.9, 0, np.where(u > 0.85, 255, r["max_retries"]))
    r["seq"] = rng.integers(1 << 20, 1 << 40, n, dtype=np.uint64)
    z = rng.random(n) < zero_ids
    r["request_id"][z] = 0
    return r


def storable(r):
    return np.isin(r["agent_id"], FOUND) & ((r["flags"] & K.AGR_F_REPLAY) == 0) & \
        (r["path_len"].astype(np.int64) + r["hdr_len"] + r["body_len"].astype(np.int64) <= k1ref.PAYLOAD)


def make_storable(r, i, agent=None):
    r["flags"][i] &= ~np.uint32(K.AGR_F_REPLAY)
    r["path_len"][i], r["hdr_len"][i], r["body_len"][i] = 10, 20, 30
    r["agent_id"][i] = agent or FOUND[int(i) % len(FOUND)]
    if not r["request_id"][i].any():
        r["request_id"][i][0] = 1


def decorate(rig, rng, r, first, *, replays=0.05, dups=0.01, triples=0):
    """Replays (every target relation) and, with caller ids, duplicate ids and dedupe triples, placed in r (arrival first..)"""
    n = len(r)
    taken = np.zeros(n, dtype=bool)
    ref = rig.ref
    w = k1ref.grid(n, sms())[1]

    def id_of(L):
        if rig.mode == "mint":
            return np.frombuffer(mint_bytes(int(L), SECRET), dtype=np.uint8)
        return r["request_id"][L - first] if L >= first else ref.idb[L]

    def agent_of(L):
        if L >= first:
            return r["agent_id"][L - first]
        s = int(ref.slot[L])
        return next((a for a, v in rig.slots.items() if v == s), LONG)

    if rig.mode == "hash" and n > 64:
        # triples: A < B carry the same id, R > A replays it, R in A's 32-row group or (every other triple) in a later one; B in
        # the same tile, another tile of A's warp, or another CTA.  Whoever's CAS lands first, A owns the id and R is a hit.
        for k in range(triples):
            a = int(rng.integers(0, n - 40))
            if a % 32 > 29:
                a -= 2
            rr = a + int(rng.integers(1, 32 - a % 32)) if k % 2 == 0 else a + 32 - a % 32 + int(rng.integers(0, 40))
            kind = k % 3
            if kind == 0:
                b = a + int(rng.integers(1, 32 - a % 32))
            elif kind == 1:
                b = a + 32 * w
            else:
                b = a + 32 * int(rng.integers(k1ref.WARPS, max(k1ref.WARPS + 1, w)))
            if b >= n or rr >= n or rr == b or taken[[a, b, rr]].any():
                continue
            make_storable(r, a); make_storable(r, b)
            r["request_id"][b] = r["request_id"][a]
            r["flags"][rr] |= K.AGR_F_REPLAY
            r["replay_of"][rr] = r["request_id"][a]
            r["agent_id"][rr] = r["agent_id"][a]
            taken[[a, b, rr]] = True
        # duplicate ids: same tile, another tile of the same warp, another CTA, an earlier batch
        cand = np.nonzero(storable(r) & ~taken)[0]
        for _ in range(int(dups * n)):
            j = int(rng.choice(cand))
            kind = int(rng.integers(0, 4))
            i = j + int(rng.integers(1, 32)) if kind == 0 else j + 32 * w if kind == 1 else int(rng.integers(j + 1, n + 1)) if kind == 2 else -1
            if kind == 3:
                if ref.head == ref.tail:
                    continue
                src = int(rng.integers(ref.tail, ref.head))
                i, j = j, None
                if taken[i]:
                    continue
                r["request_id"][i] = ref.idb[src]
                taken[i] = True
                continue
            if i >= n or taken[i] or taken[j]:
                continue
            r["request_id"][i] = r["request_id"][j]
            taken[[i, j]] = True
    # replays
    for _ in range(int(replays * n)):
        i = int(rng.integers(0, n))
        if taken[i]:
            continue
        kind = int(rng.integers(0, 8))
        if kind == 0 and ref.head > ref.tail:                       # an earlier batch
            L = int(rng.integers(ref.tail, ref.head))
        elif kind == 1 and ref.tail > 0:                            # a released row (or a row of the previous lap)
            L = int(rng.integers(max(0, ref.tail - 5000), ref.tail))
        elif kind == 2 and i % 32:                                  # the same tile, earlier
            L = first + i - int(rng.integers(1, i % 32 + 1))
        elif kind == 3 and i >= 32:                                 # an earlier tile
            L = first + int(rng.integers(0, i - i % 32))
        elif kind == 4 and i + 1 < n:                               # a later row
            L = first + int(rng.integers(i + 1, n))
        elif kind == 5:                                             # itself
            L = first + i
        elif kind == 6:                                             # an id nobody carries
            r["flags"][i] |= K.AGR_F_REPLAY
            r["replay_of"][i] = rng.integers(0, 256, 16, dtype=np.uint8)
            taken[i] = True
            continue
        else:
            L = first + int(rng.integers(0, i + 1))
        r["flags"][i] |= K.AGR_F_REPLAY
        r["replay_of"][i] = id_of(L)
        if rng.random() < 0.85:
            r["agent_id"][i] = agent_of(L)
        taken[i] = True
    if rig.mode == "mint" and n > 1 and not taken[0] and not taken[n - 1]:
        # the batch's first row and a replay of it: the earliest target that counts as "this batch" (k1_begin's olog < first_log)
        make_storable(r, 0)
        r["flags"][n - 1] |= K.AGR_F_REPLAY
        r["replay_of"][n - 1] = id_of(first)
        r["agent_id"][n - 1] = r["agent_id"][0]
        taken[[0, n - 1]] = True
    if rng.random() < 0.5 and n > 2:                                # an untracked replay (replay_of zero)
        i = int(np.nonzero(~taken)[0][0]) if (~taken).any() else 0
        r["flags"][i] |= K.AGR_F_REPLAY
        r["replay_of"][i] = 0
    return r


# ------------------------------------------------------------------------------------------------------- drivers
def ingest(rig, r, path="ex"):
    """one batch through `path`; checks everything against the reference.  Returns the reference output."""
    e, n = rig.e, len(r)
    launches = e.stats()["k1_launches"]
    v = None
    if path == "ex":
        v, ids = np.zeros(n, dtype=A.verdict_dtype), np.zeros((n, 16), dtype=np.uint8)
        first = e.ingest_ex(r, v, ids)
    elif path == "rows":
        first = e.reserve_rows(n)
        e.fill_rows(first, r)
        v = e.ingest_rows(first, n)
    elif path == "async":
        first = e.reserve_rows(n)
        e.fill_rows(first, r)
        e.ingest_rows_async(first, n)
        e.sync()
    elif path == "chunked":
        v, first = e.ingest(r)
    out = rig.ref.ingest(r, first)
    assert out["first"] == first
    rig.check_batch(out, r, v)
    if path == "ex":
        want = rig.e.mint_ids(first, n) if rig.mode == "mint" else r["request_id"]
        assert ids.tobytes() == np.ascontiguousarray(want).tobytes(), "ids"
    if path in ("ex", "rows", "async") and not e.stats()["svc_ops"]:
        got = e.stats()["k1_launches"] - launches
        chunks = -(-n // (1 << 17)) if path == "ex" else 1             # agr_ingest_ex runs K1 per 128 Ki-record chunk
        assert got == chunks * (1 if (path == "async" and rig.mode == "mint") else 2), (path, got)
    return out


def stream(rig, sizes, rng, path="ex", **kw):
    for n in sizes:
        r = decorate(rig, rng, records(rng, n), rig.ref.head, **kw)
        ingest(rig, r, path)
    rig.check_lists()
    rig.check_window()


# ------------------------------------------------------------------------------------------------------- tests
def schedule_sizes():
    w = W()
    return [31, 1, 32, 33, 14 * 32 - 1, 14 * 32 + 1, 32 * (w - 1), 32 * w, 32 * w + 5, 32 * (2 * w + 1), 32 * 3 * w, 1 << 20]


@pytest.mark.parametrize("mode", MODES)
def test_schedule(mode):
    """every tile-count edge of the grid, and first rows at 0, 1 and 31 mod 32"""
    sizes = schedule_sizes()
    firsts = np.cumsum([0] + sizes[:-1]) % 32
    assert {0, 1, 31} <= set(firsts.tolist())
    rng = np.random.default_rng(11)
    rig = Rig(mode, sum(sizes) + 64)
    try:
        stream(rig, sizes, rng, triples=200)
        for n in sizes:
            c, w = k1ref.grid(n, sms())
            assert c <= sms()
        print(f"schedule: {sms()} SMs, W = {W()}; rounds per warp up to {k1ref.schedule(1 << 20, sms())[1].max() + 1}")
    finally:
        rig.close()


@pytest.mark.parametrize("extra", [0, 1, 31])
@pytest.mark.parametrize("mode", MODES)
def test_slab_end(mode, extra):
    """slab_rows = 32k + extra; the last batch ends exactly at the slab end, and a tile straddles the 4096-row chunk edge"""
    rows = 32 * 200 + extra
    sizes = [4090, 1, 700, rows - 4791]
    rng = np.random.default_rng(20 + extra)
    rig = Rig(mode, rows)
    try:
        stream(rig, sizes, rng, triples=20)
        assert rig.ref.head == rows
    finally:
        rig.close()


@pytest.mark.parametrize("mode", MODES)
def test_ring_laps(mode):
    """a ring of 32k + 31 rows over five laps: pad rows at a lap's end, batches at physical row 0, arrival numbers far from the
    row.  Between laps the sweep drops the older 60 % of the live rows (created_at rises with arrival), so the rest stays live
    across the lap and its pad: replays name live rows of the previous lap as well as released ones"""
    rows = 32 * 300 + 31
    rng = np.random.default_rng(30)
    rig = Rig(mode, rows, ring=True)
    pads = 0
    try:
        ttl = 1 << 20
        for lap in range(5):
            sizes = [2000, 33, 1000 + 7 * lap, 1, 900]
            for n in sizes:
                first = rig.ref.head
                r = decorate(rig, rng, records(rng, n), first, triples=10)
                r["seq"] = (1 << 30) + 16 * (first + np.arange(n, dtype=np.uint64))
                at = first % rows
                out = ingest(rig, r)
                if at + n > rows:
                    assert out["first"] % rows == 0 and out["first"] == first + rows - at   # padded to the next lap
                    pads += 1
            rig.check_lists()
            rig.check_window()
            cut = rig.ref.tail + (rig.ref.head - rig.ref.tail) * 6 // 10
            now = (1 << 30) + 16 * cut + ttl
            assert rig.e.expire(now, ttl) == rig.ref.expire(now, ttl)
            assert rig.e.reclaim() == rig.ref.reclaim()
            assert rig.ref.tail < rig.ref.head
            rig.check_counters()
            rig.check_lists()
        assert rig.ref.tail > rows and pads >= 2
    finally:
        rig.close()


@pytest.mark.parametrize("mode", MODES)
def test_persistence_off(mode):
    rng = np.random.default_rng(40)
    rig = Rig(mode, 1 << 14, persistence=False)
    try:
        stream(rig, [1000, 33, 2000], rng)
        assert rig.ref.ctr["stored"] == 0
    finally:
        rig.close()


def test_small_index_collisions():
    """caller ids: table_slots the smallest power of two >= 1.25 x slab_rows, ids that share the last home slots so their
    probe chains run across the table's end, duplicates of them, zero ids"""
    rows = 3000
    slots = 4096
    rng = np.random.default_rng(50)
    pool = rng.integers(0, 256, (200000, 16), dtype=np.uint8)
    home = k1ref.hash_id(pool) & np.uint64(slots - 1)
    coll = pool[home >= slots - 3][:40]
    assert len(coll) >= 30
    rig = Rig("hash", rows, table_slots=slots)
    try:
        for n in (900, 1000, 1100):
            r = records(rng, n, zero_ids=0.01)
            pos = rng.choice(n, 2 * len(coll), replace=False)
            for k, p in enumerate(pos):
                make_storable(r, p)
                r["request_id"][p] = coll[k % len(coll)]      # each colliding id twice a batch (and again next batch)
            r = decorate(rig, rng, r, rig.ref.head, dups=0.01, triples=40)
            ingest(rig, r)
        rig.check_lists()
        rig.check_window()
    finally:
        rig.close()


@pytest.mark.parametrize("mode", MODES)
def test_back_to_back(mode):
    """batches launched through agr_ingest_rows_async with no sync in between (the next K1 starts under programmatic dependent
    launch), each replaying rows of the one before"""
    rng = np.random.default_rng(60)
    sizes = [32 * W() + 17, 5000, 1, 32 * 2 * W() + 3, 40000]
    rig = Rig(mode, sum(sizes) + 64)
    try:
        e = rig.e
        batches = []
        for n in sizes:                                             # every batch in its rows first (agr_fill_rows synchronises)
            first = e.reserve_rows(n)
            r = decorate(rig, rng, records(rng, n), first, replays=0.1, triples=50)
            e.fill_rows(first, r)
            batches.append((first, r, rig.ref.ingest(r, first)))
        for first, r, _ in batches:
            e.ingest_rows_async(first, len(r))
        e.sync()
        for first, r, out in batches:
            rig.check_batch(out, r)
        assert e.stats()["k1_launches"] == len(sizes) * (1 if mode == "mint" else 2)
        rig.check_lists()
        rig.check_window()
    finally:
        rig.close()


PATHS = ("async", "rows", "ex", "chunked")


@pytest.mark.parametrize("mode", MODES)
def test_output_paths(mode):
    """the same batches through the four entry points: identical words everywhere, and 1 or 2 K1 launches per batch.  Caller
    ids: one batch without duplicate ids (k1_post visits the marked rows only) and one with (every row)"""
    rng = np.random.default_rng(70)
    sizes = [3000, (1 << 17) + 4000, 700]
    recs = []
    probe = Rig(mode, sum(sizes) + 64)
    try:
        for k, n in enumerate(sizes):
            r = decorate(probe, rng, records(rng, n, zero_ids=0 if k == 0 else 0.002), probe.ref.head,
                         dups=0 if k == 0 else 0.01, triples=0 if k == 0 else 30)
            probe.ref.ingest(r)
            recs.append(r)
    finally:
        probe.close()
    words = {}
    for path in PATHS:
        rig = Rig(mode, sum(sizes) + 64)
        try:
            for r in recs:
                ingest(rig, r, path)
            rig.check_lists()
            head = rig.ref.head
            words[path] = [rig.e.debug_read(w, 0, head).tobytes() for w in ("route", "state", "cksum")]
        finally:
            rig.close()
    for path in PATHS[1:]:
        assert words[path] == words[PATHS[0]], path


def _service_rig(mode, ring):
    return Rig(mode, 32 * 400 + 31 if ring else 1 << 14, ring=ring, combine=True)


def _tickets(rig, r):
    """records submitted one ticket each, all before the first is collected; the reference takes each run of consecutive rows"""
    e = rig.e
    ts = [e.submit_ingest(r[i]) for i in range(len(r))]
    res = [e.poll(t) for t in ts]
    assert all(x["result"] == 0 for x in res)
    rid = np.array([x["rid"] for x in res], dtype=np.int64)
    order = np.argsort(rid, kind="stable")
    assert (order == np.arange(len(r))).all(), "rows follow submission order"
    cuts = np.nonzero(np.diff(rid) != 1)[0] + 1
    for a, b in zip(np.concatenate([[0], cuts]), np.concatenate([cuts, [len(r)]])):
        out = rig.ref.ingest(r[a:b], int(rid[a]))
        got = np.concatenate([x["verdict"] for x in res[a:b]])
        rig.check_batch(out, r[a:b], got)
        want = rig.e.mint_ids(int(rid[a]), b - a) if rig.mode == "mint" else r["request_id"][a:b]
        assert b"".join(x["request_id"] for x in res[a:b]) == np.ascontiguousarray(want).tobytes()


@pytest.mark.parametrize("ring", [False, True], ids=["append", "ring"])
@pytest.mark.parametrize("mode", MODES)
def test_service_kernel(mode, ring):
    """the record half of k_svc: calls of n <= 32 records and tickets many of which share a service batch, with the same
    relations as above, checked word by word, including k_svc's own checksum"""
    rng = np.random.default_rng(80 + ring)
    rig = _service_rig(mode, ring)
    try:
        for n in (1, 7, 31, 32, 32, 20):
            r = decorate(rig, rng, records(rng, n), rig.ref.head, replays=0.2)
            ingest(rig, r)
        for k in range(6):
            r = records(rng, 120)
            r = decorate(rig, rng, r, rig.ref.head, replays=0.1, dups=0.05, triples=20)
            _tickets(rig, r)
        rig.check_lists()
        rig.check_window()
    finally:
        rig.close()


@pytest.mark.parametrize("mode", MODES)
def test_service_kernel_promoted_owner(mode):
    """A row A that is the only stored row of its chunk, in a service batch with a later row B of the same caller id (B in the
    next chunk) and a replay R of it.  Whichever CAS lands first, A ends up stored and R is a hit.  Before each group, a sweep
    leaves the chunk's bound at "no stored row", so the bound k_svc leaves must cover A; a release must stop at A, and a sweep
    when A is due must drop it.  32 groups, A on lanes 31, 30, 15 and 0 of its warp (B on the next lane: another warp for 31)."""
    rows = k1ref.CHUNK * 33
    rig = Rig(mode, rows, ring=True, combine=True)
    try:
        rng = np.random.default_rng(90)
        for g in range(32):
            j = (31, 30, 15, 0)[g % 4]
            a_row = k1ref.CHUNK * (g + 1) - 1
            start = a_row - j
            fill = records(rng, start - rig.ref.head, agents=np.full(start - rig.ref.head, NAMES.index(LONG)))
            fill["seq"] = 1
            assert len(fill) > 32
            ingest(rig, fill)                                       # not found (batch path): bounds at the fillers' time
            assert rig.e.expire(1 << 30, 1) == rig.ref.expire(1 << 30, 1)   # ... swept: "no stored row"
            assert rig.e.reclaim() == rig.ref.reclaim()
            r = records(rng, 64, agents=np.full(64, NAMES.index(LONG)))
            r["seq"] = 1 << 50
            a, b, rr = j, j + 1, j + 5
            make_storable(r, a, b"agent-run"); make_storable(r, b, b"agent-run")
            r["request_id"][b] = r["request_id"][a]
            r["seq"][a], r["seq"][b] = (1 << 40) + g, 1 << 41
            r["flags"][rr] |= K.AGR_F_REPLAY
            r["replay_of"][rr] = r["request_id"][a] if mode == "hash" else np.frombuffer(mint_bytes(a_row, SECRET), dtype=np.uint8)
            r["agent_id"][rr] = b"agent-run"
            _tickets(rig, r)                                         # words, verdicts and the chunk bound (check_cmin)
            assert rig.ref.state[a_row] & k1ref.ST_STORED and rig.ref.route[a_row + 5] >> 26 & K.AGR_VF_KNOWN
            assert rig.e.reclaim() == rig.ref.reclaim() and rig.ref.tail <= a_row   # the earliest stored A stops it
            rig.check_window()
        rig.check_lists()
        now, ttl = 1 << 41, 1 << 39                                  # every A is due, nothing else is stored
        assert rig.e.expire(now, ttl) == rig.ref.expire(now, ttl) == 32
        assert rig.e.reclaim() == rig.ref.reclaim()
        rig.check_counters()
    finally:
        rig.close()


@pytest.mark.parametrize("mode", MODES)
def test_chunk_straddle_bound(mode):
    """a tile across a chunk edge whose rows past the edge hold the earliest created_at of the next chunk: the tile must lower
    both chunks' bounds (k1_note_time's second atomicMin)"""
    rig = Rig(mode, k1ref.CHUNK * 3, ring=True)
    rng = np.random.default_rng(95)
    try:
        for first in (k1ref.CHUNK - 16, 2 * k1ref.CHUNK - 1):
            n0 = first - rig.ref.head
            ingest(rig, records(rng, n0, agents=np.full(n0, NAMES.index(LONG))))
            r = records(rng, 96, agents=np.full(96, NAMES.index(b"agent-run")))
            for i in range(96):
                make_storable(r, i, b"agent-run")
            edge = (first // k1ref.CHUNK + 1) * k1ref.CHUNK - first     # first row of the next chunk, inside tile 0
            r["seq"] = np.where(np.arange(96) < edge, 1 << 35, 1 << 36)
            r["seq"][edge:32] = 1 << 33                                  # the next chunk's earliest rows sit in tile 0
            ingest(rig, r)
            rig.check_cmin(first, 96)
    finally:
        rig.close()
