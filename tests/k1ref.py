"""Plain reference of the fixed-stride ingest (K1: k1_ingest_tma + k1_post, and the record half of the service kernel), written
from the reference server's proxyToAgentHandler + StoreRequest (oracle/model.py) and the engine's documented extensions to it
(caller ids unique per engine, the 416 B payload, minted ids, the ring).  Nothing here comes from the engine: it is built from
the records, the agent table (names, statuses and the slots agr_agent_slot reports) and the configuration.  tests/test_k1_ref.py
checks it against oracle/model.py, the C restatement (oracle/cpu_ref.c) and hand-worked rows.

  dedupe_hits   the dedupe-hit rule alone (AGR_VF_KNOWN), over a whole stream
  Ref           every word K1 leaves behind, batch after batch: verdicts, route / state / checksum / mtime words, the counters,
                the pending list of every agent, who owns each caller id and how many ids the dedupe index holds; plus the
                ring's expire and reclaim as far as K1's words are concerned
  cksum         the record checksum over all 128 words
  grid          CTAs, warps, and which tiles each warp runs
  hash_id, hash_agent   numpy restatements of agr_hash_id / agr_hash_agent, only to BUILD colliding ids and agent names

The rules (a row is one record of a batch, L its arrival number):
  - not found: its agent id is all zero, unknown or dropped -> NOT_FOUND, 404, slot 0x7fffff, no flags, state 0;
  - stored: persistence is on, it is not replay-flagged, path + headers + body <= 416 (else BAD_LEN), and (caller ids) its id is
    non-zero and no row of earlier arrival still in the dedupe index carries it (else DUP_ID); minted ids never collide;
  - replay-flagged (found): REPLAY; TRACKED when replay_of is non-zero; KNOWN when replay_of names a row of earlier arrival that is
    stored (at the end of this row's batch) with the same agent slot.  Caller ids: the row the index names for the id (its owner).
    Minted ids: the row the id was minted for, if it is in the live window;
  - code: a running agent -> FORWARD (0); else QUEUED (202) when persistence is on and the row is stored or a tracked replay,
    UNAVAILABLE (503) otherwise;
  - state of a stored row: PENDING | INQ | STORED | max_retries << 16 (0 reads 3), INFLIGHT when its agent is running."""
import numpy as np

from agentainer_lab_b200 import constants as K

PAYLOAD = 512 - 96             # payload bytes of a fixed-stride record
TILE = 32                      # records per K1 tile
WARPS = 14                     # warps per K1 CTA
CHUNK = 4096                   # rows per TTL-sweep chunk
RT_SLOT_NONE = 0x7FFFFF
ST_INQ, ST_INFLIGHT, ST_STORED = 0x8, 0x10, 0x20
HTTP = {K.AGR_V_FORWARD: 0, K.AGR_V_QUEUED: 202, K.AGR_V_UNAVAILABLE: 503, K.AGR_V_NOT_FOUND: 404}
COUNTERS = ("ingested", "stored", "replay_flagged", "dedupe_hits", "forwarded", "queued", "unavailable", "not_found", "dup_ids",
            "malformed")


def dedupe_hits(recs, ids, registered, persistence=True):
    """recs: records in arrival order (every batch of a stream, one after the other); ids: each row's request id (the minted
    ids with AGR_CFG_MINT_IDS, else recs["request_id"]); registered: agent ids (str) that are registered and not dropped.
    Returns (known, stored), one bool per row."""
    n = len(recs)
    reg = {a.encode() for a in registered}
    idb = np.ascontiguousarray(ids, dtype=np.uint8).tobytes()
    rob = np.ascontiguousarray(recs["replay_of"]).tobytes()
    agents = recs["agent_id"].tolist()
    replay = ((recs["flags"] & K.AGR_F_REPLAY) != 0).tolist()
    fits = (recs["path_len"].astype(np.int64) + recs["hdr_len"] + recs["body_len"] <= PAYLOAD).tolist()
    zero = bytes(16)
    known, stored = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    owner = {}                                                     # id -> agent of the stored row that carries it
    for i in range(n):
        if agents[i] not in reg:
            continue
        if replay[i]:
            t = rob[16 * i:16 * i + 16]
            known[i] = t != zero and owner.get(t) == agents[i]
        elif persistence and fits[i]:
            rid = idb[16 * i:16 * i + 16]
            if rid != zero and rid not in owner:
                owner[rid] = agents[i]
                stored[i] = True
    return known, stored


# ------------------------------------------------------------------------------------------------------- hashes
def fmix64(k):
    k = np.asarray(k, dtype=np.uint64)
    with np.errstate(over="ignore"):
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xFF51AFD7ED558CCD)
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(0xC4CEB9FE1A85EC53)
        return k ^ (k >> np.uint64(33))


def hash_id(ids):
    """agr_hash_id of n x 16 id bytes (placement in the dedupe index is hash & table_mask)"""
    w = np.ascontiguousarray(ids, dtype=np.uint8).reshape(-1, 16).view("<u8")
    with np.errstate(over="ignore"):
        return fmix64(w[:, 0] ^ (w[:, 1] * np.uint64(0x9E3779B97F4A7C15)))


def hash_agent(names):
    """agr_hash_agent of agent ids (bytes, up to 32, NUL padded) (placement in the agent table is hash & amask)"""
    a = np.zeros((len(names), 32), dtype=np.uint8)
    for i, s in enumerate(names):
        a[i, :len(s)] = np.frombuffer(s, dtype=np.uint8)
    w = a.view("<u8")
    with np.errstate(over="ignore"):
        h = w[:, 0] * np.uint64(0x9E3779B97F4A7C15)
        h ^= (w[:, 1] + np.uint64(0x165667B19E3779F9)) * np.uint64(0xC2B2AE3D27D4EB4F)
        h ^= (w[:, 2] + np.uint64(0x27D4EB2F165667C5)) * np.uint64(0xFF51AFD7ED558CCD)
        h ^= (w[:, 3] + np.uint64(0x85EBCA77C2B2AE63)) * np.uint64(0xC4CEB9FE1A85EC53)
    return fmix64(h)


# ------------------------------------------------------------------------------------------------------- grid
def grid(n, sms):
    """(CTAs, warps in the grid) of a K1 launch over n records: min(SMs, ceil(tiles / 14)) CTAs of 14 warps"""
    tiles = -(-n // TILE)
    ctas = max(1, min(sms, -(-tiles // WARPS)))
    return ctas, ctas * WARPS


def schedule(n, sms):
    """per tile t of an n-record batch: (warp, round) — warp t mod W runs it in its round t // W"""
    _, w = grid(n, sms)
    t = np.arange(-(-n // TILE))
    return t % w, t // w


def cksum(recs):
    """Per record: (sum_k (k + 1) w_k mod 2^32) << 32 | (sum_k w_k mod 2^32) over its 128 little-endian u32 words."""
    b = np.ascontiguousarray(recs).view(np.uint8).reshape(-1, 512)
    out = np.zeros(len(b), dtype=np.uint64)
    k = np.arange(1, 129, dtype=np.uint64)
    for a in range(0, len(b), 1 << 15):
        w = b[a:a + (1 << 15)].view("<u4").astype(np.uint64)
        s0 = w.sum(axis=1) & np.uint64(0xFFFFFFFF)
        s1 = (w @ k) & np.uint64(0xFFFFFFFF)
        out[a:a + len(w)] = (s1 << np.uint64(32)) | s0
    return out


# ------------------------------------------------------------------------------------------------------- the engine's words
class Ref:
    """K1's effect on one engine.  agents: {name: (slot, status)} with status an AGR_AGENT_* code or "dropped" (slots from
    Engine.agent_slot).  mint: AGR_CFG_MINT_IDS with id_secret `secret` (shard 0, generation 1)."""

    def __init__(self, agents, *, mint, secret=0, persistence=True):
        self.agents = {(n.encode() if isinstance(n, str) else n): v for n, v in agents.items()}
        self.mint, self.secret, self.persistence = mint, secret, persistence
        cap = 1 << 10
        self.state = np.zeros(cap, dtype=np.uint32)
        self.route = np.zeros(cap, dtype=np.uint32)
        self.slot = np.full(cap, RT_SLOT_NONE, dtype=np.int64)
        self.created = np.zeros(cap, dtype=np.uint64)
        self.mtime = np.zeros(cap, dtype=np.uint64)             # last SET after the ingest (a completion); 0: none
        self.idb = np.zeros((cap, 16), dtype=np.uint8)           # caller ids (hash mode)
        self.head = 0                                            # rows handed out (arrival numbers < head)
        self.tail = 0                                            # rows released (ring)
        self.owner = {}                                          # caller id -> arrival number of the row the index names
        self.index = set()                                       # ids the dedupe index holds
        self.ctr = dict.fromkeys(COUNTERS, 0)
        self.pending = {}                                        # slot -> arrival numbers of its stored rows, in order

    def _grow(self, need):
        cap = len(self.state)
        if need <= cap:
            return
        new = max(need, 2 * cap)
        for name in ("state", "route", "slot", "created", "mtime", "idb"):
            a = getattr(self, name)
            b = np.zeros((new,) + a.shape[1:], dtype=a.dtype) if name != "slot" else np.full(new, RT_SLOT_NONE, dtype=np.int64)
            b[:cap] = a
            setattr(self, name, b)

    def agent_of(self, recs):
        """(slot, status) per row; slot RT_SLOT_NONE and status -1 for a row whose agent is not found"""
        names = recs["agent_id"].tolist()
        slot = np.full(len(recs), RT_SLOT_NONE, dtype=np.int64)
        status = np.full(len(recs), -1, dtype=np.int64)
        for a in set(names):
            v = self.agents.get(a)
            if a == b"" or v is None or v[1] == "dropped":
                continue
            m = recs["agent_id"] == a
            slot[m], status[m] = v
        return slot, status

    def ingest(self, recs, first=None):
        """One K1 batch of records at arrival numbers first.. (default: the next ones).  Returns a dict of per-row arrays:
        verdict (agr_verdict), route, state, cksum, created, stored, known, and first."""
        n = len(recs)
        first = self.head if first is None else first
        assert first >= self.head
        L = first + np.arange(n, dtype=np.int64)
        self._grow(first + n)
        slot, status = self.agent_of(recs)
        found = slot != RT_SLOT_NONE
        running = status == K.AGR_AGENT_RUNNING
        replay = (recs["flags"] & K.AGR_F_REPLAY) != 0
        ro = np.ascontiguousarray(recs["replay_of"])
        tracked_rep = found & replay & ro.any(axis=1)
        want = found & self.persistence & ~replay
        lens = recs["path_len"].astype(np.int64) + recs["hdr_len"] + recs["body_len"].astype(np.int64)
        bad = want & (lens > PAYLOAD)
        cand = want & ~bad
        stored = cand.copy()
        if not self.mint:
            ids = np.ascontiguousarray(recs["request_id"])
            self.idb[first:first + n] = ids
            stored &= ids.any(axis=1)                            # a zero caller id is never stored
            idbytes = ids.tobytes()
            for i in np.nonzero(stored)[0].tolist():
                k = idbytes[16 * i:16 * i + 16]
                self.index.add(k)
                if k in self.owner:                              # the lowest arrival that carries the id owns it
                    stored[i] = False
                else:
                    self.owner[k] = first + i
        dup = cand & ~stored
        self.slot[first:first + n] = slot
        self.created[first:first + n] = recs["seq"]
        mx = recs["max_retries"].astype(np.uint32)
        mx = np.where(mx == 0, 3, mx).astype(np.uint32)
        st = (K.AGR_ST_PENDING | ST_INQ | ST_STORED | (mx << 16) | np.where(running, ST_INFLIGHT, 0)).astype(np.uint32)
        self.state[first:first + n] = np.where(stored, st, 0)
        # dedupe hits: the target's status at the end of this batch
        known = np.zeros(n, dtype=bool)
        rob = ro.tobytes()
        for i in np.nonzero(tracked_rep)[0].tolist():
            t = self._target(rob[16 * i:16 * i + 16], first + n)
            known[i] = (t is not None and t < first + i and self.slot[t] == slot[i] and bool(self.state[t] & ST_STORED))
        tracked = stored | tracked_rep
        code = np.where(running, K.AGR_V_FORWARD,
                        np.where(self.persistence & tracked, K.AGR_V_QUEUED, K.AGR_V_UNAVAILABLE))
        code = np.where(found, code, K.AGR_V_NOT_FOUND)
        fl = (np.where(stored, K.AGR_VF_STORED | K.AGR_VF_TRACKED, 0) | np.where(bad, K.AGR_VF_BAD_LEN, 0)
              | np.where(dup, K.AGR_VF_DUP_ID, 0) | np.where(found & replay, K.AGR_VF_REPLAY, 0)
              | np.where(tracked_rep, K.AGR_VF_TRACKED, 0) | np.where(known, K.AGR_VF_KNOWN, 0))
        route = (np.where(found, slot, RT_SLOT_NONE) | (code << 23) | (fl << 26)).astype(np.uint32)
        self.route[first:first + n] = route
        v = np.zeros(n, dtype=[("code", "u1"), ("flags", "u1"), ("http_status", "<u2"), ("agent_slot", "<u4")])
        v["code"], v["flags"], v["agent_slot"] = code, fl, np.where(found, slot, RT_SLOT_NONE)
        v["http_status"] = np.vectorize(HTTP.get, otypes=[np.int64])(code) if n else 0
        c = self.ctr
        c["ingested"] += n
        c["not_found"] += int((~found).sum())
        c["stored"] += int(stored.sum())
        c["malformed"] += int(bad.sum())
        c["dup_ids"] += int(dup.sum())
        c["replay_flagged"] += int((found & replay).sum())
        c["dedupe_hits"] += int(known.sum())
        c["forwarded"] += int((code == K.AGR_V_FORWARD).sum())
        c["queued"] += int((code == K.AGR_V_QUEUED).sum())
        c["unavailable"] += int((code == K.AGR_V_UNAVAILABLE).sum())
        for s in np.unique(slot[stored]).tolist():
            self.pending.setdefault(s, []).extend(L[stored & (slot == s)].tolist())
        self.head = first + n
        return dict(first=first, verdict=v, route=route, state=self.state[first:first + n].copy(), cksum=cksum(recs),
                    created=recs["seq"].astype(np.uint64), stored=stored, known=known, found=found)

    def _target(self, key, head):
        """arrival number of the row a replay_of names, or None"""
        if key == bytes(16):
            return None
        if not self.mint:
            return self.owner.get(key)
        from mintref import decode, split
        lo, hi = split(key)
        return decode(lo, hi, self.secret, 0, 1, self.tail, head)

    # ---- views
    def index_used(self):
        return len(self.index)

    def pending_rows(self, slot):
        """arrival numbers of an agent's stored rows in list order"""
        return [r for r in self.pending.get(slot, []) if r >= self.tail and self.state[r] & ST_STORED]

    def stored_rows(self):
        lo = self.tail
        return lo + np.nonzero(self.state[lo:self.head] & ST_STORED)[0]

    # ---- the ring's TTL sweep and release
    def touch(self, rows, now):
        """a completion (StoreResponse, MarkRequestFailed) of these rows at time now: their last SET moves to now"""
        self.mtime[np.asarray(rows, dtype=np.int64)] = now

    def expire(self, now, ttl):
        """stored rows whose last SET (the completion's time, else created_at) is ttl or more before now lose ST_STORED"""
        r = self.stored_rows()
        t = np.maximum(np.where(self.mtime[r] != 0, self.mtime[r], self.created[r]), 1)
        gone = r[(now >= t) & (now - t >= ttl)]
        self.state[gone] &= ~np.uint32(ST_STORED)
        return len(gone)

    def reclaim(self):
        """the tail moves to the first row that still holds a stored record; when rows are released, the dedupe index is
        rebuilt from the stored rows left"""
        r = self.stored_rows()
        new = int(r[0]) if len(r) else self.head
        released, self.tail = new - self.tail, new
        if released and not self.mint:
            self._reindex(r)
        return released

    def restore(self, ring):
        """the dedupe index after a snapshot of this state is restored (caller ids): a ring's is rebuilt as a release rebuilds
        it, from the window's rows that hold a record, so the ids of rows that expired since the last release leave it; an
        append-only engine's index never shrinks, and it comes back as it was.  Returns index_used()."""
        if ring and not self.mint:
            self._reindex(self.stored_rows())
        return self.index_used()

    def _reindex(self, rows):
        self.owner, self.index = {}, set()
        for x in rows.tolist():
            k = self.idb[x].tobytes()
            self.owner.setdefault(k, x)
            self.index.add(k)
