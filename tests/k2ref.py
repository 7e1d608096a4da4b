"""Plain restatement of K2 (agr_complete, agr_complete_ex and the outcome half of the service kernel) for the edge tests of
tests/test_k2_edges_gpu.py.

Built only from what a test feeds the engine: the rows it ingested (agent, id, max_retries, created_at, whether the agent was
running), the agents it registered and dropped, the rows it expired and released, and the outcomes in call order.  The rules
are oracle/model.py's Manager (StoreResponse requests.go:120-194, MarkRequestFailed :228-275) on the engine's row words:
  * an outcome names a row when its id is nonzero, the row holds a stored record and the row's agent is the outcome's agent
    (the agent is part of the Redis key); anything else is a miss: AGR_ENOTFOUND for a RESPONSE or ERROR, nothing for a
    DIAL_ERR; a zero id is a silent no-op.  A dropped agent's records keep their keys (Q17), so outcomes still apply to them;
  * RESPONSE: status completed, response code, processed_at = seq, leaves pending, one completed push per RESPONSE;
  * ERROR: retry + 1 (an 8-bit counter that saturates at 255); at max_retries status failed, leaves pending and one failed
    push on this and every later ERROR; below it status pending;
  * both set the row's last-SET time to max(seq, 1) and clear the in-flight bit; with AGR_CFG_SKIP_INFLIGHT a DIAL_ERR that
    names a row clears the in-flight bit and nothing else;
  * the completed / failed logs are append-only in op order; only the first log_cap entries exist, and a call whose pushes
    would take a log past log_cap returns AGR_ENOSPC (ending exactly at log_cap does not);
  * bytes (agr_complete_ex): of a row's ops in one call the last RESPONSE's segment is its response (headers = the first
    hdr_lens[i] bytes) and the last ERROR's segment its error text; a plain agr_complete leaves the stored bytes as they were.
Rows that carry a k5ref.Rec (add_rows(..., recs=)) also follow every transition there, so their wire form can be compared
byte for byte.  The bulk path is numpy; only rows with more than one op in a call are looped over in Python.
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

import k5ref

OUT_RESPONSE, OUT_DIAL_ERR, OUT_ERROR = 1, 2, 3
ST_PENDING, ST_COMPLETED, ST_FAILED = 1, 3, 4
ENOSPC, ENOTFOUND = -4, -5
# the state word (csrc/agr_common.h)
ST_INQ, ST_INFLIGHT, ST_STORED, ST_RESPONDED, ST_RESP_RT, ST_ERR_RT = 0x8, 0x10, 0x20, 0x40, 0x80, 0x01000000
ST_RETRY_SHIFT, ST_MAX_SHIFT, AUX_ERR_SHIFT = 8, 16, 16
LIST_PENDING, LIST_COMPLETED, LIST_FAILED = 0, 1, 2
COUNTERS = ("completions", "failures", "dead_lettered", "completion_misses", "dial_errors", "log_overflow")

_KEY = np.dtype([("a", ">u8"), ("b", ">u8")])


def id_keys(ids) -> np.ndarray:
    """16-byte ids as sortable keys."""
    return np.ascontiguousarray(np.asarray(ids, dtype=np.uint8).reshape(-1, 16)).view(_KEY).reshape(-1)


class K2Ref:
    _BOOL = ("stored", "inq", "inflight", "responded", "resp_rt", "err_rt")
    _NUM = (("status", np.uint8), ("retry", np.uint8), ("maxr", np.uint8), ("code", np.uint16), ("errk", np.uint8),
            ("mtime", np.uint64), ("ptime", np.uint64), ("slot", np.int64))

    def __init__(self, log_cap: int, skip_inflight: bool = False):
        self.log_cap = log_cap
        self.skip_inflight = skip_inflight
        self.n = 0                                   # rows handed out (logical)
        self.tail = 0                                # first row not released
        self._alloc(1024)
        self.ids = np.zeros((1024, 16), dtype=np.uint8)
        self.recs: Dict[int, k5ref.Rec] = {}
        self.logs: tuple = ([], [])                  # completed, failed: rows in push order (-1: a dropped agent's hole)
        self.ctr = {k: 0 for k in COUNTERS}
        self.slots: Dict[str, int] = {}              # registered agent names (dropped ones stay: their keys survive)
        self.dropped = set()
        self._index = None

    def _alloc(self, cap):
        for name in self._BOOL:
            setattr(self, name, np.zeros(cap, dtype=bool))
        for name, dt in self._NUM:
            setattr(self, name, np.full(cap, -1, dtype=dt) if name == "slot" else np.zeros(cap, dtype=dt))

    def _grow(self, end: int) -> None:
        cap = len(self.stored)
        if end <= cap:
            return
        new = max(end, 2 * cap)
        for name in self._BOOL + tuple(n for n, _ in self._NUM) + ("ids",):
            a = getattr(self, name)
            b = np.full((new,) + a.shape[1:], -1, dtype=a.dtype) if name == "slot" else np.zeros((new,) + a.shape[1:], dtype=a.dtype)
            b[: len(a)] = a
            setattr(self, name, b)

    # ---- what the test did
    def register(self, name: str) -> int:
        if name not in self.slots:
            self.slots[name] = len(self.slots)
        return self.slots[name]

    def slot_of(self, name: str) -> int:
        """The agent slot an outcome's agent id resolves to (-1: unknown agent)."""
        return self.slots.get(name, -1)

    def drop(self, name: str) -> None:
        """agr_drop_agent: DEL the three lists (the log entries become holes, the rows leave pending); the records stay."""
        s = self.slots[name]
        self.dropped.add(s)
        live = slice(self.tail, self.n)
        self.inq[live] &= self.slot[live] != s
        self.logs = tuple([r if r < 0 or self.slot[r] != s else -1 for r in log] for log in self.logs)

    def add_rows(self, first: int, slots, ids, running, max_retries=3, created=0, ring=False,
                 recs: Optional[Sequence[k5ref.Rec]] = None) -> None:
        """Rows [first, +len(slots)) were ingested as fresh records of these agent slots (-1: unknown agent, not stored).
        running: the agent was running at ingest (the forward is in flight).  max_retries as fed (0 = the default 3)."""
        slots = np.asarray(slots, dtype=np.int64)
        k = len(slots)
        end = first + k
        assert first >= self.n
        self._grow(end)
        self.n = end
        rows = slice(first, end)
        st = slots >= 0
        self.slot[rows] = slots
        self.stored[rows] = st
        self.inq[rows] = st
        self.inflight[rows] = st & np.broadcast_to(np.asarray(running, dtype=bool), (k,))
        for name in ("responded", "resp_rt", "err_rt"):
            getattr(self, name)[rows] = False
        self.status[rows] = np.where(st, ST_PENDING, 0)
        self.retry[rows] = 0
        m = np.broadcast_to(np.asarray(max_retries, dtype=np.int64), (k,))
        self.maxr[rows] = np.where(m == 0, 3, m)
        self.code[rows] = 0
        self.errk[rows] = 0
        self.ptime[rows] = 0
        self.mtime[rows] = np.broadcast_to(np.asarray(created, dtype=np.uint64), (k,)) if ring else 0
        self.ids[rows] = ids
        if recs is not None:
            for i, r in enumerate(recs):
                if st[i]:
                    self.recs[first + i] = r
        self._index = None

    def expire(self, rows) -> None:
        rows = np.asarray(rows, dtype=np.int64)
        self.stored[rows] = False
        for r in rows.tolist():
            if r in self.recs:
                self.recs[r].stored = False

    def reclaim(self, end: int) -> None:
        """agr_reclaim released rows [tail, end) (none of them stored): their log entries go."""
        assert not self.stored[self.tail:end].any()
        self.inq[self.tail:end] = False
        self.logs = tuple([r for r in log if r < 0 or r >= end] for log in self.logs)
        self.tail = end
        self._index = None

    # ---- K2
    def resolve(self, ids, slots) -> np.ndarray:
        """The row each (id, agent slot) names, or -1."""
        if self._index is None:
            keys = id_keys(self.ids[self.tail:self.n])
            order = np.argsort(keys, kind="stable")
            self._index = (keys[order], order + self.tail)
        keys, rows_sorted = self._index
        q = id_keys(ids)
        pos = np.minimum(np.searchsorted(keys, q), max(len(keys) - 1, 0))
        rows = np.full(len(q), -1, dtype=np.int64)
        if len(keys):
            hit = keys[pos] == q
            rows[hit] = rows_sorted[pos[hit]]
        nz = np.asarray(ids, dtype=np.uint8).reshape(-1, 16).any(axis=1)
        ok = (rows >= 0) & nz
        r = np.where(ok, rows, 0)
        ok &= self.stored[r] & (self.slot[r] == np.asarray(slots, dtype=np.int64))
        return np.where(ok, rows, -1)

    def complete(self, ids, slots, kinds, https, seqs, segs: Optional[List[bytes]] = None, hdr_lens=None):
        """One agr_complete (segs None) or agr_complete_ex (segs: one bytes object per op) call.  Returns (results, rc)."""
        kinds = np.asarray(kinds, dtype=np.int64)
        https = np.asarray(https, dtype=np.int64)
        seqs = np.asarray(seqs, dtype=np.uint64)
        n = len(kinds)
        rows = self.resolve(ids, slots)
        nz = np.asarray(ids, dtype=np.uint8).reshape(-1, 16).any(axis=1)
        rd = (kinds == OUT_RESPONSE) | (kinds == OUT_ERROR)
        link = (rows >= 0) & (rd | ((kinds == OUT_DIAL_ERR) & self.skip_inflight))
        miss = nz & rd & (rows < 0)
        results = np.where(miss, ENOTFOUND, 0).astype(np.int32)
        self.ctr["completion_misses"] += int(miss.sum())
        self.ctr["dial_errors"] += int((kinds == OUT_DIAL_ERR).sum())
        eff = np.zeros(n, dtype=np.uint8)
        li = np.flatnonzero(link)
        lr = rows[li]
        _, inv, cnt = np.unique(lr, return_inverse=True, return_counts=True)
        one = cnt[inv] == 1
        self._apply_many(li[one], lr[one], kinds, https, seqs, eff)
        for j, r in zip(li[~one].tolist(), lr[~one].tolist()):        # (li ascending: op order)
            self._apply_many(np.array([j]), np.array([r]), kinds, https, seqs, eff)
        for j, r in zip(li.tolist(), lr.tolist()):                    # the records that carry a wire form
            rec = self.recs.get(r)
            if rec is None:
                continue
            k = int(kinds[j])
            if k == OUT_RESPONSE:
                if segs is None:
                    rec.response(int(https[j]), rec.resp_hdr, rec.resp_body, int(seqs[j]))
                else:
                    h = int(hdr_lens[j]) if hdr_lens is not None else 0
                    rec.response(int(https[j]), segs[j][:h], segs[j][h:], int(seqs[j]))
            elif k == OUT_ERROR:
                rec.error(rec.err if segs is None else segs[j])
        over = False
        self.dropped_push = np.zeros(n, dtype=bool)  # ops whose push landed past log_cap (the service kernel tells their tickets)
        for w, bit in ((0, 1), (1, 2)):
            at = np.flatnonzero(eff & bit)
            log = self.logs[w]
            room = max(self.log_cap - len(log), 0)
            log.extend(rows[at[:room]].tolist())
            self.dropped_push[at[room:]] = True
            over |= len(at) > room
        if over:
            self.ctr["log_overflow"] += 1
        return results, (ENOSPC if over else 0)

    def _apply_many(self, ops, rows, kinds, https, seqs, eff) -> None:
        """Ops on DISTINCT rows (vectorised), or one op."""
        k = kinds[ops]
        for kind in (OUT_RESPONSE, OUT_ERROR, OUT_DIAL_ERR):
            m = k == kind
            o, r = ops[m], rows[m]
            if not len(o):
                continue
            self.inflight[r] = False
            if kind == OUT_DIAL_ERR:
                continue
            self.mtime[r] = np.maximum(seqs[o], np.uint64(1))
            if kind == OUT_RESPONSE:
                self.status[r] = ST_COMPLETED
                self.code[r] = https[o]
                self.ptime[r] = seqs[o]
                self.responded[r] = True
                self.resp_rt[r] = False
                self.err_rt[r] |= self.retry[r] > 0
                self.inq[r] = False
                eff[o] |= 1
                self.ctr["completions"] += len(o)
            else:
                retry = np.minimum(self.retry[r].astype(np.int64) + 1, 255)
                self.retry[r] = retry
                self.err_rt[r] = False
                self.resp_rt[r] |= self.responded[r]
                self.errk[r] = OUT_ERROR
                dead = retry >= self.maxr[r]
                self.status[r] = np.where(dead, ST_FAILED, ST_PENDING)
                self.inq[r[dead]] = False
                eff[o[dead]] |= 2
                self.ctr["failures"] += len(o)
                self.ctr["dead_lettered"] += int(dead.sum())

    # ---- what the engine must show
    def state_words(self, rows) -> np.ndarray:
        r = np.asarray(rows, dtype=np.int64)
        w = self.status[r].astype(np.uint32)
        for name, bit in (("inq", ST_INQ), ("inflight", ST_INFLIGHT), ("stored", ST_STORED), ("responded", ST_RESPONDED),
                          ("resp_rt", ST_RESP_RT), ("err_rt", ST_ERR_RT)):
            w |= np.where(getattr(self, name)[r], bit, 0).astype(np.uint32)
        w |= self.retry[r].astype(np.uint32) << ST_RETRY_SHIFT
        w |= self.maxr[r].astype(np.uint32) << ST_MAX_SHIFT
        return w

    def aux_words(self, rows) -> np.ndarray:
        r = np.asarray(rows, dtype=np.int64)
        return self.code[r].astype(np.uint32) | (self.errk[r].astype(np.uint32) << AUX_ERR_SHIFT)

    def list(self, slot: int, which: int) -> np.ndarray:
        """agr_list of a live agent: rows whose ids LRANGE returns (pending: the stored-or-expired rows still queued)."""
        if which == LIST_PENDING:
            lo, hi = self.tail, self.n
            return np.flatnonzero(self.inq[lo:hi] & (self.slot[lo:hi] == slot)) + lo
        log = np.asarray(self.logs[which - 1], dtype=np.int64)
        return log[(log >= 0) & (self.slot[np.maximum(log, 0)] == slot)]

    def log_lens(self):
        return len(self.logs[0]), len(self.logs[1])
