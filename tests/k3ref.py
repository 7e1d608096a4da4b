"""Plain restatement of what K3 returns: the replay tick's dispatch list, agr_pending and the three agr_list views.

It is computed from what a test did to an engine, never from the engine's output:
  * the agent slot of every logical row (agents registered in order, so the slot is the registration index; -1 = the row
    holds no record: end-of-ring padding, an unknown agent),
  * the outcomes applied, in call order,
  * the agent statuses at scan time, dropped agents,
  * rows expired by agr_expire and rows released by agr_reclaim,
  * rows reserved but not filled yet (they bound every scan),
  * the time of every record and outcome (for the TTL sweep).

The rules are the reference's (oracle/model.py):
  * every stored fresh record joins its agent's pending list, whatever the agent's status;
  * RESPONSE (StoreResponse, model.py:169-183) completes the record: it leaves the pending list and its id is pushed onto the
    completed list, once per RESPONSE (a replayed id completes twice, Q7);
  * ERROR (MarkRequestFailed, model.py:198-213) adds 1 to retry_count; at max_retries it leaves the pending list and is pushed
    onto the failed list, again on every later ERROR;
  * DIAL_ERR changes nothing; an outcome for a record that is not stored (expired, released, unknown) changes nothing;
  * an expired record stays in the pending list's ids but is not returned or replayed;
  * a row's last-SET time is its record's created_at, then the time of every RESPONSE or ERROR applied to it while it is stored
    (SET ... EX restarts the TTL, Q11); sweep(now, ttl) drops a stored row when now >= t and now - t >= ttl (MiniRedis.get,
    model.py:74-80: the key expires at t + ttl; a clock behind t expires nothing);
  * a tick selects the pending, stored records of running agents with retry_count < max_retries, ordered by
    (agent slot, row) (model.py:353-376, the canonical cross-agent order Q9).
"""
from __future__ import annotations

import numpy as np

ST_PENDING, ST_PROCESSING, ST_COMPLETED, ST_FAILED = 1, 2, 3, 4
OUT_RESPONSE, OUT_DIAL_ERR, OUT_ERROR = 1, 2, 3
RUNNING = 1
LIST_PENDING, LIST_COMPLETED, LIST_FAILED = 0, 1, 2


class K3Ref:
    def __init__(self, max_retries: int = 3):
        self.max_retries = max_retries
        self.n = 0                                       # rows handed out so far (logical)
        self.tail = 0                                    # first row not released
        cap = 1024
        self.slot = np.full(cap, -1, dtype=np.int64)
        self.stored = np.zeros(cap, dtype=bool)
        self.inq = np.zeros(cap, dtype=bool)
        self.status = np.zeros(cap, dtype=np.uint8)
        self.retry = np.zeros(cap, dtype=np.uint8)
        self.err = np.zeros(cap, dtype=np.uint8)
        self.maxr = np.zeros(cap, dtype=np.uint8)
        self.resp = np.zeros(cap, dtype=np.uint16)
        self.ids = np.zeros((cap, 16), dtype=np.uint8)
        self.mtime = np.zeros(cap, dtype=np.uint64)          # last-SET time
        self.logs = ([], [])                             # completed, failed: rows in push order
        self.resv = []                                   # [first, end) reserved, not filled
        self.agent_status = {}                           # slot -> status code
        self.dropped = set()

    # ---- what the test did
    def _grow(self, end: int) -> None:
        cap = len(self.slot)
        if end <= cap:
            return
        new = max(end, 2 * cap)
        for name in ("slot", "stored", "inq", "status", "retry", "err", "maxr", "resp", "ids", "mtime"):
            a = getattr(self, name)
            b = np.zeros((new,) + a.shape[1:], dtype=a.dtype)
            if name == "slot":
                b[:] = -1
            b[: len(a)] = a
            setattr(self, name, b)

    def _per_slot(self, pred) -> np.ndarray:
        """pred(status) of every registered, not dropped agent, as a table indexed by slot (its last entry, and every slot
        that is not registered, is False)."""
        t = np.zeros(max(self.agent_status, default=-1) + 2, dtype=bool)
        for s, st in self.agent_status.items():
            t[s] = pred(st)
        return t

    def set_agents(self, slots, statuses) -> None:
        for s, st in zip(slots, statuses):
            self.agent_status[int(s)] = int(st)

    def drop_agent(self, slot: int) -> None:
        """agent.Manager.Remove: DEL the three lists; the records stay (Q17) and the slot is never reused."""
        self.dropped.add(slot)
        self.agent_status.pop(slot, None)
        hit = self.slot[: self.n] == slot
        self.inq[: self.n][hit] = False
        self.logs = tuple([r for r in log if self.slot[r] != slot] for log in self.logs)

    def skip(self, first: int) -> None:
        """Rows [n, first) hold no record (end-of-ring padding before a batch)."""
        assert first >= self.n
        self._grow(first)
        self.n = first

    def reserve(self, first: int, count: int) -> None:
        self.skip(first)
        self._grow(first + count)
        self.n = first + count
        self.resv.append((first, first + count))

    def add_rows(self, first: int, slots, ids, max_retries=None, created=None) -> None:
        """Rows [first, first + len(slots)) were ingested; slot -1 = not stored (unknown or dropped agent); created: the
        records' created_at (default 0)."""
        slots = np.asarray(slots, dtype=np.int64)
        end = first + len(slots)
        if first >= self.n:
            self.skip(first)
            self._grow(end)
            self.n = end
        else:                                            # filling (part of) a reservation
            keep = []
            for a, b in self.resv:
                keep += [(a, b)] if (b <= first or a >= end) else [p for p in ((a, first), (end, b)) if p[0] < p[1]]
            self.resv = keep
        reg = self._per_slot(lambda st: True)
        known = reg[np.clip(slots, 0, len(reg) - 1)] & (slots >= 0)   # K1 stores for every registered agent
        self.slot[first:end] = np.where(known, slots, -1)
        self.stored[first:end] = known
        self.inq[first:end] = known
        self.status[first:end] = np.where(known, ST_PENDING, 0)
        self.retry[first:end] = 0
        self.err[first:end] = 0
        self.maxr[first:end] = self.max_retries if max_retries is None else max_retries
        self.resp[first:end] = 0
        self.ids[first:end] = ids
        self.mtime[first:end] = 0 if created is None else np.asarray(created, dtype=np.uint64)

    def complete(self, rows, kinds, https, times=None) -> None:
        """Outcomes in call order (row = the record the outcome names, or -1 when it names none); times: the outcomes' times
        (default: the rows' times stay as they are)."""
        times = [None] * len(rows) if times is None else np.asarray(times, dtype=np.uint64).tolist()
        for r, k, h, t in zip(np.asarray(rows).tolist(), np.asarray(kinds).tolist(), np.asarray(https).tolist(), times):
            if r < self.tail or r >= self.n or not self.stored[r]:
                continue                                  # the key does not exist: the call fails, nothing changes
            if t is not None and k in (OUT_RESPONSE, OUT_ERROR):
                self.mtime[r] = t                         # StoreResponse / MarkRequestFailed SET the record again
            if k == OUT_RESPONSE:
                self.status[r] = ST_COMPLETED
                self.resp[r] = h
                self.inq[r] = False
                self.logs[0].append(r)
            elif k == OUT_ERROR:
                self.retry[r] = min(255, int(self.retry[r]) + 1)
                self.err[r] = OUT_ERROR
                if self.retry[r] < self.maxr[r]:
                    self.status[r] = ST_PENDING
                else:
                    self.status[r] = ST_FAILED
                    self.logs[1].append(r)
                    self.inq[r] = False

    def expire(self, mask_rows) -> int:
        """agr_expire: the records of these rows are dropped.  Returns how many were stored."""
        rows = np.asarray(mask_rows, dtype=np.int64)
        rows = rows[(rows >= self.tail) & (rows < self.n)]
        rows = rows[self.stored[rows]]
        self.stored[rows] = False
        return len(rows)

    def due(self, rows, now: int, ttl: int) -> np.ndarray:
        """Which of these rows' last SET is ttl or more before now (the model's expiry rule; Python ints: no wrap-around)."""
        t = self.mtime[np.asarray(rows, dtype=np.int64)].tolist()
        return np.array([now >= x and now - x >= ttl for x in t], dtype=bool)

    def sweep(self, now: int, ttl: int) -> int:
        """agr_expire(now, ttl): every stored row whose last SET is due is dropped.  Returns how many."""
        rows = np.flatnonzero(self.stored[self.tail:self.n]) + self.tail
        rows = rows[self.due(rows, now, ttl)]
        self.stored[rows] = False
        return len(rows)

    def bound(self) -> int:
        """Every scan stops at the first reserved row K1 has not filled."""
        return min([self.n] + [r[0] for r in self.resv])

    def reclaim(self, count=None) -> int:
        """agr_reclaim: release the rows at the tail that hold no record, up to the first stored one (or the bound).
        count: release that many instead (what an earlier scan found: agr_reclaim_async)."""
        if count is None:
            hi = self.bound()
            live = np.flatnonzero(self.stored[self.tail:hi])
            count = int(live[0]) if len(live) else hi - self.tail
        assert not self.stored[self.tail: self.tail + count].any()
        end = self.tail + count
        self.inq[self.tail:end] = False
        self.logs = tuple([r for r in log if r >= end] for log in self.logs)
        self.tail = end
        return count

    # ---- what K3 returns
    def tick(self):
        """agr_replay_scan: (rows, slots) in dispatch order."""
        lo, hi = self.tail, self.bound()
        slot = self.slot[lo:hi]
        run = self._per_slot(lambda st: st == RUNNING)
        ok = self.inq[lo:hi] & self.stored[lo:hi] & (slot >= 0)
        ok &= (self.status[lo:hi] != ST_PROCESSING) & (self.retry[lo:hi] < self.maxr[lo:hi])
        ok[ok] = run[np.minimum(slot[ok], len(run) - 1)]
        rows = np.flatnonzero(ok) + lo
        order = np.argsort(self.slot[rows], kind="stable")
        return rows[order], self.slot[rows[order]]

    def pending(self, slot: int) -> np.ndarray:
        """agr_pending: rows of the records GetPendingRequests returns, oldest first."""
        lo, hi = self.tail, self.bound()
        return np.flatnonzero(self.inq[lo:hi] & self.stored[lo:hi] & (self.slot[lo:hi] == slot)) + lo

    def list(self, slot: int, which: int) -> np.ndarray:
        """agr_list: rows whose ids LRANGE returns (pending: expired records' ids included)."""
        if which == LIST_PENDING:
            lo, hi = self.tail, self.bound()
            return np.flatnonzero(self.inq[lo:hi] & (self.slot[lo:hi] == slot)) + lo
        log = np.asarray(self.logs[which - 1], dtype=np.int64)
        return log[self.slot[log] == slot] if len(log) else log

    def header_fields(self, rows) -> dict:
        """What k3_gather patches into a returned record's header."""
        rows = np.asarray(rows, dtype=np.int64)
        return dict(status=self.status[rows], retry_count=self.retry[rows], max_retries=self.maxr[rows],
                    error_code=self.err[rows], resp_status=self.resp[rows])
