"""agr_snapshot with and without AGR_CFG_ONLINE_SNAPSHOT under load: ring + minted ids + AGR_CFG_COMBINE + AGR_CFG_TIMING,
<rows> slab rows (default 16 M) of which a quarter hold records (agr_synth_fill_rows + agr_ingest_rows), a few thousand
completions with response bytes.  During every snapshot one thread ingests batches of 64 Ki pinned records with agr_expire /
agr_reclaim_async between them, and <callers> threads ingest 32 records at a time through the ticket ring; every call's
latency is kept.  The same load also runs for as long without a snapshot.  The two arms alternate, <runs> runs each.
  python profiles/microbench/snapshot_online.py [rows, default 16777216] [runs, default 3] [callers, default 4]
The file goes to /dev/shm when it has room (so that the engine, not the disk, is what is measured), else to the temporary
directory; which one is reported, and each file is deleted after its run.  Prints one JSON line (GPU name and power limit read
in the same run)."""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K

ROWS = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 24
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
CALLERS = int(sys.argv[3]) if len(sys.argv) > 3 else 4
BULK = 1 << 16
FLAGS = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING | K.AGR_CFG_COMBINE | K.AGR_CFG_TIMING


def fill(eng, n):
    step = eng.max_batch
    for first in range(0, n, step):
        m = min(step, n - first)
        rid = eng.reserve_rows(m)
        eng.synth_fill_rows(first, rid, m, seed=7, n_agents=64)
        eng.ingest_rows(rid, m, want_verdicts=False)
    for k in range(64):
        eng.set_agent_state(A.synth_agent_id(k), "running")
    # completions with bytes on a few thousand rows (the byte slab is part of every snapshot)
    n_out = 4096
    ids = eng.mint_ids(0, n_out)
    recs = A.synth_fill_host(0, n_out, seed=7, n_agents=64)
    outs = np.zeros(n_out, dtype=A.outcome_dtype)
    outs["request_id"], outs["agent_id"], outs["kind"], outs["http_status"] = ids, recs["agent_id"], K.AGR_OUT_RESPONSE, 200
    eng.complete_ex(outs, [bytes(200)] * n_out)


class Load:
    """The bulk thread and the ticket callers; each call is stored as (end time, seconds, records accepted)."""

    def __init__(self, eng, bulk_recs, small_recs):
        self.eng, self.bulk, self.small = eng, bulk_recs, small_recs
        self.stop = threading.Event()
        self.calls = {"bulk": [], "ticket": []}
        self.enospc = {"bulk": 0, "ticket": 0}
        self.threads = [threading.Thread(target=self._bulk)] + [threading.Thread(target=self._ticket) for _ in range(CALLERS)]

    def _call(self, kind, fn, n):
        t0 = time.perf_counter()
        try:
            fn()
            ok = n
        except A.AgrError as e:
            if e.code != K.AGR_ENOSPC:
                raise
            ok = 0
            self.enospc[kind] += 1
        t1 = time.perf_counter()
        self.calls[kind].append((t1, t1 - t0, ok))
        if not ok:
            time.sleep(0.001)

    def _bulk(self):
        k = 0
        while not self.stop.is_set():
            self._call("bulk", lambda: self.eng.ingest(self.bulk, want_verdicts=False), len(self.bulk))
            k += 1
            if k % 4 == 0:
                self._call("bulk", lambda: self.eng.expire(1 << 62, 1, want_count=False), 0)   # everything is due
                self._call("bulk", lambda: self.eng.reclaim_async(), 0)

    def _ticket(self):
        while not self.stop.is_set():
            self._call("ticket", lambda: self.eng.ingest(self.small, want_verdicts=False), len(self.small))

    def start(self):
        for t in self.threads:
            t.start()

    def finish(self):
        self.stop.set()
        for t in self.threads:
            t.join()

    def window(self, t0, t1):
        """Latency of the calls that overlap [t0, t1]; records of the calls that ended inside it."""
        calls = [c for kind in self.calls for c in self.calls[kind] if c[0] - c[1] < t1 and c[0] > t0]
        lat = np.array([c[1] for c in calls]) if calls else np.zeros(1)
        return {"calls": len(calls), "records": int(sum(c[2] for c in calls if c[0] <= t1)),
                "max_call_ms": float(lat.max() * 1e3),
                "p99_call_ms": float(np.percentile(lat, 99) * 1e3)}


def d2d_ms(nbytes):
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = None
    for _ in range(5):
        e0.record(); dst.copy_(src); e1.record(); e1.synchronize()
        best = e0.elapsed_time(e1) if best is None else min(best, e0.elapsed_time(e1))
    del src, dst
    torch.cuda.empty_cache()
    return best


def one_run(online, tmpdir, bulk_recs, small_recs):
    flags = FLAGS | (K.AGR_CFG_ONLINE_SNAPSHOT if online else 0)
    out = {"arm": "online" if online else "blocking"}
    with A.Engine(slab_rows=ROWS, max_agents=256, flags=flags) as eng:
        fill(eng, ROWS // 4)
        st = eng.stats()
        path = os.path.join(tmpdir, "agr.snap")
        # warm-up: every shape of the window
        eng.ingest(bulk_recs, want_verdicts=False)
        eng.ingest(small_recs, want_verdicts=False)
        load = Load(eng, bulk_recs, small_recs)
        load.start()
        time.sleep(0.5)
        t0 = time.perf_counter()
        eng.snapshot(path)
        t1 = time.perf_counter()
        time.sleep(0.2)
        quiet0 = time.perf_counter()
        time.sleep(t1 - t0)                                        # the same window without a snapshot
        quiet1 = time.perf_counter()
        load.finish()
        size = os.path.getsize(path)
        with open(path, "rb") as f:                                # the cut's rows and log lengths: from the file's header
            hd = np.frombuffer(f.read(8 + 16 + 8 * 4), dtype="<u8")
        os.remove(path)
        out.update(snapshot_s=t1 - t0, file_bytes=size, during=load.window(t0, t1), without=load.window(quiet0, quiet1),
                   enospc_calls=dict(load.enospc), rows_used_before=int(st["rows_used"]))
        if online:
            cut_ms = eng.op_time(3)
            cut_bytes = 64 * min(int(hd[3]), ROWS) + 4 * (int(hd[5]) + int(hd[6]))   # rows_used, log_len[0], log_len[1]
            out.update(cut_ms=cut_ms, cut_bytes=cut_bytes, cut_gb_per_s=cut_bytes / cut_ms / 1e6)
            out["d2d_same_bytes_ms"] = d2d_ms(cut_bytes)
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    need = ROWS // 4 * 600 + (1 << 30)
    shm = "/dev/shm"
    where = shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 2 * need else tempfile.gettempdir()
    tmpdir = tempfile.mkdtemp(prefix="agr_snap_", dir=where)
    lib = A.load_library()
    pinned = A.binding.PinnedArray(lib, BULK, A.record_dtype)
    pinned.array[:] = A.synth_fill_host(1 << 30, BULK, seed=9, n_agents=64)
    small = A.synth_fill_host(1 << 31, 32, seed=9, n_agents=64)
    runs = []
    try:
        for _ in range(RUNS):
            for online in (False, True):
                runs.append(one_run(online, tmpdir, pinned.array, small))
    finally:
        shutil.rmtree(tmpdir, ignore_errors=True)
        pinned.free()
    print(json.dumps({"gpu": gpu, "rows": ROWS, "filled_rows": ROWS // 4, "callers": CALLERS, "bulk_batch": BULK, "file_dir": where,
                      "runs": runs}))


if __name__ == "__main__":
    main()
