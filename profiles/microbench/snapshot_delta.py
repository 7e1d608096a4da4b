"""agr_snapshot with AGR_CFG_ONLINE_SNAPSHOT against AGR_CFG_ONLINE_SNAPSHOT | AGR_CFG_DELTA_SNAPSHOT: ring + minted ids +
AGR_CFG_TIMING, <rows> slab rows (default 16 M) filled to three quarters (agr_synth_fill_rows + agr_ingest_rows).  A paced
load thread ingests 4096 records at a time and completes a small share of the rows between snapshots; one snapshot every
<period> seconds, <snaps> per run.  The two arms alternate, <runs> runs each, and which arm goes first alternates from one
pair of runs to the next.  Then one saturating run of the delta arm releases every row and fills the ring again between
snapshots (every row's words and record change), which shows the fallback to full files.
  python profiles/microbench/snapshot_delta.py [rows, default 16777216] [runs, default 3] [snaps, default 4] [period s, default 2]
Per snapshot: the kind written and its bytes, wall time, the cut's device time (agr_op_time 3); per run: the longest and p99
ingest call and the AGR_ENOSPC count.  Files go to /dev/shm when it has room, else to the temporary directory (reported);
every file is deleted at the end of its run.  Prints one JSON line (GPU name and power limit read in the same run)."""
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
SNAPS = int(sys.argv[3]) if len(sys.argv) > 3 else 4
PERIOD = float(sys.argv[4]) if len(sys.argv) > 4 else 2.0
FLAGS = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING | K.AGR_CFG_TIMING | K.AGR_CFG_ONLINE_SNAPSHOT
BATCH = 4096


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:                                              # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def fill(eng, n, index0=0):
    for first in range(0, n, eng.max_batch):
        m = min(eng.max_batch, n - first)
        rid = eng.reserve_rows(m)
        eng.synth_fill_rows(index0 + first, rid, m, seed=7, n_agents=64)
        eng.ingest_rows(rid, m, want_verdicts=False)


def make_engine(delta):
    eng = A.Engine(slab_rows=ROWS, max_agents=256, max_batch=1 << 16, flags=FLAGS | (K.AGR_CFG_DELTA_SNAPSHOT if delta else 0))
    for k in range(64):                                          # before the fill: records of unknown agents are not stored
        eng.set_agent_state(A.synth_agent_id(k), "running")
    n = ROWS * 3 // 4
    fill(eng, n)
    return eng, n


def complete(eng, lo, n, seq):
    ids = eng.mint_ids(lo, n)
    recs = A.synth_fill_host(lo, n, seed=7, n_agents=64)
    outs = np.zeros(n, dtype=A.outcome_dtype)
    outs["request_id"], outs["agent_id"], outs["kind"], outs["http_status"], outs["seq"] = ids, recs["agent_id"], K.AGR_OUT_RESPONSE, 200, seq
    rc, res = eng.complete_ex(outs, [b""] * n)
    assert rc == 0 and (res == 0).all(), np.unique(res)


def run(delta, path, saturate=False):
    eng, filled = make_engine(delta)
    stop = threading.Event()
    calls, enospc = [], [0]

    def load():
        recs = A.synth_fill_host(filled, BATCH, seed=8, n_agents=64)
        while not stop.is_set():
            t = time.perf_counter()
            try:
                eng.ingest(recs)
            except A.AgrError as e:
                if e.code != K.AGR_ENOSPC:
                    raise
                enospc[0] += 1
            calls.append(time.perf_counter() - t)
            time.sleep(0.01)
    th = threading.Thread(target=load)
    th.start()
    snaps = []
    try:
        for k in range(SNAPS):
            if saturate and k:                                       # every row released and the ring filled again
                eng.expire(1 << 62, 1)
                eng.reclaim()
                fill(eng, filled, (k + 1) * ROWS)
            elif not saturate:                                       # 0.5 % of the rows completed
                share = max(BATCH, filled // 200)
                lo = (k * 7919 * BATCH) % max(1, filled - share)
                for o in range(0, share, 1 << 16):
                    complete(eng, lo + o, min(1 << 16, share - o), 10 + k)
            time.sleep(PERIOD)
            p = "%s.%d" % (path, k)
            t = time.perf_counter()
            eng.snapshot(p)
            wall = time.perf_counter() - t
            with open(p, "rb") as f:
                kind = f.read(8).decode()
            snaps.append({"kind": kind, "bytes": os.path.getsize(p), "wall_s": round(wall, 3), "cut_ms": round(eng.op_time(3), 3)})
    finally:
        stop.set()
        th.join()
        for k in range(SNAPS):
            if os.path.exists("%s.%d" % (path, k)):
                os.remove("%s.%d" % (path, k))
        eng.close()
    lat = np.array(calls) * 1e3
    return {"delta": delta, "saturate": saturate, "snapshots": snaps, "ingest_calls": len(lat),
            "ingest_max_ms": round(float(lat.max()), 2) if len(lat) else None,
            "ingest_p99_ms": round(float(np.percentile(lat, 99)), 2) if len(lat) else None, "enospc": enospc[0]}


def main():
    name, limit = gpu_info()
    need = ROWS * 600 * 2
    shm = shutil.disk_usage("/dev/shm").free > need if os.path.isdir("/dev/shm") else False
    where = tempfile.mkdtemp(dir="/dev/shm" if shm else None)
    path = os.path.join(where, "agr.snap")
    out = {"gpu": name, "power_limit": limit, "rows": ROWS, "files_in": "/dev/shm" if shm else tempfile.gettempdir(), "runs": []}
    try:
        for r in range(RUNS):
            for delta in ((False, True) if r % 2 == 0 else (True, False)):
                out["runs"].append(run(delta, path))
        out["runs"].append(run(True, path, saturate=True))
    finally:
        shutil.rmtree(where, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
