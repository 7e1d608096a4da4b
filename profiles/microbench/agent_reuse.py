"""Agent slot reuse (DESIGN.md section 5): what a registration costs once the agent table is full.
  scan:  agr_set_agent_state of a new id right after an agr_drop_agent: the free list is empty and the window has to be scanned
         (k_slot_refs over the route words of every live row).  The window holds <rows> rows of 2048 agents (synthetic
         records, 512 B rows, engine-minted ids, decided by K1); 4096 agents are registered, half of them without rows, and each
         timed call follows the removal of one of those, so every call scans the whole window and finds exactly one free slot.
         Reported: the wall time of the call (host clock, the call ends with a stream synchronise), and the device time of
         k_slot_refs from a separate torch.profiler run (CUDA activities) over the same calls.
  list:  agr_set_agent_state of a new id while the free list of the last scan still has entries (no scan): wall time.
Windows of 1 Mi, 16 Mi and 128 Mi rows by default; a window the card has no room for is reported as not measured.  Bytes per
row read by the scan: 4 (the route word).  Prints one JSON line with the GPU name and power limit read in the same run.
  python profiles/microbench/agent_reuse.py [rows ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K

WINDOWS = [int(x) for x in sys.argv[1:]] or [1 << 20, 1 << 24, 1 << 27]
AGENTS, WITH_ROWS, CALLS = 4096, 2048, 20
FLAGS = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def fill(rows):
    B = 1 << 20
    eng = A.Engine(device=0, slab_rows=rows, max_agents=AGENTS, max_batch=B, flags=FLAGS, log_entries=1 << 20, resp_bytes=1 << 20)
    names = [A.synth_agent_id(k) for k in range(AGENTS)]
    eng.set_agent_states(names, ["stopped"] * AGENTS)
    for first in range(0, rows, B):
        n = min(B, rows - first)
        r = eng.reserve_rows(n)
        eng.synth_fill_rows(first, r, n, n_agents=WITH_ROWS)
        eng.ingest_rows(r, n, want_verdicts=False)
    eng.sync()
    return eng, names


def timed_scans(eng, names, k0, calls):
    """calls registrations that each scan: drop one agent without rows, register a new id in its slot"""
    wall = []
    for i in range(calls):
        eng.drop_agent(names[WITH_ROWS + k0 + i])
        t = time.perf_counter()
        s = eng.set_agent_state(f"fresh-{k0 + i}", "running")
        wall.append(time.perf_counter() - t)
        assert s == WITH_ROWS + k0 + i, s
    return wall


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = dict(gpu=gpu_info(), bytes_per_row=4, windows=[])
    for rows in WINDOWS:
        rec = dict(rows=rows)
        try:
            eng, names = fill(rows)
        except A.AgrError as e:
            rec["not_measured"] = f"engine of {rows} rows does not fit: {e}"
            out["windows"].append(rec)
            continue
        try:
            timed_scans(eng, names, 0, 2)                                  # warm-up (first launch, scratch allocation)
            wall = timed_scans(eng, names, 2, CALLS)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                timed_scans(eng, names, 2 + CALLS, CALLS)
            k = [e for e in prof.events() if "k_slot_refs" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
            dev = [e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3 for e in k]
            # list: 200 agents without rows removed, one registration scans, the next ones take the list
            base = 2 + 2 * CALLS
            for i in range(200):
                eng.drop_agent(names[WITH_ROWS + base + i])
            eng.set_agent_state("list-0", "running")
            lw = []
            for i in range(1, 150):
                t = time.perf_counter()
                eng.set_agent_state(f"list-{i}", "running")
                lw.append(time.perf_counter() - t)
            kernel_ms = float(np.median(dev)) if dev else None
            rec.update(scan_call_ms_median=1e3 * float(np.median(wall)), scan_call_ms_min=1e3 * float(np.min(wall)),
                       k_slot_refs_ms_median=kernel_ms, k_slot_refs_launches=len(dev),
                       k_slot_refs_gbs=(4 * rows / (kernel_ms * 1e-3) / 1e9) if kernel_ms else None,
                       list_call_us_median=1e6 * float(np.median(lw)))
        finally:
            eng.close()
        out["windows"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
