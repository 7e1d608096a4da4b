"""Single-request round trips of VARIABLE-LENGTH records (AGR_CFG_VARLEN): bench_callers mode `var`, the ticket arm (AGR_CFG_COMBINE:
8 threads x 512 tickets in flight, agr_submit_ingest -> agr_poll -> agr_submit_complete -> agr_poll) against the locked arm a
variable-length deployment has without the ring (64 threads, agr_ingest_var(n = 1) -> agr_complete(n = 1)), the two arms
alternating for every body size so that both see the same state of the shared host.  Body sizes: fixed ones, and `mix` (log-uniform
128 B - 4 KiB, BASELINE config 5).
  python profiles/microbench/ticket_var.py [seconds per run, default 1.0] [rounds, default 2]
Prints one JSON line (GPU name and power limit read in the same run); writes nothing."""
import json
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import agentainer_lab_b200 as A

SECONDS = sys.argv[1] if len(sys.argv) > 1 else "1.0"
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 2
BODIES = ["128", "1024", "4096", "8000", "mix"]
ARMS = {"ticket": ["8", "512"], "locked": ["64", "0"]}     # threads, tickets in flight per thread

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
exe = os.path.join(os.path.dirname(A.build_host()), "bench_callers")
runs = {f"{a}_{b}": [] for b in BODIES for a in ARMS}
for _ in range(ROUNDS):
    for b in BODIES:
        for a, (threads, inflight) in ARMS.items():
            p = subprocess.run([exe, threads, SECONDS, "0", "mint", "256", inflight, "var", "0" if b == "mix" else b],
                               capture_output=True, text=True, timeout=600)
            d = json.loads(p.stdout.strip().splitlines()[-1])
            assert p.returncode == 0 and d["errors"] == 0, (a, b, p.stderr[-2000:])
            runs[f"{a}_{b}"].append({k: d[k] for k in ("round_trips_per_s", "p50_us", "p99_us", "record_bytes_mean", "svc_batches")})
print(json.dumps({"gpu": gpu, "arms": {a: {"threads": int(t), "inflight_per_thread": int(i)} for a, (t, i) in ARMS.items()},
                  "seconds": float(SECONDS), "rounds": ROUNDS, "runs": runs}))
