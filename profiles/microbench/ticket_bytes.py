"""Single-request round trips that keep their response, through tickets: bench_callers with 8 threads x 512 tickets in flight,
64 B of headers + <body> B of body per response, in mode `fused` (agr_submit_complete_ex up to AGR_OUT_INLINE_BYTES, above it
the locked agr_complete_ex(n = 1)) and mode `large` (agr_submit_complete_large up to AGR_OUT_TICKET_MAX_BYTES), the two modes
alternating for every body size so that both see the same state of the shared host.
  python profiles/microbench/ticket_bytes.py [seconds per run, default 1.0] [rounds, default 2]
Prints one JSON line (GPU name and power limit read in the same run); writes nothing."""
import json
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import agentainer_lab_b200 as A

SECONDS = sys.argv[1] if len(sys.argv) > 1 else "1.0"
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 2
BODIES = [256, 1024, 2048, 4096, 16000]
MODES = ["fused", "large"]

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
exe = os.path.join(os.path.dirname(A.build_host()), "bench_callers")
runs = {f"{m}_{b}": [] for b in BODIES for m in MODES}
for _ in range(ROUNDS):
    for b in BODIES:
        for m in MODES:
            p = subprocess.run([exe, "8", SECONDS, "0", "mint", "256", "512", m, str(b)], capture_output=True, text=True, timeout=600)
            d = json.loads(p.stdout.strip().splitlines()[-1])
            assert p.returncode == 0 and d["errors"] == 0, (m, b, p.stderr[-2000:])
            runs[f"{m}_{b}"].append({"round_trips_per_s": d["round_trips_per_s"], "p50_us": d["p50_us"], "p99_us": d["p99_us"],
                                     "ops_per_batch": d["ops_per_batch"]})
print(json.dumps({"gpu": gpu, "threads": 8, "inflight_per_thread": 512, "hdr_bytes": 64, "seconds": float(SECONDS), "rounds": ROUNDS,
                  "runs": runs}))
