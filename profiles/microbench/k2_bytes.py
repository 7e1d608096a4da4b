"""K2 with and without the bytes StoreResponse keeps, on the same batch of outcomes (CUDA-event device time, AGR_CFG_TIMING).
  python profiles/microbench/k2_bytes.py [outcomes, default 1 M] [segment bytes, default 320] [repeats, default 5]
Ingests `outcomes` records of the C3 synthetic stream (engine-minted ids), then completes them `repeats` times, alternating
agr_complete (k2_link + k2_apply + k2_append) and agr_complete_ex with a segment of 64 B of headers + the rest body per outcome
(k2_link + k2_apply_bytes + k2_append + k2_copy_bytes), all from pinned buffers.  The first round of each is warm-up (it sizes
the staging buffers).  Device time covers the kernels only; the uploads are not in it.  Algorithmic bytes per outcome: 72 for
agr_complete (64 B outcome + 4 B state RMW + 4 B list append), 72 + 2 x segment with bytes (the segment read from the staged
batch and written to the response byte slab).  Prints one JSON line; writes nothing."""
import json
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 20
SEG = int(sys.argv[2]) if len(sys.argv) > 2 else 320
REP = int(sys.argv[3]) if len(sys.argv) > 3 else 5
PEAK = 3.35e12                                                 # H100 SXM data sheet HBM3 bandwidth, B/s

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
eng = A.Engine(device=0, slab_rows=B, max_agents=1024, max_batch=B, log_entries=4 * (REP + 1) * B, resp_bytes=(REP + 1) * B * ((SEG + 15) // 16 * 16),
               flags=K.AGR_CFG_PERSISTENCE | K.AGR_CFG_TIMING | K.AGR_CFG_MINT_IDS)
nanos0 = 1700000000000000000
for k in range(256):
    eng.set_agent_state(A.synth_agent_id(k, agent_nanos0=nanos0), "running")
synth = dict(seed=2, n_agents=256, zipf_milli=1200, dup_permille=100, agent_nanos0=nanos0)
first = eng.reserve_rows(B)
eng.synth_fill_rows(0, first, B, mint_base=first, **synth)
eng.ingest_rows_async(first, B)
eng.sync()
host = A.synth_fill_host(0, B, mint=(eng, first), **synth)
outs = eng.pinned(B, A.outcome_dtype)
outs.array["request_id"] = eng.mint_ids(first, B)
outs.array["agent_id"] = host["agent_id"]
outs.array["kind"] = K.AGR_OUT_RESPONSE
outs.array["http_status"] = 200
outs.array["seq"] = 8 * B
rep = (host["flags"] & 1) != 0
outs.array["request_id"][rep] = host["replay_of"][rep]
unit = np.frombuffer(b"H" * 63 + b"\n" + b"b" * (SEG - 64), dtype=np.uint8)
blob, offs, hlen = eng.pinned(B * SEG, np.uint8), eng.pinned(B + 1, np.uint64), eng.pinned(B, np.uint32)
blob.array.reshape(B, SEG)[:] = unit
offs.array[:] = np.arange(B + 1, dtype=np.uint64) * SEG
hlen.array[:] = 64
plain, with_bytes = [], []
for r in range(REP + 1):
    eng.complete(outs.array, want_results=False)
    t = eng.op_time(0)
    rc, _ = eng.complete_ex(outs.array, (blob.array, offs.array), hlen.array, want_results=False)
    assert rc == 0
    tb = eng.op_time(0)
    if r:
        plain.append(t)
        with_bytes.append(tb)
st = eng.stats()
assert st["log_overflow"] == 0
got = eng.get_response_body(host["agent_id"][0].decode(), bytes(outs.array["request_id"][0]))
assert got == unit.tobytes() or rep[0]
for a in (outs, blob, offs, hlen):
    a.free()
eng.close()
mp, mb = float(np.median(plain)), float(np.median(with_bytes))
print(json.dumps({"gpu": gpu, "outcomes": B, "segment_bytes": SEG, "repeats": REP,
                  "k2_complete": {"ms": plain, "median_ms": mp, "outcomes_per_s": B / (mp * 1e-3),
                                  "frac_of_peak": 72 * B / (mp * 1e-3) / PEAK},
                  "k2_complete_bytes": {"ms": with_bytes, "median_ms": mb, "outcomes_per_s": B / (mb * 1e-3),
                                        "algorithmic_bytes_per_outcome": 72 + 2 * SEG,
                                        "GBps": (72 + 2 * SEG) * B / (mb * 1e-3) / 1e9,
                                        "frac_of_peak": (72 + 2 * SEG) * B / (mb * 1e-3) / PEAK}}))
