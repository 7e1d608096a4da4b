"""Long variable-length records (stored length over AGR_VAR_MAX_RECORD) on one GPU.

Measures, each as one JSON line with the GPU name and power limit read in the same run:
  1. K1v + the long-record checksum pass over batches of only 64 KiB and of only 1 MiB records, staged and LSU forms: kernel
     time by CUDA events (agr_kernel_time brackets both), GB/s of algorithmic bytes (stored length + 8 per record, SURVEY 8d),
     and that rate as a share of the data sheet's 3.35 TB/s and of the LDG.128 ceiling stream_read.cu measures on the card;
  2. a C5-shaped batch (128 B - 4 KiB bodies) with and without 1 % of 256 KiB records, as kernel time per byte;
  3. agr_verify over long rows (warp per row);
  4. the locked agr_ingest_var(n = 1) rate for 64 KiB records while 8 threads submit small records as tickets, and the
     ticket rate left to them (against the ticket rate alone).

Run from the repository root: python profiles/microbench/large_records.py [--out DIR]; without --out it writes nothing."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import agentainer_lab_b200 as A                      # noqa: E402
import k1vref as kr                                   # noqa: E402
import longref as L                                   # noqa: E402
from agentainer_lab_b200 import constants as K        # noqa: E402

P, V, CB, TM = K.AGR_CFG_PERSISTENCE, K.AGR_CFG_VARLEN, K.AGR_CFG_COMBINE, K.AGR_CFG_TIMING
DATASHEET = 3.35e12
OUT = []


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else ("unknown", "unknown")
    return {"gpu": name, "power_limit": power}


CARD = None


def emit(what, **kw):
    line = json.dumps({"what": what, **CARD, **kw})
    print(line, flush=True)
    OUT.append(line)


def ldg_ceiling():
    """best LDG.128 rate (GB/s) of stream_read.cu, compiled into a temporary directory"""
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "stream_read")
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe,
                        os.path.join(ROOT, "profiles", "microbench", "stream_read.cu"), "-lcuda"], check=True)
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    rates = [float(m) for m in re.findall(r"ldg\.128.*?([0-9.]+) GB/s", out)]
    return max(rates), out


def batch(lens, rng, agents=("agent-a",)):
    h = kr.headers(len(lens), list(agents), rng)
    kr.fit_lens(h, lens, rng)
    return L.blob_from(h, lens, rng)


def k1v_rate(lens, form, reps, rng, ceiling):
    lens = np.asarray(lens, dtype=np.int64)
    blob, offs = batch(lens, rng)
    nb = int(offs[-1])
    with A.Engine(flags=P | V | TM | K.AGR_CFG_MINT_IDS, slab_rows=len(lens) * (reps + 2) + 64, max_agents=8,
                  vslab_bytes=nb * (reps + 2) + (1 << 20), max_record_bytes=max(8192, int(lens.max())), k1_variant=form) as e:
        e.set_agent_state("agent-a", "stopped")
        e.ingest_var(blob, offs)                                     # warm-up
        e.kernel_time()
        for _ in range(reps):
            e.ingest_var(blob, offs)
        ms, n = e.kernel_time()
    alg = (nb + 8 * len(lens)) * reps
    rate = alg / (ms * 1e-3)
    return ms / reps, rate, nb


def main():
    global CARD
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for large_records.jsonl and the raw stream_read output (default: stdout only)")
    args = ap.parse_args()
    CARD = card()
    rng = np.random.default_rng(1)
    ceiling, raw = ldg_ceiling()
    emit("ldg_ceiling", gbps=ceiling)
    # 1. only long records
    for size, n in ((65536, 2048), (1 << 20, 128)):
        for form in (0, 0x20):
            ms, rate, nb = k1v_rate([size] * n, form, 20, rng, ceiling)
            emit("k1v_long_only", record=size, records=n, batch_bytes=nb, form="lsu" if form else "staged", kernel_ms=ms,
                 alg_gbps=rate / 1e9, share_datasheet=rate / DATASHEET, share_ldg_ceiling=rate / 1e9 / ceiling)
    # 1b. where the time of one 1 MiB-record batch goes: every kernel of the ingest step, by torch.profiler
    import torch
    from torch.profiler import ProfilerActivity, profile
    blob, offs = batch([1 << 20] * 128, rng)
    with A.Engine(flags=P | V | K.AGR_CFG_MINT_IDS, slab_rows=4096, max_agents=8, vslab_bytes=len(blob) * 6, max_record_bytes=1 << 20) as e:
        e.set_agent_state("agent-a", "stopped")
        e.ingest_var(blob, offs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(4):
                e.ingest_var(blob, offs)
            torch.cuda.synchronize()
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" or getattr(ev, "device_time_total", 0):
            emit("k1v_long_breakdown", record=1 << 20, records=128, kernel=ev.key[:60], calls=ev.count,
                 avg_us=getattr(ev, "device_time_total", 0) / max(ev.count, 1))
    # 2. C5-shaped batch with and without 1 % of 256 KiB records
    base = kr.HDR + np.exp(rng.uniform(np.log(128), np.log(4096), 20000)).astype(np.int64) // 16 * 16
    mixed = base.copy()
    mixed[rng.choice(len(mixed), len(mixed) // 100, replace=False)] = 256 << 10
    for name, lens in (("c5", base), ("c5_1pct_256k", mixed)):
        for form in (0, 0x20):
            ms, rate, nb = k1v_rate(lens, form, 20, rng, ceiling)
            emit("k1v_c5", batch=name, batch_bytes=nb, form="lsu" if form else "staged", kernel_ms=ms, ns_per_byte=ms * 1e6 / nb,
                 alg_gbps=rate / 1e9)
    # 3. agr_verify over long rows
    for size, n in ((65536, 2048), (1 << 20, 128)):
        blob, offs = batch([size] * n, rng)
        with A.Engine(flags=P | V, slab_rows=n + 64, max_agents=8, vslab_bytes=len(blob) + (1 << 20), max_record_bytes=size) as e:
            e.set_agent_state("agent-a", "stopped")
            e.ingest_var(blob, offs)
            e.verify()
            t = time.perf_counter()
            for _ in range(10):
                rows, bad = e.verify()
            dt = (time.perf_counter() - t) / 10
            assert bad == 0
        emit("verify_long_rows", record=size, rows=rows, call_ms=dt * 1e3, gbps=len(blob) / dt / 1e9)
    # 4. locked long calls next to ticket callers
    long_blob, long_offs = batch([65536], rng)
    small = [batch([int(s)], rng) for s in rng.integers(8, 64, 64) * 16]

    def run(with_long, secs=3.0):
        with A.Engine(flags=P | V | CB | K.AGR_CFG_MINT_IDS, slab_rows=1 << 21, max_agents=8, vslab_bytes=8 << 30,
                      max_record_bytes=1 << 20) as e:
            e.set_agent_state("agent-a", "stopped")
            stop = threading.Event()
            counts = [0] * 9

            def ticket(k):
                j = 0
                while not stop.is_set():
                    b, _ = small[(k * 7 + j) % len(small)]
                    e.poll(e.submit_ingest(b))
                    counts[k] += 1; j += 1

            def locked():
                while not stop.is_set():
                    e.ingest_var(long_blob, long_offs)
                    counts[8] += 1
            th = [threading.Thread(target=ticket, args=(k,)) for k in range(8)] + ([threading.Thread(target=locked)] if with_long else [])
            for t in th:
                t.start()
            time.sleep(0.5)
            c0, t0 = list(counts), time.perf_counter()
            time.sleep(secs)
            c1, t1 = list(counts), time.perf_counter()
            stop.set()
            for t in th:
                t.join()
        dt = t1 - t0
        return sum(c1[:8]) - sum(c0[:8]), c1[8] - c0[8], dt
    tk0, _, dt0 = run(False)
    tk1, lk1, dt1 = run(True)
    emit("locked_long_next_to_tickets", ticket_rate_alone=tk0 / dt0, ticket_rate_with_long=tk1 / dt1, long_rate=lk1 / dt1,
         long_record=65536, ticket_threads=8)
    if args.out is None:
        return
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "large_records.jsonl"), "w") as f:
        f.write("\n".join(OUT) + "\n")
    with open(os.path.join(args.out, "large_records_stream_read.txt"), "w") as f:
        f.write(raw)


if __name__ == "__main__":
    main()
