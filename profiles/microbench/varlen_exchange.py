"""Variable-length engines (AGR_CFG_VARLEN) fed in the fixed 512-byte form: K1v over device-resident 512-byte slots against
agr_ingest_var of the same records from a pinned blob, and agr_ingest_sharded at world 1 against agr_ingest_var.
  resident: reserve_rows + synth_fill_rows + ingest_rows_async per step, K1v device time from agr_kernel_time (AGR_CFG_TIMING)
            and the step's wall time;
  blob:     agr_ingest_var of the same 512-byte records (offsets 512 i) from pinned host memory: K1v device time and wall time;
  sharded:  agr_ingest_sharded (NCCL, world 1) of the same records from pinned memory against agr_ingest_var: wall time.
With two or more GPUs, the exchange over two ranks with 5 % cross-shard replays per step is timed too (one process per GPU).
Prints one JSON line per measurement, each with the GPU name and power limit read in the same run.
  python profiles/microbench/varlen_exchange.py [records per step, default 1048576] [steps, default 10]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch      # (before the library loads libnccl.so.2 into the global namespace: torch's CUDA library resolves its own)

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K

N = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 20
STEPS = int(sys.argv[2]) if len(sys.argv) > 2 else 10
FLAGS = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING | K.AGR_CFG_VARLEN | K.AGR_CFG_TIMING
N_AGENTS = 64


def card(device=0):
    q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else ("unknown", "unknown")
    return {"gpu": name, "power_limit": power}


def make_engine(device=0):
    e = A.Engine(device=device, slab_rows=8 * N, max_batch=2 * N, vslab_bytes=8 * N * 512, max_agents=256, flags=FLAGS)
    for k in range(N_AGENTS):
        e.set_agent_state(A.synth_agent_id(k), "running")
    return e


def release(e):
    e.expire(1 << 62, 1)
    e.reclaim()


def emit(what, **kw):
    print(json.dumps(dict(bench="varlen_exchange", what=what, records=N, steps=STEPS, **kw, **card())), flush=True)


def resident_vs_blob():
    with make_engine() as e:
        pin = e.pinned(N)
        offs = np.arange(N + 1, dtype=np.uint32) * 512
        res = {}
        for form in ("resident", "blob"):
            wall = 0.0
            for s in range(STEPS + 2):                               # two warm-up steps
                if s == 2:
                    e.kernel_time()
                    wall = 0.0
                release(e)
                if form == "blob":
                    pin.array[:] = A.synth_fill_host(s * N, N, seed=7, n_agents=N_AGENTS)
                e.sync()
                t = time.perf_counter()
                if form == "resident":
                    f = e.reserve_rows(N)
                    e.synth_fill_rows(s * N, f, N, seed=7, n_agents=N_AGENTS)
                    e.ingest_rows_async(f, N)
                    e.sync()
                else:
                    blob = pin.array.view(np.uint8).reshape(-1)
                    e.ingest_var(blob, offs)
                wall += time.perf_counter() - t
            ms, launches = e.kernel_time()
            res[form] = dict(k1v_ms_per_step=ms / max(launches, 1), k1v_launches=launches, wall_ms_per_step=1e3 * wall / STEPS,
                             k1v_gbps=N * 520 / (ms / max(launches, 1)) / 1e6)
        emit("k1v_resident_slots_vs_pinned_blob", **res)


def sharded_vs_var():
    import ctypes
    try:
        ctypes.CDLL("libnccl.so.2")
    except OSError as ex:
        emit("ingest_sharded_world1", note=f"not measured: libnccl.so.2 cannot be loaded ({ex})")
        return
    with make_engine() as e, make_engine() as twin:
        e.comm_init(A.comm_unique_id(), 0, 1)
        pin = e.pinned(N)
        offs = np.arange(N + 1, dtype=np.uint32) * 512
        res = {}
        for name, eng in (("ingest_sharded", e), ("ingest_var", twin)):
            wall = 0.0
            for s in range(STEPS + 2):
                release(eng)
                pin.array[:] = A.synth_fill_host(s * N, N, seed=9, n_agents=N_AGENTS)
                t = time.perf_counter()
                if name == "ingest_sharded":
                    eng.ingest_sharded(pin.array)
                else:
                    eng.ingest_var(pin.array.view(np.uint8).reshape(-1), offs)
                if s >= 2:
                    wall += time.perf_counter() - t
            res[name] = dict(wall_ms_per_step=1e3 * wall / STEPS)
        emit("ingest_sharded_world1_vs_ingest_var", **res)


def _rank(rank, world, port, q):
    import torch.distributed as dist
    from agentainer_lab_b200.sharding import make_rank_batch, owned_agents
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    uid = [A.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    own = owned_agents(world, 16)
    e = A.Engine(device=rank, slab_rows=8 * N, max_batch=2 * N, vslab_bytes=8 * N * 512, max_agents=256, flags=FLAGS)
    e.comm_init(uid[0], rank, world)
    for a in own[rank]:
        e.set_agent_state(a, "running")
    batches = [make_rank_batch(rank, world, own, N, seed=3 + s, p_cross_replay=0.05, first_index=s * N) for s in range(STEPS + 2)]
    wall = 0.0
    for s, b in enumerate(batches):
        release(e)
        dist.barrier()
        t = time.perf_counter()
        e.ingest_sharded(b)
        if s >= 2:
            wall += time.perf_counter() - t
    q.put((rank, 1e3 * wall / STEPS))
    dist.barrier()
    dist.destroy_process_group()
    e.close()


def exchange_two_gpus():
    if torch.cuda.device_count() < 2:
        emit("exchange_two_gpus", note="not measured: fewer than two GPUs")
        return
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, 29571, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(sorted(q.get(timeout=600) for _ in procs))
    for p in procs:
        p.join(timeout=60)
    emit("exchange_two_gpus_5pct_cross_replays", wall_ms_per_step_by_rank=res)


if __name__ == "__main__":
    resident_vs_blob()
    sharded_vs_var()
    exchange_two_gpus()
