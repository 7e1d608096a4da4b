"""agr_restore into other capacities (DESIGN.md section 5): wall time of the restore and device time of its relocation kernels
(agr_op_time 4), for a ring restored into its own geometry, into 2x slab_rows and into about 0.6x slab_rows, and converted
into the other record form at the same slab_rows.
  fixed:      <rows> slab rows (default 4 Mi) filled through two laps in batches of rows / 4, every row completed with 48 B of
              response bytes, everything but the last two batches expired and released: the window is half the ring; also
              restored as an AGR_CFG_VARLEN ring ("varlen");
  var:        AGR_CFG_VARLEN, rows / 4 slab rows, records of 128 B - 4 KiB (C5-like bodies), the same laps and responses, byte
              rings scaled along with slab_rows;
  var_small:  AGR_CFG_VARLEN, rows / 4 slab rows, bodies of 128 - 400 B (records that fit a 512 B row), restored into 2x
              slab_rows and as a fixed-stride ring ("fixed").
Moved bytes = read + written: the window's per-row words (64 B, 76 B with AGR_CFG_VARLEN) on each side, its 512 B rows on each
fixed-stride side, the live record bytes on each variable-length side, and the packed response bytes; a conversion from 512 B
rows also reads one 32 B header sector per row (the record lengths).  Reported as GB/s over the relocation's device time and as a share of
3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth).  The snapshot goes to /dev/shm when it has room, else to the temporary
directory.  Prints one JSON line (GPU name and power limit read in the same run).
  python profiles/microbench/restore_resize.py [rows, default 4194304] [runs, default 3]"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import agentainer_lab_b200 as A
from agentainer_lab_b200 import constants as K

ROWS = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 22
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
FLAGS = K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | K.AGR_CFG_RING | K.AGR_CFG_TIMING
RESP = 48
AGENTS = [A.synth_agent_id(k).encode() for k in range(64)]


def var_blob(rng, first, n, body_hi):
    """n variable-length records (96 B header + 8 B path + body, 16 B rounded) with bodies of 128 B - body_hi."""
    body = rng.integers(128, body_hi + 1, n)
    size = 96 + ((8 + body + 15) & ~15)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(size)
    blob = np.zeros(int(offs[-1]), dtype=np.uint8)
    h = np.zeros(n, dtype=A.header_dtype)
    h["agent_id"] = np.array(AGENTS)[np.arange(n) % 64]
    h["seq"] = 1_700_000_000_000_000_000 + first + np.arange(n, dtype=np.uint64)
    h["path_len"], h["body_len"], h["status"], h["max_retries"] = 8, body, K.AGR_ST_PENDING, 3
    idx = offs[:-1, None].astype(np.int64) + np.arange(96)
    blob[idx] = h.view(np.uint8).reshape(n, 96)
    return blob, offs.astype(np.uint32), size


def compact_bytes(first_index, n):
    """the compact record bytes of synth_fill rows [first_index, + n)"""
    r = A.synth_fill_host(first_index, n, seed=7, n_agents=64)
    return int((96 + ((r["path_len"].astype(np.int64) + r["hdr_len"] + r["body_len"] + 15) & ~15)).sum())


def fill(eng, S, var, rng, body_hi):
    """Two laps in batches of S / 4 and one more batch; returns the window's record bytes (stored with AGR_CFG_VARLEN, compact
    otherwise) and rows."""
    B = S // 4
    sizes = []
    for k in range(10):
        if k < 9:                                                  # all but the last two batches are released
            eng.expire(1 << 62, 1)
            eng.reclaim()
        if var:
            blob, offs, size = var_blob(rng, k * B, B, body_hi)
            _, _, first = eng.ingest_var(blob, offs)
            sizes.append(int(size.sum()))
        else:
            first = eng.reserve_rows(B)
            eng.synth_fill_rows(k * B, first, B, seed=7, n_agents=64)
            eng.ingest_rows(first, B, want_verdicts=False)
        if k == 0:
            for a in range(64):
                eng.set_agent_state(A.synth_agent_id(a), "running")
        outs = np.zeros(B, dtype=A.outcome_dtype)
        outs["request_id"] = eng.mint_ids(first, B)
        outs["agent_id"] = np.array(AGENTS)[np.arange(B) % 64] if var else A.synth_fill_host(k * B, B, seed=7, n_agents=64)["agent_id"]
        outs["kind"], outs["http_status"], outs["seq"] = K.AGR_OUT_RESPONSE, 200, 1 << 61
        eng.complete_ex(outs, [bytes(RESP)] * B)
    return sum(sizes[-2:]) if var else compact_bytes(8 * B, 2 * B), 2 * B


def moved_bytes(var_s, var_t, window, rec_bytes):
    side = lambda v: rec_bytes if v else window * 512
    rec = window * 32 + 2 * rec_bytes if (var_t and not var_s) else side(var_s) + side(var_t)
    return window * ((76 if var_s else 64) + (76 if var_t else 64)) + rec + 2 * window * RESP


def case(form, S, tmp, targets, body_hi=4096):
    rng = np.random.default_rng(5)
    var = form != "fixed"
    per_row = 5 * 1024 if form == "var" else 512                   # (2.3x / 2x what a window of half the ring takes at most)
    vslab = lambda s, v: s * per_row if v else 0
    kw = lambda v: dict(max_agents=128, id_secret=0x5EED, flags=FLAGS | (K.AGR_CFG_VARLEN if v else 0))
    with A.Engine(slab_rows=S, vslab_bytes=vslab(S, var), resp_bytes=S * 64, **kw(var)) as eng:
        rec_bytes, window = fill(eng, S, var, rng, body_hi)
        path = os.path.join(tmp, "resize.snap")
        eng.snapshot(path)
    out = []
    for name, S2, var2 in targets:
        walls, kern = [], []
        moved = moved_bytes(var, var2, window, rec_bytes)
        for _ in range(RUNS):
            t0 = time.perf_counter()
            with A.Engine(restore_from=path, slab_rows=S2, vslab_bytes=vslab(S2, var2), resp_bytes=S2 * 64, **kw(var2)) as back:
                back.sync()
                walls.append(time.perf_counter() - t0)
                if name != "same":
                    kern.append(back.op_time(4))
        r = {"into": name, "slab_rows": S2, "restore_wall_s": round(min(walls), 3)}
        if kern:
            ms = min(kern)
            r.update(relocation_ms=round(ms, 3), moved_bytes=moved, gb_s=round(moved / ms / 1e6, 1),
                     share_of_3_35_tb_s=round(moved / ms / 1e6 / 3350, 3))
        out.append(r)
    os.remove(path)
    return {"form": form, "slab_rows": S, "window_rows": window, "record_bytes": rec_bytes, "runs": out}


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    shm = "/dev/shm"
    need = ROWS * 700
    tmp = tempfile.mkdtemp(dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 2 * need else None)
    try:
        res = [case("fixed", ROWS, tmp, [("same", ROWS, False), ("2x", 2 * ROWS, False), ("0.6x", int(ROWS * 0.6), False),
                                         ("varlen", ROWS, True)]),
               case("var", ROWS // 4, tmp, [("same", ROWS // 4, True), ("2x", ROWS // 2, True), ("0.6x", int(ROWS // 4 * 0.6), True)]),
               case("var_small", ROWS // 4, tmp, [("2x", ROWS // 2, True), ("fixed", ROWS // 4, False)], body_hi=400)]
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"bench": "restore_resize", "gpu": q.stdout.strip(), "file_dir": os.path.dirname(tmp), "cases": res}))


if __name__ == "__main__":
    main()
