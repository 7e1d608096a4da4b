"""Plain reader of the two snapshot file formats of csrc/agr_snapshot.cu: a full file (AGRSNAP3) and a delta (AGRDELT1), and
what a delta should hold given the full files of its parent's cut and of its own.  Needs no GPU."""
import numpy as np

from agentainer_lab_b200 import constants as K
from k1ref import fmix64

R, V = K.AGR_CFG_RING, K.AGR_CFG_VARLEN
BLOCK_ROWS, LOG_BLOCK = 256, 1024

# mirrors struct snap_header in csrc/agr_engine.h
HEADER = np.dtype([("magic", "S8"), ("flags", "<u4"), ("n_agents", "<u4"), ("shard", "<u4"), ("gen", "<u4"),
                   ("rows_used", "<u8"), ("vused", "<u8"), ("log_len", "<u8", (2,)), ("id_secret", "<u8"), ("scan_lo", "<u8"),
                   ("resp_used", "<u8"), ("expired_total", "<u8"), ("tail", "<u8"), ("released_total", "<u8"), ("slab_rows", "<u8"),
                   ("vtail", "<u8"), ("vcap", "<u8"), ("resp_tail", "<u8"), ("resp_cap", "<u8")])
WORDS = ("state", "route", "aux", "cksum", "voff", "vlen", "resp_off", "resp_len", "resp_hlen", "err_off", "err_len", "ptime", "mtime")
# mirrors struct delta_header in csrc/agr_snapshot.cu
DELTA = np.dtype([("magic", "S8"), ("cut", HEADER), ("file_bytes", "<u8"), ("parent_digest", "<u8", (2,)), ("digest", "<u8", (2,)),
                  ("block_rows", "<u4"), ("log_block", "<u4"), ("rows_lo", "<u8"), ("rows_hi", "<u8"), ("resp_lo", "<u8"),
                  ("resp_hi", "<u8"), ("n_blocks", "<u8"), ("n_log_blocks", "<u8", (2,)), ("parent_path_len", "<u4"), ("pad", "<u4")])


def sections(hd):
    """(name, dtype, count) of every section after the agent table, in file order (the AGRSNAP3 layout)."""
    ring, var = bool(hd["flags"] & R), bool(hd["flags"] & V)
    rows = int(min(hd["rows_used"], hd["slab_rows"])) if ring else int(hd["rows_used"])
    slab = (int(min(hd["vused"], hd["vcap"])) if ring else int(hd["vused"])) if var else rows * 512
    resp = int(min(hd["resp_used"], hd["resp_cap"])) if ring else int(hd["resp_used"])
    return [("slab", np.uint8, slab), ("state", "<u4", rows), ("route", "<u4", rows), ("aux", "<u4", rows), ("cksum", "<u8", rows),
            ("voff", "<u8", rows if var else 0), ("vlen", "<u4", rows if var else 0),
            ("completed_log", "<u4", int(hd["log_len"][0])), ("failed_log", "<u4", int(hd["log_len"][1])),
            ("resp", np.uint8, resp), ("resp_off", "<u8", rows), ("resp_len", "<u4", rows), ("resp_hlen", "<u4", rows),
            ("err_off", "<u8", rows), ("err_len", "<u4", rows), ("ptime", "<u8", rows), ("mtime", "<u8", rows)]


LOGS = ("completed_log", "failed_log")
PHI, DIGEST_C = 0x9E3779B97F4A7C15, 0x632BE59BD9B4E019
U64 = (1 << 64) - 1


def digest_sections(hd, sec):
    """(section id, bytes) of what the compare cut sums: every per-row word section that holds bytes, then the two logs; the
    id is the section's place in the file's section table (so the logs are 7 and 8)."""
    names = [name for name, _, _ in sections(hd)]
    out = [(k, sec[name].tobytes()) for k, name in enumerate(names) if name in WORDS and len(sec[name])]
    return out + [(names.index(name), sec[name].tobytes()) for name in LOGS]


def digest(hd, sec, key):
    """The 128-bit keyed digest of k_snap_cmp over the sections of a full file (parse): per section s, with the key
    fmix64(key ^ ((s + 1) << 56)), every 16 B piece i (a short last piece zero-padded) as two little-endian u64 a, b adds
    fmix64(fmix64(t ^ a) ^ b) to the first sum and fmix64(fmix64((t + C) ^ b) ^ a) to the second, t = fmix64(skey + i * phi);
    both sums mod 2^64.  The sum does not depend on the order the device adds pieces in."""
    h = [0, 0]
    u = np.uint64
    for s, b in digest_sections(hd, sec):
        n = (len(b) + 15) // 16
        if n == 0:
            continue
        w = np.frombuffer(b + bytes(16 * n - len(b)), dtype="<u8").reshape(n, 2)
        a, bb = w[:, 0], w[:, 1]
        skey = fmix64(u((int(key) ^ ((s + 1) << 56)) & U64))
        with np.errstate(over="ignore"):
            t = fmix64(skey + np.arange(n, dtype=u) * u(PHI))
            h0 = fmix64(fmix64(t ^ a) ^ bb)
            h1 = fmix64(fmix64((t + u(DIGEST_C)) ^ bb) ^ a)
        h[0] = (h[0] + int(h0.sum(dtype=u))) & U64
        h[1] = (h[1] + int(h1.sum(dtype=u))) & U64
    return tuple(h)


def parse(data: bytes):
    hd = np.frombuffer(data, dtype=HEADER, count=1)[0]
    at = HEADER.itemsize + 33 * int(hd["n_agents"])
    agents = data[HEADER.itemsize: at]
    sec = {}
    for name, dt, count in sections(hd):
        sec[name] = np.frombuffer(data, dtype=dt, count=count, offset=at)
        at += sec[name].nbytes
    assert at == len(data)
    return hd, agents, sec


def runs(lo, hi, cap, ring):
    if hi <= lo:
        return []
    p = lo % cap if ring else lo
    n0 = min(hi - lo, cap - p) if ring else hi - lo
    return [(p, n0)] + ([(0, hi - lo - n0)] if hi - lo > n0 else [])


def parse_delta(data: bytes):
    """The fields of an AGRDELT1 file; every byte of it is accounted for."""
    dh = np.frombuffer(data, dtype=DELTA, count=1)[0]
    assert dh["magic"] == b"AGRDELT1" and int(dh["file_bytes"]) == len(data)
    assert (int(dh["block_rows"]), int(dh["log_block"])) == (BLOCK_ROWS, LOG_BLOCK)
    hd = dh["cut"]
    ring, var = bool(hd["flags"] & R), bool(hd["flags"] & V)
    at = DELTA.itemsize
    n = int(dh["parent_path_len"])
    out = {"dh": dh, "hd": hd, "parent": data[at: at + n].decode()}
    at += n
    out["agents"] = data[at: at + 33 * int(hd["n_agents"])]
    at += len(out["agents"])
    unit = 1 if var else 512
    cap = int(hd["vcap"]) if var else int(hd["slab_rows"])
    out["rows"] = []
    for p, k in runs(int(dh["rows_lo"]), int(dh["rows_hi"]), cap, ring):
        out["rows"].append((p * unit, data[at: at + k * unit])); at += k * unit
    out["resp"] = []
    for p, k in runs(int(dh["resp_lo"]), int(dh["resp_hi"]), int(hd["resp_cap"]), ring):
        out["resp"].append((p, data[at: at + k])); at += k
    secs = {name: (dt, count) for name, dt, count in sections(hd)}
    words = [w for w in WORDS if secs[w][1]]
    rows = secs["state"][1]

    def blocks(names, count, per, nb):
        nonlocal at
        lst = np.frombuffer(data, dtype="<u4", count=nb, offset=at).astype(np.int64)
        at += 4 * nb
        assert np.all(np.diff(lst) > 0) and (nb == 0 or lst[-1] * per < count)
        got = []
        for b in lst:
            r = min(per, count - b * per)
            sl = {}
            for w in names:
                dt = np.dtype(secs[w][0])
                sl[w] = np.frombuffer(data, dtype=dt, count=r, offset=at); at += r * dt.itemsize
            got.append((int(b), sl))
        return lst, got
    out["wl"], out["words"] = blocks(words, rows, BLOCK_ROWS, int(dh["n_blocks"]))
    out["ll"], out["logs"] = [], []
    for j, name in enumerate(("completed_log", "failed_log")):
        lst, got = blocks([name], secs[name][1], LOG_BLOCK, int(dh["n_log_blocks"][j]))
        out["ll"].append(lst); out["logs"].append(got)
    assert at == len(data)
    return out


def apply(sec_p, d):
    """The sections the delta brings its parent's sections (sec_p) to."""
    sec = {}
    for name, dt, count in sections(d["hd"]):
        a = np.zeros(count, dtype=dt)
        old = sec_p[name]
        k = min(count, len(old))
        a[:k] = old[:k]
        sec[name] = a
    for name, pieces in (("slab", d["rows"]), ("resp", d["resp"])):
        for p, b in pieces:
            sec[name][p: p + len(b)] = np.frombuffer(b, dtype=np.uint8)
    for b, sl in d["words"]:
        for w, v in sl.items():
            sec[w][b * BLOCK_ROWS: b * BLOCK_ROWS + len(v)] = v
    for j, name in enumerate(("completed_log", "failed_log")):
        for b, sl in d["logs"][j]:
            v = sl[name]
            sec[name][b * LOG_BLOCK: b * LOG_BLOCK + len(v)] = v
    return sec


def expected_blocks(sec_a, hd_a, sec_b, hd_b):
    """Blocks where two consecutive full files differ, plus those reaching past the earlier file's rows / log length."""
    Ra, Rb = len(sec_a["state"]), len(sec_b["state"])
    dirty = set(range(Ra // BLOCK_ROWS, (Rb + BLOCK_ROWS - 1) // BLOCK_ROWS))
    for w in WORDS:
        a, b = sec_a[w], sec_b[w]
        if len(b) == 0:
            continue
        diff = np.nonzero(a[: min(len(a), len(b))] != b[: len(a)])[0]
        dirty |= set((diff // BLOCK_ROWS).tolist())
    logs = []
    for name in ("completed_log", "failed_log"):
        a, b = sec_a[name], sec_b[name]
        d = set(range(len(a) // LOG_BLOCK, (len(b) + LOG_BLOCK - 1) // LOG_BLOCK))
        k = min(len(a), len(b))
        d |= set((np.nonzero(a[:k] != b[:k])[0] // LOG_BLOCK).tolist())
        logs.append(sorted(d))
    return sorted(b for b in dirty if b * BLOCK_ROWS < Rb), logs


def _mark(mask, at, n):
    """mask[at[k]: at[k] + n[k]] = True for every k"""
    n = np.asarray(n, dtype=np.int64)
    if n.sum():
        start = np.cumsum(n) - n
        mask[np.repeat(np.asarray(at, dtype=np.int64), n) + np.arange(int(n.sum())) - np.repeat(start, n)] = True


def referenced(sec, hd, var):
    """Byte masks of the slab and the response bytes that some row of the cut's window refers to (everything else there
    is unspecified: outside the window, skipped at a lap's end, or never written by either engine, such as 16 B padding),
    and the physical rows of the window that hold a row (state != 0)."""
    ring = bool(hd["flags"] & R)
    S, used, tail = int(hd["slab_rows"]), int(hd["rows_used"]), int(hd["tail"])
    L = np.arange(tail, used, dtype=np.int64)
    live = L % S if ring else L
    live = live[sec["state"][live] != 0]
    slab = np.zeros(len(sec["slab"]), dtype=bool)
    resp = np.zeros(len(sec["resp"]), dtype=bool)
    if var:
        _mark(slab, sec["voff"][live], sec["vlen"][live])
    else:
        slab.reshape(-1, 512)[live] = True
    for off, ln in (("resp_off", "resp_len"), ("err_off", "err_len")):
        _mark(resp, sec[off][live], sec[ln][live])
    return slab, resp, live.tolist()
