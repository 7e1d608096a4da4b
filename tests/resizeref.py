"""Plain reference of a restore that relocates (agr_restore into other capacities, DESIGN.md section 5): from a full file's
parsed form (snapfile.parse) to the full file the relocated engine writes right after the restore.  Needs no GPU."""
import numpy as np

from agentainer_lab_b200 import constants as K
from snapfile import R, V, WORDS, sections


class NoSpace(Exception):
    """What agr_restore refuses with AGR_ENOSPC: the live state does not fit the new capacities."""


def r16(x):
    return (int(x) + 15) & ~15


def src_phys(hd, L):
    return L % int(hd["slab_rows"]) if int(hd["flags"]) & R else L


def src_logical(hd, p):
    """Row id of physical row p in the source's window."""
    if not int(hd["flags"]) & R:
        return p
    S, tail = int(hd["slab_rows"]), int(hd["tail"])
    return tail + (p - tail % S) % S


def _header(hd, flags, slab_rows, vcap, resp_cap, var, rec_total, rsp_total):
    out = np.zeros(1, dtype=hd.dtype)[0]
    for name in hd.dtype.names:
        out[name] = hd[name]
    out["flags"] = flags & (K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | V | R)
    out["slab_rows"], out["vcap"], out["resp_cap"] = slab_rows, vcap if var else 0, resp_cap
    out["vused"], out["vtail"] = rec_total, 0
    out["resp_used"], out["resp_tail"] = rsp_total, 0
    return out


def _gather(dst, src, dst_at, src_at, n):
    """dst[dst_at[k]: + n[k]] = src[src_at[k]: + n[k]] for every k, in one indexed copy"""
    n = np.asarray(n, dtype=np.int64)
    total = int(n.sum())
    if total == 0:
        return
    start = np.cumsum(n) - n
    step = np.arange(total, dtype=np.int64) - np.repeat(start, n)
    dst[np.repeat(np.asarray(dst_at, dtype=np.int64), n) + step] = src[np.repeat(np.asarray(src_at, dtype=np.int64), n) + step]


def relocate(hd, agents, sec, flags, slab_rows, vcap, resp_cap):
    """(header, agent table, sections) of the full file an engine of these flags and capacities writes right after restoring
    the file (hd, agents, sec) with relocation.  Raises NoSpace for what agr_restore refuses with AGR_ENOSPC.  The same rules
    as relocate_loop, one array operation per step, so that windows of 2^19 rows and more take seconds."""
    var = bool(int(hd["flags"]) & V)
    tail, used = int(hd["tail"]), int(hd["rows_used"])
    if used - tail > slab_rows:
        raise NoSpace("window")
    L = np.arange(tail, used, dtype=np.int64)
    ps = L % int(hd["slab_rows"]) if int(hd["flags"]) & R else L
    pt = L % slab_rows
    live = sec["state"][ps] != 0
    vlen = np.where(live, sec["vlen"][ps].astype(np.int64), 0) if var else None
    # per window row: its response segment then its error segment, each from a 16 B boundary; dead rows take no bytes
    seg = np.stack([np.where(live, sec[ln][ps].astype(np.int64), 0) for ln in ("resp_len", "err_len")], axis=1).reshape(-1)
    seg16 = (seg + 15) & ~15
    rec_total = int(vlen.sum()) if var else 0
    rsp_total = int(seg16.sum())
    if var and rec_total > vcap:
        raise NoSpace("vslab_bytes")
    if rsp_total > resp_cap:
        raise NoSpace("resp_bytes")

    out = _header(hd, flags, slab_rows, vcap, resp_cap, var, rec_total, rsp_total)
    new = {name: np.zeros(count, dtype=dt) for name, dt, count in sections(out)}
    for w in WORDS:
        if len(new[w]):
            new[w][pt] = sec[w][ps]
    if var:
        rec_at = np.cumsum(vlen) - vlen
        new["voff"][pt] = np.where(live, rec_at, 0)
        _gather(new["slab"], sec["slab"], rec_at, sec["voff"][ps], vlen)
    else:
        new["slab"].reshape(-1, 512)[pt] = sec["slab"].reshape(-1, 512)[ps]
    rsp_at = np.cumsum(seg16) - seg16
    src_at = np.stack([sec["resp_off"][ps], sec["err_off"][ps]], axis=1).reshape(-1).astype(np.int64)
    at = np.where(seg > 0, rsp_at, 0).reshape(-1, 2)
    new["resp_off"][pt], new["err_off"][pt] = at[:, 0], at[:, 1]
    _gather(new["resp"], sec["resp"], rsp_at, src_at, seg)
    for name in ("completed_log", "failed_log"):
        e = sec[name].astype(np.int64)
        none = e == 0xFFFFFFFF
        if int(hd["flags"]) & R:
            S = int(hd["slab_rows"])
            e = tail + (e - tail % S) % S
        new[name][:] = np.where(none, 0xFFFFFFFF, e % slab_rows)
    return out, agents, new


def relocate_loop(hd, agents, sec, flags, slab_rows, vcap, resp_cap):
    """relocate, one row at a time: the form the rules are easiest to read in (and the one relocate is checked against)."""
    var = bool(int(hd["flags"]) & V)
    tail, used = int(hd["tail"]), int(hd["rows_used"])
    if used - tail > slab_rows:
        raise NoSpace("window")
    window = list(range(tail, used))
    live = [L for L in window if sec["state"][src_phys(hd, L)] != 0]
    rec_total = sum(int(sec["vlen"][src_phys(hd, L)]) for L in live) if var else 0
    rsp_total = sum(r16(sec["resp_len"][src_phys(hd, L)]) + r16(sec["err_len"][src_phys(hd, L)]) for L in live)
    if var and rec_total > vcap:
        raise NoSpace("vslab_bytes")
    if rsp_total > resp_cap:
        raise NoSpace("resp_bytes")

    out = _header(hd, flags, slab_rows, vcap, resp_cap, var, rec_total, rsp_total)
    new = {name: np.zeros(count, dtype=dt) for name, dt, count in sections(out)}
    slab = new["slab"]
    rec_at = rsp_at = 0
    for L in window:
        ps, pt = src_phys(hd, L), L % slab_rows
        for w in WORDS:
            if len(new[w]):
                new[w][pt] = sec[w][ps]
        is_live = sec["state"][ps] != 0
        if var:
            new["voff"][pt] = rec_at if is_live else 0
            if is_live:
                n, o = int(sec["vlen"][ps]), int(sec["voff"][ps])
                slab[rec_at: rec_at + n] = sec["slab"][o: o + n]
                rec_at += n
        else:
            slab[pt * 512: (pt + 1) * 512] = sec["slab"][ps * 512: (ps + 1) * 512]
        new["resp_off"][pt] = new["err_off"][pt] = 0
        if is_live:
            for off, ln in (("resp_off", "resp_len"), ("err_off", "err_len")):
                n = int(sec[ln][ps])
                if n:
                    o = int(sec[off][ps])
                    new[off][pt] = rsp_at
                    new["resp"][rsp_at: rsp_at + n] = sec["resp"][o: o + n]
                rsp_at += r16(n)
    for name in ("completed_log", "failed_log"):
        new[name][:] = [e if e == 0xFFFFFFFF else src_logical(hd, int(e)) % slab_rows for e in sec[name]]
    return out, agents, new


def content(hd, sec):
    """Per live row id: its words without the byte offsets, its record (512 B row or record bytes), response and error bytes.
    What a relocation keeps."""
    var = bool(int(hd["flags"]) & V)
    out = {}
    for L in range(int(hd["tail"]), int(hd["rows_used"])):
        p = src_phys(hd, L)
        if sec["state"][p] == 0:
            continue
        words = tuple(int(sec[w][p]) for w in WORDS if len(sec[w]) and w not in ("voff", "resp_off", "err_off"))
        rec = bytes(sec["slab"][int(sec["voff"][p]): int(sec["voff"][p]) + int(sec["vlen"][p])]) if var else bytes(sec["slab"][p * 512: (p + 1) * 512])
        segs = tuple(bytes(sec["resp"][int(sec[o][p]): int(sec[o][p]) + int(sec[n][p])]) for o, n in (("resp_off", "resp_len"), ("err_off", "err_len")))
        out[L] = (words, rec, segs)
    return out


def log_rows(hd, sec):
    """The completed / failed logs as row ids."""
    return [[None if e == 0xFFFFFFFF else src_logical(hd, int(e)) for e in sec[name]] for name in ("completed_log", "failed_log")]
