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


def relocate(hd, agents, sec, flags, slab_rows, vcap, resp_cap):
    """(header, agent table, sections) of the full file an engine of these flags and capacities writes right after restoring
    the file (hd, agents, sec) with relocation.  Raises NoSpace for what agr_restore refuses with AGR_ENOSPC."""
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

    out = np.zeros(1, dtype=hd.dtype)[0]
    for name in hd.dtype.names:
        out[name] = hd[name]
    out["flags"] = flags & (K.AGR_CFG_PERSISTENCE | K.AGR_CFG_MINT_IDS | V | R)
    out["slab_rows"], out["vcap"], out["resp_cap"] = slab_rows, vcap if var else 0, resp_cap
    out["vused"], out["vtail"] = rec_total, 0
    out["resp_used"], out["resp_tail"] = rsp_total, 0

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
