"""Plain reference of a restore that converts the record form (agr_restore of a snapshot into a ring of the other form,
DESIGN.md section 5): the source is first rewritten in the target's form at its own geometry, then relocated by the rules of
resizeref.  Fixed-stride to variable-length: a live row becomes its compact record, the row's first
96 + round16(path_len + hdr_len + body_len) bytes.  Variable-length to fixed-stride: a live record becomes a 512 B row, its
bytes then zeros.  Every per-row word moves unchanged.  Needs no GPU."""
import numpy as np

from resizeref import NoSpace, _gather, r16, relocate, relocate_loop, src_phys
from snapfile import R, V

REC, HDR = 512, 96

__all__ = ["NoSpace", "NotRepresentable", "compact_len", "convert", "convert_loop", "bad_rows"]


class NotRepresentable(Exception):
    """What agr_restore refuses with AGR_EINVAL: a live record longer than the fixed form's 512 B row."""


def compact_len(row):
    """The compact length of one 512 B row's record (capped at the row)."""
    row = bytes(row[:84])
    n = int.from_bytes(row[76:78], "little") + int.from_bytes(row[78:80], "little") + int.from_bytes(row[80:84], "little")
    return min(HDR + r16(n), REC)


def _compact_lens(slab, ps):
    """compact_len of the 512 B rows ps of a fixed-stride slab"""
    h = np.ascontiguousarray(slab.reshape(-1, REC)[ps, 76:84]).view("<u2").astype(np.int64)
    n = h[:, 0] + h[:, 1] + h[:, 2] + (h[:, 3] << 16)
    return np.minimum(HDR + ((n + 15) & ~15), REC)


def _window(hd, sec):
    """row ids of the window, their physical rows, and which hold a record"""
    tail, used = int(hd["tail"]), int(hd["rows_used"])
    L = np.arange(tail, used, dtype=np.int64)
    ps = L % int(hd["slab_rows"]) if int(hd["flags"]) & R else L
    return L, ps, sec["state"][ps] != 0


def _recast(hd, sec, var_t):
    """(header, sections) to fill in: the source's, with the other form's record sections"""
    out = np.zeros(1, dtype=hd.dtype)[0]
    for name in hd.dtype.names:
        out[name] = hd[name]
    rows = len(sec["state"])
    new = dict(sec)
    if var_t:
        out["flags"] = int(hd["flags"]) | V
        new["voff"], new["vlen"] = np.zeros(rows, dtype="<u8"), np.zeros(rows, dtype="<u4")
    else:
        out["flags"] = int(hd["flags"]) & ~V
        out["vcap"] = out["vused"] = out["vtail"] = 0
        new["voff"], new["vlen"] = np.zeros(0, dtype="<u8"), np.zeros(0, dtype="<u4")
        new["slab"] = np.zeros(rows * REC, dtype=np.uint8)
    return out, new


def _refuse_oversize(L, ps, live, vlen):
    big = np.nonzero(live & (vlen[ps] > REC))[0] if len(L) else []
    if len(big):
        raise NotRepresentable("%d live records are longer than 512 B (the first: row %d, %d B)" % (len(big), int(L[big[0]]), int(vlen[ps[big[0]]])))


def to_form(hd, sec, var_t):
    """The source (hd, sec) in the record form var_t at its own geometry: fixed-stride rows as records at their own place
    (voff = physical row * 512, vlen = compact length; 0 for rows that hold none), or records as 512 B rows.  Array form."""
    L, ps, live = _window(hd, sec)
    out, new = _recast(hd, sec, var_t)
    if var_t:
        new["voff"][ps] = ps * REC
        new["vlen"][ps] = np.where(live, _compact_lens(sec["slab"], ps) if len(ps) else 0, 0)
        out["vcap"] = len(sec["slab"])
    else:
        _refuse_oversize(L, ps, live, sec["vlen"])
        _gather(new["slab"], sec["slab"], ps * REC, sec["voff"][ps], np.where(live, sec["vlen"][ps], 0))
    return out, new


def to_form_loop(hd, sec, var_t):
    """to_form, one row at a time"""
    L, ps, live = _window(hd, sec)
    out, new = _recast(hd, sec, var_t)
    if not var_t:
        _refuse_oversize(L, ps, live, sec["vlen"])
    for x in range(int(hd["tail"]), int(hd["rows_used"])):
        p = src_phys(hd, x)
        if sec["state"][p] == 0:
            continue
        if var_t:
            new["voff"][p], new["vlen"][p] = p * REC, compact_len(sec["slab"][p * REC: (p + 1) * REC])
        else:
            o, n = int(sec["voff"][p]), int(sec["vlen"][p])
            new["slab"][p * REC: p * REC + n] = sec["slab"][o: o + n]
    if var_t:
        out["vcap"] = len(sec["slab"])
    return out, new


def _check_window(hd, slab_rows):
    if int(hd["rows_used"]) - int(hd["tail"]) > slab_rows:
        raise NoSpace("window")


def convert(hd, agents, sec, flags, slab_rows, vcap, resp_cap):
    """(header, agent table, sections) of the full file an engine of these flags (the other record form than hd's) and
    capacities writes right after restoring the file (hd, agents, sec).  Raises NoSpace / NotRepresentable for what
    agr_restore refuses with AGR_ENOSPC / AGR_EINVAL, in its order: the window, oversized records, then the byte rings."""
    _check_window(hd, slab_rows)
    h2, s2 = to_form(hd, sec, bool(flags & V))
    return relocate(h2, agents, s2, flags, slab_rows, vcap, resp_cap)


def convert_loop(hd, agents, sec, flags, slab_rows, vcap, resp_cap):
    """convert, one row at a time (the form it is checked against)"""
    _check_window(hd, slab_rows)
    h2, s2 = to_form_loop(hd, sec, bool(flags & V))
    return relocate_loop(h2, agents, s2, flags, slab_rows, vcap, resp_cap)


def bad_rows(hd, sec):
    """Row ids of a fixed-stride file's live rows whose bytes past their compact length are not zero: after a conversion to
    variable-length records their checksum no longer matches (agr_verify counts them)."""
    L, ps, live = _window(hd, sec)
    if not len(L):
        return []
    rows = sec["slab"].reshape(-1, REC)[ps]
    past = np.arange(REC)[None, :] >= _compact_lens(sec["slab"], ps)[:, None]
    return L[live & ((rows != 0) & past).any(axis=1)].tolist()
