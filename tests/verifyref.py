"""Plain reference of the integrity sweep (agr_verify / k_verify, csrc/agr_kernels.cu), built from the per-row words and the
slab bytes of an engine: which physical rows the sweep examines, how many it reports as checked, and which it must count as
bad.  The checksum itself is k1ref.cksum (512-byte rows) and k1vref.cksum (variable-length records).

The rules:
  - the sweep covers the physical rows [0, rows_span) that are not rows of an undecided reservation (agr_reserve_rows not yet
    followed by agr_ingest_rows); rows_checked is the number of rows it covers;
  - of those it examines every row on an append-only engine, and only the rows whose state has ST_STORED on a ring;
  - a row's bytes are its 512-byte row, or [voff, voff + vlen) of the byte slab on a variable-length engine (vlen 0: no
    bytes, checksum 0);
  - an examined row is bad when agr_cksum_pack(c0, c1) over its little-endian u32 words differs from its checksum word,
    c0 = sum w_k and c1 = sum (k + 1) w_k, both mod 2^32.

Nothing here needs a GPU."""
from typing import NamedTuple

import numpy as np

import k1ref
import k1vref

ST_STORED = k1ref.ST_STORED
REC = 512


class Sweep(NamedTuple):
    checked: int            # rows_checked: rows in the swept ranges
    examined: np.ndarray    # physical rows whose checksum is compared
    bad: np.ndarray         # physical rows the sweep counts


def reserved_rows(resv, span, slab_rows=None, ring=False) -> np.ndarray:
    """bool mask over the physical rows [0, span) of the undecided reservations; resv: (first, end) runs of logical rows, which
    on a ring lie at row mod slab_rows (a run may wrap there)"""
    m = np.zeros(span, dtype=bool)
    for first, end in resv:
        lr = np.arange(first, end, dtype=np.int64)
        p = lr % slab_rows if ring else lr
        m[p[p < span]] = True
    return m


def record_cksums(rows, slab, voff=None, vlen=None) -> np.ndarray:
    """the checksum of the bytes of each physical row in `rows`: its 512-byte row, or its [voff, voff + vlen) bytes"""
    rows = np.asarray(rows, dtype=np.int64)
    slab = np.asarray(slab, dtype=np.uint8)
    if voff is None:
        return k1ref.cksum(slab.reshape(-1, REC)[rows]) if len(rows) else np.zeros(0, np.uint64)
    out = np.zeros(len(rows), dtype=np.uint64)
    at = np.asarray(voff, dtype=np.int64)[rows]
    ln = np.asarray(vlen, dtype=np.int64)[rows]
    has = np.nonzero(ln > 0)[0]
    if len(has):
        n = ln[has]
        offs = np.concatenate([[0], np.cumsum(n)])
        idx = np.repeat(at[has], n) + np.arange(int(offs[-1])) - np.repeat(offs[:-1], n)
        out[has] = k1vref.cksum(slab[idx], offs)
    return out


def sweep(state, cksum, slab, *, span, ring, resv=(), slab_rows=None, voff=None, vlen=None) -> Sweep:
    """What agr_verify reports.  state / cksum (and voff / vlen on a variable-length engine): the per-row words by physical
    row; slab: the slab (fixed stride, 512 B per physical row) or the byte slab; span: rows_span (rows_used, or at most
    slab_rows on a ring); resv: the undecided reservations as (first, end) logical rows."""
    skip = reserved_rows(resv, span, slab_rows, ring)
    cover = ~skip
    look = cover & ((np.asarray(state[:span]) & ST_STORED) != 0) if ring else cover
    rows = np.nonzero(look)[0]
    got = record_cksums(rows, slab, voff, vlen)
    bad = rows[got != np.asarray(cksum, dtype=np.uint64)[rows]]
    return Sweep(int(cover.sum()), rows, bad)
