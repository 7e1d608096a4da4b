"""Plain reference of the variable-length ingest (K1v, csrc/agr_k1_var.cu), built only from what a test feeds the engine.

  wire form     headers(), fit_lens(), blob_from(), layout(): numpy-vectorised builders of a batch (blob + offsets) that
                follow the contract of include/agentainer_gpu.h (lengths multiples of 16 in [96, 8192], offsets[0] = 0)
  tile_owners   "tile t owns the records that start in [t * 8192, (t + 1) * 8192)", and the facts about each tile that
                decide which code path the two forms of K1v take (records per tile, stage span, sweep rows, starts per row)
  grid          how the two forms spread the tiles over CTAs and warps
  cksum         the record checksum: (sum (k + 1) w_k mod 2^32) << 32 | (sum w_k mod 2^32) over the record's u32 words
  twin_records  each record as a 512 B agr_record whose K1 decision equals the variable-length record's: same header, and
                path + headers + body <= 416 exactly when the record fits its own stored payload
  readback      the bytes agr_get_record_var / agr_replay_scan_var hand back for a record, given its row's live words

Nothing here reads engine output, and nothing needs a GPU."""
import numpy as np

from agentainer_lab_b200 import constants as K
from agentainer_lab_b200.binding import header_dtype, record_dtype

TILE = 8192                  # bytes of blob per tile (VT_TILE)
STAGE = 12800                # staged form: bytes of a tile's records that land in the warp's stage (VT_STAGE)
MAXCNT = TILE // 96 + 2      # most records that can start in one tile, plus one (VT_MAXCNT = 87)
HDR = 96
MAXREC = K.AGR_VAR_MAX_RECORD
ROW = 32                     # LSU form: 16 B chunks per sweep row (one per lane)
STAGED_WARPS, LSU_WARPS, LSU_CTAS_PER_SM = 16, 8, 5
PAYLOAD_FIXED = 512 - HDR    # 416


# ------------------------------------------------------------------------------------------------------- wire form
def check_wire(offsets) -> None:
    o = np.asarray(offsets, dtype=np.int64)
    lens = np.diff(o)
    assert len(o) >= 1 and o[0] == 0, "offsets[0] must be 0"
    assert (lens % 16 == 0).all() and (lens >= HDR).all() and (lens <= MAXREC).all(), "lengths: multiples of 16 in [96, 8192]"


def layout(spec) -> np.ndarray:
    """Record lengths from a list of steps: ("rec", length) appends one record; ("to", offset) appends records (8192 B
    where they fit, never shorter than 96 B) so that the next record starts exactly at offset."""
    lens, at = [], 0
    for kind, v in spec:
        if kind == "rec":
            lens.append(v); at += v
            continue
        gap = v - at
        assert gap == 0 or (gap >= HDR and gap % 16 == 0), (v, at)
        while gap > 0:
            take = min(gap, MAXREC)
            if 0 < gap - take < HDR:
                take = gap - HDR
            lens.append(take); at += take; gap -= take
    out = np.array(lens, dtype=np.int64)
    check_wire(np.concatenate([[0], np.cumsum(out)]))
    return out


def headers(n, agents, rng, *, seq0=1, agent_of=None) -> np.ndarray:
    """n headers: random non-zero caller ids, agent agents[agent_of[i]] (default round robin), seq = seq0 + i, method POST,
    max_retries a mix of 0 (= 3) and 1..7, and junk in the output-only bytes 80..95 after body_len, which the engine ignores
    on input and patches or passes through on output.  Lengths are set by fit_lens()."""
    h = np.zeros(n, dtype=header_dtype)
    h["request_id"] = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    h["request_id"][:, 0] |= 1
    names = np.array([a.encode() for a in agents], dtype="S32")
    h["agent_id"] = names[np.arange(n) % len(agents) if agent_of is None else np.asarray(agent_of)]
    h["seq"] = seq0 + np.arange(n, dtype=np.uint64)
    h["flags"] = K.METHOD_CODES["POST"] << K.AGR_F_METHOD_SHIFT
    h["status"] = rng.integers(0, 256, n)
    h["retry_count"] = rng.integers(0, 256, n)
    h["max_retries"] = np.where(rng.random(n) < 0.3, 0, rng.integers(1, 8, n))
    h["error_code"] = rng.integers(1, 256, n)
    h["resp_status"] = rng.integers(1, 65536, n)
    h["reserved0"] = rng.integers(0, 65536, n)
    h["reserved1"] = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    return h


def fit_lens(h, lens, rng) -> None:
    """path_len / hdr_len / body_len of every record so that 96 + round16(path + headers + body) == its stored length."""
    pay = np.asarray(lens, dtype=np.int64) - HDR
    slack = np.where(pay > 0, rng.integers(0, 16, len(pay)), 0)
    total = pay - np.minimum(slack, np.maximum(pay - 1, 0))
    path = np.minimum(total, rng.integers(1, 64, len(pay)))
    hdr = np.minimum(total - path, rng.integers(0, 200, len(pay)))
    h["path_len"], h["hdr_len"], h["body_len"] = path, hdr, total - path - hdr


def blob_from(h, lens, rng):
    """The batch: records back to back, header h[i] then payload bytes (random, pad included) of record i."""
    lens = np.asarray(lens, dtype=np.int64)
    offs = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    check_wire(offs)
    assert offs[-1] < 1 << 32
    blob = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    blob[(offs[:-1, None] + np.arange(HDR)[None, :]).ravel()] = h.view(np.uint8).reshape(len(h), HDR).ravel()
    return blob, offs.astype(np.uint32)


def header_of(blob, offsets) -> np.ndarray:
    o = np.asarray(offsets, dtype=np.int64)
    return blob[(o[:-1, None] + np.arange(HDR)[None, :]).ravel()].reshape(-1, HDR).copy().view(header_dtype)[:, 0]


def fits(h, lens) -> np.ndarray:
    """K1's length test: path + headers + body fit the stored payload (sum in 64 bits: the fields cannot wrap)."""
    s = h["path_len"].astype(np.int64) + h["hdr_len"].astype(np.int64) + h["body_len"].astype(np.int64)
    return s <= np.asarray(lens, dtype=np.int64) - HDR


# ------------------------------------------------------------------------------------------------------- tiles
class Tiles:
    """tile_owners(offsets): first[0..ntiles] (first[ntiles] = n) and, per tile t with cnt[t] records:
      span[t]       bytes from its first start to the end of its last record (so[cnt] - so[0] in the kernel)
      over[t]       span > STAGE: the staged form's 1-D copy stops at STAGE bytes
      nglobal[t]    records whose end lies beyond the copied bytes: the staged form sums them through global loads
      sweep[t]      chunks the LSU form's linear sweep covers (span / 16)
    and per record i: tile[i], chunk[i] / end_chunk[i] (start and end in the tile's sweep), row[i] = chunk[i] // 32."""

    def __init__(self, offsets):
        o = np.asarray(offsets, dtype=np.int64)
        n = len(o) - 1
        self.n = n
        self.ntiles = int((o[-1] + TILE - 1) // TILE)
        bounds = np.arange(self.ntiles, dtype=np.int64) * TILE
        self.first = np.concatenate([np.searchsorted(o[:-1], bounds, side="left"), [n]]).astype(np.int64)
        self.cnt = np.diff(self.first)
        has = self.cnt > 0
        so0 = np.where(has, o[np.minimum(self.first[:-1], n)], 0)
        self.span = np.where(has, o[self.first[1:]] - so0, 0)
        self.over = self.span > STAGE
        self.sweep = self.span // 16
        self.tile = (o[:-1] // TILE).astype(np.int64)
        base = so0[self.tile]
        self.chunk = (o[:-1] - base) // 16
        self.end_chunk = (o[1:] - base) // 16
        self.row = self.chunk // ROW
        self.global_read = (o[1:] - base) > np.minimum(self.span[self.tile], STAGE)
        self.nglobal = np.bincount(self.tile[self.global_read], minlength=self.ntiles)

    def starts_per_row(self) -> np.ndarray:
        """(tile, row, starts) for every sweep row that holds at least one record start."""
        key = self.tile * 64 + self.row
        u, c = np.unique(key, return_counts=True)
        return np.stack([u // 64, u % 64, c], axis=1)


def tile_owners(offsets) -> Tiles:
    return Tiles(offsets)


def grid(ntiles, sms, lsu):
    """(CTAs, warps per CTA) of a launch over ntiles tiles (agr_launch_k1_var); tile t goes to warp t mod (CTAs * warps),
    i.e. CTA (t mod (CTAs * warps)) // warps, and every warp takes every (CTAs * warps)-th tile after its first."""
    w = LSU_WARPS if lsu else STAGED_WARPS
    ctas = max(1, min(sms * (LSU_CTAS_PER_SM if lsu else 1), (ntiles + w - 1) // w))
    return ctas, w


def tiles_per_warp(ntiles, sms, lsu) -> float:
    c, w = grid(ntiles, sms, lsu)
    return ntiles / (c * w)


def cta_of(tile, ntiles, sms, lsu):
    c, w = grid(ntiles, sms, lsu)
    return (np.asarray(tile) % (c * w)) // w


# ------------------------------------------------------------------------------------------------------- checksum
def cksum(blob, offsets) -> np.ndarray:
    """Per record: (sum_k (k + 1) w_k mod 2^32) << 32 | (sum_k w_k mod 2^32), w = its little-endian u32 words."""
    o = np.asarray(offsets, dtype=np.int64)
    n = len(o) - 1
    out = np.zeros(n, dtype=np.uint64)
    step = 1 << 14
    for a in range(0, n, step):
        b = min(n, a + step)
        w = np.asarray(blob[o[a]: o[b]]).view("<u4").astype(np.uint64)
        starts = (o[a:b] - o[a]) // 4
        k = np.arange(len(w), dtype=np.uint64) - np.repeat(starts.astype(np.uint64), np.diff(o[a: b + 1]) // 4)
        s0 = np.add.reduceat(w, starts) & 0xFFFFFFFF
        s1 = np.add.reduceat(w * (k + 1), starts) & 0xFFFFFFFF
        out[a:b] = (s1 << np.uint64(32)) | s0
    return out


# ------------------------------------------------------------------------------------------------------- twin
def twin_records(blob, offsets) -> np.ndarray:
    """Fixed-stride twins: every header byte kept; path / headers / body lengths shrunk so that their sum is <= 416 exactly
    when the record fits its own stored payload (stored length - 96), else raised above 416 when they are not already.
    The payload bytes are zero: K1's decision never reads them."""
    o = np.asarray(offsets, dtype=np.int64)
    h = header_of(blob, o)
    lens = np.diff(o)
    ok = fits(h, lens)
    p, q, b = (h[f].astype(np.int64) for f in ("path_len", "hdr_len", "body_len"))
    p2 = np.where(ok, np.minimum(p, PAYLOAD_FIXED), p)
    q2 = np.where(ok, np.minimum(q, PAYLOAD_FIXED - p2), q)
    b2 = np.where(ok, np.minimum(b, PAYLOAD_FIXED - p2 - q2), np.where(p + q + b > PAYLOAD_FIXED, b, PAYLOAD_FIXED + 1 - p - q))
    t = np.zeros(len(h), dtype=record_dtype)
    t.view(np.uint8).reshape(len(h), 512)[:, :HDR] = h.view(np.uint8).reshape(len(h), HDR)
    t["path_len"], t["hdr_len"], t["body_len"] = p2, q2, b2
    assert ((t["path_len"].astype(np.int64) + t["hdr_len"] + t["body_len"].astype(np.int64) <= PAYLOAD_FIXED) == ok).all()
    return t


# ------------------------------------------------------------------------------------------------------- read-back
ST_STATUS, ST_RETRY_SHIFT, ST_MAX_SHIFT, AUX_ERR_SHIFT = 0x7, 8, 16, 16


def readback(blob, offsets, state, aux, ids=None) -> np.ndarray:
    """The records of blob as agr_get_record_var / agr_replay_scan_var return them (same layout as blob), given each
    row's live state and aux words and, in mint mode, its minted id (n x 16, else None):
      bytes  0..15  the minted id (mint mode), bytes 84..87 status | retry << 8 | max << 16 | error << 24 of the live row,
      bytes 88..89  the stored response status, every other byte as ingested.
    A record ingested with max_retries = 0 reads back 3 (requests.go:95): K1 puts 3 into the state word."""
    o = np.asarray(offsets, dtype=np.int64)[:-1]
    out = np.array(blob, dtype=np.uint8, copy=True)
    st, ax = np.asarray(state, dtype=np.uint32), np.asarray(aux, dtype=np.uint32)
    w84 = (st & ST_STATUS) | (((st >> ST_RETRY_SHIFT) & 0xFF) << 8) | (((st >> ST_MAX_SHIFT) & 0xFF) << 16) | (((ax >> AUX_ERR_SHIFT) & 0xFF) << 24)
    out[(o[:, None] + 84 + np.arange(4)[None, :]).ravel()] = w84.astype("<u4").view(np.uint8)
    out[(o[:, None] + 88 + np.arange(2)[None, :]).ravel()] = (ax & 0xFFFF).astype("<u2").view(np.uint8)
    if ids is not None:
        out[(o[:, None] + np.arange(16)[None, :]).ravel()] = np.asarray(ids, dtype=np.uint8).ravel()
    return out


def stored_state(h, running) -> np.ndarray:
    """State word K1 gives a record it stores: pending, in the pending list, stored, max_retries (0 -> 3), and in flight
    when its agent is running."""
    mx = h["max_retries"].astype(np.uint32)
    mx = np.where(mx == 0, 3, mx).astype(np.uint32)
    return (1 | 0x8 | 0x20 | (mx << ST_MAX_SHIFT) | np.where(np.asarray(running), 0x10, 0)).astype(np.uint32)


def gather(blob, offsets, idx):
    """records idx (in that order) of blob, packed back to back, and their offsets"""
    o = np.asarray(offsets, dtype=np.int64)
    idx = np.asarray(idx, dtype=np.int64)
    lens = o[idx + 1] - o[idx]
    go = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum(lens, out=go[1:])
    src = np.repeat(o[idx] - go[:-1], lens) + np.arange(int(go[-1]), dtype=np.int64)
    return np.asarray(blob)[src], go
