"""Plain reference of the checksum pass for LONG variable-length records (stored length over AGR_VAR_MAX_RECORD,
k1v_long_sums in csrc/agr_k1_var.cu), and batch builders that allow such records.

  piece_cksums  a record's checksum assembled the way the pass computes it: the record cut into pieces of piece_words u32
                words, each piece summing s0 = sum w and s1 = sum (k + 1) w with k the word's index IN THE RECORD, the pieces'
                sums added mod 2^32 and packed (s1 << 32 | s0).  Equal to verifyref.record_cksums / k1vref.cksum of the
                whole record for any cut, since sums mod 2^32 do not depend on the order they are taken in.
  stored_len    the stored length a header gives, capped at a limit (binding.var_record_len with an engine's max_record_bytes)
  blob_from     k1vref.blob_from without its 8 KiB bound on a record's length

Nothing here reads engine output, and nothing needs a GPU."""
import numpy as np

import k1vref

PIECE_WORDS = 8192 // 4          # words per piece of k1v_long_sums (VT_TILE bytes)
M32 = np.uint64(0xFFFFFFFF)


def piece_cksums(blob, offsets, piece_words=PIECE_WORDS) -> np.ndarray:
    """per record of the batch: the packed checksum from its pieces of piece_words words"""
    o = np.asarray(offsets, dtype=np.int64)
    out = np.zeros(len(o) - 1, dtype=np.uint64)
    for i in range(len(o) - 1):
        w = np.asarray(blob[o[i]: o[i + 1]]).view("<u4")
        s0 = s1 = np.uint64(0)
        for p in range(0, len(w), piece_words):
            x = w[p: p + piece_words].astype(np.uint64)
            k1 = np.arange(p + 1, p + 1 + len(x), dtype=np.uint64)
            s0 = (s0 + (x.sum() & M32)) & M32
            s1 = (s1 + (((x * k1) & M32).sum() & M32)) & M32
        out[i] = (s1 << np.uint64(32)) | s0
    return out


def stored_len(h, cap) -> np.ndarray:
    p = h["path_len"].astype(np.int64) + h["hdr_len"].astype(np.int64) + h["body_len"].astype(np.int64)
    return np.minimum(cap, k1vref.HDR + (p + 15) // 16 * 16)


def blob_from(h, lens, rng):
    """The batch: records back to back, header h[i] then random payload bytes (pad included) of record i."""
    lens = np.asarray(lens, dtype=np.int64)
    assert (lens % 16 == 0).all() and (lens >= k1vref.HDR).all()
    offs = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    assert offs[-1] < 1 << 32
    blob = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    blob[(offs[:-1, None] + np.arange(k1vref.HDR)[None, :]).ravel()] = h.view(np.uint8).reshape(len(h), k1vref.HDR).ravel()
    return blob, offs.astype(np.uint32)
