"""Plain restatement of the engine-minted request ids (DESIGN section 3.1) in Python integers: what agr_mint_id computes and
how a lookup places a presented id in the live window.  The tests check the C header and the kernels against it; nothing here
comes from the engine."""

M64 = (1 << 64) - 1
M60 = (1 << 60) - 1
M40 = (1 << 40) - 1
ROW_LIMIT = 1 << 52            # rows (arrival numbers) an engine hands out; ids are unique below it
C1, C2 = 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9


def fmix64(k):
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M64
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M64
    return k ^ (k >> 33)


def perm60(x):
    x &= M60
    x = (x * C1) & M60
    x ^= x >> 29
    x = (x * C2) & M60
    return x ^ (x >> 31)


def perm60_inv(y):
    y &= M60
    y ^= y >> 31
    y = (y * pow(C2, -1, 1 << 60)) & M60
    y ^= y >> 29
    y ^= y >> 58
    return (y * pow(C1, -1, 1 << 60)) & M60


def packed(row, shard=0, gen=1):
    """The 60-bit value an id encodes: row mod 2^40, the shard, and the generation field gen ^ (row >> 40)."""
    return (row & M40) | ((shard & 0xFF) << 40) | (((gen ^ (row >> 40)) & 0xFFF) << 48)


def mint(row, secret, shard=0, gen=1):
    """(lo, hi) of the id of `row`: lo = the keyed permutation of packed() around the UUIDv4 version nibble, hi = a keyed hash
    of the same value with the RFC 4122 variant bits."""
    x = packed(row, shard, gen)
    y = perm60(x ^ (secret & M60))
    lo = (y & ((1 << 52) - 1)) | (0x4 << 52) | ((y >> 52) << 56)
    hi = fmix64(((((x + 0x632BE59BD9B4E019) & M64) * 0x9E3779B97F4A7C15) & M64) ^ (secret >> 7))
    return lo, (hi & ~0xC0 & M64) | 0x80


def mint_bytes(row, secret, shard=0, gen=1):
    lo, hi = mint(row, secret, shard, gen)
    return lo.to_bytes(8, "little") + hi.to_bytes(8, "little")


def mint_many(first, n, secret, shard=0, gen=1):
    import numpy as np
    return np.frombuffer(b"".join(mint_bytes(first + i, secret, shard, gen) for i in range(n)), dtype=np.uint8).reshape(n, 16)


def decode(lo, hi, secret, shard, gen, tail, head):
    """Row of the window [tail, head) (head - tail < 2^40) the id (lo, hi) was minted for, or None."""
    if (lo >> 52) & 0xF != 0x4:
        return None
    y = (lo & ((1 << 52) - 1)) | ((lo >> 56) << 52)
    x = perm60_inv(y) ^ (secret & M60)
    row = tail + (((x & M40) - tail) % (1 << 40))
    if row >= head or mint(row, secret, shard, gen) != (lo, hi):
        return None
    return row


def split(idbytes):
    b = bytes(idbytes)
    return int.from_bytes(b[:8], "little"), int.from_bytes(b[8:], "little")
