"""Plain reference of K4, the multi-GPU exchange's binning (agr_k4.cu): Python ints and numpy, no engine code.

An item is `item_bytes` bytes with a 32 B agent id at `agent_off` (records: 512 B at 32; outcomes: 64 B at 16).  Its owner is
FNV-1a 64 over the id's bytes up to the first NUL, mod G.  Items are placed owner-major and stable: item i goes to
goff[owner] + (earlier items with the same owner).  In place (records already in their slab rows) this shard's own items stay
where they are, the send buffer holds the peers' items only, and positions of owners above `me` move down by gtotal[me]; the
rows of the items that leave are holes at this shard."""
import numpy as np

FNV_OFFSET = 0xCBF29CE484222325
FNV_PRIME = 0x100000001B3
M64 = (1 << 64) - 1


def fnv1a64(b: bytes) -> int:
    """FNV-1a 64 of `b` up to its first NUL byte."""
    h = FNV_OFFSET
    for c in b:
        if c == 0:
            break
        h = ((h ^ c) * FNV_PRIME) & M64
    return h


def owners(raw: np.ndarray, agent_off: int, G: int) -> np.ndarray:
    """owner of every item of `raw` ((n, item_bytes) uint8); each distinct id is hashed once."""
    if len(raw) == 0:
        return np.zeros(0, np.uint8)
    ids = np.ascontiguousarray(raw[:, agent_off: agent_off + 32]).view("V32").ravel()
    uniq, inv = np.unique(ids, return_inverse=True)
    own = np.array([fnv1a64(bytes(u)) % G for u in uniq], dtype=np.uint8)
    return own[inv.ravel()]


def partition(owner, G: int, me: int, inplace: bool) -> dict:
    """gtotal[G], goff[G + 1] and every item's position, as K4 lays them out: a stable sort by owner."""
    owner = np.asarray(owner, dtype=np.int64)
    gtotal = np.bincount(owner, minlength=G).astype(np.int64)
    goff = np.concatenate([[0], np.cumsum(gtotal)])
    perm = np.empty(len(owner), np.int64)
    perm[np.argsort(owner, kind="stable")] = np.arange(len(owner))
    if inplace:
        perm[owner > me] -= gtotal[me]
    return dict(gtotal=gtotal.astype(np.uint32), goff=goff.astype(np.uint32), perm=perm.astype(np.uint32))


def expected(raw: np.ndarray, agent_off: int, G: int, me: int, inplace: bool) -> dict:
    """Everything agr_debug_k4 returns for `raw`, byte for byte: owner, perm, gtotal, goff, the send and local buffers (n items
    each, zero where nothing is written), the items after the pass (unchanged), and the rows that become holes."""
    n, ib = raw.shape
    own = owners(raw, agent_off, G)
    part = partition(own, G, me, inplace)
    send = np.zeros((n, ib), np.uint8)
    local = np.zeros((n, ib), np.uint8)
    peer = own != me
    send[part["perm"][peer]] = raw[peer]
    if not inplace:
        local[part["perm"][~peer].astype(np.int64) - int(part["goff"][me])] = raw[~peer]
    holes = peer if inplace else np.zeros(n, bool)
    return dict(owner=own, send=send, local=local, items=raw.copy(), holes=holes, **part)


def unpermute(owner, perm, goff, me: int, inplace: bool, local_res: np.ndarray, remote_res: np.ndarray) -> np.ndarray:
    """Results back in item order: an own item's result from local_res (by item in place, by local position otherwise), a
    peer's from remote_res at its owner-major position."""
    owner, perm = np.asarray(owner), np.asarray(perm, np.int64)
    mine = owner == me
    out = np.zeros(len(owner), dtype=local_res.dtype)
    out[~mine] = remote_res[perm[~mine]]
    out[mine] = local_res[np.nonzero(mine)[0] if inplace else perm[mine] - int(goff[me])]
    return out
