"""Plain reference of where a variable-length engine puts the 512-byte slots of the rows agr_reserve_rows hands out: each
reservation takes its slots back to back from the byte slab's cursor; in ring mode a reservation never wraps (the rest of
the lap is skipped) and fits only while everything from the tail to its end stays within one lap, as agr_ingest_var's blobs."""
SLOT = 512


def slot_layout(cap: int, ring: bool, ops) -> list:
    """ops: ("reserve", n) with n >= 1, or ("release_all",) (every row so far expired and reclaimed: the tail reaches the
    cursor).  Per op: the physical byte offset of the reservation's first slot, "ENOSPC" or "EINVAL"; None for a release."""
    used = tail = 0
    out = []
    for op in ops:
        if op[0] == "release_all":
            tail = used
            out.append(None)
            continue
        need = op[1] * SLOT
        if not ring:
            if used + need > cap:
                out.append("ENOSPC")
                continue
            out.append(used)
            used += need
            continue
        if need > cap // 2:
            out.append("EINVAL")
            continue
        at = used % cap
        pad = cap - at if at + need > cap else 0
        if used + pad + need - tail > cap:
            out.append("ENOSPC")
            continue
        used += pad
        out.append(used % cap)
        used += need
    return out
