"""Executable model of vlscan_last_rows (the N newest selected rows, `/select/logsql/query?limit=N`) and its brute-force definition (tests only).

A block is (mn, mx, ts, sel): its header minimum and maximum, the timestamps of its rows (non-decreasing) and its selected rows ascending.
"""

SIGN = 1 << 63
M64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
GEN_T0, GEN_STEP = 1700000000000000000, 1000000   # the generator's timestamps column: VLSCAN_GEN_T0, VLSCAN_GEN_STEP


def gen_timestamps(cfg, block_id):
    """The timestamps of block `block_id` of a generated data set with the timestamps column (columns_mask bit 4).  Bits 12..16 = k interleave
    S = 2^k blocks: row i of block b at GEN_T0 + ((b // S) * S * R + i * S + b % S) * GEN_STEP; k = 0 is one row every GEN_STEP from GEN_T0
    (vlohits.gen_timestamps)."""
    first = block_id * cfg.rows_per_block
    rows = min(cfg.rows_per_block, cfg.total_rows - first)
    s = 1 << ((cfg.columns_mask >> 12) & 31)
    base = (block_id // s) * s * cfg.rows_per_block + block_id % s
    return [GEN_T0 + (base + i * s) * GEN_STEP for i in range(rows)]


def brute_force(blocks, limit, floor=I64_MIN):
    """getLastNRows over the selected rows with ts >= floor, ordered by (ts, block, row): the last `limit` of them, ascending"""
    rows = sorted((b[2][r], bi, r) for bi, b in enumerate(blocks) for r in b[3] if b[2][r] >= floor)
    return rows[max(0, len(rows) - limit):]


def radix_select(keys, limit):
    """The limit-th largest of the int64 keys [(key, weight)], 8 passes of 8 bits over the sign-flipped keys, as k_radix_hist / k_radix_pick do
    -> (key, how many keys equal to it are needed), or None when the weights add up to less than the limit"""
    cur = [((k & M64) ^ SIGN, w) for k, w in keys if w]
    if sum(w for _, w in cur) < limit:
        return None
    prefix, k = 0, limit
    for p in range(8):
        shift = 56 - 8 * p
        hist = [0] * 256
        for u, w in cur:
            hist[(u >> shift) & 255] += w
        above, d = 0, 255
        while d > 0 and above + hist[d] < k:
            above += hist[d]
            d -= 1
        prefix |= d << shift
        k -= above
        cur = [(u, w) for u, w in cur if (u >> shift) & 255 == d]
    key = prefix ^ SIGN
    return (key - (1 << 64) if key >> 63 else key), k


class HeaderMismatch(Exception):
    pass


def model(blocks, limit, floor=I64_MIN):
    """The device algorithm -> (rows ascending, blocks whose timestamps are decoded).  Raises HeaderMismatch where the call fails."""
    sel = radix_select([(b[0], len(b[3])) for b in blocks if b[3] and b[0] >= floor], limit)
    t_lo = floor if sel is None else sel[0]
    cands, decoded = [], 0
    for bi, (mn, mx, ts, rows) in enumerate(blocks):
        if not rows or mx < t_lo:
            continue
        flat = mn == mx
        if not flat:
            decoded += 1
            if any(t < mn or t > mx for t in ts):
                raise HeaderMismatch(bi)
        for r in rows:
            t = mn if flat else ts[r]
            if t >= t_lo:
                cands.append((t, bi, r))
    if sel is not None and len(cands) < limit:
        raise HeaderMismatch(None)
    top = radix_select([(t, 1) for t, _, _ in cands], limit)
    if top is None:
        chosen = cands
    else:
        tn, k = top
        ties = [c for c in cands if c[0] == tn]
        chosen = [c for c in cands if c[0] > tn] + ties[len(ties) - k:]
    return sorted(chosen), decoded
