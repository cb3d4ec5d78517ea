"""Glue between the oracle's encoded blocks and the product's vlscan_block descriptors (tests only)."""
import os

import numpy as np

import vloracle
from victorialogs_b200 import scan as vs


def oracle_block_to_desc(blk, stage="ondisk"):
    """vloracle.Block -> dict accepted by victorialogs_b200.scan.HostBlocks"""
    cols = []
    for name, value in blk.consts:
        cols.append(dict(field=name, kind="const", value=value))
    for c in blk.columns:
        d = dict(field=c.name, kind="values", value_type=c.value_type, min_value=c.min_value, max_value=c.max_value, dict=c.dict, bloom=c.bloom)
        if stage == "ondisk":
            d["values_block"] = c.values_block
        else:
            d["lens_items"], d["data"] = vloracle.decode_values_block(c.values_block)
        cols.append(d)
    d = dict(rows=blk.rows, columns=cols)
    try:
        d["timestamps"] = blk.timestamps_block()   # (encoded bytes, marshalType, minTimestamp, maxTimestamp)
    except ValueError:
        pass
    return d


def field_names_of(blocks):
    names = []
    for b in blocks:
        for n, _ in b.consts:
            if n not in names:
                names.append(n)
        for c in b.columns:
            if c.name not in names:
                names.append(c.name)
    return names


def host_blocks_from_oracle(blocks, stage="ondisk"):
    return vs.HostBlocks(field_names_of(blocks) or [b"_msg"], [oracle_block_to_desc(b, stage) for b in blocks])


ACCOUNTING = ("blocks", "rows", "rows_matched", "blocks_matched", "values_bytes", "bloom_probe_bytes", "bitmap_bytes", "columns_read")


def scan_batch_both_ways(ctx, prog, hb):
    """vlscan_scan_batch staged in one go and staged bloom-first (headers + bloom filters, probe pass, then only the values some filter can reach):
    the same bitmaps, counts and accounting.  -> the results of the one-go call"""
    out = {}
    old = os.environ.get("VLSCAN_BLOOM_FIRST")
    try:
        for mode in ("0", "2"):
            os.environ["VLSCAN_BLOOM_FIRST"] = mode
            words, counts, st = ctx.scan_batch(prog, hb)
            out[mode] = (words.copy(), counts.copy(), st)
    finally:
        if old is None:
            os.environ.pop("VLSCAN_BLOOM_FIRST", None)
        else:
            os.environ["VLSCAN_BLOOM_FIRST"] = old
    (w0, c0, s0), (w2, c2, s2) = out["0"], out["2"]
    assert np.array_equal(w0, w2) and np.array_equal(c0, c2), "bloom-first staging changed the result bitmaps"
    for k in ACCOUNTING:
        assert getattr(s0, k) == getattr(s2, k), ("bloom-first staging changed the accounting", k, getattr(s0, k), getattr(s2, k))
    assert s0.staged_columns == 0 and s0.pruned_columns == 0
    return w0, c0, s0


def numeric_and_special_columns(n=300):
    """one block's columns of every kind: uint8 / uint16 / uint32 / uint64 / int64, ipv4, iso8601, dict, const and a string column"""
    return [
        ("u8", [b"%d" % (i % 200) for i in range(n)]),
        ("u16", [b"%d" % (i * 37 % 60000) for i in range(n)]),
        ("u32", [b"%d" % (i * 104729 % 4000000000) for i in range(n)]),
        ("u64", [b"%d" % (i * 1234567890123 + 5000000000) for i in range(n)]),
        ("i64", [b"%d" % ((i - 150) * 987654321) for i in range(n)]),
        ("ip", [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)]),
        ("ts", [b"2024-03-%02dT12:%02d:%02d.%03dZ" % (1 + i % 28, i % 60, (i * 7) % 60, i % 1000) for i in range(n)]),
        ("lvl", [[b"info", b"warn", b"error", b"ERROR", b"debug"][i % 5] for i in range(n)]),
        ("cst", [b"same value"] * n),
        ("msg", [b"row %d has status %d" % (i, 200 + i % 5) for i in range(n)]),
    ]


def float64_columns(n=300):
    """a float64 column (f) next to a string column (k)"""
    fvals = [b"%d.%d" % (i * 7 - 900, i % 97) for i in range(n - 8)] + [b"9007199254740991", b"0.00000015", b"-0.000123", b"123456789.125", b"0.5", b"-12.25", b"12.50", b"125"]
    return [("f", fvals), ("k", [b"k%d" % i for i in range(n)])]


def gpu_rows(ctx, flt, blocks, stage="ondisk"):
    """run the product end to end through vlscan_scan_batch -> list of matching row lists, counts, stats"""
    hb = host_blocks_from_oracle(blocks, stage)
    prog = vs.Program(flt)
    words, counts, st = scan_batch_both_ways(ctx, prog, hb)
    per = vs.split_bitmaps(words, [b.rows for b in blocks])
    return [vloracle.bitmap_rows(np.ascontiguousarray(w), b.rows) for w, b in zip(per, blocks)], counts, st
