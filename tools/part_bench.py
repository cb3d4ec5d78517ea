#!/usr/bin/env python3
"""Time the part directory reader end to end on a part of >= 10 GB: open -> block descriptors -> vlscan_scan_batch.

The part is written by the oracle's restatement of the reference writer (`oracle/vlo_part.h`, test infrastructure: it plays
blockStreamWriter here, it is not on the timed path), from blocks of the deterministic generator, on many host threads.  The timed part is
the product only: `vlscan_part_open` (metadata inflated by the device decoder), `vlscan_part_blocks` (block headers -> column headers ->
bloom / values byte ranges) and `vlscan_scan_batch` on descriptors that point into the mmap()ed files - pageable memory, packed into the
pinned staging ring by the host threads.

    python tools/part_bench.py --rows 220000000 --dir /tmp/vlpart_bench --out part_bench.json
"""
import argparse
import json
import os
import shutil
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=220_000_000)
    ap.add_argument("--dir", default="/tmp/vlpart_bench")
    ap.add_argument("--threads", type=int, default=min(64, os.cpu_count() or 8))
    ap.add_argument("--batch-blocks", type=int, default=16384)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import bench
    import vloracle as oracle
    from victorialogs_b200 import scan as vs

    wl = bench.WORKLOADS["C3"]
    rpb = wl["rows_per_block"]
    rows = args.rows - args.rows % rpb
    nb = rows // rpb
    cfg = oracle.GenConfig(seed=bench.SEED, total_rows=rows, rows_per_block=rpb, hot_block_permille=1000, hit_row_permille=60, columns_mask=wl["mask"])
    t0 = time.time()
    if os.path.isdir(args.dir):
        shutil.rmtree(args.dir)
    w = oracle.PartWriter()
    ts0 = 1_700_000_000_000_000_000

    def make(b):
        blk = oracle.Block.generated(cfg, b)
        blk.set_timestamps(ts0 + (b * rpb + np.arange(blk.rows, dtype=np.int64)) * 1000)
        return blk

    with ThreadPoolExecutor(args.threads) as ex:
        for lo in range(0, nb, 1024):
            for blk in ex.map(make, range(lo, min(nb, lo + 1024))):
                w.add_block((0, 0, 1, 1), blk)     # one stream, blocks in time order
    files = w.finalize()
    oracle.save_part(files, args.dir)
    part_bytes = sum(len(v) for v in files.values())
    del files, w
    t_write = time.time() - t0
    print("wrote %d blocks / %d rows, %.2f GB in %.1f s" % (nb, rows, part_bytes / 1e9, t_write), file=sys.stderr, flush=True)

    ctx = vs.Ctx(0)
    F = vs.Filter
    flt = wl["tree"](F)
    prog = vs.Program(flt)
    fields = prog.fields()
    t = time.time()
    part = vs.Part(args.dir, ctx=ctx)
    t_open = time.time() - t
    assert part.nblocks == nb
    runs = []
    for p in range(args.passes):
        t_desc = t_scan = 0.0
        matched = h2d = 0
        t_all = time.time()
        for lo in range(0, nb, args.batch_blocks):
            t = time.time()
            hb = part.blocks(fields, lo, min(nb, lo + args.batch_blocks))
            t_desc += time.time() - t
            t = time.time()
            words, counts, st = ctx.scan_batch(prog, hb)
            t_scan += time.time() - t
            matched += int(np.asarray(counts).sum())
            h2d += int(st.h2d_bytes)
        t_all = time.time() - t_all
        runs.append({"pass": p, "seconds": t_all, "describe_seconds": t_desc, "scan_batch_seconds": t_scan, "matched": matched, "h2d_bytes": h2d,
                     "rows_per_s": rows / t_all, "h2d_gbs": h2d / 1e9 / t_all})
        print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    # the same rows generated on the device and scanned resident: the match count must agree
    want = None
    try:
        gcfg = vs.GenConfig(seed=bench.SEED, total_rows=rows, rows_per_block=rpb, hot_block_permille=1000, hit_row_permille=60, columns_mask=wl["mask"])
        sub = min(nb, 20000)
        batch = ctx.generate(gcfg, 0, sub)
        st = ctx.scan_resident(prog, batch)
        want_sub = int(st.rows_matched)
        batch.free()
        hb = part.blocks(fields, 0, sub)
        _, counts, _ = ctx.scan_batch(prog, hb)
        want = {"blocks": sub, "resident_generated": want_sub, "from_part": int(np.asarray(counts).sum())}
        assert want["resident_generated"] == want["from_part"], want
    finally:
        part.close()
    out = {"what": "part directory reader end to end: vlscan_part_open + vlscan_part_blocks + vlscan_scan_batch over mmap()ed (pageable) files",
           "workload": "C3: %s" % wl["logsql"], "rows": rows, "blocks": nb, "part_bytes": part_bytes, "batch_blocks": args.batch_blocks,
           "write_seconds (oracle writer, not the product)": t_write, "open_seconds": t_open, "passes": runs, "parity": want,
           "host_threads": int(os.environ.get("VLSCAN_HOST_THREADS", "0")) or "default (min(16, cores))"}
    print(json.dumps(out))
    if args.out:
        json.dump(out, open(args.out, "w"), indent=1)
    ctx.close()
    shutil.rmtree(args.dir, ignore_errors=True)


if __name__ == "__main__":
    main()
