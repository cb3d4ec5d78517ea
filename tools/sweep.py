#!/usr/bin/env python3
"""C5 of BASELINE.json: selectivity / block-clustering sweep of the scan on one H100 (resident inputs).

For every (workload, hot_block_permille, hit_row_permille) point: generate the data set on the device, run W warm-up + K timed scans
(CUDA events on the ctx stream), and report rows/s, ms/step, how many blocks the bloom pre-pass pruned ("bloom-only" blocks: their
values are never read) versus fully decoded, algorithmic bytes and the achieved HBM GB/s of the step and of the dominant kernel.

Vocabulary rows all carry the entry the workload's query looks for (`columns_mask` bits 8..11, the generator's focus knob), so
hit_row_permille x hot_block_permille IS the row selectivity of the leading leaf: the sweep reaches 0.5 and 1.0, not just the 8 % a uniform
draw over the 12 vocabulary entries allows.

    python tools/sweep.py --rows 100000000 --out sweep.json
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="C1,C2,C3,C4")
    ap.add_argument("--no-focus", action="store_true", help="uniform vocabulary draw (the round-1 sweep)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import bench
    from victorialogs_b200 import scan as vs
    peak, _ = bench.hbm_peak()
    ctx = vs.Ctx(0)
    stream = torch.cuda.ExternalStream(ctx.stream, device=0)
    results = []
    for name in args.workloads.split(","):
        wl = bench.WORKLOADS[name]
        rows = args.rows - args.rows % wl["rows_per_block"]
        nb = rows // wl["rows_per_block"]
        prog = vs.Program(wl["tree"](vs.Filter))
        focus = 0 if args.no_focus else {"C1": 1, "C2": 2, "C3": 4, "C4": 3}[name]   # error / timeout / conn 10.0.0.7 refused / GET /api/v1/items
        for hot in (1000, 300, 50):
            for hit in (1, 10, 100, 500, 1000):
                cfg = vs.GenConfig(seed=bench.SEED, total_rows=rows, rows_per_block=wl["rows_per_block"], hot_block_permille=hot, hit_row_permille=hit, columns_mask=wl["mask"] | (focus << 8))
                batch = ctx.generate(cfg, 0, nb)
                for _ in range(args.warmup):
                    ctx.scan_resident(prog, batch, want_stats=False)
                ctx.sync()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    ctx.scan_resident(prog, batch, want_stats=False)
                e1.record(stream)
                ctx.sync()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                st = ctx.last_scan_stats()
                step_bytes = st.values_bytes + st.bloom_probe_bytes + st.bitmap_bytes
                r = {"workload": name, "logsql": wl["logsql"], "rows": rows, "blocks": nb, "hot_block_permille": hot, "hit_row_permille": hit, "vocabulary_focus": focus,
                     "selectivity": st.rows_matched / rows, "rows_per_s": rows / (ms / 1e3), "ms_per_step": ms, "blocks_matched": int(st.blocks_matched),
                     "columns_read": int(st.columns_read), "values_bytes": int(st.values_bytes), "bloom_probe_bytes": int(st.bloom_probe_bytes),
                     "step_hbm_gbs": step_bytes / 1e9 / (ms / 1e3), "scan_kernel_gbs": (st.scan_kernel_bytes / 1e9) / (st.scan_kernel_ms / 1e3) if st.scan_kernel_ms > 0 else None,
                     "scan_kernel_frac_of_peak": ((st.scan_kernel_bytes / 1e9) / (st.scan_kernel_ms / 1e3) / peak) if st.scan_kernel_ms > 0 else None}
                results.append(r)
                print(json.dumps(r), flush=True)
                batch.free()
    if args.out:
        json.dump(results, open(args.out, "w"), indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
