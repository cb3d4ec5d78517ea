#!/usr/bin/env python3
"""Times the per-query aggregations on on-disk blocks two ways, on one GPU.

    python tools/stage_selected_bench.py [--rows 100000000] [--steps 5] [--warmup 1]

Data: generated rows (3000 per block) with `_msg`, `level`, `path`, `status` and a timestamps column, vocabulary rows in 2 blocks of 100
(hot_block_permille 20) so that the bloom filters rule out most blocks for `_msg:"error"`, re-encoded into the on-disk form
(vlscan_host_blocks_compress) in pinned host memory.  Per request it reports the median wall-clock time (ending in a device sync) and the
host->device bytes of
  (a) vlscan_batch_upload of the filter and output fields + vlscan_scan_resident + the call (the only way before vlscan_scan_batch_keep), and
  (b) vlscan_scan_batch_keep + vlscan_stage_selected + the call (for the newest rows: the call without fields, vlscan_stage_selected of the
      returned rows' blocks, the call with fields),
both given the same descriptors with only the filter and output fields' columns, as a caller would pass them.  (a) frees its batch inside
the timed region (a worker has to, batch after batch); (b) reuses the ctx's memory.  The script asserts that both give the same answer on every call.  Prints one JSON line with the card's name, power limit and SM clock.  Nothing is
written to the repository."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SEED = 20251015
RPB = 3000
FIELDS = ["_msg", "level", "path", "status"]
MINUTE = 60 * 10 ** 9
REQUESTS = (   # (LogsQL, filter, aggregation, fields the aggregation reads)
    ('_msg:"error" | last 1000 rows with _msg, path, status', lambda F: F.phrase("_msg", "error"), "last_rows", ["_msg", "path", "status"]),
    ('_msg:"error" | facets', lambda F: F.phrase("_msg", "error"), "facets", ["_msg", "level", "path", "status"]),
    ('_msg:"error" | hits by (_time:1m, path)', lambda F: F.phrase("_msg", "error"), "hits", ["path"]),
    ("* | hits by (level)", lambda F: F.noop(), "hits_level", ["level"]),
)


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")]


def call(ctx, kind, fields):
    if kind == "facets":
        return ctx.facets(fields + ["_time"])
    if kind == "hits":
        return ctx.hits_stats(MINUTE, 0, 0, tuple(fields))
    if kind == "hits_level":
        return ctx.hits_stats(10 ** 18, 0, 0, tuple(fields))
    return ctx.last_rows(1000, fields)


def restrict(vs, disk, fields):
    """the descriptors of `disk` with only the columns of `fields` (path (a) uploads exactly the fields the request reads)"""
    import ctypes as C
    names = [f.encode() for f in fields]
    idx = {disk.field_names.index(f): i for i, f in enumerate(names)}
    keep, blocks = [], (vs.CBlock * disk.nblocks)()
    for b in range(disk.nblocks):
        blk = disk.blocks[b]
        mine = [vs.CColumn.from_buffer_copy(blk.cols[k]) for k in range(blk.ncols) if blk.cols[k].field in idx]
        for c in mine:
            c.field = idx[c.field]
        arr = (vs.CColumn * max(len(mine), 1))(*mine)
        keep.append(arr)
        blocks[b] = blk
        blocks[b].ncols = len(mine)
        blocks[b].cols = C.cast(arr, C.POINTER(vs.CColumn))
    sub = vs.HostBlocks.__new__(vs.HostBlocks)
    sub.field_names, sub.blocks, sub.nblocks, sub.rows, sub._keep = names, blocks, disk.nblocks, disk.rows, (keep, disk)
    return sub


def workload(ctx, vs, disk, steps, warmup):
    out = {}
    for logsql, mk, kind, fields in REQUESTS:
        prog = vs.Program(mk(vs.Filter))
        need = sorted({f.decode() for f in prog.fields()} | set(fields), key=lambda f: FIELDS.index(f))
        sub = restrict(vs, disk, need)

        def path_a():
            st = vs.CStats()
            batch = ctx.upload(sub, stats=st)
            ctx.scan_resident(prog, batch, want_stats=False)
            r = call(ctx, kind, fields)
            batch.free()
            ctx.sync()
            return r, st.h2d_bytes

        def path_b():
            words, counts, st = ctx.scan_batch_keep(prog, sub)
            h2d = st.h2d_bytes
            if kind == "last_rows":
                chosen = sorted({b for _, b, _, _ in ctx.last_rows(1000)})
                h2d += ctx.stage_selected(sub, fields, blocks=chosen)["h2d_bytes"]
            else:
                h2d += ctx.stage_selected(sub, fields)["h2d_bytes"]
            r = call(ctx, kind, fields)
            ctx.sync()
            return r, h2d

        res = {}
        for name, fn in (("a_upload_resident", path_a), ("b_keep_stage_selected", path_b)):
            ms, answers, h2d = [], [], 0
            for i in range(warmup + steps):
                t0 = time.perf_counter()
                r, h2d = fn()
                dt = 1000 * (time.perf_counter() - t0)
                if i >= warmup:
                    ms.append(dt)
                answers.append(r)
            res[name] = {"median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3), "h2d_bytes": int(h2d)}
            res.setdefault("_answers", []).extend(answers)
        first = res["_answers"][0]
        res["equal"] = all(a == first for a in res.pop("_answers"))
        assert res["equal"], logsql
        words, counts, _ = ctx.scan_batch(prog, sub)
        res["blocks_with_hits"] = int((counts[:disk.nblocks] > 0).sum())
        res["blocks"] = int(disk.nblocks)
        res["timed_runs"] = steps
        out[logsql] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from victorialogs_b200 import scan as vs
    if vs.device_count() == 0:
        raise SystemExit("stage_selected_bench.py: no CUDA device; libvlscan has no CPU fallback")
    name, power, max_sm = smi("name", "power.limit", "clocks.max.sm")
    ctx = vs.Ctx(0)
    nb = args.rows // RPB
    cfg = vs.GenConfig(seed=SEED, total_rows=nb * RPB, rows_per_block=RPB, hot_block_permille=20, hit_row_permille=50, columns_mask=0x1F)
    t0 = time.perf_counter()
    gen = ctx.generate(cfg, 0, nb)
    host = ctx.download(gen)
    gen.free()
    disk = host.compress()   # its blocks still point at the timestamps in `host`, which stays alive
    t_prep = time.perf_counter() - t0
    clocks, done = [], threading.Event()

    def sample():   # SM clock while the workload runs (read-only query)
        while not done.wait(0.5):
            clocks.append(int(float(smi("clocks.sm")[0])))

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    out = workload(ctx, vs, disk, args.steps, args.warmup)
    done.set()
    t.join()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_during": sorted(set(clocks)), "rows": nb * RPB,
                      "rows_per_block": RPB, "on_disk_host_bytes": int(disk.bytes), "prepare_seconds": round(t_prep, 1), "requests": out}), flush=True)


if __name__ == "__main__":
    main()
