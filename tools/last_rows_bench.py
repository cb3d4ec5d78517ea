#!/usr/bin/env python3
"""Times the N newest selected rows that `/select/logsql/query?limit=N` returns (vlscan_last_rows), on one GPU.

    python tools/last_rows_bench.py [--steps 20] [--warmup 3]

100 M generated rows (2000 per block, `_msg` + `level` + a timestamps column) stay resident.  Time-ordered data puts row i at
VLSCAN_GEN_T0 + i ms; the interleaved data set (columns_mask bits 12..16 = 16) lets 2^16 blocks overlap in time, so no block can be pruned by
its header.  For each query (limit 1000) it reports the median wall-clock time of the scan alone, of scan + vlscan_last_rows, and of scan +
vlscan_gather_timestamps + a numpy top-N + vlscan_gather_values of the requested fields for every selected row (what a caller does without
the call), the bytes each path copies back, the blocks whose timestamps were decoded, and whether both paths gave the same rows on every
call.  Prints one JSON line with the card's name, power limit and SM clock.  Nothing is written to the repository."""
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
SEED = 20250718
ROWS = 100_000_000
RPB = 2000
LIMIT = 1000
QUERIES = (   # (LogsQL, filter, fields, interleaving k)
    ('_msg:"error" | limit 1000', lambda F: F.phrase("_msg", "error"), ("_msg", "level"), 0),
    ("* | limit 1000 (time-ordered blocks)", lambda F: F.noop(), ("level",), 0),
    ("* | limit 1000 (2^16 interleaved blocks)", lambda F: F.noop(), ("level",), 16),
)


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")]


def workload(ctx, vs, np, steps, warmup):
    import ctypes as C
    L = vs.lib()
    nb = ROWS // RPB
    cap_rows, cap_bytes = LIMIT, 1 << 24
    d_ts, d_blk, d_row = np.zeros(cap_rows, dtype=np.int64), np.zeros(cap_rows, dtype=np.uint32), np.zeros(cap_rows, dtype=np.uint32)
    d_bytes, d_offs, d_info = np.zeros(cap_bytes, dtype=np.uint8), np.zeros(cap_rows * 4 + 1, dtype=np.uint64), (C.c_uint64 * 4)()

    def device_path(fields):   # vlscan_last_rows into preallocated arrays; the result list is built outside the timed region
        q, keep = vs.last_query(LIMIT, fields)
        ctx._check(L.vlscan_last_rows(ctx.h, C.byref(q), d_ts.ctypes.data_as(C.c_void_p), d_blk.ctypes.data_as(C.c_void_p), d_row.ctypes.data_as(C.c_void_p), C.c_uint64(cap_rows),
                                      d_bytes.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), d_offs.ctypes.data_as(C.c_void_p), d_info))
        n, nf = int(d_info[0]), len(fields)
        return n, d_ts[:n].copy(), d_blk[:n].copy(), d_row[:n].copy(), d_bytes[:int(d_info[1])].tobytes(), d_offs[:n * nf + 1].copy(), nf

    def device_list(r):
        n, ts, blk, row, raw, offs, nf = r
        return [(int(ts[i]), int(blk[i]), int(row[i]), tuple(raw[int(offs[i * nf + f]):int(offs[i * nf + f + 1])] for f in range(nf))) for i in range(n)]

    def gather_texts(batch, field):   # vlscan_gather_values into flat numpy buffers
        n = int(batch.rows)
        offs, hoffs, total = np.zeros(n + 1, dtype=np.uint64), np.zeros(nb + 1, dtype=np.uint64), C.c_uint64()
        buf = np.zeros(1, dtype=np.uint8)
        for _ in range(2):
            rc = L.vlscan_gather_values(ctx.h, field.encode(), C.c_size_t(len(field)), buf.ctypes.data_as(C.c_void_p), C.c_uint64(buf.size), offs.ctypes.data_as(C.c_void_p),
                                        C.c_uint64(n), C.byref(total), hoffs.ctypes.data_as(C.c_void_p))
            if rc and total.value > buf.size:
                buf = np.zeros(total.value, dtype=np.uint8)
                continue
            ctx._check(rc)
            break
        hits = int(hoffs[-1])
        return buf[:total.value], offs[:hits + 1], 8 * (hits + 1) + total.value + 8 * (nb + 1)

    def host_path(batch, fields):
        """every selected row's _time to the host, the N newest by (ts, hit order = block, row) in numpy, then every selected row's field texts"""
        ts, hoffs = ctx.gather_timestamps(batch)
        d2h = 8 * ts.size + 8 * (nb + 1)
        if ts.size > LIMIT:
            tn = ts[np.argpartition(ts, ts.size - LIMIT)[ts.size - LIMIT:]].min()
            cand = np.nonzero(ts >= tn)[0]
        else:
            cand = np.arange(ts.size)
        chosen = cand[np.argsort(ts[cand], kind="stable")][-LIMIT:]
        texts = []
        for f in fields:
            buf, offs, nbytes = gather_texts(batch, f)
            d2h += nbytes
            texts.append([bytes(buf[int(offs[i]):int(offs[i + 1])]) for i in chosen])
        return (ts[chosen], chosen, hoffs, texts), d2h

    def host_list(r, hit_rows):
        ts, chosen, hoffs, texts = r[0]
        blk = np.searchsorted(hoffs, chosen, side="right") - 1
        return [(int(ts[j]), int(blk[j]), int(hit_rows[chosen[j]]), tuple(t[j] for t in texts)) for j in range(len(chosen))]

    out = {"rows": ROWS, "blocks": nb, "limit": LIMIT, "note": "times are the median wall-clock time per call including the scan, its synchronisation and the "
           "copies back into preallocated arrays (turning the rows into Python objects is not timed)"}
    batch, batch_k = None, None
    for logsql, tree, fields, k in QUERIES:
        if batch is None or batch_k != k:
            if batch is not None:
                batch.free()
            cfg = vs.GenConfig(seed=SEED, total_rows=ROWS, rows_per_block=RPB, hot_block_permille=300, hit_row_permille=50,
                               columns_mask=1 | 2 | vs.GEN_TIMESTAMPS | vs.gen_streams(k))
            batch, batch_k = ctx.generate(cfg, 0, nb), k
        prog = vs.Program(tree(vs.Filter))
        res = {}

        def scan():
            ctx.scan_resident(prog, batch, want_stats=False)

        def timed(fn, n, warm):
            for _ in range(warm):
                fn()
            ctx.sync()
            ms, outs = [], []
            for _ in range(n):
                t0 = time.perf_counter()
                r = fn()
                ctx.sync()
                ms.append(1000 * (time.perf_counter() - t0))
                outs.append(r)
            return statistics.median(ms), outs

        res["scan_ms"], _ = timed(scan, steps, warmup)
        res["scan_last_rows_ms"], dev = timed(lambda: (scan(), device_path(fields))[1], steps, warmup)
        info = dict(rows=int(d_info[0]), value_bytes=int(d_info[1]), selected=int(d_info[2]), blocks_decoded=int(d_info[3]))
        host_steps = max(1, min(steps, 3))   # seconds per call at 1e8 selected rows: fewer runs, one warm-up
        res["scan_gather_numpy_ms"], host = timed(lambda: (scan(), host_path(batch, fields))[1], host_steps, 1)
        hit_rows, _ = ctx.fetch_hits(batch)
        want = device_list(dev[0])
        res["equal"] = all(device_list(d) == want for d in dev) and all(host_list(h, hit_rows) == want for h in host)
        res["rows_returned"] = len(want)
        res["selected_rows"] = info["selected"]
        res["blocks_decoded"] = info["blocks_decoded"]
        res["d2h_bytes_last_rows"] = 16 * info["rows"] + 8 * (info["rows"] * len(fields) + 1) + info["value_bytes"]
        res["d2h_bytes_gather"] = host[0][1]
        res["timed_runs"] = {"scan": steps, "last_rows": steps, "gather_numpy": host_steps}
        out[logsql] = res
        del hit_rows
    batch.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    from victorialogs_b200 import scan as vs
    if vs.device_count() == 0:
        raise SystemExit("last_rows_bench.py: no CUDA device; libvlscan has no CPU fallback")
    name, power, max_sm = smi("name", "power.limit", "clocks.max.sm")
    ctx = vs.Ctx(0)
    clocks, done = [], threading.Event()

    def sample():   # SM clock while the workload runs (read-only query)
        while not done.wait(0.5):
            clocks.append(int(float(smi("clocks.sm")[0])))

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    out = workload(ctx, vs, np, args.steps, args.warmup)
    done.set()
    t.join()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_during": sorted(set(clocks)), "last_rows": out}), flush=True)


if __name__ == "__main__":
    main()
