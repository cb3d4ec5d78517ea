#!/usr/bin/env python3
"""Times the hits histogram that /select/logsql/hits adds to every query, `stats by (_time:step, fields) count()`, on one GPU.

    python tools/hits_bench.py [--steps 20] [--warmup 3]

100 M generated rows (2000 per block, `_msg` + `level` + a timestamps column: row i at VLSCAN_GEN_T0 + i ms, so a block spans 2 s) stay
resident.  For each of two queries it reports the median wall-clock time of the scan alone, of scan + vlscan_hits_stats, and of scan +
vlscan_gather_timestamps / vlscan_gather_values + bucketing and counting in numpy (what a caller does without the aggregation), the bytes
each path copies back, and whether both paths gave the same groups on every call.  Prints one JSON line with the card's name, power limit
and SM clock.  Nothing is written to the repository."""
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


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")]


HITS_ROWS = 100_000_000
HITS_QUERIES = (   # (LogsQL, filter, step ns, by-fields): the first spans a bucket boundary in most blocks, the second in almost none
    ('_msg:"error" | stats by (_time:1s) count() hits', lambda F: F.phrase("_msg", "error"), 10 ** 9, ()),
    ("* | stats by (_time:1h, level) count() hits", lambda F: F.noop(), 3600 * 10 ** 9, ("level",)),
)


def hits_workload(ctx, vs, np, steps, warmup):
    """`/select/logsql/hits` on 100 M generated rows (2000 per block, 1 ms apart, so a block spans 2 s): per query the scan alone, the scan +
    vlscan_hits_stats, and the scan + gather `_time` and the by-field + bucketing and counting in numpy; every run of both paths must give
    the same groups.  D2H bytes are those of the result arrays each path copies back."""
    import ctypes as C
    rpb = 2000
    cfg = vs.GenConfig(seed=SEED, total_rows=HITS_ROWS, rows_per_block=rpb, hot_block_permille=300, hit_row_permille=50, columns_mask=1 | 2 | vs.GEN_TIMESTAMPS)
    nb = HITS_ROWS // rpb
    batch = ctx.generate(cfg, 0, nb)
    L = vs.lib()

    def gather_texts(field):   # vlscan_gather_values into flat numpy buffers (a list of 1e8 Python bytes objects would dominate the time)
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

    cap_groups, cap_bytes = 1 << 20, 1 << 24
    d_buckets, d_counts = np.zeros(cap_groups, dtype=np.int64), np.zeros(cap_groups, dtype=np.uint64)
    d_keys, d_offs, d_info = np.zeros(cap_bytes, dtype=np.uint8), np.zeros(cap_groups * 4 + 1, dtype=np.uint64), (C.c_uint64 * 4)()

    def device_path(step, by):   # vlscan_hits_stats into preallocated arrays; the result list is built outside the timed region
        q, keep = vs.hits_query(step, 0, 0, by)
        ctx._check(L.vlscan_hits_stats(ctx.h, C.byref(q), d_buckets.ctypes.data_as(C.c_void_p), d_counts.ctypes.data_as(C.c_void_p), C.c_uint64(cap_groups),
                                       d_keys.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), d_offs.ctypes.data_as(C.c_void_p), d_info))
        g, nby = int(d_info[0]), len(by)
        return g, d_buckets[:g].copy(), d_counts[:g].copy(), d_keys[:int(d_info[1])].tobytes(), d_offs[:g * nby + 1].copy(), nby

    def device_list(r):
        g, buckets, counts, raw, offs, nby = r
        return [(int(buckets[i]), tuple(raw[int(offs[i * nby + f]):int(offs[i * nby + f + 1])] for f in range(nby)), int(counts[i])) for i in range(g)]

    def host_path(step, by):
        ts, _ = ctx.gather_timestamps(batch)
        d2h = 8 * ts.size + 8 * (nb + 1)
        bucket = ts - np.mod(ts, step)
        b0 = int(bucket.min()) if ts.size else 0
        bidx = (bucket - b0) // step
        code, texts = np.zeros(ts.size, dtype=np.int64), [()]
        for f in by:   # factorize the field's text (<= 8 bytes here: packed into one u64 per row)
            buf, offs, nbytes = gather_texts(f)
            d2h += nbytes
            lens = np.diff(offs).astype(np.int64)
            if lens.size and lens.max() > 8:
                raise RuntimeError("bench host path packs texts of at most 8 bytes")
            packed = np.zeros(ts.size, dtype=np.uint64)
            for k in range(8):
                m = lens > k
                packed[m] |= buf[(offs[:-1][m] + k).astype(np.int64)].astype(np.uint64) << np.uint64(8 * (7 - k))
            uniq, inv = np.unique(packed, return_inverse=True)
            first = np.zeros(uniq.size, dtype=np.int64)
            first[inv[::-1]] = np.arange(ts.size)[::-1]
            names = [bytes(buf[int(offs[j]):int(offs[j + 1])]) for j in first]
            code = code * uniq.size + inv
            texts = [t + (nm,) for t in texts for nm in names]
        ncodes = len(texts)
        cnt = np.bincount(bidx * ncodes + code, minlength=0)
        nz = np.nonzero(cnt)[0]
        return (step, b0, ncodes, texts, nz, cnt[nz]), d2h

    def host_list(r):
        step, b0, ncodes, texts, nz, cnt = r[0]
        return sorted((b0 + int(i // ncodes) * step, texts[int(i % ncodes)], int(c)) for i, c in zip(nz, cnt))

    out = {"rows": int(batch.rows), "blocks": nb, "note": "timestamps: row i at %d + i ms; times are the median wall-clock time per call including "
           "the scan, its synchronisation and the copies back into preallocated arrays (turning the groups into Python objects is not timed)" % vs.GEN_T0}
    for logsql, tree, step, by in HITS_QUERIES:
        prog = vs.Program(tree(vs.Filter))
        res = {}

        def scan():
            ctx.scan_resident(prog, batch, want_stats=False)

        def timed(fn, k, warm):
            for _ in range(warm):
                fn()
            ctx.sync()
            ms, outs = [], []
            for _ in range(k):
                t0 = time.perf_counter()
                r = fn()
                ctx.sync()
                ms.append(1000 * (time.perf_counter() - t0))
                outs.append(r)
            return statistics.median(ms), outs

        res["scan_ms"], _ = timed(scan, steps, warmup)
        res["scan_hits_stats_ms"], dev = timed(lambda: (scan(), device_path(step, by))[1], steps, warmup)
        info = dict(groups=int(d_info[0]), key_bytes=int(d_info[1]), rows=int(d_info[2]), blocks_decoded=int(d_info[3]))
        host_steps = max(1, min(steps, 3))   # tens of seconds per call at 1e8 selected rows: fewer runs, one warm-up
        res["scan_gather_numpy_ms"], host = timed(lambda: (scan(), host_path(step, by))[1], host_steps, 1)
        want = device_list(dev[0])
        res["equal"] = all(device_list(d) == want for d in dev) and all(host_list(h) == want for h in host)
        res["groups"] = len(want)
        res["selected_rows"] = int(info["rows"])
        res["blocks_decoded"] = int(info["blocks_decoded"])
        res["d2h_bytes_hits_stats"] = 16 * info["groups"] + 8 * (info["groups"] * len(by) + 1) + info["key_bytes"]
        res["d2h_bytes_gather"] = host[0][1]
        res["timed_runs"] = {"scan": steps, "hits_stats": steps, "gather_numpy": host_steps}
        out[logsql] = res
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
        raise SystemExit("hits_bench.py: no CUDA device; libvlscan has no CPU fallback")
    name, power, max_sm = smi("name", "power.limit", "clocks.max.sm")
    ctx = vs.Ctx(0)
    clocks, done = [], threading.Event()

    def sample():   # SM clock while the workload runs (read-only query)
        while not done.wait(0.5):
            clocks.append(int(float(smi("clocks.sm")[0])))

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    out = hits_workload(ctx, vs, np, args.steps, args.warmup)
    done.set()
    t.join()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_during": sorted(set(clocks)), "hits": out}), flush=True)


if __name__ == "__main__":
    main()
