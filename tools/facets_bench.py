#!/usr/bin/env python3
"""Times the facets state that /select/logsql/facets asks for (`| facets`), on one GPU.

    python tools/facets_bench.py [--steps 20] [--warmup 3] [--rows 100000000]

Generated rows (2000 per block; `_msg`, `level` (dict), `path` (~10^5 distinct strings), `status` (uint16) and a timestamps column) stay
resident.  For `_msg:"error"` and `*`, with fields `_msg, level, path, status, _time`, at the default max_values_per_field and at 200000, it
reports the median wall-clock time of the scan + vlscan_facets and the bytes that call copies back.  The path without it, scan + gather of every
field and of `_time` to the host, is timed for its gathers alone (a lower bound: the facets count in numpy comes on top) and for the selective
query is also finished on the host with tests/facets_model.py, whose answer must equal the device's.  Prints one JSON line with the card's
name, power limit and SM clock.  Nothing is written to the repository."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
SEED = 20250718
FIELDS = ["_msg", "level", "path", "status", "_time"]
QUERIES = (('_msg:"error" | facets', lambda F: F.phrase("_msg", "error"), True), ("* | facets", lambda F: F.noop(), False))


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")]


def workload(ctx, vs, steps, warmup, rows):
    import facets_model as fm
    rpb = 2000
    nb = rows // rpb
    cfg = vs.GenConfig(seed=SEED, total_rows=nb * rpb, rows_per_block=rpb, hot_block_permille=300, hit_row_permille=50, columns_mask=0x1F)
    batch = ctx.generate(cfg, 0, nb)

    def gather_flat(field):   # vlscan_gather_values into flat numpy buffers (10^8 Python bytes objects would dominate the time)
        import ctypes as C
        import numpy as np
        n = int(batch.rows)
        offs, hoffs, total, buf = np.zeros(n + 1, dtype=np.uint64), np.zeros(nb + 1, dtype=np.uint64), C.c_uint64(), np.zeros(1, dtype=np.uint8)
        for _ in range(2):
            rc = vs.lib().vlscan_gather_values(ctx.h, field.encode(), C.c_size_t(len(field)), buf.ctypes.data_as(C.c_void_p), C.c_uint64(buf.size),
                                               offs.ctypes.data_as(C.c_void_p), C.c_uint64(n), C.byref(total), hoffs.ctypes.data_as(C.c_void_p))
            if rc and total.value > buf.size:
                buf = np.zeros(total.value, dtype=np.uint8)
                continue
            ctx._check(rc)
            break
        return buf[:total.value], offs[:int(hoffs[-1]) + 1]

    def timed(fn, k, warm):
        for _ in range(warm):
            fn()
        ctx.sync()
        ms, outs = [], []
        for _ in range(k):
            t0 = time.perf_counter()
            outs.append(fn())
            ctx.sync()
            ms.append(1000 * (time.perf_counter() - t0))
        return statistics.median(ms), outs

    out = {"rows": int(batch.rows), "blocks": nb, "fields": FIELDS,
           "note": "median wall-clock time per call including the scan and its synchronisation; gather_ms is the scan + the gathers of every field and "
                   "_time alone, without the facets count on the host"}
    for logsql, tree, finish_on_host in QUERIES:
        prog = vs.Program(tree(vs.Filter))
        res = {}
        for mv in (0, 200000):
            info = {}
            ms, states = timed(lambda: (ctx.scan_resident(prog, batch, want_stats=False), ctx.facets(FIELDS, mv, info=info))[1], steps, warmup)
            r = {"scan_facets_ms": ms, "equal_runs": all(s == states[0] for s in states), "selected_rows": int(info["rows"]),
                 "blocks_decoded": int(info["blocks_decoded"]), "entries": int(info["entries"]),
                 "kept": [f for f in FIELDS if states[0][f] is not None],
                 "d2h_bytes_facets": len(FIELDS) * 9 + 8 + int(info["entries"]) * 17 + 8 + int(info["value_bytes"])}
            res["max_values_per_field=%d" % mv] = r
            res["_state_%d" % mv] = states[0]
        host_steps = max(1, min(steps, 2))

        def gather():
            ctx.scan_resident(prog, batch, want_stats=False)
            ts, _ = ctx.gather_timestamps(batch)
            return ts, {f: gather_flat(f) for f in FIELDS if f != "_time"}
        res["scan_gather_ms"], g = timed(gather, host_steps, 1)
        ts, cols = g[0]
        res["d2h_bytes_gather"] = 8 * ts.size + sum(8 * offs.size + buf.size for buf, offs in cols.values()) + 8 * (nb + 1) * len(FIELDS)
        if finish_on_host:
            for mv in (0, 200000):
                sh = fm.Shard(mv, 0)
                cells = {f: ("text", [bytes(buf[int(offs[i]):int(offs[i + 1])]) for i in range(ts.size)]) for f, (buf, offs) in cols.items()}
                cells["_time"] = ("time", [int(x) for x in ts])
                sh.block(cells, list(range(ts.size)))
                res["max_values_per_field=%d" % mv]["equal_host"] = sh.state(FIELDS) == res["_state_%d" % mv]
        for k in [k for k in res if k.startswith("_state")]:
            del res[k]
        out[logsql] = res
    batch.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=100_000_000)
    args = ap.parse_args()
    from victorialogs_b200 import scan as vs
    if vs.device_count() == 0:
        raise SystemExit("facets_bench.py: no CUDA device; libvlscan has no CPU fallback")
    name, power, max_sm = smi("name", "power.limit", "clocks.max.sm")
    ctx = vs.Ctx(0)
    clocks, done = [], threading.Event()

    def sample():
        while not done.wait(0.5):
            clocks.append(int(float(smi("clocks.sm")[0])))

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    out = workload(ctx, vs, args.steps, args.warmup, args.rows)
    done.set()
    t.join()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_during": sorted(set(clocks)), "facets": out}), flush=True)


if __name__ == "__main__":
    main()
