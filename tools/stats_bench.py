#!/usr/bin/env python3
"""Times `stats by (_time:step, fields) count(), sum(status), avg(status)` (vlscan_hits_sums) on one GPU, with plain and bucketed by-fields, and
`stats by (_time:step, fields) histogram(status)` (vlscan_hits_vmranges).

    python tools/stats_bench.py [--steps 20] [--warmup 3]

100 M generated rows (2000 per block, `_msg`, `level` (dict), `path`, `status` (uint16) and a timestamps column: row i at VLSCAN_GEN_T0 + i ms)
stay resident.  For each of three queries it reports the median wall-clock time of the scan alone, of scan + vlscan_hits_sums, and of scan +
vlscan_gather_timestamps / vlscan_gather_values + bucketing, parsing and summing in numpy (what a caller does without the aggregation), the
bytes each path copies back, and whether both paths gave the same groups, rows and counts (and sums within 2^-40 of the host's) on every call.
The two histogram queries are timed the same way against gather + numpy, where numpy maps each distinct value through vlscan_vmrange_index and
counts per (group, vmrange); their hits must be equal.
Prints one JSON line with the card's name, power limit and SM clock.  Nothing is written to the repository."""
import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from hits_bench import SEED, smi  # noqa: E402

ROWS = 100_000_000
QUERIES = (   # (LogsQL, filter, step ns, by-fields, value fields, by-field buckets)
    ('_msg:"error" | stats by (_time:1s) sum(status), avg(status)', lambda F: F.phrase("_msg", "error"), 10 ** 9, (), ("status",), None),
    ("* | stats by (_time:1h, level) count(), avg(status)", lambda F: F.noop(), 3600 * 10 ** 9, ("level",), ("status",), None),
    # a dashboard panel `| stats by (status:100) count(), avg(status)` as /select/logsql/stats_query_range sends it
    ("* | stats by (_time:1h, status:100) count(), avg(status)", lambda F: F.noop(), 3600 * 10 ** 9, ("status",), ("status",), [(100.0, 0.0, 0)]),
)
VMR_QUERIES = (   # (LogsQL, filter, step ns, by-fields, value field): the shapes of a Grafana heatmap panel
    ("* | stats by (_time:1h, level) histogram(status)", lambda F: F.noop(), 3600 * 10 ** 9, ("level",), "status"),
    ('_msg:"error" | stats by (_time:1s) histogram(status)', lambda F: F.phrase("_msg", "error"), 10 ** 9, (), "status"),
)


def workload(ctx, vs, np, steps, warmup, rows=ROWS):
    import ctypes as C
    rpb = 2000
    nb = rows // rpb
    cfg = vs.GenConfig(seed=SEED, total_rows=nb * rpb, rows_per_block=rpb, hot_block_permille=300, hit_row_permille=50, columns_mask=0x1F)
    batch = ctx.generate(cfg, 0, nb)
    L = vs.lib()

    def gather_texts(field):   # vlscan_gather_values into flat numpy buffers
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

    def packed(buf, offs):   # texts of at most 8 bytes, one u64 per row
        lens = np.diff(offs).astype(np.int64)
        if lens.size and lens.max() > 8:
            raise RuntimeError("bench host path packs texts of at most 8 bytes")
        out = np.zeros(lens.size, dtype=np.uint64)
        for k in range(8):
            m = lens > k
            out[m] |= buf[(offs[:-1][m] + k).astype(np.int64)].astype(np.uint64) << np.uint64(8 * (7 - k))
        return out, lens

    cap_groups, cap_bytes = 1 << 20, 1 << 24
    d_buckets, d_counts = np.zeros(cap_groups, dtype=np.int64), np.zeros(cap_groups, dtype=np.uint64)
    d_sums, d_vcounts = np.zeros(cap_groups * 4, dtype=np.float64), np.zeros(cap_groups * 4, dtype=np.uint64)
    d_keys, d_offs, d_info = np.zeros(cap_bytes, dtype=np.uint8), np.zeros(cap_groups * 4 + 1, dtype=np.uint64), (C.c_uint64 * 4)()

    def decimal(p, lens):   # the packed decimal integer texts -> their values
        num = np.zeros(lens.size, dtype=np.float64)
        for k in range(8):   # most significant byte first
            m = lens > k
            num[m] = num[m] * 10 + ((p[m] >> np.uint64(8 * (7 - k))) & np.uint64(0xFF)).astype(np.float64) - 48
        return num

    def device_path(step, by, values, buckets):
        q, keep = vs.hits_query(step, 0, 0, by)
        bks = vs.by_buckets(buckets, len(by))
        vn = [v.encode() for v in values]
        varr, vlens = (C.c_char_p * len(vn))(*vn), (C.c_size_t * len(vn))(*[len(v) for v in vn])
        ctx._check(L.vlscan_hits_sums_bucketed(ctx.h, C.byref(q), bks, varr, vlens, C.c_uint32(len(vn)), d_buckets.ctypes.data_as(C.c_void_p), d_counts.ctypes.data_as(C.c_void_p),
                                      d_sums.ctypes.data_as(C.c_void_p), d_vcounts.ctypes.data_as(C.c_void_p), C.c_uint64(cap_groups),
                                      d_keys.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), d_offs.ctypes.data_as(C.c_void_p), d_info))
        g, nby, nv = int(d_info[0]), len(by), len(vn)
        return g, d_buckets[:g].copy(), d_counts[:g].copy(), d_sums[:g * nv].copy(), d_vcounts[:g * nv].copy(), d_keys[:int(d_info[1])].tobytes(), d_offs[:g * nby + 1].copy(), nby

    def device_list(r):
        g, buckets, counts, sums, vcounts, raw, offs, nby = r
        return [(int(buckets[i]), tuple(raw[int(offs[i * nby + f]):int(offs[i * nby + f + 1])] for f in range(nby)), int(counts[i]), float(sums[i]), int(vcounts[i]))
                for i in range(g)]

    def host_groups(step, by, buckets):
        """gather `_time` and the by-fields -> (bucket index, first bucket, key code, key texts by code), D2H bytes"""
        ts, _ = ctx.gather_timestamps(batch)
        d2h = 8 * ts.size + 8 * (nb + 1)
        bucket = ts - np.mod(ts, step)
        b0 = int(bucket.min()) if ts.size else 0
        bidx = (bucket - b0) // step
        code, texts = np.zeros(ts.size, dtype=np.int64), [()]
        for f, bk in zip(by, buckets or [None] * len(by)):
            buf, offs, nbytes = gather_texts(f)
            d2h += nbytes
            p, lens = packed(buf, offs)
            if bk:
                v = decimal(p, lens).astype(np.int64)
                uniq, inv = np.unique(v - v % int(bk[0]), return_inverse=True)
                names = [b"%d" % u for u in uniq]
            else:
                uniq, inv = np.unique(p, return_inverse=True)
                first = np.zeros(uniq.size, dtype=np.int64)
                first[inv[::-1]] = np.arange(ts.size)[::-1]
                names = [bytes(buf[int(offs[j]):int(offs[j + 1])]) for j in first]
            code = code * uniq.size + inv
            texts = [t + (nm,) for t in texts for nm in names]
        return (bidx, b0, code, texts), d2h

    def host_path(step, by, values, buckets):
        """gather `_time`, the by-field and the value field; `status` texts are decimal integers here (a uint16 column), so int parsing
        stands for tryParseFloat64, and a bucketed `status` is truncateUint64 of that integer"""
        (bidx, b0, code, texts), d2h = host_groups(step, by, buckets)
        buf, offs, nbytes = gather_texts(values[0])
        d2h += nbytes
        num = decimal(*packed(buf, offs))
        ncodes = len(texts)
        key = bidx * ncodes + code
        cnt = np.bincount(key)
        sm = np.bincount(key, weights=num)
        nz = np.nonzero(cnt)[0]
        return (step, b0, ncodes, texts, nz, cnt[nz], sm[nz]), d2h

    def host_list(r):
        step, b0, ncodes, texts, nz, cnt, sm = r[0]
        return sorted((b0 + int(i // ncodes) * step, texts[int(i % ncodes)], int(c), float(s), int(c)) for i, c, s in zip(nz, cnt, sm))

    def same(a, b):
        return len(a) == len(b) and all(x[:3] == y[:3] and x[4] == y[4] and abs(x[3] - y[3]) <= 2.0 ** -40 * abs(y[3]) for x, y in zip(a, b))

    out = {"rows": int(batch.rows), "blocks": nb, "note": "times are the median wall-clock time per call including the scan, its synchronisation and the copies "
           "back into preallocated arrays (turning the groups into Python objects is not timed)"}
    for logsql, tree, step, by, values, buckets in QUERIES:
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
        res["scan_hits_sums_ms"], dev = timed(lambda: (scan(), device_path(step, by, values, buckets))[1], steps, warmup)
        groups, key_bytes, selected = int(d_info[0]), int(d_info[1]), int(d_info[2])
        host_steps = max(1, min(steps, 3))
        res["scan_gather_numpy_ms"], host = timed(lambda: (scan(), host_path(step, by, values, buckets))[1], host_steps, 1)
        want = device_list(dev[0])
        res["equal"] = all(device_list(d) == want for d in dev) and all(same(want, host_list(h)) for h in host)
        res["groups"] = groups
        res["selected_rows"] = selected
        res["d2h_bytes_hits_sums"] = 16 * groups + 16 * groups * len(values) + 8 * (groups * len(by) + 1) + key_bytes
        res["d2h_bytes_gather"] = host[0][1]
        res["timed_runs"] = {"scan": steps, "hits_sums": steps, "gather_numpy": host_steps}
        out[logsql] = res
    nvr = vs.VMRANGES
    d_eoffs, d_ranges, d_hits, v_info = np.zeros(cap_groups + 1, dtype=np.uint64), np.zeros(cap_groups * 8, dtype=np.uint16), np.zeros(cap_groups * 8, dtype=np.uint64), (C.c_uint64 * 6)()

    def device_vmr(step, by, value):
        q, keep = vs.hits_query(step, 0, 0, by)
        varr, vlens = (C.c_char_p * 1)(value.encode()), (C.c_size_t * 1)(len(value))
        ctx._check(L.vlscan_hits_vmranges(ctx.h, C.byref(q), None, varr, vlens, C.c_uint32(1), d_buckets.ctypes.data_as(C.c_void_p), d_counts.ctypes.data_as(C.c_void_p),
                                          C.c_uint64(cap_groups), d_keys.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), d_offs.ctypes.data_as(C.c_void_p),
                                          d_eoffs.ctypes.data_as(C.c_void_p), d_ranges.ctypes.data_as(C.c_void_p), d_hits.ctypes.data_as(C.c_void_p), C.c_uint64(d_ranges.size), v_info))
        g, e, nby = int(v_info[0]), int(v_info[4]), len(by)
        return (g, d_buckets[:g].copy(), d_counts[:g].copy(), d_keys[:int(v_info[1])].tobytes(), d_offs[:g * nby + 1].copy(), d_eoffs[:g + 1].copy(), d_ranges[:e].copy(),
                d_hits[:e].copy(), nby)

    def device_vmr_list(r):
        g, buckets, counts, raw, offs, eoffs, ranges, hits, nby = r
        return [(int(buckets[i]), tuple(raw[int(offs[i * nby + f]):int(offs[i * nby + f + 1])] for f in range(nby)), int(counts[i]),
                 tuple((int(ranges[k]), int(hits[k])) for k in range(int(eoffs[i]), int(eoffs[i + 1])))) for i in range(g)]

    def host_vmr(step, by, value):
        """gather + numpy: the by-field keys of host_groups, the value field's distinct numbers through vlscan_vmrange_index, one bincount"""
        (bidx, b0, code, texts), d2h = host_groups(step, by, None)
        buf, offs, nbytes = gather_texts(value)
        d2h += nbytes
        uniq, inv = np.unique(decimal(*packed(buf, offs)), return_inverse=True)
        idx = np.array([vs.vmrange_index(u) for u in uniq.tolist()], dtype=np.int64)[inv]
        key = bidx * len(texts) + code
        rows = np.bincount(key)
        ok = idx >= 0
        cnt = np.bincount(key[ok] * nvr + idx[ok])
        nz = np.nonzero(cnt)[0]
        return (step, b0, len(texts), texts, rows, nz, cnt[nz]), d2h

    def host_vmr_list(r):
        step, b0, ncodes, texts, rows, nz, cnt = r[0]
        ents = {}
        for k, c in zip(nz.tolist(), cnt.tolist()):
            ents.setdefault(k // nvr, []).append((k % nvr, c))
        return sorted((b0 + int(i // ncodes) * step, texts[int(i % ncodes)], int(rows[i]), tuple(ents.get(i, ()))) for i in np.nonzero(rows)[0].tolist())

    for logsql, tree, step, by, value in VMR_QUERIES:
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
        res["scan_hits_vmranges_ms"], dev = timed(lambda: (scan(), device_vmr(step, by, value))[1], steps, warmup)
        groups, key_bytes, selected, entries = int(v_info[0]), int(v_info[1]), int(v_info[2]), int(v_info[4])
        host_steps = max(1, min(steps, 3))
        res["scan_gather_numpy_ms"], host = timed(lambda: (scan(), host_vmr(step, by, value))[1], host_steps, 1)
        want = device_vmr_list(dev[0])
        res["equal"] = all(device_vmr_list(d) == want for d in dev) and all(host_vmr_list(h) == want for h in host)
        res["groups"] = groups
        res["entries"] = entries
        res["selected_rows"] = selected
        res["d2h_bytes_hits_vmranges"] = 16 * groups + 8 * (groups * len(by) + 1) + key_bytes + 16 * entries   # the compacted (key, count) entries
        res["d2h_bytes_gather"] = host[0][1]
        res["timed_runs"] = {"scan": steps, "hits_vmranges": steps, "gather_numpy": host_steps}
        out[logsql] = res
    batch.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=ROWS)
    args = ap.parse_args()
    import numpy as np
    from victorialogs_b200 import scan as vs
    if vs.device_count() == 0:
        raise SystemExit("stats_bench.py: no CUDA device; libvlscan has no CPU fallback")
    name, power, max_sm = smi("name", "power.limit", "clocks.max.sm")
    ctx = vs.Ctx(0)
    clocks, done = [], threading.Event()

    def sample():
        while not done.wait(0.5):
            clocks.append(int(float(smi("clocks.sm")[0])))

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    out = workload(ctx, vs, np, args.steps, args.warmup, args.rows)
    done.set()
    t.join()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": max_sm, "sm_clock_mhz_during": sorted(set(clocks)), "stats": out}), flush=True)


if __name__ == "__main__":
    main()
