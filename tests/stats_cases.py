"""The reference's sum / avg / `stats by (_time:...)` tables (tests/golden/stats_cases.json, transcribed by
tests/golden/extract_stats_cases.py) as inputs of this project's `stats by (_time:step, f...) count(), sum(v...), avg(v...)`: the query is
parsed into (step, offset, by-fields, functions), the rows become oracle blocks, and a backend's groups are formatted as the pipe writes its
result rows.  Cases with `if (...)` filters or `*` arguments are not of that shape and are skipped."""
import datetime
import decimal
import json
import math
import os
import re

import stats_model as sm

HERE = os.path.dirname(os.path.abspath(__file__))
UNITS = {"h": 3600 * 10 ** 9, "d": 86400 * 10 ** 9}


def load():
    return json.load(open(os.path.join(HERE, "golden", "stats_cases.json")))


def parse(q):
    """-> (step, offset, by-fields without _time, has _time, [(func, [fields], result name)]) or None when the query is not of the shape"""
    m = re.fullmatch(r"stats (?:by \((.*?)\) )?(.*)", q)
    step, off, by, has_time = 10 ** 18, 0, [], False
    for item in (m.group(1).split(", ") if m.group(1) else []):
        t = re.fullmatch(r"_time:(\d+)([hd])(?: offset (\d+)([hd]))?", item)
        if t:
            step, has_time = int(t.group(1)) * UNITS[t.group(2)], True
            off = int(t.group(3)) * UNITS[t.group(4)] if t.group(3) else 0
        elif item.startswith("_time"):
            return None
        else:
            by.append(item)
    funcs = []
    for f in m.group(2).split(", "):
        g = re.fullmatch(r"(sum|avg|count)\(([^)]*)\) as (\w+)", f)
        if not g or (g.group(1) != "count" and "*" in g.group(2)):
            return None
        funcs.append((g.group(1), g.group(2).split(", "), g.group(3)))
    return step, off, by, has_time, funcs


def ts_of(v):
    d = datetime.datetime.strptime(v[:19], "%Y-%m-%dT%H:%M:%S").replace(tzinfo=datetime.timezone.utc)
    frac = v[20:-1] if "." in v else ""
    return int(d.timestamp()) * 10 ** 9 + int((frac + "000000000")[:9])


def fmt_time(ns):
    return datetime.datetime.fromtimestamp(ns // 10 ** 9, datetime.timezone.utc).strftime("%Y-%m-%dT%H:%M:%SZ")


def fmt_float(x):
    """strconv.AppendFloat(x, 'f', -1, 64)"""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "+Inf" if x > 0 else "-Inf"
    s = format(decimal.Decimal(repr(x)), "f")
    return s.rstrip("0").rstrip(".") if "." in s else s


def blocks_of(oracle, rows, one_per_row):
    """oracle blocks of the rows: one per run of rows with the same field names (or one per row), _time as the timestamps (0 without it)
    -> [(block, {name: texts}, timestamps)]"""
    runs = []
    for row in rows:
        names = [n for n, _ in row]
        if one_per_row or not runs or runs[-1][0] != names:
            runs.append((names, []))
        runs[-1][1].append(dict(row))
    out = []
    for names, rs in runs:
        cols = {n: [r[n].encode() for r in rs] for n in names if n != "_time"}
        ts = [ts_of(r["_time"]) if "_time" in r else 0 for r in rs]
        blk = oracle.Block.from_columns(list(cols.items()), rows=len(rs)).set_timestamps(ts)
        out.append((blk, cols, ts))
    return out


def result_rows(groups, parsed):
    """groups {(bucket, keys): (rows, [(sum, count) per value field of `values_of(parsed)`])} -> the pipe's result rows, sorted"""
    step, off, by, has_time, funcs = parsed
    values = values_of(parsed)
    out = []
    for (bucket, keys), (rows, vals) in groups.items():
        row = dict(zip(by, [k.decode() for k in keys]))
        if has_time:
            row["_time"] = fmt_time(bucket)
        for func, fields, name in funcs:
            if func == "count":
                row[name] = str(rows)
                continue
            s, c = math.nan, 0
            for f in fields:
                fs, fc = vals[values.index(f)]
                c += fc
                if not math.isnan(fs):
                    s = fs if math.isnan(s) else s + fs
            row[name] = fmt_float(s if func == "sum" else (0.0 if math.isnan(s) else s) / c if c else math.nan)
        out.append(sorted(row.items()))
    return sorted(out)


def values_of(parsed):
    vals = []
    for func, fields, _ in parsed[4]:
        if func != "count":
            vals += [f for f in fields if f not in vals]
    return vals


def expected_rows(case):
    return sorted(sorted((n, v) for n, v in row) for row in case["expected"])


def model_groups(oracle, blocks, flt, step, off, cal, by, values):
    """the Python restatement's groups over [(block, texts, timestamps)] -> {(bucket, keys): (rows, [(sum, count)])}"""
    import vlohits
    mb = [model_block(oracle, b, c, t, flt) for b, c, t in blocks]
    want = sm.stats(mb, lambda t: vlohits.truncate_timestamp(t, step, off, cal), by, values)
    return {k: (g.rows, list(zip(g.sums, g.counts))) for k, g in want.items()}


def model_block(oracle, blk, cols, ts, flt):
    """the stats_model form of an oracle block: its column kinds as the oracle's writer chose them, the texts it was built from"""
    kinds = {c.name.decode(): sm.VT_KIND[c.value_type] for c in blk.columns}
    out = {name: (kinds[name], vals) for name, vals in cols.items() if name in kinds}
    for name, v in blk.consts:
        out[name.decode()] = ("const", v)
    return {"ts": ts, "rows": oracle.bitmap_rows(blk.search(flt), blk.rows), "cols": out}
