"""Python restatement of `stats by (_time:step offset off, f1, ...) count(), sum(v...), avg(v...)` over the selected rows of a batch, per block
as pipeStatsProcessorShard.writeBlock feeds it (lib/logstorage/pipe_stats.go:552-626, 700-730): a block whose selected rows all have one key
goes through blockResultColumn.sumValues (block_result.go:2501-2600), any other block row by row through getFloatValueAtRow (:2402-2448).
Float adds happen in the reference's order: rows in order inside a block, blocks in order.

A block is {"ts": [int ns per row], "rows": [selected row indices, ascending], "cols": {name: (kind, payload)}} with kind "const" (payload: the
value) or one of KINDS (payload: the text of every row, as the block stores it; a float64 row may instead be the double the cell holds, for
values such as NaN, +-Inf or subnormals that no text of the writer's reaches).  Parsers: the oracle's tryParseFloat64 and tryParseNumber
(oracle/vlo_mathnum.h, through tests/vlostats.py); the engine's own parser is not used here.
"""
import math

KINDS = ("string", "dict", "uint8", "uint16", "uint32", "uint64", "int64", "float64", "ipv4", "iso8601")
# valueType codes of the oracle's columns (lib/logstorage/values_encoder.go)
VT_KIND = {1: "string", 2: "dict", 3: "uint8", 4: "uint16", 5: "uint32", 6: "uint64", 7: "float64", 8: "ipv4", 9: "iso8601", 10: "int64"}
NAN = float("nan")


def _f64(s):
    import vlostats
    return vlostats.try_parse_float64(s)


def _num(s):
    import vlostats
    return vlostats.try_parse_number(s)


def _cell_f64(v):
    """a float64 row: its text through tryParseFloat64, or the double itself"""
    return v if isinstance(v, float) else _f64(v)[0]


def sum_values(kind, payload, rows):
    """blockResultColumn.sumValues over the selected rows -> (sum, count)"""
    n = len(rows)
    if kind == "const":
        f, ok = _f64(payload)
        return (f * n, n) if ok else (0.0, 0)
    vals = [payload[r] for r in rows]
    s, c = 0.0, 0
    if kind in ("string", "dict"):
        for v in vals:
            f, ok = _num(v)
            if ok and not (kind == "dict" and math.isnan(f)):
                s += f
                c += 1
        return s, c
    if kind in ("uint8", "uint16", "uint32"):
        return float(sum(int(v) for v in vals) & (2 ** 64 - 1)), n
    if kind in ("uint64", "int64"):
        for v in vals:
            s += float(int(v))
        return s, n
    if kind == "float64":
        for v in vals:
            f = _cell_f64(v)
            if not math.isnan(f):
                s += f
        return s, n
    return 0.0, 0


def value_at_row(kind, payload, r):
    """getFloatValueAtRow -> (number, ok)"""
    if kind == "const":
        return _f64(payload)
    v = payload[r]
    if kind in ("string", "dict"):
        return _f64(v)
    if kind in ("uint8", "uint16", "uint32", "uint64", "int64"):
        return float(int(v)), True
    if kind == "float64":
        f = _cell_f64(v)
        return f, not math.isnan(f)
    return 0.0, False


def text(col, r):
    if col is None:
        return b""
    kind, payload = col
    return payload if kind == "const" else payload[r]


class Group:
    __slots__ = ("rows", "sums", "counts", "abs", "ints")

    def __init__(self, nv):
        self.rows, self.sums, self.counts, self.abs, self.ints = 0, [NAN] * nv, [0] * nv, [0.0] * nv, [True] * nv

    def add(self, f, x, count):
        """statsSumProcessor.updateState / statsAvgProcessor: x joins the sum when count > 0"""
        self.counts[f] += count
        if count:
            self.sums[f] = x if math.isnan(self.sums[f]) else self.sums[f] + x
            if not math.isnan(x):
                self.abs[f] += abs(x)
                self.ints[f] = self.ints[f] and math.isfinite(x) and x == int(x)


def stats(blocks, bucket_of, by, values):
    """-> {(bucket, key texts): Group}; bucket_of(ts) is truncateTimestamp with the query's step, offset and calendar"""
    out = {}
    nv = len(values)
    for blk in blocks:
        rows = blk["rows"]
        if not rows:
            continue
        cols = blk["cols"]
        keys = [(bucket_of(blk["ts"][r]), tuple(text(cols.get(f), r) for f in by)) for r in rows]
        if all(k == keys[0] for k in keys):
            g = out.setdefault(keys[0], Group(nv))
            g.rows += len(rows)
            for f, name in enumerate(values):
                col = cols.get(name) if name != "_time" else None
                if col is not None:
                    x, c = sum_values(col[0], col[1], rows)
                    g.add(f, x, c)
            continue
        for k, r in zip(keys, rows):
            g = out.setdefault(k, Group(nv))
            g.rows += 1
            for f, name in enumerate(values):
                col = cols.get(name) if name != "_time" else None
                if col is not None:
                    x, ok = value_at_row(col[0], col[1], r)
                    if ok:
                        g.add(f, x, 1)
    return out


def close(got, want, absum, ints):
    """the device's sum against the model's: equal when every number is an integer and the total stays below 2^53, else within
    2^-40 * sum |x| (the two add in different orders); NaN on both sides when there were no numbers; a zero has the model's sign"""
    if math.isnan(want) or math.isnan(got):
        return math.isnan(want) and math.isnan(got)
    if math.isinf(want) or math.isinf(got):
        return want == got
    if got == 0.0 and want == 0.0:
        return math.copysign(1.0, got) == math.copysign(1.0, want)
    if ints and absum < 2.0 ** 53:
        return got == want
    return abs(got - want) <= 2.0 ** -40 * absum
