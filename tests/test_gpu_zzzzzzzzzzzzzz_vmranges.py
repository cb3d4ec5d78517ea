"""GPU parity for `stats by (_time:step, f:bucket, ...) histogram(v...)` (vlscan_hits_vmranges) against the C++ restatement from the reference
Go (tests/vmrange_oracle via tests/vlovmrange.py), which computes every index from Histogram.Update's formula: every column kind (numeric
strings with durations, byte sizes, hex, `1_000`, "NaN", "-1" and ""; float64 rows with NaN, +-Inf, -0 and subnormals; uint64 max; negative
int64; const and dict cells), the values at every vmrange boundary and next to it as float64 rows and as texts, all six timestamp marshal types,
0-4 by-fields with and without buckets, 1-4 value fields, the header fast path on and off, a kept batch staged late, a table that grows, and
the merge of two halves.  Groups, keys and rows must be those of vlscan_hits_stats_bucketed, hits exact."""
import math
import random
import struct

import numpy as np
import pytest

import vlovmrange
import vmrange_model as vm

pytestmark = pytest.mark.gpu

HOUR = 3600 * 10 ** 9
T0 = 1_700_000_000_000_000_000


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


@pytest.fixture(scope="module")
def edges():
    """the least double of every index 1..487 (from the model's formula) and its neighbours"""
    from test_vmranges_cpu import model_bounds
    out = []
    for u in model_bounds():
        out += [vm.f64_of_bits(u + d) for d in (-2, -1, 0, 1)]
    return out


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def columns(rng, bi, n, edges):
    texts = [b"7", b"250", b"-3", b"12.5", b"1.5s", b"1KiB", b"0x1F", b"1_000", b"NaN", b"-1", b"", b"abc", b"2h5m", b"-0", b"1e-9", b"1e18",
             b"Inf", b"-Inf", b"0.000001", b"3.05", b"10.1.2.3"]
    e = [edges[(bi * 131 + i * 17) % len(edges)] for i in range(n)]
    cols = {
        "u8": [b"%d" % (i * 7 % 250) for i in range(n)],
        "u16": [b"%d" % ((i * 37 % 60000) if bi % 3 else 200 + i % 3) for i in range(n)],   # every third block: one index in the header
        "u32": [b"%d" % (i * 1000003 % 4000000000) for i in range(n)],
        "u64": [b"%d" % (18446744073709551615 - i * 977) for i in range(n)],
        "i64": [b"%d" % ((i - n // 2) * 987654321) for i in range(n)] if bi % 2 else [b"%d" % (10 ** 12 + i) for i in range(n)],
        "f64": [b"%d.%d" % (i * 7 - 900, 1 + i % 97) for i in range(n)],
        "ip": [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)],
        "iso": [b"2024-03-%02dT12:%02d:%02d.%03dZ" % (1 + i % 28, i % 60, (i * 7) % 60, i % 1000) for i in range(n)],
        "str": [rng.choice(texts) for _ in range(n)],
        "etxt": [repr(x).encode() + (b"" if i else b" ") for i, x in enumerate(e)],   # the boundary values as texts (row 0 keeps it a string column)
        "dict": [[b"201", b"1e-9", b"-0", b"abc", b"1s"][(i * 5 // 7) % (5 if bi % 2 else 3)] for i in range(n)],
        "cst": [[b"1234", b"1KiB", b"-5", b"1e18"][bi % 4]] * n,
        "lvl": [[b"info", b"warn", b"error"][(i * 3 // 5) % 3] for i in range(n)],
        "code": [b"%d" % (200 + (i * 3) % 20) for i in range(n)] if bi % 2 == 0 else [b"x" if i == 0 else b"%d" % (200 + i % 80) for i in range(n)],
    }
    if bi % 4 == 3:
        del cols["u32"]
    return cols, e


def mix(env, seed, edges, nblocks=10):
    """blocks of every kind; the float64 column `ef` holds boundary values, specials and NaN rows, and in every fourth block one value
    between NaN rows (its header maps to one index, and the NaN rows must still count nothing)"""
    from test_gpu_zzzzz_hits import nearest_delta, series, zstd_compress
    oracle, vs, pu, ctx = env
    rng = random.Random(seed)
    blocks, descs, t = [], [], T0
    specials = [math.nan, math.inf, -math.inf, -0.0, 0.0, 5e-324, 2.2250738585072009e-308, -1.5, 1e-9, 1e18, 1.7976931348623157e308]
    for bi in range(nblocks):
        n = rng.choice([1, 64, 65, 300, 1500])
        ts = series(rng, ["const", "step", "jitter", "bursty"][bi % 4], n, 10 ** 12)
        ts = [v - ts[0] + t for v in ts]
        t = ts[-1] + rng.choice([1, HOUR, 40 * HOUR])
        cols, e = columns(rng, bi, n, edges)
        ef = [2.5 if i % 4 else math.nan for i in range(n)] if bi % 4 == 1 else [specials[i % len(specials)] if i % 3 == 0 else e[i] for i in range(n)]
        cols["ef"] = [b"%d.5" % i for i in range(n)]   # n distinct texts: a float64 column, its rows replaced below
        blk = oracle.Block.from_columns(list(cols.items())).set_timestamps(ts)
        d = pu.oracle_block_to_desc(blk)
        col = next((c for c in d["columns"] if c["field"] in ("ef", b"ef")), None)
        if col is not None and col["kind"] == "values" and col["value_type"] == 7:
            col["values_block"] = oracle.marshal_strings_block([struct.pack(">d", v) for v in ef])
            fin = [v for v in ef if not math.isnan(v)] or [0.0]
            col["min_value"], col["max_value"] = f64_bits(min(fin)), f64_bits(max(fin))
        if n >= 2 and bi % 5 == 3:
            raw = nearest_delta(ts)
            d["timestamps"] = (raw, 6, ts[0], ts[-1]) if bi % 10 == 3 else (zstd_compress(raw), 4, ts[0], ts[-1])
        blocks.append(blk)
        descs.append(d)
    return blocks, descs


def check(env, blocks, descs, flt, step, by, values, buckets=None, words=None, info=None):
    oracle, vs, pu, ctx = env
    words = words or [b.search(flt) for b in blocks]
    want = vlovmrange.vmranges(descs, words, step, 0, 0, by, buckets, values)
    info = {} if info is None else info
    got = ctx.hits_vmranges(step, 0, 0, by, values, buckets=buckets, info=info)
    assert [(b, k) for b, k, _, _ in got] == sorted(want), (by, values, buckets)
    for b, k, rows, vals in got:
        wrows, wvals = want[(b, k)]
        assert rows == wrows, (b, k)
        assert vals == wvals, (b, k, by, values)
    assert [(b, k, r) for b, k, r, _ in got] == ctx.hits_stats(step, 0, 0, by, buckets=buckets)
    assert info["entries"] == sum(len(m) for _, _, _, vals in got for m in vals)
    return got


VALUES = ["u8", "u16", "u32", "u64", "i64", "f64", "ef", "ip", "iso", "str", "etxt", "dict", "cst", "code", "lvl", "nope", "_time"]


def test_every_kind(env, edges):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 1, edges, nblocks=12)
    kinds = {(c["field"] if isinstance(c["field"], str) else c["field"].decode(), c["kind"], c.get("value_type")) for d in descs for c in d["columns"]}
    for name, vt in (("u8", 3), ("u16", 4), ("u32", 5), ("u64", 6), ("f64", 7), ("ef", 7), ("ip", 8), ("iso", 9), ("i64", 10), ("dict", 2), ("str", 1), ("etxt", 1)):
        assert (name, "values", vt) in kinds, name
    assert ("cst", "const", None) in kinds
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    for of, gf in ((oracle.Filter.noop(), vs.Filter.noop()), (oracle.Filter.phrase("lvl", "error"), vs.Filter.phrase("lvl", "error"))):
        ctx.scan_resident(vs.Program(gf), batch)
        for v in VALUES:
            check(env, blocks, descs, of, 10 ** 18, (), (v,))
            check(env, blocks, descs, of, HOUR, ("lvl",), (v,))
    batch.free()


def test_boundaries_in_every_bucket(env, edges):
    """every boundary and its neighbours, as float64 rows and as texts, in one group: all 488 indexes appear"""
    oracle, vs, pu, ctx = env
    vals = list(edges) + [0.0, -0.0, math.inf]
    n = len(vals)
    blk = oracle.Block.from_columns([("f", [b"%d.5" % i for i in range(n)]), ("s", [repr(x).encode() for x in vals])]).set_timestamps([T0 + i for i in range(n)])
    d = pu.oracle_block_to_desc(blk)
    col = next(c for c in d["columns"] if c["field"] in ("f", b"f"))
    col["values_block"] = oracle.marshal_strings_block([struct.pack(">d", v) for v in vals])
    col["min_value"], col["max_value"] = f64_bits(0.0), f64_bits(math.inf)
    batch = ctx.upload(vs.HostBlocks([b"f", b"s"], [d]))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    got = check(env, [blk], [d], oracle.Filter.noop(), 10 ** 18, (), ("f", "s"))
    (_, _, _, (hf, hs)), = got
    assert sorted(hf) == list(range(488))
    want = {}
    for x in vals:
        vm.update(want, x)
    assert hf == want
    batch.free()


def test_by_fields_values_and_buckets(env, edges):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 2, edges, nblocks=10)
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    rng = random.Random(7)
    specs = {"code": (100, 0, 0), "u16": (1000, 0, 0), "f64": (100, 0, 0), "str": (10, 0, 0), "ip": (256, 0, 0), "iso": (HOUR, 0, 0), "lvl": None, "dict": (100, 0, 0)}
    for it in range(30):
        by = tuple(rng.sample(sorted(specs), rng.randint(0, 4)))
        buckets = [specs[f] if rng.random() < 0.6 else None for f in by] if by and it % 3 else None
        values = tuple(rng.sample(VALUES, rng.randint(1, 4)))
        check(env, blocks, descs, oracle.Filter.noop(), rng.choice([HOUR, 24 * HOUR, 10 ** 18]), by, values, buckets)
    batch.free()


def test_header_fast_path(env):
    """uint cells whose header minimum and maximum map to one index count without reading rows; float64 and negative int64 cells never"""
    oracle, vs, pu, ctx = env
    blocks, descs = [], []
    for bi, u in enumerate((lambda i: 200 + i % 15, lambda i: 200 + i * 36, lambda i: 1100 + i % 30)):   # one index, many, one
        n = 50
        cols = [("u", [b"%d" % u(i) for i in range(n)]), ("i", [b"%d" % (2 * 10 ** 12 + i) for i in range(n)]),
                ("ineg", [b"%d" % (i - 3) for i in range(n)]), ("f", [b"%d.25" % (200 + i % 10) for i in range(n)])]
        blk = oracle.Block.from_columns(cols).set_timestamps([T0 + bi * HOUR + i for i in range(n)])
        blocks.append(blk)
        d = pu.oracle_block_to_desc(blk)
        assert {c["field"] if isinstance(c["field"], str) else c["field"].decode(): c.get("value_type") for c in d["columns"]} == {"u": [3, 4, 4][bi], "i": 6, "ineg": 10, "f": 7}
        descs.append(d)
    batch = ctx.upload(vs.HostBlocks([b"u", b"i", b"ineg", b"f"], descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    for values, fast in ((("u",), 2), (("i",), 3), (("ineg",), 0), (("f",), 0), (("u", "i", "ineg", "f"), 5)):
        info = {}
        check(env, blocks, descs, oracle.Filter.noop(), HOUR, (), values, info=info)
        assert info["header_cells"] == fast, values
    batch.free()


def test_kept_batch_and_errors(env, edges):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 4, edges, nblocks=8)
    hb = vs.HostBlocks(pu.field_names_of(blocks), descs)
    ctx.scan_batch_keep(vs.Program(vs.Filter.phrase("lvl", "error")), hb)
    with pytest.raises(vs.VlscanError, match="str"):
        ctx.hits_vmranges(HOUR, 0, 0, (), ("str",))
    with pytest.raises(vs.VlscanError, match="histogram"):
        ctx.hits_vmranges(HOUR, 0, 0, ("lvl",), ("a*",))
    ctx.stage_selected(hb, ["str", "ef", "lvl"])
    check(env, blocks, descs, oracle.Filter.phrase("lvl", "error"), HOUR, ("lvl",), ("str", "ef"))


def test_table_grows(env):
    """200 000 groups with several indexes each: the vmrange table starts at 16 Ki slots and grows"""
    oracle, vs, pu, ctx = env
    blocks, descs, t = [], [], T0
    for bi in range(50):
        n = 4000
        ts = [t + i for i in range(n)]
        t = ts[-1] + 1
        g = [(bi * n + i) % 200_000 for i in range(n)]
        cols = [("k", [b"k%d" % x for x in g]), ("v", [b"%d" % (10 ** ((x + i) % 7)) + b"5" for i, x in enumerate(g)]), ("w", [b"%d.5" % (i % 13) for i in range(n)])]
        blk = oracle.Block.from_columns(cols).set_timestamps(ts)
        blocks.append(blk)
        descs.append(pu.oracle_block_to_desc(blk))
    batch = ctx.upload(vs.HostBlocks([b"k", b"v", b"w"], descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    info = {}
    got = check(env, blocks, descs, oracle.Filter.noop(), 10 ** 18, ("k",), ("v", "w"), info=info)
    assert info["groups"] == len(got) == 200_000 and info["entries"] > 300_000
    batch.free()


def test_halves_merge(env, edges):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 5, edges, nblocks=10)
    names = pu.field_names_of(blocks)
    by, values, buckets = ("code", "lvl"), ("str", "ef", "u64"), [(100, 0, 0), None]
    states = []
    for part in (descs[:5], descs[5:]):
        batch = ctx.upload(vs.HostBlocks(names, part))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        states.append(ctx.hits_vmranges(HOUR, 0, 0, by, values, buckets=buckets))
        batch.free()
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    whole = ctx.hits_vmranges(HOUR, 0, 0, by, values, buckets=buckets)
    assert vs.vmranges_merge(states) == {(b, k): (r, v) for b, k, r, v in whole}
    batch.free()
