"""GPU parity for bucketed by-fields, `stats by (_time:step, f:size offset off, ...) count(), sum(v), avg(v)` (vlscan_hits_stats and
vlscan_hits_sums with by_buckets), against the C++ restatement from the reference Go (tests/bucket_oracle via tests/vlobucket.py): every column
kind with and without the typed header fast path (float64 blocks with NaN rows included), const and dict entries that merge into one bucket,
1-4 by-fields mixing bucketed and plain ones, a kept batch staged late, a group table that grows, the sums' one-key-per-block path and the merge
of two halves.  Groups, keys and rows are exact; sums as in tests/test_gpu_zzzzzzzzzz_stats.py."""
import math
import random
import struct

import numpy as np
import pytest

import stats_model as sm
import vlobucket

pytestmark = pytest.mark.gpu

HOUR, DAY = 3600 * 10 ** 9, 86400 * 10 ** 9
T0 = 1_700_000_000_000_000_000


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


def columns(rng, bi, n):
    nums = [b"7", b"250", b"-3", b"12.5", b"1.5s", b"2024-03-05T12:34:56.5Z", b"10.1.2.3", b"abc", b"", b"2h5m", b"-0.01"]
    cols = {
        "u8": [b"%d" % (i * 7 % 250) for i in range(n)],
        "u16": [b"%d" % ((i * 37 % 60000) if bi % 3 else 200 + i % 90) for i in range(n)],   # every third block: one bucket of 100
        "u32": [b"%d" % (i * 1000003 % 4000000000) for i in range(n)],
        "u64": [b"%d" % (18446744073709551615 - i * 977) for i in range(n)],
        "i64": [b"%d" % ((i - n // 2) * 987654321) for i in range(n)],
        "f64": [b"%d.%d" % (i * 7 - 900, 1 + i % 97) for i in range(n)] if bi % 3 else [b"%d.25" % (1000 + i % 50) for i in range(n)],
        "ip": [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)] if bi % 3 else [b"10.9.8.%d" % (i % 200) for i in range(n)],
        "iso": [b"2024-03-%02dT12:%02d:%02d.%03dZ" % (1 + i % 28, i % 60, (i * 7) % 60, i % 1000) for i in range(n)],
        "str": [rng.choice(nums) for _ in range(n)],
        "dict": [[b"201", b"250", b"299", b"abc"][(i * 5 // 7) % (4 if bi % 2 else 3)] for i in range(n)],
        "cst": [b"1234"] * n,
        "lvl": [[b"info", b"warn", b"error"][(i * 3 // 5) % 3] for i in range(n)],
        "code": [b"%d" % (200 + (i * 3) % 20) for i in range(n)] if bi % 2 == 0 else [b"x" if i == 0 else b"%d" % (200 + i % 80) for i in range(n)],
        "v": [b"%d" % (i % 13) for i in range(n)],
    }
    if bi % 4 == 3:
        del cols["u32"]
    return cols


def mix(env, seed, nblocks=10):
    oracle, vs, pu, ctx = env
    rng = random.Random(seed)
    blocks, descs, t = [], [], T0
    for bi in range(nblocks):
        n = rng.choice([1, 64, 65, 300, 1500])
        dt = rng.choice([10 ** 6, 10 ** 9, 60 * 10 ** 9])
        ts = [t + i * dt for i in range(n)]
        t = ts[-1] + HOUR
        blk = oracle.Block.from_columns(list(columns(rng, bi, n).items())).set_timestamps(ts)
        blocks.append(blk)
        descs.append(pu.oracle_block_to_desc(blk))
    return blocks, descs


def kinds_of(descs, name):
    return {(c["kind"], c.get("value_type")) for d in descs for c in d["columns"] if c["field"] in (name, name.encode())}


def check(env, blocks, descs, flt, step, off, cal, by, buckets, values=(), words=None, info=None):
    oracle, vs, pu, ctx = env
    words = words or [b.search(flt) for b in blocks]
    want = vlobucket.stats(descs, words, step, off, cal, by, buckets, values)
    if values:
        got = ctx.hits_sums(step, off, cal, by, values, buckets=buckets, info=info)
    else:
        got = [(b, k, r, []) for b, k, r in ctx.hits_stats(step, off, cal, by, buckets=buckets, info=info)]
    assert [(b, k) for b, k, _, _ in got] == sorted(want), (by, buckets)
    for b, k, rows, vals in got:
        wrows, wvals = want[(b, k)]
        assert rows == wrows, (b, k)
        for (s, c), (ws, wc, wa, wi) in zip(vals, wvals):
            assert c == wc and sm.close(s, ws, wa, wi), (b, k, s, ws)
    return got


SPECS = {
    "u8": [(10, 0, 0), (100, 3, 0), (0.5, 0, 0)], "u16": [(100, 0, 0), (1000, -7, 0)], "u32": [(1e6, 0, 0), (3, 1e19, 0)],
    "u64": [(1e15, 0, 0), (7, 2, 0)], "i64": [(1e9, 0, 0), (1e9, -5e8, 0), (0, 0, 0)], "f64": [(100, 0, 0), (0.1, 0, 0), (0.02, 0.05, 0), (2.5, -1.25, 0)],
    "ip": [(256, 0, 0), (65536, 0, 0), (16, 3, 0)], "iso": [(HOUR, 0, 0), (DAY, 1800 * 10 ** 9, 0), (0, 0, 2), (0, 0, 3), (7 * DAY, 0, 1)],
    "str": [(100, 0, 0), (0.1, 0, 0), (HOUR, 0, 0), (256, 0, 0)], "dict": [(100, 0, 0)], "cst": [(1000, 0, 0), (10, 5, 0)],
    "code": [(100, 0, 0), (10, 0, 0)], "nope": [(10, 0, 0)],
}


def test_every_kind(env):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 1, nblocks=12)
    for name, want in (("u8", 3), ("u16", 4), ("u32", 5), ("u64", 6), ("f64", 7), ("ip", 8), ("iso", 9), ("i64", 10), ("dict", 2)):
        assert ("values", want) in kinds_of(descs, name), (name, kinds_of(descs, name))
    assert kinds_of(descs, "cst") == {("const", None)} and kinds_of(descs, "code") >= {("values", 1), ("values", 3)}
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    F, G = oracle.Filter, vs.Filter
    for of, gf in ((F.noop(), G.noop()), (F.phrase("lvl", "error"), G.phrase("lvl", "error"))):
        ctx.scan_resident(vs.Program(gf), batch)
        for name, specs in SPECS.items():
            for spec in specs:
                check(env, blocks, descs, of, 10 ** 18, 0, 0, (name,), [spec])
                check(env, blocks, descs, of, HOUR, 0, 0, (name, "lvl"), [spec, None])
    batch.free()


def test_mixed_by_fields_and_sums(env):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 2, nblocks=10)
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    rng = random.Random(7)
    names = sorted(SPECS)
    for _ in range(40):
        by = rng.sample(names, rng.randint(1, 4))
        buckets = [rng.choice(SPECS[f]) if rng.random() < 0.7 else None for f in by]
        values = rng.sample(["v", "u16", "f64", "str", "dict", "cst", "nope"], rng.randint(0, 3))
        check(env, blocks, descs, oracle.Filter.noop(), rng.choice([HOUR, DAY, 10 ** 18]), 0, 0, by, buckets, values)
    batch.free()


def test_null_and_disabled_buckets_are_the_plain_call(env):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 3, nblocks=6)
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    by = ("code", "f64", "lvl")
    plain = ctx.hits_stats(HOUR, 0, 0, by)
    assert ctx.hits_stats(HOUR, 0, 0, by, buckets=[None, None, None]) == plain
    import ctypes as C   # by_buckets NULL through the bucketed entry point
    q, keep = vs.hits_query(HOUR, 0, 0, by)
    b, c, o, kb, info = np.zeros(1 << 16, np.int64), np.zeros(1 << 16, np.uint64), np.zeros(3 << 16 | 1, np.uint64), np.zeros(1 << 22, np.uint8), (C.c_uint64 * 4)()
    ctx._check(vs.lib().vlscan_hits_stats_bucketed(ctx.h, C.byref(q), None, b.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p), C.c_uint64(1 << 16),
                                                   kb.ctypes.data_as(C.c_void_p), C.c_uint64(1 << 22), o.ctypes.data_as(C.c_void_p), info))
    keys = vs._row_texts(kb.tobytes(), o, int(info[0]), 3)
    assert [(int(b[g]), keys[g], int(c[g])) for g in range(int(info[0]))] == plain
    sums = ctx.hits_sums(HOUR, 0, 0, by, ("v",))
    assert ctx.hits_sums(HOUR, 0, 0, by, ("v",), buckets=[None] * 3) == sums
    with pytest.raises(vs.VlscanError, match="bucket rejected"):
        ctx.hits_stats(HOUR, 0, 0, by, buckets=[(math.nan, 0, 0), None, None])
    with pytest.raises(vs.VlscanError, match="bucket rejected"):
        ctx.hits_stats(HOUR, 0, 0, by, buckets=[None, (1e11, 0, 0), None])   # int64(1e11 * 10^-11) is 0
    assert ctx.hits_stats(HOUR, 0, 0, by) == plain   # the ctx stays usable
    batch.free()


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def test_float64_nan_blocks(env):
    """tryFloat64Encoding skips NaN in min / max except on row 0: NaN rows between finite values share the header's bucket; a block whose first
    row is NaN has min = max = NaN and lands in one finite bucket as a whole"""
    oracle, vs, pu, ctx = env
    nan = float("nan")
    rows = [[1.5, nan, 1.75, nan, 1.25], [nan, 5.5, 300.25, -7.5], [2.5, 2.5, nan], [nan, 4.0], [130.4, 30.3, nan, 99.9, -0.01]]
    rows = [v + [v[0]] * (12 - len(v)) for v in rows]   # 12 distinct texts below: a float64 column, not a dict
    blocks, descs = [], []
    for bi, vals in enumerate(rows):
        n = len(vals)
        blk = oracle.Block.from_columns([("f", [b"%d.5" % i for i in range(n)]), ("k", [b"k%d" % (i % 2) for i in range(n)])]).set_timestamps([T0 + bi * HOUR + i for i in range(n)])
        d = pu.oracle_block_to_desc(blk)
        col = next(c for c in d["columns"] if c["field"] in ("f", b"f"))
        assert col["value_type"] == 7
        finite = [v for i, v in enumerate(vals) if i == 0 or not math.isnan(v)]
        col["values_block"] = oracle.marshal_strings_block([struct.pack(">d", v) for v in vals])
        col["min_value"], col["max_value"] = f64_bits(min(finite) if not math.isnan(finite[0]) else nan), f64_bits(max(finite) if not math.isnan(finite[0]) else nan)
        blocks.append(blk)
        descs.append(d)
    batch = ctx.upload(vs.HostBlocks([b"f", b"k"], descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    words = [np.array([(1 << len(v)) - 1], dtype=np.uint64) for v in rows]
    for spec in [(1, 0, 0), (100, 0, 0), (0.1, 0, 0), (100, 30.3, 0), (1e6, 0, 0)]:
        check(env, blocks, descs, None, 10 ** 18, 0, 0, ("f",), [spec], words=words)
        check(env, blocks, descs, None, 10 ** 18, 0, 0, ("f", "k"), [spec, None], ("f",), words=words)
    batch.free()


def test_kept_batch_staged_late(env):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 4, nblocks=8)
    hb = vs.HostBlocks(pu.field_names_of(blocks), descs)
    prog = vs.Program(vs.Filter.phrase("lvl", "error"))
    ctx.scan_batch_keep(prog, hb)
    with pytest.raises(vs.VlscanError, match="u16"):
        ctx.hits_stats(HOUR, 0, 0, ("u16",), buckets=[(100, 0, 0)])
    ctx.stage_selected(hb, ["u16", "str", "v"])
    check(env, blocks, descs, oracle.Filter.phrase("lvl", "error"), HOUR, 0, 0, ("u16", "str"), [(100, 0, 0), (10, 0, 0)], ("v",))


def test_table_grows(env):
    """20 000 distinct bucketed keys: the table starts at 16 Ki slots, overflows and runs again"""
    oracle, vs, pu, ctx = env
    blocks, descs, t = [], [], T0
    for bi in range(10):
        n = 4000
        ts = [t + i * 10 ** 6 for i in range(n)]
        t = ts[-1] + 10 ** 6
        cols = [("k", [b"%d" % (((bi * n + i) * 7919 % 20_000) * 10 + i % 7) for i in range(n)]), ("v", [b"%d" % (i % 5) for i in range(n)])]
        blk = oracle.Block.from_columns(cols).set_timestamps(ts)
        blocks.append(blk)
        descs.append(pu.oracle_block_to_desc(blk))
    batch = ctx.upload(vs.HostBlocks([b"k", b"v"], descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    info = {}
    got = check(env, blocks, descs, oracle.Filter.noop(), 10 ** 18, 0, 0, ("k",), [(10, 0, 0)], ("v",), info=info)
    assert info["groups"] == len(got) == 20_000
    batch.free()


def test_sums_one_key_per_block(env):
    """raw values that differ but share one bucket make the block one group: its sums go through sumValues (tryParseNumber: "1KiB" and "5s"
    count), not getFloatValueAtRow"""
    oracle, vs, pu, ctx = env
    blocks, descs = [], []
    for bi, keys in enumerate(([b"201", b"250", b"299", b"2.5e2x"], [b"301", b"399", b"350", b"300"])):
        cols = [("s", keys), ("d", [b"1KiB", b"5s", b"7", b"x"])]
        blk = oracle.Block.from_columns(cols).set_timestamps([T0 + bi * 10 ** 9 + i for i in range(4)])
        blocks.append(blk)
        descs.append(pu.oracle_block_to_desc(blk))
    batch = ctx.upload(vs.HostBlocks([b"s", b"d"], descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    got = check(env, blocks, descs, oracle.Filter.noop(), 10 ** 18, 0, 0, ("s",), [(100, 0, 0)], ("d",))
    byk = {k: vals for _, k, _, vals in got}
    assert byk[(b"300",)] == [(1024 + 5e9 + 7, 3)]          # one key in block 1: sumValues
    assert byk[(b"200",)] == [(7.0, 1)]                     # block 0 has two keys: row by row, tryParseFloat64
    batch.free()


def test_halves_merge(env):
    oracle, vs, pu, ctx = env
    blocks, descs = mix(env, 5, nblocks=10)
    names = pu.field_names_of(blocks)
    args = dict(buckets=[(100, 0, 0), (256, 0, 0)])
    states = []
    for part in (descs[:5], descs[5:]):
        batch = ctx.upload(vs.HostBlocks(names, part))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        states.append(ctx.hits_sums(HOUR, 0, 0, ("str", "ip"), ("v", "f64"), **args))
        batch.free()
    merged = vs.stats_merge(states)
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    whole = ctx.hits_sums(HOUR, 0, 0, ("str", "ip"), ("v", "f64"), **args)
    assert sorted(merged) == [(b, k) for b, k, _, _ in whole]
    for b, k, rows, vals in whole:
        mrows, mvals = merged[(b, k)]
        assert mrows == rows
        for (s1, c1), (s2, c2) in zip(vals, mvals):
            assert c1 == c2 and (math.isnan(s1) and math.isnan(s2) or abs(s1 - s2) <= 2.0 ** -40 * max(abs(s1), 1.0) * rows)
    batch.free()
