"""GPU parity for `stats by (_time:step offset off, f1, ...) count(), sum(v...), avg(v...)` (vlscan_hits_sums) against the Python restatement
(tests/stats_model.py) and the C++ one over the oracle's value decode (tests/stats_oracle via tests/vlostats.py), over the oracle's blocks, selected rows and timestamps: every column kind as a value field, all six timestamp marshal
types, 0-3 by-fields and 1-4 value fields, plain, month and year buckets.  Groups, rows and counts are exact; a sum is exact when its numbers
are integers adding up to less than 2^53, else within 2^-40 * sum |x|, and a zero has the restatements' sign.  The device's exactness contract
itself is checked against exact rational sums in tests/test_gpu_zzzzzzzzzzz_stats_exact.py."""
import math
import random

import pytest

import stats_cases as sc
import stats_model as sm
import vlohits
import vlostats

pytestmark = pytest.mark.gpu

DAY = 86400 * 10 ** 9


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


model_block = sc.model_block


def block_mix(env, seed, nblocks=12, scale=10 ** 12):
    from test_gpu_zzzzz_hits import nearest_delta, series, zstd_compress
    oracle, vs, pu, ctx = env
    rng = random.Random(seed)
    blocks, descs, cols_all, stamps, t0 = [], [], [], [], 1_700_000_000_000_000_000
    for bi in range(nblocks):
        n = rng.choice([1, 64, 65, 300, 2100])
        ts = series(rng, ["const", "step", "jitter", "bursty"][bi % 4], n, scale)
        ts = [v - ts[0] + t0 for v in ts]
        t0 = ts[-1] + rng.choice([1, scale, 40 * DAY])
        cols = {
            "lvl": [[b"info", b"warn", b"error", b""][(i * 5 // 7) % 4] for i in range(n)],
            "host": [b"h%d" % (i * 3 // 100) for i in range(n)],
            "u8": [b"%d" % (i * 7 % 250) for i in range(n)],
            "u16": [b"%d" % (i * 37 % 60000) for i in range(n)],
            "u32": [b"%d" % (i * 1000003 % 4000000000) for i in range(n)],
            "u64": [b"%d" % (18446744073709551615 - i * 977) for i in range(n)],
            "i64": [b"%d" % ((i - n // 2) * 987654321) for i in range(n)],
            "f64": [b"%d.%d" % (i * 7 - 900, 1 + i % 97) for i in range(n)],
            "ip": [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)],
            "iso": [b"2024-03-%02dT12:%02d:%02d.%03dZ" % (1 + i % 28, i % 60, (i * 7) % 60, i % 1000) for i in range(n)],
            "dur": [[b"5s", b"1KiB", b"12", b"x", b"1.5", b"2h", b"-3"][(i + bi) % 7] for i in range(n)],
            "dnum": [[b"7", b"abc", b"1KiB", b"-2.5"][(i * 3 // 5) % 4] for i in range(n)],
            "cst": [b"12"] * n,
            "ckib": [b"1KiB"] * n,
            # typed (uint8) in even blocks, strings in odd ones
            "code": [b"%d" % (200 + (i * 3) % 20) for i in range(n)] if bi % 2 == 0 else [b"x" if i == 0 else b"%d" % (200 + i % 20) for i in range(n)],
        }
        if bi % 3 == 2:
            del cols["u32"]
        blk = oracle.Block.from_columns(list(cols.items())).set_timestamps(ts)
        d = pu.oracle_block_to_desc(blk)
        if n >= 2 and bi % 5 == 3:
            raw = nearest_delta(ts)
            d["timestamps"] = (raw, 6, ts[0], ts[-1]) if bi % 10 == 3 else (zstd_compress(raw), 4, ts[0], ts[-1])
        blocks.append(blk)
        descs.append(d)
        cols_all.append(cols)
        stamps.append(ts)
    return blocks, descs, cols_all, stamps


def check(env, blocks, cols_all, stamps, of, step, off, cal, by, values, info=None):
    oracle, vs, pu, ctx = env
    got = ctx.hits_sums(step, off, cal, by, values, info=info)
    mb = [model_block(oracle, b, c, t, of) for b, c, t in zip(blocks, cols_all, stamps)]
    want = sm.stats(mb, lambda t: vlohits.truncate_timestamp(t, step, off, cal), by, values)
    assert [(b, k) for b, k, _, _ in got] == sorted(want), (step, off, cal, by, values)
    for b, k, rows, vals in got:
        g = want[(b, k)]
        assert rows == g.rows
        for f, (s, c) in enumerate(vals):
            assert c == g.counts[f], (b, k, values[f])
            assert sm.close(s, g.sums[f], g.abs[f], g.ints[f]), (b, k, values[f], s, g.sums[f])
    cpp = vlostats.stats(blocks, of, step, off, cal, by, values)
    assert sorted(cpp) == [(b, k) for b, k, _, _ in got]
    for b, k, rows, vals in got:
        crows, cvals = cpp[(b, k)]
        assert rows == crows
        for (s, c), (cs, cc, ca, ci) in zip(vals, cvals):
            assert c == cc and sm.close(s, cs, ca, ci), (b, k, s, cs)
    return got, want


VALUES = ["u8", "u16", "u32", "u64", "i64", "f64", "ip", "iso", "dur", "dnum", "cst", "ckib", "code", "lvl", "nope", "_time"]


def test_differential(env):
    oracle, vs, pu, ctx = env
    blocks, descs, cols_all, stamps = block_mix(env, 41, nblocks=20)
    assert {d["timestamps"][1] for d in descs} == {1, 2, 3, 4, 5, 6}
    kinds = {k for b, c, t in zip(blocks, cols_all, stamps) for k, _ in model_block(oracle, b, c, t, oracle.Filter.noop())["cols"].values()}
    assert kinds >= {"const", "string", "dict", "uint8", "uint16", "uint32", "uint64", "int64", "float64", "ipv4", "iso8601"}, kinds
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    F, G = oracle.Filter, vs.Filter
    lo, hi = stamps[3][len(stamps[3]) // 2], stamps[15][len(stamps[15]) // 3]
    filters = [(F.noop(), G.noop()), (F.phrase("lvl", "error"), G.phrase("lvl", "error")), (F.time(lo, hi), G.time(lo, hi))]
    steps = [(10 ** 9, 0, 0), (3600 * 10 ** 9, 1800 * 10 ** 9, 0), (10 ** 18, 0, 0), (0, 0, vs.BUCKET_MONTH), (0, 4 * 3600 * 10 ** 9, vs.BUCKET_YEAR), (1000, 7, 0)]
    bys = [(), ("lvl",), ("host", "lvl"), ("code", "lvl", "dur")]
    rng = random.Random(5)
    whole = multi = 0
    for k, (of, gf) in enumerate(filters):
        ctx.scan_resident(vs.Program(gf), batch)
        for j, (step, off, cal) in enumerate(steps):
            for by in bys:
                values = rng.sample(VALUES, rng.randint(1, 4))
                before = ctx.hits_stats(step, off, cal, by)
                got, want = check(env, blocks, cols_all, stamps, of, step, off, cal, by, values)
                assert ctx.hits_stats(step, off, cal, by) == before == [(b, k2, r) for b, k2, r, _ in got]
                multi += len(got) > 1
                whole += len(got) == 1
        for values in ([v] for v in VALUES):   # every kind alone, one group per block and many
            check(env, blocks, cols_all, stamps, of, 10 ** 18, 0, 0, (), values)
            check(env, blocks, cols_all, stamps, of, 10 ** 9, 0, 0, ("host",), values)
    assert multi and whole
    batch.free()


def test_quirks_on_device(env):
    """const through tryParseFloat64 ("1KiB" is none, "12" counts rows times), strings through tryParseNumber only in one-group blocks,
    dict entries that are no number, NaN for a group without numbers, uint64 near 2^64"""
    oracle, vs, pu, ctx = env
    ts = [1_700_000_000_000_000_000 + i * 10 ** 9 for i in range(4)]
    cols = {"k": [b"a", b"a", b"b", b"b"], "s": [b"1KiB", b"5s", b"7", b"x"], "c": [b"12"] * 4, "ck": [b"1KiB"] * 4, "u": [b"18446744073709551615", b"1", b"2", b"3"]}
    blk = oracle.Block.from_columns(list(cols.items())).set_timestamps(ts)
    batch = ctx.upload(pu.host_blocks_from_oracle([blk]))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    one = ctx.hits_sums(10 ** 18, 0, 0, (), ("s", "c", "ck", "u"))
    assert len(one) == 1
    (s, sc), (c, cc), (ck, ckc), (u, uc) = one[0][3]
    assert (s, sc) == (1024 + 5e9 + 7, 3) and (c, cc) == (48.0, 4) and math.isnan(ck) and ckc == 0 and uc == 4
    two = ctx.hits_sums(10 ** 18, 0, 0, ("k",), ("s", "c"))
    assert [k for _, k, _, _ in two] == [(b"a",), (b"b",)]
    (sa, na), (ca, cna) = two[0][3]
    assert math.isnan(sa) and na == 0 and (ca, cna) == (24.0, 2)   # "1KiB" and "5s" are no tryParseFloat64 numbers
    assert two[1][3] == [(7.0, 1), (24.0, 2)]
    check(env, [blk], [cols], [ts], oracle.Filter.noop(), 10 ** 18, 0, 0, ("k",), ("s", "c", "ck", "u"))
    batch.free()


def test_halves_merge(env):
    oracle, vs, pu, ctx = env
    blocks, descs, cols_all, stamps = block_mix(env, 9, nblocks=12)
    names = pu.field_names_of(blocks)
    args = (3600 * 10 ** 9, 0, 0, ("lvl",), ("u16", "dur", "f64"))
    states = []
    for part in (descs[:6], descs[6:]):
        batch = ctx.upload(vs.HostBlocks(names, part))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        states.append(ctx.hits_sums(*args))
        batch.free()
    merged = vs.stats_merge(states)
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    whole = ctx.hits_sums(*args)
    assert sorted(merged) == [(b, k) for b, k, _, _ in whole]
    for b, k, rows, vals in whole:
        mrows, mvals = merged[(b, k)]
        assert mrows == rows
        for (s1, c1), (s2, c2) in zip(vals, mvals):
            assert c1 == c2 and (math.isnan(s1) and math.isnan(s2) or abs(s1 - s2) <= 2.0 ** -40 * max(abs(s1), 1.0) * rows)
    batch.free()


def test_many_groups_rerun_the_table(env):
    """20 000 distinct keys: the table starts at 16 Ki slots, overflows and runs again; sums stay exact"""
    oracle, vs, pu, ctx = env
    blocks, cols_all, stamps, t = [], [], [], 1_700_000_000_000_000_000
    for bi in range(20):
        n = 2000
        ts = [t + i * 10 ** 6 for i in range(n)]
        t = ts[-1] + 10 ** 6
        cols = {"k": [b"key-%06d" % ((bi * n + i) * 7919 % 20_000) for i in range(n)], "v": [b"%d" % (i * 13 + bi) for i in range(n)]}
        blocks.append(oracle.Block.from_columns(list(cols.items())).set_timestamps(ts))
        cols_all.append(cols)
        stamps.append(ts)
    batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    info = {}
    got, want = check(env, blocks, cols_all, stamps, oracle.Filter.noop(), 3600 * 10 ** 9, 0, 0, ("k",), ("v",), info=info)
    assert info["groups"] == len(want) == 20_000
    batch.free()


def test_kept_batch_and_errors(env):
    oracle, vs, pu, ctx = env
    blocks, descs, cols_all, stamps = block_mix(env, 3, nblocks=6)
    names = pu.field_names_of(blocks)
    hb = vs.HostBlocks(names, descs)
    prog = vs.Program(vs.Filter.phrase("lvl", "error"))
    ctx.scan_batch_keep(prog, hb)
    ctx.stage_selected(hb, ["lvl"])
    with pytest.raises(vs.VlscanError, match="u16"):
        ctx.hits_sums(10 ** 9, 0, 0, ("lvl",), ("u16",))
    ctx.scan_batch_keep(prog, hb)
    ctx.stage_selected(hb, ["lvl", "u16", "dur"])
    check(env, blocks, cols_all, stamps, oracle.Filter.phrase("lvl", "error"), 10 ** 9, 0, 0, ("lvl",), ("u16", "dur"))
    with pytest.raises(vs.VlscanError, match="too many value fields"):
        ctx.hits_sums(10 ** 9, 0, 0, (), ("u8", "u16", "u32", "u64", "i64"))
    with pytest.raises(vs.VlscanError, match="prefix filter"):
        ctx.hits_sums(10 ** 9, 0, 0, (), ("u*",))
    with pytest.raises(vs.VlscanError, match="no value fields"):
        ctx.hits_sums(10 ** 9, 0, 0, (), ())
    check(env, blocks, cols_all, stamps, oracle.Filter.phrase("lvl", "error"), 10 ** 9, 0, 0, ("lvl",), ("dur",))


def test_reference_tables_on_device(env):
    """TestStatsSum / TestStatsAvg and the `stats by (_time:...)` cases of TestPipeStats (tests/golden/stats_cases.json) through the device,
    with the rows in one block per run of equal field names and in one block per row"""
    oracle, vs, pu, ctx = env
    used = 0
    for case in sc.load():
        p = sc.parse(case["query"])
        if p is None:
            continue
        used += 1
        step, off, by, _, _ = p
        for one_per_row in (False, True):
            blocks = sc.blocks_of(oracle, case["rows"], one_per_row)
            batch = ctx.upload(pu.host_blocks_from_oracle([b for b, _, _ in blocks]))
            ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
            got = ctx.hits_sums(step, off, 0, by, sc.values_of(p)) if sc.values_of(p) else \
                [(b, k, r, []) for b, k, r in ctx.hits_stats(step, off, 0, by)]
            groups = {(b, k): (r, v) for b, k, r, v in got}
            assert sc.result_rows(groups, p) == sc.expected_rows(case), (case["query"], one_per_row)
            batch.free()
    assert used == 18
