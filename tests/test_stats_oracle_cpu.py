"""The reference's TestStatsSum / TestStatsAvg tables and the `stats by (_time:...)` cases of TestPipeStats (tests/golden/stats_cases.json)
through both restatements of `stats ... sum(v), avg(v)`: the C++ one over the oracle's value and timestamp decode (tests/stats_oracle) and the
Python one (tests/stats_model.py), each with the rows in one block per run of equal field names and in one block per row.  Then random blocks
of every column kind through both, which must agree."""
import math
import random

import stats_cases as sc
import vlostats


def cpp_groups(oracle, blocks, flt, step, off, cal, by, values):
    got = vlostats.stats([b for b, _, _ in blocks], flt, step, off, cal, by, values)
    return {k: (rows, [(s, c) for s, c, _, _ in vals]) for k, (rows, vals) in got.items()}


def test_reference_tables(oracle):
    used = 0
    for case in sc.load():
        p = sc.parse(case["query"])
        if p is None:
            continue
        used += 1
        step, off, by, _, _ = p
        for one_per_row in (False, True):
            blocks = sc.blocks_of(oracle, case["rows"], one_per_row)
            for backend in (cpp_groups, sc.model_groups):
                got = backend(oracle, blocks, oracle.Filter.noop(), step, off, 0, by, sc.values_of(p))
                assert sc.result_rows(got, p) == sc.expected_rows(case), (case["query"], backend.__name__, one_per_row)
    assert used == 18, used   # 30 cases; 8 have `if (...)` or `*` arguments


def test_random_blocks_agree(oracle):
    rng = random.Random(11)
    pool = {
        "u8": lambda i: b"%d" % (i % 200), "u32": lambda i: b"%d" % (i * 100003 % 4000000000), "u64": lambda i: b"%d" % (2 ** 64 - 1 - i),
        "i64": lambda i: b"%d" % ((i - 50) * 12345678901), "f64": lambda i: b"%d.%d" % (i - 40, 1 + i % 9), "ip": lambda i: b"1.2.3.%d" % (i % 256),
        "iso": lambda i: b"2024-01-%02dT00:00:00Z" % (1 + i % 28), "s": lambda i: [b"5s", b"1KiB", b"x", b"7", b"1_000", b"-2.5", b"0x10"][i % 7] + (b"" if i % 3 else b" "),
        "d": lambda i: [b"3", b"abc", b"1MB"][i % 3], "c": lambda i: b"42",
    }
    blocks, t = [], 10 ** 18
    for bi in range(12):
        n = rng.choice([1, 3, 70, 200])
        cols = {name: [gen(i + bi) for i in range(n)] for name, gen in pool.items()}
        cols["k"] = [b"k%d" % (i * 3 // n) for i in range(n)] if bi % 2 else [b"k0"] * n
        ts = [t + i * 10 ** 8 for i in range(n)]
        t = ts[-1] + rng.choice([1, 10 ** 9, 10 ** 11])
        blk = oracle.Block.from_columns(list(cols.items())).set_timestamps(ts)
        blocks.append((blk, cols, ts))
    values = list(pool) + ["nope", "_time"]
    for step, by, flt in ((10 ** 18, (), oracle.Filter.noop()), (10 ** 10, ("k",), oracle.Filter.noop()), (10 ** 18, ("k",), oracle.Filter.phrase("s", "x"))):
        a = cpp_groups(oracle, blocks, flt, step, 0, 0, by, values)
        b = sc.model_groups(oracle, blocks, flt, step, 0, 0, by, values)
        assert a.keys() == b.keys()
        for k in a:
            assert a[k][0] == b[k][0]
            for (s1, c1), (s2, c2) in zip(a[k][1], b[k][1]):
                assert c1 == c2 and (s1 == s2 or (math.isnan(s1) and math.isnan(s2))), (k, s1, s2)
