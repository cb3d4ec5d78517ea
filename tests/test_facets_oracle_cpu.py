"""CPU differential of the two restatements of `| facets`: tests/facets_model.py (Python, the bar of the GPU differential) against the C++
shard and flush of tests/facets_oracle/vlo_facets.h over oracle blocks, whose values and timestamps the C++ side decodes from the stored bytes.
Covers the reference's TestPipeFacets cases and thousands of random blocks with every column kind the oracle's writer picks, the key-class
quirks of updateStateGeneric, both length rules at max_value_len 1..22 and distinct counts at and just above max_values_per_field."""
import json
import os
import random

import pytest

import facets_model as fm
from victorialogs_b200 import scan as vs

HERE = os.path.dirname(os.path.abspath(__file__))
QUIRKS = [b"1_000", b"1000", b"_", b"-_", b"_01", b"0123", b"0_1", b"-0", b"0", b"-", b"1" + b"_" * 25, b"1" + b"_" * 26, b"-9223372036854775808",
          b"-9223372036854775809", b"18446744073709551615", b"18446744073709551616", b"12345678901", b"-7", b""]


@pytest.fixture(scope="module")
def vlofacets(oracle):
    import vlofacets
    vlofacets.lib()
    return vlofacets


def model(oracle, blocks, flt, fields, max_values=0, max_len=0):
    sh = fm.Shard(max_values, max_len)
    decoded = 0
    for blk in blocks:
        sel = oracle.bitmap_rows(blk.search(flt), blk.rows)
        if sel and "_time" in fields:
            _, _, mn, mx = blk.timestamps_block()
            decoded += mn != mx
        sh.block(fm.oracle_cells(blk, fields, oracle) if sel else {}, sel)
    return sh.state(fields), sh.rows, decoded


def test_golden_cases_against_the_oracle(oracle, vlofacets):
    for c in json.load(open(os.path.join(HERE, "golden", "facets_cases.json"))):
        blocks = [oracle.Block.from_columns([(n, [v.encode()]) for n, v in row]).set_timestamps([i]) for i, row in enumerate(c["rows"])]
        fields = sorted({n for row in c["rows"] for n, _ in row})
        state, rows, _, flushed = vlofacets.facets(blocks, oracle.Filter.noop(), fields, limit=c["limit"], keep_const_fields=c["keep_const_fields"])
        want = [tuple(w) for w in c["want"]]
        assert [(f, t.decode(), h) for f, t, h in flushed] == want, c["pipe"]
        assert [(f, t.decode(), h) for f, t, h in vs.facets_merge([(state, rows)], c["limit"], c["keep_const_fields"])] == want, c["pipe"]
        assert model(oracle, blocks, oracle.Filter.noop(), fields) == (state, rows, 0)


def random_column(rng, n):
    kind = rng.randrange(9)
    if kind == 0:
        return [rng.choice(QUIRKS) for _ in range(n)]                                        # strings with the key-class quirks
    if kind == 1:
        top = rng.choice([255, 65535, 2 ** 32 - 1, 2 ** 64 - 1])                          # uint8..uint64 (more than 8 values: not a dict)
        big = [10 ** 10 - 1, 10 ** 10] if top > 10 ** 10 else []
        return [b"%d" % rng.choice([rng.randrange(top + 1), i, top] + big) for i in range(n)]
    if kind == 2:
        return [b"%d" % rng.choice([-(1 << 63), -1, 0, (1 << 63) - 1, -12345678901, -i, rng.randrange(-10 ** 12, 10 ** 12)]) for i in range(n)]   # int64
    if kind == 3:
        return [rng.choice([b"1.5", b"-2.25", b"3", b"-0.5", b"%d.25" % i, b"-%d" % i, b"%d.0625" % -i]) for i in range(n)]   # float64
    if kind == 4:
        return [b"10.0.%d.%d" % (rng.randrange(3), i) for i in range(n)]                     # ipv4
    if kind == 5:
        return [b"2024-03-%02dT12:00:%02d.%03dZ" % (1 + rng.randrange(28), i, rng.randrange(1000)) for i in range(n)]   # iso8601
    if kind == 6:
        return [rng.choice([b"info", b"warn", b"-0", b"0", b"", b"x" * 30]) for _ in range(n)]  # dict
    if kind == 7:
        return [rng.choice(QUIRKS)] * n                                                       # const
    return [b"v%d" % rng.randrange(n * 2) for _ in range(n)]                                # many distinct strings


def random_blocks(oracle, rng):
    blocks, t = [], rng.choice([-10 ** 18, 0, 1_700_000_000_000_000_000])
    for _ in range(rng.randint(1, 5)):
        n = rng.choice([1, 3, rng.randint(12, 60)])
        cols = [(name, random_column(rng, n)) for name in ("a", "b", "c") if rng.random() < 0.85]
        cols.append(("lvl", [rng.choice([b"info", b"error"]) for _ in range(n)]))
        step = rng.choice([0, 1, 10 ** 6, 10 ** 9 + 7])
        ts = [t + i * step + (rng.randrange(3) if step else 0) for i in range(n)]
        ts.sort()
        t = ts[-1] + rng.randrange(10 ** 9)
        blocks.append(oracle.Block.from_columns(cols).set_timestamps(ts))
    return blocks


def test_model_against_the_oracle_on_random_blocks(oracle, vlofacets):
    rng = random.Random(1234)
    fields = ["a", "b", "c", "lvl", "_time", "absent"]
    seen, nblocks = set(), 0
    for case in range(700):
        blocks = random_blocks(oracle, rng)
        nblocks += len(blocks)
        flt = rng.choice([oracle.Filter.noop(), oracle.Filter.phrase("lvl", "error")])
        max_len = rng.choice([0, rng.randint(1, 22)])
        sizes = [len(set(fm.oracle_cells(b, ["a"], oracle).get("a", ("const", b""))[1])) for b in blocks]
        max_values = rng.choice([0, 1, 2, 3, max(sizes), max(sizes) + 1, rng.randint(1, 40)])
        got, rows, decoded, _ = vlofacets.facets(blocks, flt, fields, max_values, max_len)
        assert model(oracle, blocks, flt, fields, max_values, max_len) == (got, rows, decoded), case
        for b in blocks:
            seen |= {c.value_type for c in b.columns}
        seen |= {("dropped", f) for f, st in got.items() if st is None}
        seen |= {("class", e[0]) for st in got.values() if st for e in st}
    assert nblocks > 2000
    assert {1, 2, 3, 4, 5, 6, 7, 8, 9, 10} <= seen, sorted(x for x in seen if isinstance(x, int))
    assert {("class", 0), ("class", 1), ("class", 2), ("dropped", "a"), ("dropped", "_time")} <= seen


def test_quirky_texts_in_the_oracle(oracle, vlofacets):
    blk = oracle.Block.from_columns([("k", QUIRKS)]).set_timestamps(list(range(len(QUIRKS))))
    got = vlofacets.facets([blk], oracle.Filter.noop(), ["k"], 0, 0)[0]["k"]
    keys = {(c, t) for c, t, _ in got}
    assert (fm.U64, b"1000") in keys and (fm.U64, b"1") in keys and (fm.NEG, b"0") in keys and (fm.U64, b"0") in keys
    assert (fm.STR, b"0123") in keys and (fm.STR, b"0_1") in keys and (fm.STR, b"-") in keys and (fm.STR, b"1" + b"_" * 26) in keys
    assert (fm.NEG, b"-9223372036854775808") in keys and (fm.STR, b"-9223372036854775809") in keys and (fm.STR, b"18446744073709551616") in keys
    assert dict(((c, t), h) for c, t, h in got)[(fm.U64, b"1000")] == 2          # "1_000" and "1000"
    assert dict(((c, t), h) for c, t, h in got)[(fm.NEG, b"0")] == 2             # "-0" and "-_"
