"""The restatement of `stats ... sum(v), avg(v)` (tests/stats_model.py) on hand-made blocks, with the reference's quirks pinned: a const value
goes through tryParseFloat64 and counts once per row, strings and dict entries go through tryParseNumber only when the block is one group
(sumValues) and through tryParseFloat64 row by row otherwise, uint8..uint32 add as uint64, a float64 NaN counts in sumValues only, and a
group without numbers sums to NaN.  Also the cross-batch merge of the per-batch states."""
import math
import sys

import pytest

import stats_model as sm


def one(cols, rows=None, n=4, by=(), values=("v",), keys=None):
    blk = {"ts": [10 ** 18 + i for i in range(n)], "rows": list(range(n)) if rows is None else rows, "cols": dict(cols)}
    if keys is not None:
        blk["cols"]["k"] = ("string", keys)
        by = ("k",)
    return sm.stats([blk], lambda t: 0, by, values)


def test_const_goes_through_try_parse_float64(oracle):
    g = one({"v": ("const", b"12")})[(0, ())]
    assert (g.rows, g.sums, g.counts) == (4, [48.0], [4])
    g = one({"v": ("const", b"1KiB")})[(0, ())]
    assert math.isnan(g.sums[0]) and g.counts == [0]
    g = one({"v": ("const", b"1.5")}, keys=[b"a", b"a", b"b", b"b"])[(0, (b"a",))]
    assert (g.sums, g.counts) == ([3.0], [2])


def test_const_integer_above_2_53(oracle):
    g = one({"v": ("const", b"18446744073709551615")})[(0, ())]
    assert (g.sums, g.counts) == ([4 * 2.0 ** 64], [4])


def test_strings_parse_by_block_shape(oracle):
    vals = [b"1KiB", b"5s", b"7", b"x"]
    g = one({"v": ("string", vals)})[(0, ())]
    assert (g.sums, g.counts) == ([1024 + 5e9 + 7], [3])
    out = one({"v": ("string", vals)}, keys=[b"a", b"a", b"b", b"b"])
    assert math.isnan(out[(0, (b"a",))].sums[0]) and out[(0, (b"a",))].counts == [0]
    assert (out[(0, (b"b",))].sums, out[(0, (b"b",))].counts) == ([7.0], [1])


def test_dict_entries_that_are_no_number(oracle):
    g = one({"v": ("dict", [b"abc", b"2", b"1KiB", b"abc"])})[(0, ())]
    assert (g.sums, g.counts) == ([1026.0], [2])
    out = one({"v": ("dict", [b"abc", b"2", b"1KiB", b"abc"])}, keys=[b"a", b"b", b"a", b"b"])
    assert math.isnan(out[(0, (b"a",))].sums[0]) and (out[(0, (b"b",))].sums, out[(0, (b"b",))].counts) == ([2.0], [1])


def test_integers_and_floats(oracle):
    g = one({"v": ("uint64", [b"18446744073709551615", b"1", b"2", b"3"])})[(0, ())]
    assert g.sums == [float(2 ** 64)] and g.counts == [4]
    g = one({"v": ("uint32", [b"4294967295"] * 4)})[(0, ())]
    assert g.sums == [4 * 4294967295.0]
    g = one({"v": ("int64", [b"-5", b"3", b"-9223372036854775808", b"0"])})[(0, ())]
    assert g.sums == [-5.0 + 3.0 - 9223372036854775808.0] and g.counts == [4]
    g = one({"v": ("float64", [b"1.25", b"2.5", b"-0.75", b"3"])})[(0, ())]
    assert g.sums == [6.0]


def test_nothing_from_ipv4_iso8601_time_or_absent(oracle):
    for col in (("ipv4", [b"1.2.3.4"] * 4), ("iso8601", [b"2024-01-01T00:00:00Z"] * 4)):
        g = one({"v": col})[(0, ())]
        assert math.isnan(g.sums[0]) and g.counts == [0]
    g = one({"v": ("uint8", [b"1"] * 4)}, values=("_time", "nope", "v"))[(0, ())]
    assert math.isnan(g.sums[0]) and math.isnan(g.sums[1]) and g.counts == [0, 0, 4] and g.sums[2] == 4.0


def test_selected_rows_only(oracle):
    g = one({"v": ("uint16", [b"1", b"10", b"100", b"1000"])}, rows=[1, 3])[(0, ())]
    assert (g.rows, g.sums, g.counts) == (2, [1010.0], [2])


def test_close_bounds():
    assert sm.close(3.0, 3.0, 3.0, True) and not sm.close(3.0 + 2 ** -40, 3.0, 3.0, True)
    assert sm.close(0.1 + 0.2, 0.3, 0.5, False) and not sm.close(0.31, 0.3, 0.5, False)
    assert sm.close(math.nan, math.nan, 0.0, True) and not sm.close(0.0, math.nan, 0.0, True)
    assert sm.close(-0.0, -0.0, 0.0, True) and not sm.close(0.0, -0.0, 0.0, True) and not sm.close(-0.0, 0.0, 0.0, False)


def test_signed_zero_sums(oracle):
    """the reference's sum is -0 only when every term it adds is -0: a row-path "-0" and a const "-0" (f * rows) stay -0, sumValues' total
    over strings starts at +0"""
    g = one({"v": ("string", [b"-0", b"x"])}, n=2, keys=[b"a", b"b"])[(0, (b"a",))]
    assert math.copysign(1.0, g.sums[0]) < 0 and g.sums[0] == 0.0 and g.counts == [1]
    g = one({"v": ("const", b"-0")})[(0, ())]
    assert math.copysign(1.0, g.sums[0]) < 0 and g.counts == [4]
    g = one({"v": ("string", [b"-0", b"-0", b"x", b"y"])})[(0, ())]
    assert math.copysign(1.0, g.sums[0]) > 0 and g.counts == [2]


def test_exact_sum_reference():
    """the exact reference of tests/test_gpu_zzzzzzzzzzz_stats_exact.py on hand-computed cases"""
    import test_gpu_zzzzzzzzzzz_stats_exact as sx

    def terms(*xs):
        t = sx.Terms()
        t.count = len(xs)
        for x in xs:
            t.add(x)
        return t

    tiny, big = 2.0 ** -1074, sys.float_info.max
    assert sx.exact(terms(2.0 ** 53, 1.0)) == 2.0 ** 53                       # the tie 2^53 + 1 goes to the even 2^53
    assert sx.exact(terms(2.0 ** 53, 1.0, 2.0)) == 2.0 ** 53 + 4               # 2^53 + 3 rounds up
    assert sx.exact(terms(2.0 ** 60, 1.0, -(2.0 ** 60))) == 1.0
    assert sx.exact(terms(tiny, tiny, tiny)) == 3 * tiny                        # subnormal totals are exact
    assert sx.exact(terms(2.0 ** -1023, 2.0 ** -1023)) == 2.0 ** -1022
    assert sx.exact(terms(2.0 ** -1022, -tiny)) == 2.0 ** -1022 - tiny
    assert sx.exact(terms(big, big)) == math.inf and sx.exact(terms(-big, -big)) == -math.inf
    assert sx.exact(terms(big, 2.0 ** 970)) == math.inf                        # 2^1024 - 2^970: the tie goes to the even 2^1024
    assert sx.exact(terms(big, 2.0 ** 969)) == big
    assert sx.exact(terms(big, big, -big)) == big
    for xs, sign in (((-0.0,), -1), ((-0.0, -0.0), -1), ((-0.0, 0.0), 1), ((1.0, -1.0), 1)):
        assert math.copysign(1.0, sx.exact(terms(*xs))) == sign, xs
    assert math.isnan(sx.exact(terms(math.inf, -math.inf))) and math.isnan(sx.exact(sx.Terms()))
    assert sx.check_sum(2.0 ** 53, terms(2.0 ** 53, 1.0)) == "exact"
    assert sx.check_sum(0.0, terms(2.0 ** 93, 1.0, -(2.0 ** 93))) == "bound"    # 1 is below the unit 2^(93 - 92)
    with pytest.raises(AssertionError):
        sx.check_sum(2.0 ** 53 + 2, terms(2.0 ** 53, 1.0))
    with pytest.raises(AssertionError):
        sx.check_sum(-0.0, terms(-0.0, 0.0))
    assert sx.order_free(terms(1.0, 2.0, -0.5)) and not sx.order_free(terms(2.0 ** 60, 1.0))


def test_stats_merge():
    from victorialogs_b200 import scan as vs
    a = [(0, (b"x",), 3, [(math.nan, 0), (5.0, 2)]), (1, (), 1, [(1.0, 1), (2.0, 1)])]
    b = [(0, (b"x",), 2, [(4.0, 1), (math.nan, 0)])]
    m = vs.stats_merge([a, b])
    assert m[(0, (b"x",))] == (5, [(4.0, 1), (5.0, 2)]) and m[(1, ())] == (1, [(1.0, 1), (2.0, 1)])
    m = vs.stats_merge([b, b])
    assert m[(0, (b"x",))][1][0] == (8.0, 2) and math.isnan(m[(0, (b"x",))][1][1][0])
