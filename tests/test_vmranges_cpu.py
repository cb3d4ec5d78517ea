"""`histogram(v)` without a device: the host build of the kernels' vmrange mapping (vlscan_vmrange_index) against the Python restatement of
Histogram.Update (tests/vmrange_model.py) at every bucket boundary and around it, at powers of ten, special values and a million seeded
doubles; the vmrange texts and their independence from how Pow(10, 1/18) rounds; the reference's TestStatsHistogram JSON; the C++ restatement
(tests/vmrange_oracle) against the Python one on random blocks of every column kind; the merge; the ABI's argument errors."""
import ctypes as C
import json
import math
import os
import random

import numpy as np
import pytest

import vlovmrange
import vmrange_model as vm
from victorialogs_b200 import scan as vs

HERE = os.path.dirname(os.path.abspath(__file__))


def model_bounds():
    """bound k - 1: the least double whose model index reaches k, by bisection on the bit patterns"""
    out = []
    for k in range(1, vm.VMRANGES):
        lo, hi = 0, 0x7FF0000000000000
        while hi - lo > 1:
            m = (lo + hi) // 2
            if vm.vmrange_index(vm.f64_of_bits(m)) >= k:
                hi = m
            else:
                lo = m
        out.append(hi)
    return out


@pytest.fixture(scope="module")
def bounds():
    return model_bounds()


def test_index_at_every_boundary(bounds):
    assert len(set(bounds)) == vm.VMRANGES - 1
    for k, u in enumerate(bounds):
        for d in range(-64, 65):
            x = vm.f64_of_bits(u + d)
            want = vm.vmrange_index(x)
            assert want == (k + 1 if d >= 0 else k) or d not in (-1, 0), (k, d)
            assert vs.vmrange_index(x) == want, (k, d, x)
            if abs(d) <= 2:
                assert vlovmrange.index(x) == want, (k, d, x)


def test_boundaries_differ_from_correct_rounding(bounds):
    """Go's Log puts hundreds of boundaries off where a correctly rounded log10 would: the mapping must follow Go, not libm"""
    def libm_index(v):
        b = (math.log10(v) + 9) * 18
        if b < 0:
            return 0
        if b >= 486:
            return 487
        i = int(b)
        if b == i and i > 0:
            i -= 1
        return i + 1
    off = sum(1 for k, u in enumerate(bounds) if libm_index(vm.f64_of_bits(u)) != k + 1 or libm_index(vm.f64_of_bits(u - 1)) != k)
    assert off == 429, off


def test_index_powers_of_ten_and_specials():
    vals = [10.0 ** n for n in range(-12, 21)] + [float("1e%d" % n) for n in range(-12, 21)]
    vals += [0.0, -0.0, 5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308, math.inf, -math.inf, math.nan, -1.0, -5e-324, -1e300,
             1e-9, 1e18, 1.8446744073709552e19, 1.7976931348623157e308]
    for x in vals:
        assert vs.vmrange_index(x) == vm.vmrange_index(x) == vlovmrange.index(x), x
    assert vs.vmrange_index(1e-9) == 1 and vs.vmrange_index(1e18) == 487 and vs.vmrange_index(math.inf) == 487
    assert vs.vmrange_index(-0.0) == 0 and vs.vmrange_index(0.0) == 0 and vs.vmrange_index(5e-324) == 0
    assert vs.vmrange_index(math.nan) == -1 and vs.vmrange_index(-5e-324) == -1
    assert vs.vmrange_index(1.0) == 162 and vm.vmrange_text(162) == "8.799e-01...1.000e+00"   # 10^n: the bucket whose upper end it is


def test_index_seeded_doubles():
    rng = np.random.default_rng(20261019)
    a = 10.0 ** rng.uniform(-12, 20, 500_000)
    b = rng.integers(0, 0x7FF0000000000000, 500_000, dtype=np.uint64).view(np.float64)
    for x in np.concatenate([a, b]).tolist():
        assert vs.vmrange_index(x) == vm.vmrange_index(x), x


def test_texts():
    want = vm.vmrange_texts()
    got = [vs.vmrange_text(i) for i in range(vm.VMRANGES)]
    assert got == want
    assert got[0] == "0...1.000e-09" and got[1] == "1.000e-09...1.136e-09" and got[-1] == "1.000e+18...+Inf" and got[-2].endswith("...1.000e+18")
    for i in range(1, vm.VMRANGES - 1):   # ascending, adjacent
        assert got[i].split("...")[0] == got[i - 1].split("...")[1]
    with pytest.raises(ValueError):
        vs.vmrange_text(vm.VMRANGES)


def test_texts_do_not_depend_on_pow_rounding():
    m = vm.bits_of_f64(vm.bucket_multiplier())
    want = vm.vmrange_texts()
    for d in range(-16, 17):
        assert vm.vmrange_texts(vm.f64_of_bits(m + d)) == want, d


def test_reference_table():
    cases = json.load(open(os.path.join(HERE, "golden", "histogram_cases.json")))
    assert len(cases) == 1
    for case in cases:
        assert case["query"] == "stats histogram(a) as x"
        st = {}
        for row in case["rows"]:
            for name, value in row:
                if name == "a":
                    x, ok = vlovmrange.parse_number(value)
                    if ok:
                        vm.update(st, x)
        assert vm.finalize(st) == case["expected"][0][0][1]
    assert vm.finalize({}) == "]"


def test_less_natural_orders_the_texts():
    texts = [t.encode() for t in vm.vmrange_texts()]
    assert vm.less_natural(b"1.896e+00...2.154e+00", b"2.783e+00...3.162e+00")
    assert vm.less_natural(b"1.000e+00...1.136e+00", b"2.154e-01...2.448e-01")   # mantissas first: not numeric order
    assert vm.less_natural(b"1.000e+00...1.136e+00", b"1.000e-09...1.136e-09")   # "+" sorts before "-"
    assert not any(vm.less_natural(t, t) for t in texts)


def model_number(col, r):
    """stats_histogram.go's number of row r of a generated column -> (x, ok)"""
    kind, texts = col
    if kind in ("ipv4", "iso8601"):
        return 0.0, False
    return vlovmrange.parse_number(texts if kind == "const" else texts[r])


VT_NAMES = {1: "string", 2: "dict", 3: "uint8", 4: "uint16", 5: "uint32", 6: "uint64", 7: "float64", 8: "ipv4", 9: "iso8601", 10: "int64"}


def random_blocks(oracle, seed):
    import parity_util as pu
    rng = random.Random(seed)
    pool = {
        "u8": lambda i: b"%d" % (i % 200), "u32": lambda i: b"%d" % (i * 100003 % 4000000000), "u64": lambda i: b"%d" % (2 ** 64 - 1 - i),
        "i64": lambda i: b"%d" % ((i - 50) * 12345678901), "f64": lambda i: b"%d.%d" % (i - 40, 1 + i % 9), "ip": lambda i: b"1.2.3.%d" % (i % 256),
        "iso": lambda i: b"2024-01-%02dT00:00:%02d.%03dZ" % (1 + i % 28, i % 60, i % 1000),
        "s": lambda i: [b"5s", b"1KiB", b"x", b"7", b"1_000", b"-2.5", b"0x10", b"", b"NaN", b"-0", b"1e-9", b"1e18", b"Inf"][i % 13],
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
        blocks.append((blk, pu.oracle_block_to_desc(blk), cols, ts))
    return blocks


def test_restatements_agree_on_random_blocks(oracle):
    values = ["u8", "u32", "u64", "i64", "f64", "ip", "iso", "s", "d", "c", "nope", "_time"]
    blocks = random_blocks(oracle, 3)
    seen = set()
    for step, by in ((10 ** 18, ()), (10 ** 10, ("k",))):
        words = [b.search(oracle.Filter.noop()) for b, _, _, _ in blocks]
        got = vlovmrange.vmranges([d for _, d, _, _ in blocks], words, step, 0, 0, by, None, values)
        want = {}
        for blk, desc, cols, ts in blocks:
            kinds = {c["field"] if isinstance(c["field"], str) else c["field"].decode(): ("const" if c["kind"] == "const" else VT_NAMES[c["value_type"]])
                     for c in desc["columns"]}
            seen.update(kinds.values())
            for r in range(blk.rows):
                key = (ts[r] // step * step, tuple(cols[f][r] for f in by))
                rows, vals = want.setdefault(key, (0, [{} for _ in values]))
                for f, name in enumerate(values):
                    if name in cols and name != "_time":
                        x, ok = model_number((kinds[name], cols[name][0] if kinds[name] == "const" else cols[name]), r)
                        if ok:
                            vm.update(vals[f], x)
                want[key] = (rows + 1, vals)
        assert got == want
    assert seen >= {"const", "string", "dict", "uint8", "uint32", "uint64", "int64", "float64", "ipv4", "iso8601"}, seen


def test_merge_of_random_splits():
    rng = random.Random(5)
    for _ in range(20):
        states = []
        whole = {}
        for _ in range(rng.randint(1, 5)):
            st = []
            for g in range(rng.randint(0, 4)):
                vals = [{rng.randrange(488): rng.randint(1, 9) for _ in range(rng.randint(0, 3))} for _ in range(2)]
                rows = rng.randint(1, 50)
                st.append((g, (b"k",), rows, vals))
                r0, v0 = whole.get((g, (b"k",)), (0, [{}, {}]))
                whole[(g, (b"k",))] = (r0 + rows, [vm.merge(a, b) for a, b in zip(v0, vals)])
            states.append(st)
        assert vs.vmranges_merge(states) == whole


def test_struct_layout_and_argument_errors():
    L = vs.lib()
    assert vs.VMRANGES == 488
    buf = C.create_string_buffer(64)
    assert L.vlscan_vmrange_text(0, buf, 12) == -1 and L.vlscan_vmrange_text(0, buf, 13) == 13 and L.vlscan_vmrange_text(488, buf, 64) == -2
    info = (C.c_uint64 * 6)(*([7] * 6))
    q, keep = vs.hits_query(3600 * 10 ** 9)
    names = (C.c_char_p * 1)(b"v")
    lens = (C.c_size_t * 1)(1)
    # no device ctx: a loud failure, never a CPU fallback; out_info zeroed
    rc = L.vlscan_hits_vmranges(None, C.byref(q), None, names, lens, 1, None, None, 0, None, 0, None, None, None, None, 0, info)
    assert rc != 0 and list(info) == [0] * 6
    assert b"CUDA device" in L.vlscan_last_error(None)
    rc = L.vlscan_hits_vmranges(None, C.byref(q), None, names, lens, 0, None, None, 0, None, 0, None, None, None, None, 0, info)
    assert rc != 0 and b"no value fields" in L.vlscan_last_error(None)
    star, lens2 = (C.c_char_p * 1)(b"a*"), (C.c_size_t * 1)(2)
    rc = L.vlscan_hits_vmranges(None, C.byref(q), None, star, lens2, 1, None, None, 0, None, 0, None, None, None, None, 0, info)
    assert rc != 0 and b"histogram(foo*)" in L.vlscan_last_error(None)
    five = (C.c_char_p * 5)(*[b"v"] * 5)
    lens5 = (C.c_size_t * 5)(*[1] * 5)
    rc = L.vlscan_hits_vmranges(None, C.byref(q), None, five, lens5, 5, None, None, 0, None, 0, None, None, None, None, 0, info)
    assert rc != 0 and b"too many value fields for vlscan_hits_vmranges" in L.vlscan_last_error(None)
