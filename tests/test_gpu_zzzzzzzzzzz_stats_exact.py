"""The sums of vlscan_hits_sums (`stats ... sum(v), avg(v)`, DESIGN §3.13) against an exact rational reference, and the device's number
parsers bit for bit through one-number groups.

The device writes every finite number x of a (group, field) as x / u cut toward zero to an integer, u = 2^(e - 92), e the ilogb of the largest
|x| of that (group, field), adds the integers exactly and rounds once.  So when every number is a multiple of u its sum is the correctly rounded
exact sum, bit for bit (+-Inf when that rounding overflows); otherwise |sum - exact| <= 1/2 ulp(sum) + n * u.  `terms` lists the numbers the
device adds, per row as the reference reads them (a const cell of a one-group block is one f * rows), `exact` rounds their sum once from
Python integers in units of 2^-1074, and `check_sum` applies the bound and says which of the two cases it was.  Where the reference's float
adds give one result in any order (`order_free`), the device also equals both restatements (tests/stats_model.py, and tests/vlostats.py for
oracle blocks) bit for bit.  The sum is -0 only when every term the reference adds is -0: a one-group block other than a const adds
sumValues' total, which starts at +0.

Most blocks are hand-made (float64 cells hold any 8-byte payload: subnormals, DBL_MAX, NaN and +-Inf bits), laid out twice: each case as one
one-group block, and spread over multi-group blocks with its frame in another block than its small numbers."""
import math
import random
import struct
import sys
from fractions import Fraction

import pytest

import stats_model as sm

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000_000
STEP = 10 ** 18
SCALE = 2 ** 1074                      # every double is an integer multiple of 2^-1074
DBL_MAX = sys.float_info.max
OVERFLOW = (2 ** 1024 - 2 ** 970) * SCALE   # |sum| at or above it rounds to +-Inf (the tie goes to the even 2^1024)
NAN = math.nan


# ---- the exact reference -------------------------------------------------------------------------------------------------------------------

def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or bits(a) == bits(b)


def scaled(x):
    """x * 2^1074 as an integer (x finite)"""
    p, q = x.as_integer_ratio()
    return p * (SCALE // q)


def rounded(n):
    """n * 2^-1074 rounded once to the nearest double, ties to even"""
    if abs(n) >= OVERFLOW:
        return math.inf if n > 0 else -math.inf
    return n / SCALE   # int / int true division rounds correctly, subnormals included


def ilogb(x):
    return math.frexp(x)[1] - 1


class Terms:
    """the numbers one (group, field) adds: finite ones in xs, the count, the +-Inf / NaN flags and whether the reference adds a term that is
    not -0"""
    __slots__ = ("xs", "count", "nan", "pinf", "ninf", "pos")

    def __init__(self):
        self.xs, self.count, self.nan, self.pinf, self.ninf, self.pos = [], 0, False, False, False, False

    def add(self, x):
        if math.isnan(x):
            self.nan = True
        elif math.isinf(x):
            self.pinf, self.ninf = self.pinf or x > 0, self.ninf or x < 0
        else:
            self.xs.append(x)
        self.pos = self.pos or x != 0.0 or math.copysign(1.0, x) > 0


def _whole(t, kind, payload, rows):
    """a one-group block (sumValues): a const counts rows times as one f * rows; anything else adds per row, and its total starts at +0"""
    if kind == "const":
        f, ok = sm._f64(payload)
        if ok:
            t.count += len(rows)
            t.add(f * len(rows))
        return
    before = t.count
    for r in rows:
        v = payload[r]
        if kind in ("string", "dict"):
            f, ok = sm._num(v)
            if ok and not (kind == "dict" and math.isnan(f)):
                t.count += 1
                t.add(f)
        elif kind in ("uint8", "uint16", "uint32", "uint64", "int64"):
            t.count += 1
            t.add(float(int(v)))
        elif kind == "float64":
            f = sm._cell_f64(v)
            t.count += 1
            if not math.isnan(f):
                t.add(f)
    if t.count > before:
        t.pos = True


def terms(blocks, bucket_of, by, values):
    """the inputs of stats_model.stats -> {(bucket, key texts): [Terms per value field]}"""
    out = {}
    for blk in blocks:
        rows = blk["rows"]
        if not rows:
            continue
        cols = blk["cols"]
        keys = [(bucket_of(blk["ts"][r]), tuple(sm.text(cols.get(f), r) for f in by)) for r in rows]
        cells = [cols.get(name) if name != "_time" else None for name in values]
        if all(k == keys[0] for k in keys):
            ts = out.setdefault(keys[0], [Terms() for _ in values])
            for t, col in zip(ts, cells):
                if col is not None:
                    _whole(t, col[0], col[1], rows)
            continue
        for k, r in zip(keys, rows):
            ts = out.setdefault(k, [Terms() for _ in values])
            for t, col in zip(ts, cells):
                if col is not None:
                    x, ok = sm.value_at_row(col[0], col[1], r)
                    if ok:
                        t.count += 1
                        t.add(x)
    return out


def exact(t):
    """the sum the device must return when every number is a multiple of its unit: NaN without numbers, with a NaN or with both Infs; an Inf
    as it is; else the exact sum rounded once, -0 when every term is -0"""
    if not t.count or t.nan or (t.pinf and t.ninf):
        return NAN
    if t.pinf or t.ninf:
        return math.inf if t.pinf else -math.inf
    n = sum(scaled(x) for x in t.xs)
    if n == 0:
        return 0.0 if t.pos else -0.0
    return rounded(n)


def check_sum(s, t):
    """-> "exact" or "bound" when the device's sum s obeys the contract for the terms t, else raises"""
    want = exact(t)
    nz = [scaled(x) for x in t.xs if x != 0.0]
    if math.isnan(want) or math.isinf(want) and (t.pinf or t.ninf) or not nz:
        assert same(s, want), (s, want)
        return "exact"
    k = max(ilogb(x) for x in t.xs if x != 0.0) - 92 + 1074   # u = 2^k in units of 2^-1074
    if k <= 0 or all(v % (1 << k) == 0 for v in nz):
        assert same(s, want), (s, want, s.hex(), want.hex())
        return "exact"
    n, slack = sum(nz), len(nz) << k
    if math.isinf(s):
        assert s == rounded(n + slack if s > 0 else n - slack), (s, want)
    else:
        assert not math.isnan(s) and 2 * abs(scaled(s) - n) <= scaled(math.ulp(s)) + 2 * slack, (s, want, s.hex(), want.hex())
    return "bound"


def order_free(t):
    """True when the reference's float adds give the exact sum in any order: no NaN, not both Infs, and every finite number a multiple of
    2^m with sum |x| < 2^(m + 53), so that every partial sum is a double"""
    if t.nan or (t.pinf and t.ninf):
        return False
    nz = [scaled(x) for x in t.xs if x != 0.0]
    if not nz:
        return True
    m = min((v & -v).bit_length() - 1 for v in (abs(v) for v in nz))
    return sum(abs(v) for v in nz) < 1 << (m + 53)


# ---- hand-made blocks ----------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


_TS = {}


def timestamps(oracle, rows):
    if rows not in _TS:
        _TS[rows] = oracle.Block.from_columns([("x", [b"%d" % i for i in range(rows)])]).set_timestamps([T0] * rows).timestamps_block()
    return _TS[rows]


def _lens(texts):
    w = max(len(x) for x in texts)
    if w < 256:
        return bytes([0]) + bytes(len(x) for x in texts)
    return bytes([1]) + b"".join(struct.pack(">H", len(x)) for x in texts)


WIDTH = {"uint8": ">B", "uint16": ">H", "uint32": ">I"}


def cell(vs, name, kind, payload, rows):
    """the device column of a model cell"""
    if kind == "const":
        return dict(field=name, kind="const", value=payload)
    if kind == "float64":
        data = b"".join(struct.pack(">d", x if isinstance(x, float) else float(x)) for x in payload)
        return dict(field=name, kind="values", value_type=vs.VT_FLOAT64, lens_items=bytes([4, 8]), data=data)
    if kind in WIDTH:
        fmt = WIDTH[kind]
        return dict(field=name, kind="values", value_type={"uint8": vs.VT_UINT8, "uint16": vs.VT_UINT16, "uint32": vs.VT_UINT32}[kind],
                    lens_items=bytes([4, struct.calcsize(fmt)]), data=b"".join(struct.pack(fmt, int(v)) for v in payload))
    if kind == "string":
        return dict(field=name, kind="values", value_type=vs.VT_STRING, lens_items=_lens(payload), data=b"".join(payload))
    assert kind == "dict"
    entries = sorted(set(payload))
    return dict(field=name, kind="values", value_type=vs.VT_DICT, dict=entries, lens_items=bytes([4, 1]), data=bytes(entries.index(v) for v in payload))


def block(keys, kind, payload, rows=None):
    """a model block: `keys` one key text per row (a list) or the key of every row (a const), value field v of `kind` (a const: `rows` rows
    under a const key)"""
    n = len(payload) if kind != "const" else rows if isinstance(keys, bytes) else len(keys)
    kc = ("const", keys) if isinstance(keys, bytes) else ("string", list(keys))
    return {"ts": [T0] * n, "rows": list(range(n)), "cols": {"k": kc, "v": (kind, payload)}}


def device_sums(env, blocks):
    """model blocks uploaded as hand-made cells, grouped by k on the device -> hits_sums' groups"""
    oracle, vs, pu, ctx = env
    descs = []
    for b in blocks:
        n = len(b["rows"])
        descs.append(dict(rows=n, timestamps=timestamps(oracle, n), columns=[cell(vs, name, kind, payload, n) for name, (kind, payload) in b["cols"].items()]))
    batch = ctx.upload(vs.HostBlocks(["k", "v"], descs))
    try:
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        return ctx.hits_sums(STEP, 0, 0, ("k",), ("v",))
    finally:
        batch.free()


def run(env, blocks):
    """blocks through the device grouped by k -> {key: (sum, count)}, checked against the exact bound, the terms' counts and (order-free
    groups) the model bit for bit; -> {key: mode}"""
    got = device_sums(env, blocks)
    bucket = T0 // STEP * STEP
    want = terms(blocks, lambda t: bucket, ("k",), ("v",))
    model = None
    assert sorted(want) == [(b, k) for b, k, _, _ in got]
    modes = {}
    for b, k, rows, [(s, c)] in got:
        t = want[(b, k)][0]
        assert c == t.count, (k, c, t.count)
        modes[k[0]] = check_sum(s, t)
        if order_free(t):
            model = model or sm.stats(blocks, lambda t: bucket, ("k",), ("v",))
            assert same(s, model[(b, k)].sums[0]), (k, s, model[(b, k)].sums[0])
    return modes


def layouts(cases, filler=1.0):
    """cases {key: [numbers]} -> (one one-group block per case, the same cases over multi-group blocks: the first number of a case in one
    block, the rest in another, each beside rows of a filler group)"""
    whole = [block(k, "float64", list(xs)) for k, xs in cases.items()]
    spread = []
    for k, xs in cases.items():
        spread.append(block([k, b"~filler"], "float64", [xs[0], filler]))
        if len(xs) > 1:
            keys, vals = [], []
            for i, x in enumerate(xs[1:]):
                keys.append(k)
                vals.append(x)
                if i % 3 == 0:
                    keys.append(b"~filler")
                    vals.append(filler)
            spread.append(block(keys, "float64", vals))
    return whole, spread


def run_both(env, cases, modes=None):
    whole, spread = layouts(cases)
    for blocks in (whole, spread):
        got = run(env, blocks)
        for k, m in (modes or {}).items():
            assert got[k] == m, (k, got[k], m)


# ---- digit boundaries ----------------------------------------------------------------------------------------------------------------------

FRAMES = (-1074, -1060, -1023, -1022, -1, 0, 52, 53, 63, 64, 500, 1022, 1023)
OFFSETS = (0, 30, 31, 32, 61, 62, 63, 91, 92, 93)
SIGNS = {   # sign of the term at offset j
    "plus": lambda i, j: 1,
    "high_plus_low_minus": lambda i, j: 1 if j < 31 else -1,    # the high digit sum positive, the lower ones negative, the total positive
    "high_minus_low_plus": lambda i, j: -1 if j < 31 else 1,
    "alternating": lambda i, j: -1 if i % 2 else 1,
}


def _exact_double(m, e):
    """m * 2^e when that is a double, else None"""
    x = math.ldexp(float(m), e)
    return x if x != 0.0 and x.as_integer_ratio() == Fraction(m * 2 ** e).as_integer_ratio() else None


def boundary_terms(e, sign, fits):
    """+-2^(e - j) and full-mantissa values at the same offsets for j in OFFSETS; fits: only the numbers that are multiples of 2^(e - 92)"""
    out = []
    for i, j in enumerate(OFFSETS):
        for m, low in ((1, e - j), ((1 << 53) - 1, e - j - 52)):
            if fits and low < e - 92:
                continue
            x = _exact_double(m, low)
            if x is not None:
                out.append(SIGNS[sign](i, j) * x)
    if not fits and _exact_double(1, e - 93):
        out.append(SIGNS[sign](0, 99) * math.ldexp(1.0, e - 93))
    return out


def test_digit_boundaries(env):
    cases, modes = {}, {}
    for e in FRAMES:
        for sign in SIGNS:
            for fits in (True, False):
                xs = boundary_terms(e, sign, fits)
                key = b"e%d-%s-%s" % (e, sign.encode(), b"fits" if fits else b"cut")
                assert max(ilogb(abs(x)) for x in xs) == e
                cases[key] = xs
                below = any(x % math.ldexp(1.0, e - 92) for x in xs) if e - 92 >= -1074 else False
                modes[key] = "bound" if below else "exact"
    assert sum(m == "bound" for m in modes.values()) >= 30 and sum(m == "exact" for m in modes.values()) >= 60
    run_both(env, cases, modes)


# ---- cancellation, range, overflow -----------------------------------------------------------------------------------------------------------

def test_cancellation_and_range(env):
    tiny = math.ldexp(1.0, -1074)
    cases = {
        b"cancel-10": [2.0 ** 10, 1.0, -2.0 ** 10],
        b"cancel-60": [2.0 ** 60, 1.0, -2.0 ** 60],      # exact 1 on the device, 0 in the reference's row order
        b"cancel-92": [2.0 ** 92, 1.0, -2.0 ** 92],
        b"cancel-93": [2.0 ** 93, 1.0, -2.0 ** 93],      # 1 is below the unit 2: cut to 0
        b"span": [1.0, 2.0 ** -100, -(2.0 ** -150), 2.0 ** -200, 3.0 * 2.0 ** -60],
        b"tie-2^53": [2.0 ** 53, 1.0],
        b"tie-2^53-up": [2.0 ** 53, 1.0, 2.0],
        b"subnormals": [tiny, 3 * tiny, math.ldexp(1.0, -1030), -math.ldexp(5.0, -1060), math.ldexp(1.0, -1023) - tiny],
        b"subnormals-to-normal": [math.ldexp(1.0, -1023), math.ldexp(1.0, -1023), tiny],
        b"subnormal-cancel": [tiny, -tiny, math.ldexp(1.0, -1050), -math.ldexp(1.0, -1050)],
        b"max+max": [DBL_MAX, DBL_MAX],
        b"-max-max": [-DBL_MAX, -DBL_MAX],
        b"max+max-max": [DBL_MAX, DBL_MAX, -DBL_MAX],    # the reference's order overflows to +Inf first
        b"max+half-ulp": [DBL_MAX, 2.0 ** 970],          # the tie at 2^1024 - 2^970 rounds to +Inf
        b"max+quarter-ulp": [DBL_MAX, 2.0 ** 969],
        b"near-2^1024": [2.0 ** 1023, 2.0 ** 1022, 2.0 ** 1021, -(2.0 ** 970)],
    }
    modes = {k: "exact" for k in cases}
    modes[b"cancel-93"] = modes[b"span"] = "bound"
    run_both(env, cases, modes)
    t = Terms()
    t.count = 3
    for x in cases[b"max+max-max"]:
        t.add(x)
    assert exact(t) == DBL_MAX
    g = sm.stats([block(b"a", "float64", cases[b"max+max-max"])], lambda ts: 0, ("k",), ("v",))[(0, (b"a",))]
    assert g.sums == [math.inf]
    assert exact_of([DBL_MAX, 2.0 ** 970]) == math.inf and exact_of([DBL_MAX, 2.0 ** 969]) == DBL_MAX


def exact_of(xs):
    t = Terms()
    t.count = len(xs)
    for x in xs:
        t.add(x)
    return exact(t)


def test_const_cells(env):
    """a const of a one-group block is one f * rows; elsewhere one f per row.  tryParseFloat64 takes at most 27 characters, so no const
    reaches a product that overflows: "1e308" is no number there"""
    consts = [(b"c-big", b"99999999999999999999999999", 7), (b"c-neg", b"-12345678901234567890.5", 3), (b"c-1e308", b"1e308", 4),
              (b"c-frac", b"0.1", 5), (b"c-2^53", b"9007199254740993", 3)]
    whole = [block(k, "const", v, rows=n) for k, v, n in consts]
    spread = [block([k, b"~z"] * n, "const", v) for k, v, n in consts]
    for blocks in (whole, spread):
        modes = run(env, blocks)
        assert {modes[k] for k, _, _ in consts} == {"exact"}


# ---- NaN, Inf and signed zeros -------------------------------------------------------------------------------------------------------------

def _nan(payload):
    return struct.unpack(">d", struct.pack(">Q", payload))[0]


def test_special_values(env):
    qnan, snan, nnan = _nan(0x7FF8000000000000), _nan(0x7FF0000000000001), _nan(0xFFF8000000000123)
    inf = math.inf
    cases = {
        b"nan": [1.0, qnan, 2.0],
        b"nans-only": [snan, nnan],
        b"+inf": [1.0, inf, -5.0],
        b"-inf": [-inf, 3.0],
        b"+inf-inf": [inf, 1.0, -inf],
        b"inf-nan": [inf, qnan],
        b"max+inf": [DBL_MAX, DBL_MAX, inf],
    }
    run_both(env, cases)
    # NaN rows count in a one-group block only
    modes = run(env, [block(b"n1", "float64", [qnan, 1.0, snan]), block([b"n2", b"n2", b"n3"], "float64", [qnan, 1.0, nnan])])
    assert modes == {b"n1": "exact", b"n2": "exact", b"n3": "exact"}


def test_signed_zeros(env):
    nz = -0.0
    modes = run(env, [
        block([b"rows-neg", b"z"], "float64", [nz, 1.0]),                  # a row-path -0 alone: -0
        block([b"rows-neg2", b"z", b"rows-neg2"], "float64", [nz, 1.0, nz]),
        block([b"rows-neg2", b"z"], "float64", [nz, 2.0]),
        block([b"rows-mixed", b"rows-mixed", b"z"], "float64", [nz, 0.0, 1.0]),   # -0 + +0: +0
        block([b"rows-cancel", b"rows-cancel", b"z"], "float64", [1.5, -1.5, 1.0]),   # exact cancellation: +0
        block(b"whole-f64", "float64", [nz, nz]),                          # sumValues starts at +0: +0
        block(b"whole-str", "string", [b"-0", b"-0.0", b"x"]),
        block(b"whole-dict", "dict", [b"-0", b"x", b"-0"]),
        block(b"whole-u8", "uint8", [b"0", b"0"]),
        block(b"const-neg", "const", b"-0", rows=3),                               # f * rows of -0: -0
        block([b"const-rows", b"z2"], "const", b"-0"),                     # per row: -0 for each group
        block([b"str-rows", b"z"], "string", [b"-0", b"7"]),
        block([b"mix-const", b"mix-const"], "const", b"-0"),
        block([b"mix-const", b"z"], "float64", [0.0, 1.0]),
    ])
    assert set(modes.values()) == {"exact"}


def test_signed_zeros_against_both_restatements(env):
    """the oracle's own blocks: a "-0" text read row by row, a const "-0" (f * rows) and a "-0" in a one-group string block"""
    import stats_cases as sc
    import vlostats
    oracle, vs, pu, ctx = env
    cols = [{"k": [b"a", b"b"], "v": [b"-0", b"x"]}, {"k": [b"c", b"c"], "v": [b"-0", b"-0"]}, {"k": [b"d"] * 10, "v": [b"-0"] + [b"x%d" % i for i in range(9)]},
            {"k": [b"e", b"f", b"e"], "v": [b"-0", b"y", b"-0.0"]}]
    blocks = [oracle.Block.from_columns(list(c.items())).set_timestamps([T0] * len(c["k"])) for c in cols]
    kinds = [{c.name: c.value_type for c in b.columns}.get(b"v") for b in blocks]
    assert kinds[0] in (1, 2) and kinds[1] is None and kinds[2] == 1, kinds   # strings / dict, const, strings
    got = _device_groups(env, blocks)
    bucket = T0 // STEP * STEP
    cpp = vlostats.stats(blocks, oracle.Filter.noop(), STEP, 0, 0, ("k",), ("v",))
    model = sc.model_groups(oracle, [(b, c, [T0] * len(c["k"])) for b, c in zip(blocks, cols)], oracle.Filter.noop(), STEP, 0, 0, ("k",), ("v",))
    want = {b"a": -0.0, b"c": -0.0, b"d": 0.0, b"e": -0.0}
    for k, w in want.items():
        s = got[k][0]
        assert same(s, w) and same(cpp[(bucket, (k,))][1][0][0], w) and same(model[(bucket, (k,))][1][0][0], w), (k, s)


# ---- large groups --------------------------------------------------------------------------------------------------------------------------

def test_large_group_digit_sums(env):
    """2^20 numbers per group, each a multiple of u = 2^(E - 92): the high digit of one kind, the low and middle digits of others, so that every
    digit sum reaches 2^45 in magnitude, one with the total's sign and one against it; half the rows in one-group blocks, half row by row"""
    rng = random.Random(7)
    E, n, per = 200, 1 << 20, 1 << 16
    unit = E - 92
    groups = {}
    for key, sgn in ((b"big+", 1), (b"big-", -1)):
        vs_ = []
        for i in range(n):
            m = rng.randrange(1 << 52, 1 << 53)
            kind = i % 3
            v = m << 40 if kind == 0 else -m if kind == 1 else (m << 20) * rng.choice((1, -1))
            vs_.append(sgn * v)
        trunc = lambda v, s: abs(v) >> s if v >= 0 else -(abs(v) >> s)
        d0 = sum(trunc(v, 62) for v in vs_)
        d1 = sum(trunc(v - (trunc(v, 62) << 62), 31) for v in vs_)
        d2 = sum(v - (trunc(v, 31) << 31) for v in vs_)
        assert min(abs(d0), abs(d1), abs(d2)) >= 2 ** 45 and sgn * d0 > 0 and sgn * d2 < 0, (d0, d1, d2)
        groups[key] = [math.ldexp(float(v), unit) for v in vs_]
    blocks = []
    for key, xs in groups.items():
        half = len(xs) // 2
        for o in range(0, half, per):
            blocks.append(block(key, "float64", xs[o:o + per]))
        for o in range(half, len(xs), per):
            part = xs[o:o + per]
            blocks.append(block([key] * (len(part) - 1) + [b"~z"], "float64", part))   # the last row in another group
    modes = run(env, blocks)
    assert modes[b"big+"] == modes[b"big-"] == "exact"


# ---- small unsigned integers ---------------------------------------------------------------------------------------------------------------

def test_small_uints_bit_for_bit(env):
    rng = random.Random(11)
    blocks = []
    for kind, hi in (("uint8", 255), ("uint16", 65535), ("uint32", 4294967295)):
        for n in (1, 2, 63, 300, 5000):
            blocks.append(block(b"%s-%d" % (kind.encode(), n), kind, [b"%d" % rng.randrange(hi + 1) for _ in range(n - 1)] + [b"%d" % hi]))
    modes = run(env, blocks)
    assert set(modes.values()) == {"exact"} and len(modes) == 15


# ---- the device's number parsers -----------------------------------------------------------------------------------------------------------

def parser_texts():
    import test_mathnum_cpu as tm
    rng = random.Random(20261017)
    out = [s.encode("utf-8", "surrogateescape") for s in tm.FIXED]
    out += [tm.random_text(rng).encode("utf-8", "surrogateescape") for _ in range(3000)]
    seen, uniq = set(), []
    for s in out:
        if s not in seen and not s.startswith(b"~"):
            seen.add(s)
            uniq.append(s)
    return uniq


FILL = [b"~f%d" % i for i in range(9)]   # no number under either parser


def _device_groups(env, blocks):
    oracle, vs, pu, ctx = env
    batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    got = ctx.hits_sums(STEP, 0, 0, ("k",), ("v",))
    batch.free()
    return {k[0]: v[0] for _, k, _, v in got}


def _parity(env, blocks, cols, want):
    """device vs the parser (want {key: (sum, count)}) and vs both restatements, bit for bit"""
    import stats_cases as sc
    import vlostats
    oracle = env[0]
    got = _device_groups(env, blocks)
    bucket = T0 // STEP * STEP
    cpp = vlostats.stats(blocks, oracle.Filter.noop(), STEP, 0, 0, ("k",), ("v",))
    model = sc.model_groups(oracle, [(b, c, [T0] * len(c["k"])) for b, c in zip(blocks, cols)], oracle.Filter.noop(), STEP, 0, 0, ("k",), ("v",))
    bad = []
    for k, (ws, wc) in want.items():
        s, c = got[k]
        ms, mc = model[(bucket, (k,))][1][0]
        cs, cc = cpp[(bucket, (k,))][1][0][:2]
        if not (c == wc == mc == cc and same(s, ws) and same(ms, ws) and same(cs, ws)):
            bad.append((k, (s, c), (ws, wc), (ms, mc), (cs, cc)))
    assert not bad, bad[:10]


def _value_kinds(blocks):
    return {{c.name: c.value_type for c in b.columns}.get(b"v") for b in blocks}


def test_parser_row_path(env):
    """one row per group in multi-group blocks: getFloatValueAtRow's tryParseFloat64 (the device's parse_f64_internal)"""
    import vlostats
    oracle = env[0]
    texts = parser_texts()
    blocks, cols, want = [], [], {}
    for o in range(0, len(texts), 500):
        part = texts[o:o + 500]
        c = {"k": [b"r%05d" % (o + i) for i in range(len(part))], "v": part}
        blocks.append(oracle.Block.from_columns(list(c.items())).set_timestamps([T0] * len(part)))
        cols.append(c)
        for k, s in zip(c["k"], part):
            x, ok = vlostats.try_parse_float64(s)
            want[k] = (x, 1) if ok else (NAN, 0)
    assert _value_kinds(blocks) == {1}
    assert sum(c for _, c in want.values()) > 250 and sum(c == 0 for _, c in want.values()) > 2000
    _parity(env, blocks, cols, want)


def test_parser_one_group_strings(env):
    """one number per one-group block of strings: sumValues' tryParseNumber (the device's parse_number), added to sumValues' +0"""
    import vlostats
    oracle = env[0]
    blocks, cols, want = [], [], {}
    for i, s in enumerate(parser_texts()):
        c = {"k": [b"s%05d" % i] * 10, "v": [s] + FILL}
        blocks.append(oracle.Block.from_columns(list(c.items())).set_timestamps([T0] * 10))
        cols.append(c)
        x, ok = vlostats.try_parse_number(s)
        want[c["k"][0]] = (0.0 + x, 1) if ok else (NAN, 0)
    assert _value_kinds(blocks) == {1}
    assert sum(c for _, c in want.values()) > 1000
    _parity(env, blocks, cols, want)


def test_parser_dict_cells(env):
    """the same through dict cells: tryParseNumber per entry in one-group blocks (an entry that is no number, here ~f0, is NaN and none),
    tryParseFloat64 of the entry row by row"""
    import vlostats
    oracle = env[0]
    blocks, cols, want = [], [], {}
    for i, s in enumerate(parser_texts()):
        pair = [({"k": [b"w%05d" % i] * 3, "v": [s, FILL[0], s]}), {"k": [b"p%05d" % i, b"q%05d" % i], "v": [s, FILL[0]]}]
        made = [oracle.Block.from_columns(list(c.items())).set_timestamps([T0] * len(c["k"])) for c in pair]
        if _value_kinds(made) != {2}:   # a text too long for a dictionary
            continue
        blocks += made
        cols += pair
        x, ok = vlostats.try_parse_number(s)
        want[b"w%05d" % i] = (0.0 + x + x, 2) if ok and not math.isnan(x) else (NAN, 0)
        x, ok = vlostats.try_parse_float64(s)
        want[b"p%05d" % i] = (x, 1) if ok else (NAN, 0)
        want[b"q%05d" % i] = (NAN, 0)
    assert _value_kinds(blocks) == {2} and len(blocks) > 2 * 3000
    _parity(env, blocks, cols, want)
