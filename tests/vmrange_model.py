"""Python restatement of `histogram(v)` (lib/logstorage/stats_histogram.go) and of the metrics.Histogram parts it uses
(github.com/VictoriaMetrics/metrics histogram.go): Update's index, initBucketRanges' texts, finalizeStats' JSON and the merge of states.
Python floats are IEEE doubles rounded like Go's float64 operations, so the index is computed from the formula, step by step, with Go's
portable math.Log (math/log.go) restated below; the engine's boundary table is not used here.
"""
import math
import struct

VMRANGES = 488
# math/log.go
LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
L1, L2, L3, L4 = 6.666666666666735130e-01, 3.999999999940941908e-01, 2.857142874366239149e-01, 2.222219843214978396e-01
L5, L6, L7 = 1.818357216161805012e-01, 1.531383769920937332e-01, 1.479819860511658591e-01
SQRT2_HALF = 0.70710678118654752440
INV_LN10 = float.fromhex("0x1.bcb7b1526e50ep-2")   # 1 / Ln10, the untyped constant rounded once


def go_log(x):
    if math.isnan(x) or x == math.inf:
        return x
    if x < 0:
        return math.nan
    if x == 0:
        return -math.inf
    f1, ki = math.frexp(x)
    if f1 < SQRT2_HALF:
        f1 *= 2
        ki -= 1
    f = f1 - 1
    k = float(ki)
    s = f / (2 + f)
    s2 = s * s
    s4 = s2 * s2
    t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)))
    t2 = s4 * (L2 + s4 * (L4 + s4 * L6))
    R = t1 + t2
    hfsq = 0.5 * f * f
    return k * LN2_HI - ((hfsq - (s * (hfsq + R) + k * LN2_LO)) - f)


def vmrange_index(v):
    """Histogram.Update: -1 for a skipped number (NaN, v < 0), 0 lower, 1 + bucket index, 487 upper"""
    if math.isnan(v) or v < 0:
        return -1
    b = (go_log(v) * INV_LN10 - (-9)) * 18
    if b < 0:
        return 0
    if b >= 486:
        return VMRANGES - 1
    idx = int(b)
    if b == float(idx) and idx > 0:
        idx -= 1
    return idx + 1


def _e3(v):
    return "%.3e" % v   # Go's %.3e: exact decimal rounding, at least two exponent digits


def bucket_multiplier():
    return 10 ** (1 / 18)


def vmrange_texts(multiplier=None):
    """lowerBucketRange, bucketRanges (initBucketRanges), upperBucketRange, by index"""
    m = bucket_multiplier() if multiplier is None else multiplier
    v = 1e-9
    out = ["0..." + _e3(v)]
    for _ in range(486):
        start = _e3(v)
        v *= m
        out.append(start + "..." + _e3(v))
    out.append(_e3(1e18) + "...+Inf")
    return out


_TEXTS = None


def vmrange_text(index):
    global _TEXTS
    if _TEXTS is None:
        _TEXTS = vmrange_texts()
    return _TEXTS[index]


def update(state, v):
    """Histogram.Update into {index: hits}"""
    i = vmrange_index(v)
    if i >= 0:
        state[i] = state.get(i, 0) + 1


def merge(a, b):
    """statsHistogramProcessor.mergeState: hits add"""
    out = dict(a)
    for i, h in b.items():
        out[i] = out.get(i, 0) + h
    return out


def less_natural(a, b):
    """stringsutil.LessNatural over bytes, transcribed step by step"""
    rev = False
    while True:
        if len(a) > len(b):
            a, b = b, a
            rev = not rev
        i = 0
        while i < len(a):
            ca, cb = a[i], b[i]
            if 48 <= ca <= 57:
                if 48 <= cb <= 57:
                    break
                return not rev
            if 48 <= cb <= 57:
                return rev
            if ca != cb:
                return cb < ca if rev else ca < cb
            i += 1
        a, b = a[i:], b[i:]
        if not a:
            return False if rev else len(b) > 0
        nums = []
        for s in (a, b):
            j, n = 1, s[0] - 48
            while j < len(s) and 48 <= s[j] <= 57:
                if n > (2 ** 64 - 1 - 9) // 10:
                    return b < a if rev else a < b
                n = n * 10 + s[j] - 48
                j += 1
            nums.append((n, j))
        (na, ia), (nb, ib) = nums
        if na != nb:
            return nb < na if rev else na < nb
        if ia != ib:
            return ib < ia if rev else ia < ib
        a, b = a[ia:], b[ib:]


def finalize(state):
    """finalizeStats: the JSON of {index: hits}, vmranges ordered by LessNatural"""
    import functools
    names = {vmrange_text(i).encode(): h for i, h in state.items() if h}
    order = sorted(names, key=functools.cmp_to_key(lambda x, y: -1 if less_natural(x, y) else (1 if less_natural(y, x) else 0)))
    if not order:
        return "]"   # dst[:len(dst)-1] drops the '[' when there is no bucket
    return "[" + ",".join('{"vmrange":"%s","hits":%d}' % (r.decode(), names[r]) for r in order) + "]"


def f64_of_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def bits_of_f64(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]
