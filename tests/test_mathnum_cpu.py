"""Host build of the device's parseMathNumber (victorialogs_b200/csrc/vl_mathnum.cuh, exported as vlscan_parse_math_number) against the
oracle's restatement (oracle/vlo_mathnum.h, which leans on strtod for the strconv.ParseFloat part): bit-for-bit equal doubles on the value
syntaxes of filter_range_test.go / filter_le_field_test.go, on hand-picked rounding cases (halfway, denormal, overflow, long digit strings) and
on seeded random strings of every form the function knows."""
import math
import random
import struct

from victorialogs_b200 import scan as vs


def bits(f):
    return struct.unpack("<Q", struct.pack("<d", f))[0]


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or bits(a) == bits(b)


FIXED = ["", "0", "-0", "1", "-1", "123", "1_000", "1__0", "_1", "1_", "00", "01", "0.5", "-0.5", ".5", "5.", "1.2.3", "10.20.30.40", "256.1.1.1", "1.1.1.1", "255.255.255.255",
         "1e5", "1E5", "1e+5", "1e-5", "1.5e300", "1e308", "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1e309", "2e308", "4.9e-324", "2.4703282292062327e-324",
         "2.4703282292062328e-324", "5e-324", "1e-400", "0e999", "9007199254740993", "9007199254740992.5", "9007199254740993.0e0", "0.1", "0.2", "0.30000000000000004", "123456789012345678901234567890",
         "1" + "0" * 400, "0." + "0" * 400 + "1", "1." + "0" * 900 + "1e5", "8.98846567431158e307", "2.2250738585072011e-308", "2.2250738585072014e-308", "+5", "+.5", "-.5e1", "+inf", "-inf", "inf", "Infinity",
         "-INFINITY", "infinit", "nan", "NaN", "0x10", "0X1F", "0x1p3", "0x1.8p1", "0x.8p0", "0x1p-1074", "0x1p-1075", "0x1.0000000000000800p0", "0x1.00000000000008p0", "0x1.00000000000018p0", "0x1p1024", "0x1p1023",
         "0x", "0xg", "0b101", "0o17", "017", "08", "0x_1", "0_1", "1_000.5", "1_0e1_0", "1e", "e5", "1e5x", "--1", "1-", "1h", "1h30m", "1.5h", "-2d", "1w", "1y", "5ms", "5µs", "5ns", "5us", "1h5", "h", "1KB", "1KiB",
         "1.5MiB", "10GB", "1TiB", "1.5", "1.5K", "1K5", "5B", "1KB2MB", "1.1B", "2024-03-05T12:04:28Z", "2024-03-05T12:04:28.123456789Z", "2024-03-05 12:04:28", "2024-03-05T12:04:28+02:00",
         "2024-03-05T12:04:28.5-07:30", "2024-03-05T12:04:28.1234567890Z", "1677-01-01T00:00:00Z", "2262-12-31T23:59:59Z", "2263-01-01T00:00:00Z", "2024-13-45T25:61:61Z", "2024-03-05T12:04:28+25:00",
         "2024-03-05T12:04", "10.0.0.7", "1.2.3", "1.2.3.4.5", "999.1.1.1", "1.1.1.1a", "abc", " 1", "1 ", "18446744073709551615", "18446744073709551616", "-9223372036854775808", "9223372036854775807",
         "9223372036854775808", "0x7fffffffffffffff", "0x8000000000000000", "-0x8000000000000000", "1" * 27, "1" * 28, "0." + "1" * 25, "99999999999999999999999999.5", "1e23", "8.5e22", "6.02214076e23"]


def test_fixed_cases(oracle):
    for s in FIXED:
        a, b = vs.parse_math_number(s), oracle.lib().vlo_parse_math_number(s.encode(), len(s.encode()))
        assert same(a, b), (s, a, b)


def test_reference_table_values(oracle):
    """every column value of filter_range_test.go and filter_le_field_test.go"""
    from golden_util import load_filter_cases
    seen = set()
    for c in load_filter_cases("filter_cases_next.json"):
        if c["filter"]["kind"] not in ("range", "le_field"):
            continue
        for _, vals in c["columns"]:
            seen.update(vals)
    assert len(seen) > 50
    for v in sorted(seen):
        a, b = vs.parse_math_number(v), oracle.lib().vlo_parse_math_number(v, len(v))
        assert same(a, b), (v, a, b)


def random_text(rng):
    """one seeded string of a form the number parsers know (or nearly do)"""
    k = rng.randrange(12)
    d = lambda n: "".join(rng.choice("0123456789") for _ in range(n))
    if k == 0:
        return d(rng.randrange(1, 25))
    if k == 1:
        return rng.choice(["", "-", "+"]) + d(rng.randrange(0, 20)) + "." + d(rng.randrange(0, 20))
    if k == 2:
        return rng.choice(["", "-", "+"]) + d(rng.randrange(1, 22)) + rng.choice(["", "." + d(rng.randrange(1, 22))]) + rng.choice("eE") + rng.choice(["", "-", "+"]) + d(rng.randrange(1, 4))
    if k == 3:   # near the limits of the exponent range
        return d(rng.randrange(1, 19)) + "e" + str(rng.choice([-330, -325, -324, -323, -310, -308, 300, 305, 307, 308, 309]) - rng.randrange(0, 18))
    if k == 4:   # long digit strings: rounding far beyond 17 digits
        return d(rng.randrange(17, 60)) + rng.choice(["", "." + d(rng.randrange(1, 40))]) + rng.choice(["", "e" + str(rng.randrange(-40, 40))])
    if k == 5:
        h = lambda n: "".join(rng.choice("0123456789abcdefABCDEF") for _ in range(n))
        return rng.choice(["", "-"]) + "0x" + h(rng.randrange(0, 18)) + rng.choice(["", "." + h(rng.randrange(0, 18))]) + rng.choice(["", "p" + rng.choice(["", "-", "+"]) + d(rng.randrange(1, 5))])
    if k == 6:
        return "".join(d(rng.randrange(1, 4)) + rng.choice(["", "." + d(rng.randrange(1, 3))]) + rng.choice(["h", "m", "s", "ms", "µs", "ns", "d", "w", "y", "x", ""]) for _ in range(rng.randrange(1, 4)))
    if k == 7:
        return "".join(d(rng.randrange(1, 5)) + rng.choice(["", "." + d(1)]) + rng.choice(["B", "K", "KB", "KiB", "Ki", "M", "MiB", "G", "GB", "T", "TiB", "Q", ""]) for _ in range(rng.randrange(1, 3)))
    if k == 8:
        return "%04d-%02d-%02d%s%02d:%02d:%02d%s%s" % (rng.choice([1676, 1677, 1970, 2024, 2262, 2263]), rng.randrange(0, 14), rng.randrange(0, 33), rng.choice("T tx"), rng.randrange(0, 26), rng.randrange(0, 62),
                                                      rng.randrange(0, 62), rng.choice(["", "." + d(rng.randrange(1, 11))]), rng.choice(["", "Z", "+01:00", "-23:59", "+24:60", "+1:00", "z"]))
    if k == 9:
        return ".".join(str(rng.choice([0, 1, 9, 10, 99, 127, 255, 256, 1000])) for _ in range(rng.choice([3, 4, 4, 4, 5])))
    if k == 10:
        return "".join(rng.choice("0123456789_.-+eExXpPbBoOinfINF ") for _ in range(rng.randrange(0, 12)))
    return bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 9))).decode("latin-1")


def test_random_strings(oracle):
    rng = random.Random(20250924)
    O = oracle.lib()
    for _ in range(60000):
        s = random_text(rng).encode("utf-8", "surrogateescape") if rng.random() < 0.97 else bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 12)))
        a, b = vs.parse_math_number(s), O.vlo_parse_math_number(s, len(s))
        assert same(a, b), (s, a, b)
