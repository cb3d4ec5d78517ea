"""Bucketed by-fields on the CPU: vlscan_bucket_text (the host build of getBucketedValue the hits kernels run) and the C++ restatement
(tests/bucket_oracle) against the reference's TestTruncate* tables wherever a text reaches them, against each other on random texts and bucket
sizes, and the restatement against the bucketed TestPipeStats cases (tests/golden/bucketed_by_cases.json)."""
import json
import math
import os
import random
import struct

import numpy as np
import pytest

import vlobucket
from victorialogs_b200 import scan as vs

CASES = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bucketed_by_cases.json")))
HOUR, DAY = 3600 * 10 ** 9, 86400 * 10 ** 9


def both(text, size, offset=0.0, calendar=0):
    """the engine's and the restatement's bucketed text, which must agree"""
    got = vs.bucket_text(text, size, offset, calendar)
    assert got == vlobucket.bucket_text(text, size, offset, calendar), (text, size, offset, calendar)
    return got


def f64_text(x):
    return vs.format_float64(struct.unpack("<Q", struct.pack("<d", x))[0])


def test_by_bucket_layout():
    # include/vlscan.h, x86-64 SysV: two doubles, two uint32
    import ctypes as C
    assert C.sizeof(vs.ByBucket) == 24 and vs.ByBucket.calendar.offset == 16 and vs.ByBucket.enabled.offset == 20


def test_truncate_int64_table_through_texts():
    for n, size, off, want in CASES["int64"]:
        assert both(n, float(size), float(off)) == want.encode()


def test_truncate_float64_table_through_texts():
    for n, size, off, want in CASES["float64"]:
        text = n if "." in n else n + ".0"   # an integer text would take the int64 path: "130.0" is a tryParseFloat64 number of the same value
        assert both(text, float(size), float(off)) == f64_text(float(want)), (n, size, off, want)


def test_truncate_uint32_table_through_ipv4_texts():
    ip = lambda n: b"%d.%d.%d.%d" % (n >> 24, (n >> 16) & 255, (n >> 8) & 255, n & 255)
    for n, size, off, want in CASES["uint32"]:
        assert both(ip(int(n)), float(size), float(off)) == ip(int(want))


def test_texts_of_every_kind():
    assert both(b"", 100) == b"" and both(b"abc", 100) == b"abc" and both(b"+5", 100) == b"+5"
    assert both(b"-", 100) == b"0"   # tryParseDuration takes "-" as a zero duration
    assert both(b"1_234", 100) == b"1200" and both(b"-1", 100) == b"-100" and both(b"-9223372036854775808", 7) != b""
    assert both(b"1.5s", 10 ** 9) == b"1s" and both(b"-2h5m", HOUR) == b"-3h" and both(b"1h30m", HOUR, 1800 * 10 ** 9) == b"1h30m"
    assert both(b"10.1.2.3", 256) == b"10.1.2.0" and both(b"10.1.200.3", 65536) == b"10.1.0.0"
    assert both(b"2024-03-05T12:34:56.123456789Z", HOUR) == b"2024-03-05T12:00:00Z"
    assert both(b"2024-03-05T12:34:56+02:00", DAY) == b"2024-03-05T00:00:00Z"
    assert both(b"2024-03-05T12:34:56Z", 0, 0, vs.BUCKET_MONTH) == b"2024-03-01T00:00:00Z"
    assert both(b"2024-03-05T12:34:56Z", 0, 0, vs.BUCKET_YEAR) == b"2024-01-01T00:00:00Z"
    assert both(b"2024-03-06T12:34:56Z", 7 * DAY, 0, vs.BUCKET_WEEK) == b"2024-03-04T00:00:00Z"   # a Monday
    assert both(b"17", 0, 0, vs.BUCKET_MONTH) == b"17"          # month / year leave the size 0: an integer by month is size 1
    assert both(b"17", 0.1) == b"17" and both(b"1.37", 0.1) == b"1.3"   # int64(0.1) = 0 counts as 1; the float path keeps 0.1
    assert both(b"17", 10, -3) == b"17" and both(b"16", 10, -3) == b"7"
    assert both(b"1e3", 100) == b"1e3"                          # no parser of getBucketedValue takes an exponent
    assert both(b"1KiB", 100) == b"1KiB"                        # nor a byte size


def test_rejected_buckets():
    for size, off in ((math.nan, 0), (math.inf, 0), (1, math.inf), (1, -math.nan)):
        for f in (vs.bucket_text, vlobucket.bucket_text):
            with pytest.raises(ValueError):
                f(b"5", size, off)
    rejected = []
    for size in [1e300, 1e-300, 5e-324, 1.7976931348623157e308, 3e-7, 1e22, 0.3, 7.0, 1e-7] + [10.0 ** k for k in range(-30, 31)]:
        outs = []
        for f in (vs.bucket_text, vlobucket.bucket_text):
            try:
                outs.append(f(b"1.5", size))
            except ValueError:
                outs.append(None)
        assert outs[0] == outs[1], size
        if outs[0] is None:
            rejected.append(size)
    assert rejected, "no size with int64(size * 10^-e) == 0 among the probes"


def random_text(rng):
    k = rng.randrange(9)
    if k == 0:
        return b"%d" % rng.randrange(-10 ** 12, 10 ** 12)
    if k == 1:
        return b"%d.%0*d" % (rng.randrange(-5000, 5000), rng.randrange(1, 6), rng.randrange(0, 10 ** 5))
    if k == 2:
        return rng.choice([b"1_000", b"12_34.5_6", b"-0", b"-0.0", b"0", b"00", b"007", b"18446744073709551616", b"9223372036854775807"])
    if k == 3:
        z = rng.choice([b"Z", b"+02:00", b"-05:30", b""])
        frac = rng.choice([b"", b".5", b".123456789", b".000"])
        return b"20%02d-%02d-%02dT%02d:%02d:%02d%s%s" % (rng.randrange(100), rng.randrange(1, 13), rng.randrange(1, 29), rng.randrange(24), rng.randrange(60), rng.randrange(60), frac, z)
    if k == 4:
        return b"%d.%d.%d.%d" % tuple(rng.randrange(256) for _ in range(4))
    if k == 5:
        return rng.choice([b"1.5s", b"-2h5m", b"3d4h", b"1w2d3h4m5.25s", b"250ms", b"17\xc2\xb5s", b"9ns", b"1y", b"-0s", b"5m30s"])
    if k == 6:
        return rng.choice([b"abc", b"", b"-", b"-x", b"1e5", b"0x10", b"1KiB", b"1..2", b".5", b"5.", b" 5"])
    if k == 7:
        return b"-%d" % rng.randrange(10 ** 19)
    return b"%d.%d" % (rng.randrange(10 ** 9), rng.randrange(10 ** 9))


def random_bucket(rng):
    size = rng.choice([1, 2, 7, 10, 100, 1024, 256, 65536, 0.1, 0.25, 0.02, 1.5, 1e9, HOUR, DAY, 7 * DAY, 0, -5, 3.3e-5, 2.5e12, 1e19, 1e20])
    off = rng.choice([0, 0, 3, -3, 0.05, -1.25, 1800 * 10 ** 9, -HOUR, 2 ** 31, 1e19, -1e19])
    cal = rng.choice([0, 0, 0, vs.BUCKET_WEEK, vs.BUCKET_MONTH, vs.BUCKET_YEAR])
    return size, off, cal


def test_engine_against_restatement_random():
    rng = random.Random(20261018)
    for _ in range(20000):
        size, off, cal = random_bucket(rng)
        text = random_text(rng)
        try:
            both(text, size, off, cal)
        except ValueError:
            with pytest.raises(ValueError):
                vlobucket.bucket_text(text, size, off, cal)


def test_pipe_stats_cases_on_the_restatement(oracle):
    import parity_util as pu
    sizes = {"x:1KiB": 1024.0, "ip:/24": 256.0}
    for case in CASES["pipe_stats"]:
        spec = case["query"].split("by (")[1].split(")")[0]
        field = spec.split(":")[0]
        rows = [{k: v for k, v in r} for r in case["rows"]]
        names = sorted({k for r in rows for k in r})
        blk = oracle.Block.from_columns([(n, [r.get(n, "").encode() for r in rows]) for n in names]).set_timestamps([10 ** 9 * i for i in range(len(rows))])
        d = pu.oracle_block_to_desc(blk)
        words = np.array([(1 << len(rows)) - 1], dtype=np.uint64)
        got = vlobucket.stats([d], [words], 10 ** 18, 0, 0, [field], [(sizes[spec], 0.0, 0)])
        want = {dict(e)[field].encode(): int(dict(e)["rows"]) for e in case["expected"]}
        assert {k[1][0]: v[0] for k, v in got.items()} == want, case["query"]
