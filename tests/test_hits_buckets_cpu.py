"""CPU suite for the `_time` buckets of the hits aggregation (`stats by (_time:step offset off, ...) count()`, block_result.go:760-848):
the host build of the device routine (vlscan_truncate_timestamp) and the oracle's restatement against the reference's own table
(TestTruncateTimestamp, tests/golden/bucket_cases.json) and against a plain Python integer / datetime model on random inputs, including
int64 wrap-around at both ends.  Also the ABI of vlscan_hits_stats: struct layout, argument checks and the loud failure without a device."""
import ctypes as C
import datetime
import json
import os
import random

import pytest

import vlohits
from victorialogs_b200 import scan as vs

HERE = os.path.dirname(os.path.abspath(__file__))
DAY = 86400 * 10 ** 9
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
EPOCH = datetime.date(1970, 1, 1)


def wrap(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


def model(ts, step, offset, calendar):
    """truncateTimestamp with Python integers: Go's int64 sums wrap, `%` of a positive step made non-negative is Python's floor `%`."""
    if step <= 0:
        step = 1
    if calendar == vs.BUCKET_WEEK:
        offset = wrap(offset + 4 * DAY)
    t = wrap(ts - offset)
    if calendar in (vs.BUCKET_MONTH, vs.BUCKET_YEAR):
        d = EPOCH + datetime.timedelta(days=t // DAY)
        first = datetime.date(d.year, 1 if calendar == vs.BUCKET_YEAR else d.month, 1)
        res = (first - EPOCH).days * DAY
    else:
        res = t - t % step
    return wrap(res + offset)


def golden():
    cases = json.load(open(os.path.join(HERE, "golden", "bucket_cases.json")))
    assert len(cases) == 29
    return cases


def test_reference_table_host_build():
    for c in golden():
        got = vs.truncate_timestamp(c["ts_ns"], c["step_ns"], c["offset_ns"], c["calendar"])
        assert got == c["want_ns"], c


def test_reference_table_oracle():
    for c in golden():
        assert vlohits.truncate_timestamp(c["ts_ns"], c["step_ns"], c["offset_ns"], c["calendar"]) == c["want_ns"], c


def test_reference_table_model():
    for c in golden():
        assert model(c["ts_ns"], c["step_ns"], c["offset_ns"], c["calendar"]) == c["want_ns"], c


def random_cases(n, seed):
    rng = random.Random(seed)
    year = 366 * DAY
    out = []
    for _ in range(n):
        kind = rng.randrange(6)
        if kind == 0:
            ts = rng.randint(I64_MIN, I64_MAX)
        elif kind == 1:
            ts = I64_MAX - rng.randrange(year)                  # within a year of the ends
        elif kind == 2:
            ts = I64_MIN + rng.randrange(year)
        elif kind == 3:
            ts = rng.randint(-10 * year, 10 * year)               # around the epoch, negative included
        else:
            ts = 1_700_000_000_000_000_000 + rng.randint(-year, year)
        sk = rng.randrange(6)
        if sk == 0:
            step = 1
        elif sk == 1:
            step = rng.choice([10 ** 3, 10 ** 6, 10 ** 9, 60 * 10 ** 9, 3600 * 10 ** 9, DAY, 7 * DAY])
        elif sk == 2:
            step = rng.randint(1, 10 ** 12)
        elif sk == 3:
            step = rng.randint(1 << 62, I64_MAX)                  # larger than any span
        elif sk == 4:
            step = rng.randint(-5, 0)                              # treated as 1
        else:
            step = rng.randint(2, 1 << 40)
        ok = rng.randrange(5)
        if ok == 0:
            offset = 0
        elif ok == 1:
            offset = rng.randint(-abs(step), abs(step))
        elif ok == 2:
            offset = rng.randint(-50, 50) * max(abs(step), 1) + rng.randint(-3, 3)   # larger than the step
        elif ok == 3:
            offset = rng.randint(-30 * DAY, 30 * DAY)
        else:
            offset = rng.randint(I64_MIN, I64_MAX)
        out.append((ts, step, offset, rng.randrange(4)))
    return out


def test_random_against_model():
    cases = random_cases(100_000, 5)
    for ts, step, offset, cal in cases:
        want = model(ts, step, offset, cal)
        assert vs.truncate_timestamp(ts, step, offset, cal) == want, (ts, step, offset, cal)
        assert vlohits.truncate_timestamp(ts, step, offset, cal) == want, (ts, step, offset, cal)


def test_hits_query_layout():
    # include/vlscan.h, x86-64 SysV: two int64, two uint32, two pointers
    assert C.sizeof(vs.HitsQuery) == 8 + 8 + 4 + 4 + 8 + 8
    assert vs.HitsQuery.by_names.offset == 24 and vs.HitsQuery.by_name_lens.offset == 32


def test_generator_constants_agree():
    assert (vs.GEN_TIMESTAMPS, vs.GEN_T0, vs.GEN_STEP) == (vlohits.GEN_TIMESTAMPS, vlohits.GEN_T0, vlohits.GEN_STEP)
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "vlscan.h")).read()
    assert "#define VLSCAN_GEN_T0 %dll" % vs.GEN_T0 in hdr and "#define VLSCAN_GEN_STEP %dll" % vs.GEN_STEP in hdr


def _call_without_ctx(by):
    q, keep = vs.hits_query(10 ** 9, 0, vs.BUCKET_PLAIN, by)
    L = vs.lib()
    info = (C.c_uint64 * 4)(7, 7, 7, 7)
    b = (C.c_int64 * 4)(); c = (C.c_uint64 * 4)(); o = (C.c_uint64 * 32)(); kb = C.create_string_buffer(64)
    rc = L.vlscan_hits_stats(None, C.byref(q), b, c, C.c_uint64(4), kb, C.c_uint64(64), o, info)
    return rc, L.vlscan_last_error(None).decode(), list(info)


def test_hits_stats_fails_loudly_without_a_device():
    rc, err, info = _call_without_ctx(["level"])
    assert rc != 0 and "CUDA device" in err
    assert info == [0, 0, 0, 0]


def test_hits_stats_rejects_bad_queries():
    rc, err, _ = _call_without_ctx(["_time"])
    assert rc < 0 and "_time" in err
    rc, err, _ = _call_without_ctx(["a", "b", "c", "d", "e"][:vs.HITS_MAX_BY + 1])
    assert rc < 0 and "by-fields" in err
    q, keep = vs.hits_query(1, 0, 4, [])
    assert vs.lib().vlscan_hits_stats(None, C.byref(q), None, None, C.c_uint64(0), None, C.c_uint64(0), None, None) < 0
    assert "calendar" in vs.lib().vlscan_last_error(None).decode()
