#!/usr/bin/env python3
"""Transcribe the reference's TestTruncateTimestamp (lib/logstorage/block_result_test.go) into tests/golden/bucket_cases.json: the `_time`
buckets of `stats by (_time:step offset off)`, every case as the test writes it (RFC 3339 texts, bucket and offset strings) and as
nanoseconds (step 0 for month / year, calendar 0 plain, 1 week, 2 month, 3 year).  Uses the Go-literal tokenizer of extract_go_fixtures.py;
run in the build container only, /root/reference is not needed at test time."""
import datetime
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_go_fixtures import OUT, REF, extract_f_calls  # noqa: E402

RFC3339 = re.compile(r"^(\d{4})-(\d\d)-(\d\d)T(\d\d):(\d\d):(\d\d)(?:\.(\d{1,9}))?(Z|[+-]\d\d:\d\d)$")
DURATION_UNITS = {"ns": 1, "us": 10 ** 3, "µs": 10 ** 3, "ms": 10 ** 6, "s": 10 ** 9, "m": 60 * 10 ** 9, "h": 3600 * 10 ** 9,
                  "d": 86400 * 10 ** 9, "w": 7 * 86400 * 10 ** 9, "y": 365 * 86400 * 10 ** 9}
BUCKET_NAMES = {"nanosecond": 1, "microsecond": 10 ** 3, "millisecond": 10 ** 6, "second": 10 ** 9, "minute": 60 * 10 ** 9, "hour": 3600 * 10 ** 9,
                "day": 86400 * 10 ** 9, "week": 7 * 86400 * 10 ** 9}


def rfc3339_ns(s):
    m = RFC3339.match(s)
    assert m, s
    y, mo, d, hh, mi, ss = (int(x) for x in m.groups()[:6])
    frac = (m.group(7) or "").ljust(9, "0")
    days = (datetime.date(y, mo, d) - datetime.date(1970, 1, 1)).days
    ns = (((days * 24 + hh) * 60 + mi) * 60 + ss) * 10 ** 9 + int(frac)
    z = m.group(8)
    if z != "Z":
        sign = 1 if z[0] == "+" else -1
        ns -= sign * (int(z[1:3]) * 3600 + int(z[4:6]) * 60) * 10 ** 9
    return ns


def duration_ns(s):
    neg = s.startswith("-")
    parts = re.findall(r"(\d+)(ns|us|µs|ms|s|m|h|d|w|y)", s.lstrip("-"))
    assert "".join(a + b for a, b in parts) == s.lstrip("-"), s
    v = sum(int(a) * DURATION_UNITS[b] for a, b in parts)
    return -v if neg else v


def main():
    out = []
    for args in extract_f_calls(os.path.join(REF, "block_result_test.go"), "TestTruncateTimestamp"):
        ts, bucket, offset, want = (a.decode() for a in args)
        calendar = {"week": 1, "month": 2, "year": 3}.get(bucket, 0)
        step = 0 if bucket in ("month", "year") else BUCKET_NAMES.get(bucket) or duration_ns(bucket)
        out.append({"ts": ts, "bucket": bucket, "offset": offset, "want": want, "ts_ns": rfc3339_ns(ts), "step_ns": step,
                    "offset_ns": duration_ns(offset) if offset else 0, "calendar": calendar, "want_ns": rfc3339_ns(want)})
    print("TestTruncateTimestamp", len(out))
    json.dump(out, open(os.path.join(OUT, "bucket_cases.json"), "w"), indent=0, ensure_ascii=False)


if __name__ == "__main__":
    main()
