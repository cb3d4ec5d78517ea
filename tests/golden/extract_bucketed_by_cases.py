#!/usr/bin/env python3
"""Transcribe the reference's bucketed by-field fixtures into tests/golden/bucketed_by_cases.json: TestTruncateFloat64 / TestTruncateInt64 /
TestTruncateUint64 / TestTruncateUint32 (lib/logstorage/block_result_test.go) as [n, bucketSize, offset, expected] per kind, and the cases of
TestPipeStats (pipe_stats_test.go) that bucket a by-field other than `_time` (`by (x:1KiB)`, `by (ip:/24)`) as {query, rows, expected}.  Run in
the build container only: /root/reference is not needed at test time."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_go_fixtures import OUT, REF, extract_f_calls  # noqa: E402
from extract_stats_cases import cases  # noqa: E402


def main():
    out = {}
    for kind in ("Float64", "Int64", "Uint64", "Uint32"):
        calls = extract_f_calls(os.path.join(REF, "block_result_test.go"), "TestTruncate" + kind)
        assert calls and all(len(c) == 4 and all(a[0] == "num" for a in c) for c in calls), kind
        out[kind.lower()] = [[a[1] for a in c] for c in calls]   # the numbers as written: float cases keep their decimal text
    pipe = cases(os.path.join(REF, "pipe_stats_test.go"), "TestPipeStats", lambda q: "by (" in q and ":" in q.split("by (")[1].split(")")[0] and "_time:" not in q)
    assert {c["query"] for c in pipe} >= {"stats by (x:1KiB) count(*) as rows", "stats by (ip:/24) count(*) as rows"}, [c["query"] for c in pipe]
    out["pipe_stats"] = pipe
    json.dump(out, open(os.path.join(OUT, "bucketed_by_cases.json"), "w"), indent=1)
    print({k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
