#!/usr/bin/env python3
"""Transcribe the reference's TestStatsHistogram (lib/logstorage/stats_histogram_test.go) into tests/golden/histogram_cases.json as
{query, rows, expected} per case.  Usage: extract_histogram_cases.py <VictoriaLogs checkout>/lib/logstorage"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_stats_cases import cases  # noqa: E402


def main(ref_dir):
    out = cases(os.path.join(ref_dir, "stats_histogram_test.go"), "TestStatsHistogram")
    assert out, "no TestStatsHistogram cases"
    json.dump(out, open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "histogram_cases.json"), "w"), indent=1)
    print(len(out), "cases")


if __name__ == "__main__":
    main(sys.argv[1])
