"""Transcribes the reference's TestStatsSum (lib/logstorage/stats_sum_test.go), TestStatsAvg (stats_avg_test.go) and the
`stats by (_time:...)` cases of TestPipeStats (pipe_stats_test.go) into stats_cases.json: [{source, query, rows, expected}], every row a list
of [name, value].  Run it with the reference tree's lib/logstorage directory as the argument."""
import json
import os
import re
import sys

TOKEN = re.compile(r'\s*(`[^`]*`|"(?:[^"\\]|\\.)*"|\[\]\[\]Field|\{|\}|,|\)|f\()', re.S)


def tokens(src):
    pos, out = 0, []
    while pos < len(src):
        m = TOKEN.match(src, pos)
        if not m:
            pos += 1
            continue
        out.append(m.group(1))
        pos = m.end()
    return out


def lit(t):
    return t[1:-1] if t[0] == "`" else json.loads(t)


def rows(ts, i):
    """[][]Field{ {{"a", `1`}, ...}, ... } at ts[i] -> (rows, next index)"""
    assert ts[i] == "[][]Field" and ts[i + 1] == "{", ts[i:i + 3]
    i += 2
    out = []
    while ts[i] != "}":
        if ts[i] == ",":
            i += 1
            continue
        assert ts[i] == "{"
        i += 1
        row = []
        while ts[i] != "}":
            if ts[i] == ",":
                i += 1
                continue
            assert ts[i] == "{" and ts[i + 2] == ",", ts[i:i + 5]
            row.append([lit(ts[i + 1]), lit(ts[i + 3])])
            assert ts[i + 4] == "}", ts[i:i + 5]
            i += 5
        out.append(row)
        i += 1
    return out, i + 1


def cases(path, func, want=lambda q: True):
    src = open(path).read()
    start = src.index("func %s(t *testing.T)" % func)
    end = src.find("\nfunc ", start + 1)
    ts = tokens(src[start:end if end > 0 else len(src)])
    out = []
    for i, t in enumerate(ts):
        if t != "f(" or not (ts[i + 1][0] in "`\"" and ts[i + 2] == "," and ts[i + 3] == "[][]Field"):
            continue
        q = lit(ts[i + 1])
        r, j = rows(ts, i + 3)
        assert ts[j] == ","
        e, _ = rows(ts, j + 1)
        if want(q):
            out.append({"source": "%s %s" % (os.path.basename(path), func), "query": q, "rows": r, "expected": e})
    return out


def main(ref_dir):
    out = cases(os.path.join(ref_dir, "stats_sum_test.go"), "TestStatsSum") + cases(os.path.join(ref_dir, "stats_avg_test.go"), "TestStatsAvg")
    out += cases(os.path.join(ref_dir, "pipe_stats_test.go"), "TestPipeStats", lambda q: "_time:" in q)
    json.dump(out, open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "stats_cases.json"), "w"), indent=1)
    print(len(out), "cases")


if __name__ == "__main__":
    main(sys.argv[1])
