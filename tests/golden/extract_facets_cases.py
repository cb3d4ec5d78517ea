#!/usr/bin/env python3
"""Transcribe the reference's TestPipeFacets (lib/logstorage/pipe_facets_test.go) into tests/golden/facets_cases.json: the pipe text, its limit
and keep_const_fields, the input rows as [[name, value], ...] and the expected [field_name, field_value, hits] rows.  Uses the Go-literal
tokenizer of extract_go_fixtures.py; run in the build container only, /root/reference is not needed at test time."""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_go_fixtures import OUT, REF, extract_f_calls  # noqa: E402


def main():
    out = []
    # the tokenizer reads one level of slice type: `[][]Field{` becomes `[]Rows{`, the same composite literal
    src = open(os.path.join(REF, "pipe_facets_test.go"), encoding="utf-8").read().replace("[][]Field{", "[]Rows{")
    with tempfile.NamedTemporaryFile("w", suffix=".go", delete=False) as tmp:
        tmp.write(src)
    try:
        calls = extract_f_calls(tmp.name, "TestPipeFacets")
    finally:
        os.unlink(tmp.name)
    for pipe, rows, want in calls:
        words = pipe.decode().split()
        assert words[0] == "facets" and set(words[2:]) <= {"keep_const_fields"}, words
        limit = int(words[1]) if len(words) > 1 and words[1].isdigit() else 10
        got_rows = [[[f[0].decode(), f[1].decode()] for f in row] for row in rows]
        got_want = []
        for row in want:
            d = {f[0].decode(): f[1].decode() for f in row}
            got_want.append([d["field_name"], d["field_value"], int(d["hits"])])
        out.append({"pipe": pipe.decode(), "limit": limit, "keep_const_fields": "keep_const_fields" in words, "rows": got_rows, "want": got_want})
    print("TestPipeFacets", len(out))
    json.dump(out, open(os.path.join(OUT, "facets_cases.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
