"""CPU suite for the facets state of a batch (vlscan_facets, `| facets`, lib/logstorage/pipe_facets.go): the reference's TestPipeFacets cases
through the model and facets_merge, the key-class and length quirks of updateStateGeneric / updateStateUint64 / updateStateInt64, random splits
of a batch merging to the whole, and the ABI: struct layout, argument checks, loud failure without a device."""
import ctypes as C
import json
import os
import random

import facets_model as fm
from victorialogs_b200 import scan as vs

HERE = os.path.dirname(os.path.abspath(__file__))


def golden_cases():
    return json.load(open(os.path.join(HERE, "golden", "facets_cases.json")))


def rows_to_blocks(rows):
    """one block per input row, every field a const cell (the row's value); all rows selected"""
    return [({name: ("const", value.encode()) for name, value in row}, [0]) for row in rows]


def model_state(blocks, fields, max_values=0, max_len=0):
    sh = fm.Shard(max_values, max_len)
    for cells, sel in blocks:
        sh.block(cells, sel)
    return sh.state(fields), sh.rows


def test_golden_cases_through_the_model():
    cases = golden_cases()
    assert len(cases) == 3
    for c in cases:
        fields = sorted({name for row in c["rows"] for name, _ in row})
        state, rows = model_state(rows_to_blocks(c["rows"]), fields)
        got = vs.facets_merge([(state, rows)], c["limit"], c["keep_const_fields"])
        assert [(f, t.decode(), h) for f, t, h in got] == [tuple(w) for w in c["want"]], c["pipe"]


def test_key_classes():
    K = fm.generic_key
    assert K(b"1_000") == (fm.U64, 1000) and K(b"_") == (fm.U64, 0) and K(b"_01") == (fm.U64, 1)
    assert K(b"0123") == (fm.STR, b"0123") and K(b"0_1") == (fm.STR, b"0_1") and K(b"0") == (fm.U64, 0)
    assert K(b"-0") == (fm.NEG, 0) and K(b"-_") == (fm.NEG, 0) and K(b"-") == (fm.STR, b"-")
    assert K(b"-9223372036854775808") == (fm.NEG, -(1 << 63)) and K(b"-9223372036854775809") == (fm.STR, b"-9223372036854775809")
    assert K(b"18446744073709551615") == (fm.U64, (1 << 64) - 1) and K(b"18446744073709551616")[0] == fm.STR
    assert K(b"1" + b"_" * 26)[0] == fm.STR and K(b"1" + b"_" * 25) == (fm.U64, 1)
    # "-0" and the uint64 0 are two entries that both print as 0; "1_000" and a uint16 1000 are one
    sh = fm.Shard()
    sh.block({"f": ("text", [b"-0", b"0", b"1_000", b"-_"]), "g": ("uint", [1000, 7, 1000, 7])}, [0, 1, 2, 3])
    sh.block({"f": ("uint", [1000]), "g": ("text", [b"1_000"])}, [0])
    st = sh.state(["f", "g"])
    assert st["f"] == [(fm.NEG, b"0", 2), (fm.U64, b"1000", 2), (fm.U64, b"0", 1)]
    assert st["g"] == [(fm.U64, b"1000", 3), (fm.U64, b"7", 2)]


def test_length_rules():
    for L in range(1, 23):
        sh = fm.Shard(0, L)
        sh.block({"u": ("uint", [12345678901]), "i": ("int", [-(1 << 63)]), "j": ("int", [-5]), "t": ("text", [b"x" * 11]),
                  "c": ("const", b"y" * 12)}, [0])
        st = sh.state(["u", "i", "j", "t", "c"])
        assert (st["u"] is None) == (L <= 19), L          # uint64StringLen(11 digits) = 20, checked only while L <= 20
        assert (st["i"] is None) == (L <= 20), L          # int64StringLen(MinInt64) = 21, checked only while L <= 21
        assert (st["j"] is None) == (L < 2), L
        assert (st["t"] is None) == (L < 11) and (st["c"] is None) == (L < 12), L
    # a long dict entry without selected rows is never looked at; an empty text is skipped
    sh = fm.Shard(0, 3)
    sh.block({"d": ("dict", [b"abc", b"too long", b""], [0, 0, 1, 2]), "e": ("text", [b"", b"", b"ok", b""])}, [0, 1, 3])
    st = sh.state(["d", "e"])
    assert st["d"] == [(fm.STR, b"abc", 2)] and st["e"] == []
    sh = fm.Shard(0, 3)
    sh.block({"d": ("dict", [b"abc", b"too long", b""], [0, 0, 1, 2])}, [2])
    assert sh.state(["d"])["d"] is None


def test_distinct_limit_is_exact():
    for m in (1, 2, 5, 1000):
        for extra in (0, 1):
            n = m + extra
            sh = fm.Shard(m, 0)
            sh.block({"f": ("text", [b"v%d" % i for i in range(n)])}, list(range(n)))
            assert (sh.state(["f"])["f"] is None) == bool(extra), (m, extra)


def test_rfc3339_nano():
    assert fm.rfc3339_nano(1700000000000000000) == b"2023-11-14T22:13:20Z"
    assert fm.rfc3339_nano(1700000000500000000) == b"2023-11-14T22:13:20.5Z"
    assert fm.rfc3339_nano(-1) == b"1969-12-31T23:59:59.999999999Z"
    assert fm.rfc3339_nano(-(1 << 63)) == b"1677-09-21T00:12:43.145224192Z"
    assert fm.rfc3339_nano((1 << 63) - 1) == b"2262-04-11T23:47:16.854775807Z"


def random_cells(rng, rows):
    cells = {}
    vocab = [b"", b"0", b"00", b"1_000", b"1000", b"-0", b"-_", b"_", b"-7", b"abc", b"x" * rng.randint(1, 30), b"18446744073709551616", b"-9223372036854775808"]
    for name in ("c", "d", "u", "i", "t", "ts"):
        kind = rng.randrange(6)
        if kind == 0:
            continue
        if name == "ts":
            t = rng.choice([0, 1700000000000000000, -5])
            cells[name] = ("time", sorted(t + rng.randrange(4) * rng.choice([1, 10 ** 9, 10 ** 6]) for _ in range(rows)))
        elif kind == 1:
            cells[name] = ("const", rng.choice(vocab[1:]))
        elif kind == 2:
            ents = rng.sample(vocab, rng.randint(1, 8))
            cells[name] = ("dict", ents, [rng.randrange(len(ents)) for _ in range(rows)])
        elif kind == 3:
            cells[name] = ("uint", [rng.choice([0, 7, 1000, 10 ** 10, (1 << 64) - 1, rng.randrange(50)]) for _ in range(rows)])
        elif kind == 4:
            cells[name] = ("int", [rng.choice([0, -1, -(1 << 63), (1 << 63) - 1, rng.randrange(-50, 50)]) for _ in range(rows)])
        else:
            cells[name] = ("text", [rng.choice(vocab) for _ in range(rows)])
    return cells


def test_random_splits_merge_to_the_whole():
    rng = random.Random(77)
    fields = ["c", "d", "u", "i", "t", "ts"]
    for case in range(400):
        blocks = []
        for _ in range(rng.randint(1, 6)):
            rows = rng.randint(1, 12)
            blocks.append((random_cells(rng, rows), [r for r in range(rows) if rng.random() < 0.7]))
        mv, ml = rng.choice([0, 1, 2, 3, 6, 20]), rng.choice([0, 1, 2, 5, 19, 20, 21, 22])
        whole, rows = model_state(blocks, fields, mv, ml)
        cut = rng.randint(0, len(blocks))
        parts = [model_state(blocks[:cut], fields, mv, ml), model_state(blocks[cut:], fields, mv, ml)]
        for limit, keep in ((10, False), (3, True), (1 << 30, False)):
            assert vs.facets_merge(parts, limit, keep, mv) == vs.facets_merge([(whole, rows)], limit, keep, mv), case


def test_facets_query_layout():
    # include/vlscan.h, x86-64 SysV: u64, u64, u32 (+ 4 bytes padding), two pointers
    assert C.sizeof(vs.FacetsQuery) == 40
    assert vs.FacetsQuery.max_values_per_field.offset == 0 and vs.FacetsQuery.max_value_len.offset == 8 and vs.FacetsQuery.nfields.offset == 16
    assert vs.FacetsQuery.field_names.offset == 24 and vs.FacetsQuery.field_name_lens.offset == 32
    q, keep = vs.facets_query(["level", "", "_time"], 5, 7)
    assert (q.max_values_per_field, q.max_value_len, q.nfields) == (5, 7, 3)


def _call_without_ctx(fields, q=True):
    query, keep = vs.facets_query(fields)
    info = (C.c_uint64 * 4)(*[7] * 4)
    d = (C.c_uint8 * 8)(); fo = (C.c_uint64 * 9)(); h = (C.c_uint64 * 4)(); cl = (C.c_uint8 * 4)(); vo = (C.c_uint64 * 5)(); vb = C.create_string_buffer(64)
    rc = vs.lib().vlscan_facets(None, C.byref(query) if q else None, d, fo, h, cl, C.c_uint64(4), vb, C.c_uint64(64), vo, info)
    return rc, vs.lib().vlscan_last_error(None).decode(), list(info)


def test_facets_fails_loudly_without_a_device():
    rc, err, info = _call_without_ctx(["level", "", "_time"])
    assert rc != 0 and "CUDA device" in err
    assert info == [0, 0, 0, 0]


def test_facets_rejects_bad_queries():
    for fields, word in (([], "at least one"), (["a", "a"], "duplicate"), (["", "_msg"], "duplicate"), (["_stream"], "_stream"), (["x", "_stream_id"], "_stream_id")):
        rc, err, _ = _call_without_ctx(fields)
        assert rc < 0 and word in err, (fields, err)
    rc, err, _ = _call_without_ctx(["a"], q=False)
    assert rc < 0 and "query" in err
