"""Typed and dict cells in the layouts the upload accepts besides one value per row, through every reader of a cell: gathered values, hits by
the field, newest rows, facets, and eq_field / le_field against a strings copy of the same values.

A single-copy cell (rows >= 2, const lens equal to the data length: every row is the whole payload, lib/logstorage/encoding.go:113-120) gives
its one value in every row.  A cell whose stored length is not its type's width fails with the reference's "unexpected length for binary
representation of a number" and leaves the ctx usable.  The blocks are small: a reader that ignored the layout would read past the payload
into its padding, never past the arena."""
import calendar
import struct

import pytest

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000_000_000
ISO_NS = calendar.timegm((2024, 3, 1, 12, 0, 0)) * 10 ** 9 + 123_000_000
WIDTH_MSG = "unexpected length for binary representation of a number"


def cases(vs):
    """(name, value type, encoded value, its text, dict entries)"""
    return [
        ("uint8", vs.VT_UINT8, bytes([200]), b"200", None),
        ("uint16", vs.VT_UINT16, struct.pack(">H", 300), b"300", None),
        ("uint32", vs.VT_UINT32, struct.pack(">I", 70000), b"70000", None),
        ("uint64", vs.VT_UINT64, struct.pack(">Q", 5_000_000_000), b"5000000000", None),
        ("int64", vs.VT_INT64, struct.pack(">Q", 9), b"-5", None),   # zig-zag of -5
        ("float64", vs.VT_FLOAT64, struct.pack(">d", 1.5), b"1.5", None),
        ("ipv4", vs.VT_IPV4, bytes([10, 1, 2, 3]), b"10.1.2.3", None),
        ("iso8601", vs.VT_ISO8601, struct.pack(">Q", ISO_NS), b"2024-03-01T12:00:00.123Z", None),
        ("dict", vs.VT_DICT, bytes([1]), b"error", [b"warn", b"error"]),
    ]


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    ctx = vs.Ctx(0)
    yield oracle, vs, ctx
    ctx.close()


def upload(env, rows, f_col, text, g_col=None):
    """one block: field `f` as given, field `s` the strings copy `text` in every row, field `g` when given, timestamps T0 + row"""
    oracle, vs, ctx = env
    ts = oracle.Block.from_columns([("x", [b"%d" % i for i in range(rows)])]).set_timestamps([T0 + i for i in range(rows)]).timestamps_block()
    cols = [dict(field="f", kind="values", **f_col), dict(field="s", kind="values", value_type=vs.VT_STRING, lens_items=bytes([4, len(text)]), data=text * rows)]
    if g_col:
        cols.append(dict(field="g", kind="values", **g_col))
    return ctx.upload(vs.HostBlocks(["f", "s", "g"], [dict(rows=rows, columns=cols, timestamps=ts)]))


def row_values(vs, vt, rows):
    """rows distinct encoded values of type vt (dict: ids 0 and 1 in turn)"""
    def one(i):
        if vt == vs.VT_UINT8:
            return bytes([200 + i])
        if vt == vs.VT_IPV4:
            return bytes([10, 1, 2, 3 + i])
        if vt == vs.VT_DICT:
            return bytes([i % 2])
        if vt == vs.VT_INT64:
            v = i - 5
            return struct.pack(">Q", ((v << 1) ^ (v >> 63)) & (2 ** 64 - 1))
        fmt = {vs.VT_UINT16: (">H", 300), vs.VT_UINT32: (">I", 70000), vs.VT_UINT64: (">Q", 5_000_000_000), vs.VT_ISO8601: (">Q", ISO_NS)}.get(vt)
        return struct.pack(">d", 1.5 + i) if vt == vs.VT_FLOAT64 else struct.pack(fmt[0], fmt[1] + i * (10 ** 6 if vt == vs.VT_ISO8601 else 1))
    return [one(i) for i in range(rows)]


def matched(env, flt, batch):
    oracle, vs, ctx = env
    ctx.scan_resident(vs.Program(flt), batch)
    return int(ctx.fetch()[1].sum())


@pytest.mark.parametrize("case", range(9))
def test_single_copy_cell_gives_its_value_in_every_row(env, case):
    oracle, vs, ctx = env
    name, vt, enc, text, dct = cases(vs)[case]
    rows = 4
    batch = upload(env, rows, dict(value_type=vt, dict=dct, lens_items=bytes([4, len(enc)]), data=enc), text)
    assert matched(env, vs.Filter.noop(), batch) == rows
    assert ctx.gather_values("f")[0] == [text] * rows, name
    assert ctx.hits_stats(10 ** 9, by=("f",)) == [(T0, (text,), rows)], name
    assert ctx.hits_stats(1, by=("f",)) == [(T0 + i, (text,), 1) for i in range(rows)], name
    assert [(t, r, v) for t, _, r, v in ctx.last_rows(rows, ("f",))] == [(T0 + i, i, (text,)) for i in range(rows)], name
    assert [(t, h) for _, t, h in ctx.facets(["f"])["f"]] == [(text, rows)], name
    assert matched(env, vs.Filter.eq_field("f", "s"), batch) == rows, name
    assert matched(env, vs.Filter.le_field("f", "s"), batch) == rows, name
    assert matched(env, vs.Filter.le_field("f", "s", exclude_equal=True), batch) == 0, name
    batch.free()


@pytest.mark.parametrize("case", range(9))
def test_same_type_single_copy_cells_compare_their_values(env, case):
    """eq_field / le_field between two cells of one value type: their encoded values (typed) or dictionary entries (dict)"""
    oracle, vs, ctx = env
    name, vt, enc, text, dct = cases(vs)[case]
    rows = 4
    col = dict(value_type=vt, dict=dct, lens_items=bytes([4, len(enc)]), data=enc)
    batch = upload(env, rows, col, text, g_col=col)
    assert matched(env, vs.Filter.eq_field("f", "g"), batch) == rows, name
    assert matched(env, vs.Filter.le_field("f", "g"), batch) == rows, name
    assert matched(env, vs.Filter.le_field("f", "g", exclude_equal=True), batch) == 0, name
    batch.free()


@pytest.mark.parametrize("case", range(9))
def test_per_row_lens_cell_reads_like_const_lens(env, case):
    """a typed or dict cell whose lens items are stored per row (as the writer does for a one-row block) reads through its row offsets:
    ten rows, so rows 8 and 9 need the offset of the second group of eight"""
    oracle, vs, ctx = env
    name, vt, enc, text, dct = cases(vs)[case]
    rows, w = 10, len(enc)
    vals = b"".join(row_values(vs, vt, rows))
    got = []
    for lens in (bytes([4, w]), bytes([0]) + bytes([w] * rows)):
        batch = upload(env, rows, dict(value_type=vt, dict=dct, lens_items=lens, data=vals), text)
        assert matched(env, vs.Filter.noop(), batch) == rows
        got.append((ctx.gather_values("f")[0], ctx.hits_stats(10 ** 9, by=("f",)), ctx.hits_stats(1, by=("f",)), ctx.last_rows(rows, ("f",)),
                    ctx.facets(["f"])))
        batch.free()
    assert len(set(got[0][0])) == (2 if vt == vs.VT_DICT else rows), name
    assert got[1] == got[0], name
    one = upload(env, 1, dict(value_type=vt, dict=dct, lens_items=bytes([0, w]), data=enc), text)
    assert matched(env, vs.Filter.noop(), one) == 1
    assert ctx.gather_values("f")[0] == [text] and ctx.hits_stats(10 ** 9, by=("f",)) == [(T0, (text,), 1)], name
    assert [(t, h) for _, t, h in ctx.facets(["f"])["f"]] == [(text, 1)], name
    one.free()


@pytest.mark.parametrize("case", range(9))
def test_width_mismatch_fails_and_leaves_the_ctx_usable(env, case):
    oracle, vs, ctx = env
    name, vt, enc, text, dct = cases(vs)[case]
    rows, stored = 4, (2 if len(enc) == 1 else len(enc) // 2)   # rows * (width - stored) <= 32
    batch = upload(env, rows, dict(value_type=vt, dict=dct, lens_items=bytes([4, stored]), data=bytes(rows * stored)), text)
    assert matched(env, vs.Filter.noop(), batch) == rows
    calls = [lambda: ctx.gather_values("f"), lambda: ctx.hits_stats(10 ** 9, by=("f",)), lambda: ctx.hits_stats(1, by=("f",)),
             lambda: ctx.last_rows(rows, ("f",)), lambda: ctx.facets(["f"])]
    for call in calls:
        with pytest.raises(vs.VlscanError, match=WIDTH_MSG):
            call()
        assert ctx.gather_values("s")[0] == [text] * rows, name
    for flt in (vs.Filter.eq_field("f", "s"), vs.Filter.le_field("f", "s")):
        with pytest.raises(vs.VlscanError, match=WIDTH_MSG):
            ctx.scan_resident(vs.Program(flt), batch)
        assert matched(env, vs.Filter.noop(), batch) == rows
        assert ctx.gather_values("s")[0] == [text] * rows, name
    batch.free()
