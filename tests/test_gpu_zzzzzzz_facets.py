"""GPU parity for the facets state of a batch (vlscan_facets; `| facets`, lib/logstorage/pipe_facets.go:162-307) against both restatements,
tests/facets_model.py and the C++ shard of tests/facets_oracle/vlo_facets.h, fed from the oracle's own blocks: its bitmaps, and the values and
timestamps decoded from the stored bytes.  Bar: the same
kept / dropped fields, the same entries with the same classes, texts, hits and order; the blocks whose timestamps were decoded are exactly the
blocks with hits whose minimum and maximum timestamps differ."""
import ctypes as C
import json
import os

import pytest

import facets_model as fm
import vlofacets
import vlohits
from test_gpu_zzzzz_hits import block_mix

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


def model(oracle, blocks, flt, fields, max_values=0, max_len=0):
    sh = fm.Shard(max_values, max_len)
    decoded = 0
    for blk in blocks:
        sel = oracle.bitmap_rows(blk.search(flt), blk.rows)
        if sel and "_time" in fields:
            _, _, mn, mx = blk.timestamps_block()
            decoded += mn != mx
        sh.block(fm.oracle_cells(blk, fields, oracle) if sel else {}, sel)
    return sh.state(fields), sh.rows, decoded


def run_both(env, blocks, of, fields, max_values=0, max_len=0):
    oracle, vs, pu, ctx = env
    info = {}
    got = ctx.facets(fields, max_values, max_len, info=info)
    want, rows, decoded = model(oracle, blocks, of, fields, max_values, max_len)
    assert vlofacets.facets(blocks, of, fields, max_values, max_len)[:3] == (want, rows, decoded)
    assert got == want, (fields, max_values, max_len)
    assert info["rows"] == rows and info["blocks_decoded"] == decoded
    return got, info


def test_differential_against_oracle(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = block_mix(env, 41, nblocks=20)
    assert {d["timestamps"][1] for d in descs} == {1, 2, 3, 4, 5, 6}
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    F, G = oracle.Filter, vs.Filter
    lo, hi = stamps[3][len(stamps[3]) // 2], stamps[15][len(stamps[15]) // 3]
    filters = [(F.noop(), G.noop()), (F.phrase("lvl", "error"), G.phrase("lvl", "error")), (F.time(lo, hi), G.time(lo, hi)), (F.phrase("msg", "absent"), G.phrase("msg", "absent"))]
    fields = ["msg", "u16", "i64", "f64", "ip", "ts", "lvl", "cst", "code", "_time", "nope"]
    seen = set()
    for of, gf in filters:
        ctx.scan_resident(vs.Program(gf), batch)
        for mv, ml in ((0, 0), (3, 0), (20, 0), (200000, 0), (0, 3), (0, 4), (0, 8), (0, 19), (0, 20), (0, 21), (0, 24), (0, 29), (50, 12), (2 ** 64 - 1, 0)):
            got, info = run_both(env, blocks, of, fields, mv, ml)
            seen |= {(f, st is None) for f, st in got.items()}
            seen.add(("decoded", info["blocks_decoded"] > 0))
    assert all((f, d) in seen for f in fields[:-1] for d in (False, True)), sorted(seen)
    assert ("decoded", True) in seen
    batch.free()


def test_flat_time_blocks_are_not_decoded(env):
    oracle, vs, pu, ctx = env
    blocks = [oracle.Block.from_columns([("k", [b"a", b"b", b"-0", b"0"] * 25)]).set_timestamps([1_700_000_000_000_000_000 + b * 10 ** 9] * 100) for b in range(6)]
    blocks.append(oracle.Block.from_columns([("k", [b"c"] * 3)]).set_timestamps([5, 6, 6]))
    batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    got, info = run_both(env, blocks, oracle.Filter.noop(), ["_time", "k"])
    assert info["blocks_decoded"] == 1
    # "-0" and "0" both print as 0 but are two entries; ties go by text, then class
    assert got["k"] == [(vs.FACET_UINT64, b"0", 150), (vs.FACET_NEGATIVE, b"0", 150), (vs.FACET_STRING, b"a", 150), (vs.FACET_STRING, b"b", 150), (vs.FACET_STRING, b"c", 3)]
    assert got["_time"][0] == (vs.FACET_STRING, b"2023-11-14T22:13:20Z", 100)
    batch.free()


QUIRKS = [b"1_000", b"1000", b"_", b"-_", b"_01", b"0123", b"0_1", b"-0", b"0", b"-", b"1" + b"_" * 25, b"1" + b"_" * 26, b"-9223372036854775808",
          b"-9223372036854775809", b"18446744073709551615", b"18446744073709551616", b"12345678901", b"-7", b""]


def test_key_class_quirks_on_device(env):
    """texts tryParseUint64 / tryParseInt64 read as numbers or not, in strings, dict and const cells, next to uint64 and int64 columns"""
    oracle, vs, pu, ctx = env
    n = len(QUIRKS)
    us, is_ = (0, 1000, 1, 12345678901, 2 ** 64 - 1, 7, 300, 65536, 9), (-(1 << 63), 0, -1, 1000, -12345678901, 5, 300, -300, 9)
    blocks = [oracle.Block.from_columns([("k", QUIRKS * 3), ("u", [b"%d" % us[r % 9] for r in range(3 * n)]),
                                         ("i", [b"%d" % is_[r % 9] for r in range(3 * n)])]).set_timestamps(list(range(3 * n))),
              oracle.Block.from_columns([("k", [b"1_000", b"-0", b"0", b"0123", b"-_", b"_01"]), ("u", [b"-0"] * 6), ("i", [b"_"] * 6)]).set_timestamps([5] * 6),
              oracle.Block.from_columns([("k", [b"18446744073709551615"] * 4)]).set_timestamps([1, 2, 3, 4])]
    assert {c.value_type for c in blocks[0].columns} == {1, 6, 10}
    assert {c.value_type for c in blocks[1].columns if c.name == b"k"} == {2} and blocks[1].consts and blocks[2].consts
    batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    for ml in (0, 1, 2, 4, 10, 11, 19, 20, 21, 22, 26, 27):
        got, _ = run_both(env, blocks, oracle.Filter.noop(), ["k", "u", "i"], 0, ml)
    got, _ = run_both(env, blocks, oracle.Filter.noop(), ["k", "u", "i"])
    k = {(c, t): h for c, t, h in got["k"]}
    assert k[(vs.FACET_UINT64, b"1000")] == 3 * 2 + 1 and k[(vs.FACET_NEGATIVE, b"0")] == 3 * 2 + 2 and k[(vs.FACET_UINT64, b"1")] == 3 * 2 + 1
    assert (vs.FACET_STRING, b"0123") in k and (vs.FACET_STRING, b"-9223372036854775809") in k and (vs.FACET_NEGATIVE, b"-9223372036854775808") in k
    assert k[(vs.FACET_UINT64, b"18446744073709551615")] == 3 + 4
    batch.free()


def test_golden_cases_on_device(env):
    oracle, vs, pu, ctx = env
    for c in json.load(open(os.path.join(HERE, "golden", "facets_cases.json"))):
        blocks = [oracle.Block.from_columns([(n, [v.encode()]) for n, v in row]).set_timestamps([i]) for i, row in enumerate(c["rows"])]
        fields = sorted({n for row in c["rows"] for n, _ in row})
        batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        info = {}
        state = ctx.facets(fields, info=info)
        got = vs.facets_merge([(state, info["rows"])], c["limit"], c["keep_const_fields"])
        assert [(f, t.decode(), h) for f, t, h in got] == [tuple(w) for w in c["want"]], c["pipe"]
        batch.free()


def generated(env, nblocks=8, rows=2000):
    oracle, vs, pu, ctx = env
    kw = dict(seed=20250718, total_rows=nblocks * rows, rows_per_block=rows, hot_block_permille=500, hit_row_permille=100, columns_mask=0x1F)
    ocfg = oracle.GenConfig(**kw)
    oblocks = [oracle.Block.generated(ocfg, b).set_timestamps(vlohits.gen_timestamps(ocfg, b)) for b in range(nblocks)]
    return oblocks, ctx.generate(vs.GenConfig(**kw), 0, nblocks)


def test_generated_data(env):
    oracle, vs, pu, ctx = env
    oblocks, batch = generated(env)
    fields = ["_msg", "level", "path", "status", "_time"]
    for gf, of in ((vs.Filter.phrase("_msg", "error"), oracle.Filter.phrase("_msg", "error")), (vs.Filter.noop(), oracle.Filter.noop())):
        ctx.scan_resident(vs.Program(gf), batch)
        for mv in (0, 200000):
            got, info = run_both(env, oblocks, of, fields, mv)
            assert got["level"] is not None and got["status"] is not None
            if mv:
                assert got["path"] is not None and got["_time"] is not None
    batch.free()


def test_halves_merge_to_the_whole(env):
    oracle, vs, pu, ctx = env
    blocks, descs, _ = block_mix(env, 9, nblocks=12)
    names = pu.field_names_of(blocks)
    fields = ["lvl", "code", "u16", "cst", "_time", "msg"]
    parts = []
    for part in (descs[:5], descs[5:]):
        batch = ctx.upload(vs.HostBlocks(names, part))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        info = {}
        parts.append((ctx.facets(fields, 500, info=info), info["rows"]))
        batch.free()
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    info = {}
    whole = ctx.facets(fields, 500, info=info)
    for limit, keep in ((10, False), (3, True), (1 << 30, True)):
        assert vs.facets_merge(parts, limit, keep, 500) == vs.facets_merge([(whole, info["rows"])], limit, keep, 500)
    batch.free()


def test_other_calls_unchanged_after_facets(env):
    oracle, vs, pu, ctx = env
    blocks, descs, _ = block_mix(env, 5, nblocks=8)
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    ctx.scan_resident(vs.Program(vs.Filter.phrase("lvl", "warn")), batch)

    def snapshot():
        words, counts = ctx.fetch()
        return (words.tobytes(), counts.tobytes(), ctx.gather_values("msg")[0], ctx.gather_values("u16")[0], ctx.gather_timestamps()[0].tobytes(),
                ctx.hits_stats(10 ** 9, 0, 0, ("lvl",)), ctx.last_rows(7, ("msg",)))
    before = snapshot()
    ctx.facets(["msg", "u16", "lvl", "_time"])
    assert snapshot() == before
    batch.free()


def test_error_paths_leave_the_ctx_usable(env):
    oracle, vs, pu, ctx = env
    blocks, descs, _ = block_mix(env, 3, nblocks=4)
    names = pu.field_names_of(blocks)
    fresh = vs.Ctx(0)
    with pytest.raises(vs.VlscanError, match="no scan result"):
        fresh.facets(["lvl"])
    fresh.close()
    no_ts = ctx.upload(vs.HostBlocks(names, [{k: v for k, v in d.items() if k != "timestamps"} for d in descs]))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), no_ts)
    with pytest.raises(vs.VlscanError, match="timestamps"):
        ctx.facets(["lvl", "_time"])
    assert ctx.facets(["lvl"])["lvl"]
    no_ts.free()
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    for bad in (["_stream"], ["lvl", "lvl"], []):
        with pytest.raises(vs.VlscanError):
            ctx.facets(bad)
    want = ctx.facets(["msg", "lvl"], 100000)
    ents = [e for f in ("msg", "lvl") for e in want[f]]
    q, keep = vs.facets_query(["msg", "lvl"], 100000)
    info = (C.c_uint64 * 4)()
    d = (C.c_uint8 * 2)(); fo = (C.c_uint64 * 3)(); vo = (C.c_uint64 * (len(ents) + 1))()
    rc = vs.lib().vlscan_facets(ctx.h, C.byref(q), d, fo, None, None, C.c_uint64(0), None, C.c_uint64(0), vo, info)
    assert rc < 0 and info[0] == len(ents) and info[1] == sum(len(t) for _, t, _ in ents) and info[2] == sum(b.rows for b in blocks)
    assert ctx.facets(["msg", "lvl"], 100000) == want
    run_both(env, blocks, oracle.Filter.noop(), ["lvl", "_time", "msg"])
    batch.free()
