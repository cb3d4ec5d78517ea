"""GPU suite for keeping an end-to-end scan on the device (vlscan_scan_batch_keep) and staging the pipes' columns only for the blocks that need
them (vlscan_stage_selected), differential against today's path (vlscan_batch_upload of every field + vlscan_scan_resident) and against the
oracle's restatements of the hits and facets pipes.  Bar: the same bitmaps, counts, hits, gathered values and timestamps, hits groups, facets and
newest rows; only the values cells of blocks with selected rows are staged; reading a cell still on the host fails naming the field; the kept
result ends with the next scan and reuses its device memory."""
import numpy as np
import pytest

import vlohits
from test_gpu_zzzzz_hits import block_mix
from test_gpu_zzzzzzz_facets import model as facets_model

pytestmark = pytest.mark.gpu

STEP = 10 ** 9
DAY_STEP = 86400 * 10 ** 9
ACCOUNTING = ("blocks", "rows", "rows_matched", "blocks_matched", "values_bytes", "bloom_probe_bytes", "bitmap_bytes", "columns_read")
MIX_FIELDS = ["msg", "u16", "i64", "f64", "ip", "ts", "lvl", "cst", "code"]
MIX_BYS = [(), ("lvl",), ("lvl", "code"), ("msg", "u16", "ip")]
GEN_FIELDS = ["_msg", "level", "path", "status"]
GEN_BYS = [(), ("level",), ("level", "status"), ("path", "status", "_msg")]


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


@pytest.fixture(scope="module")
def mix(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = block_mix(env, 41, nblocks=20)
    assert {d["timestamps"][1] for d in descs} == {1, 2, 3, 4, 5, 6}
    return blocks, vs.HostBlocks(pu.field_names_of(blocks), descs), stamps


@pytest.fixture(scope="module")
def gen(env):
    """generated rows re-encoded into the on-disk form (vlscan_host_blocks_compress), pinned"""
    oracle, vs, pu, ctx = env
    kw = dict(seed=20251015, total_rows=12 * 3000, rows_per_block=3000, hot_block_permille=250, hit_row_permille=40, columns_mask=0x1F)
    b = ctx.generate(vs.GenConfig(**kw), 0, 12)
    host = ctx.download(b)
    b.free()
    hb = host.compress()
    hb._host = host   # the compressed descriptors still point at the downloaded timestamps
    hb.oracle_blocks = [oracle.Block.generated(oracle.GenConfig(**kw), i) for i in range(12)]
    return hb


def results(ctx, fields, bys, nblocks):
    out = {}
    words, counts = ctx.fetch()
    out["words"], out["counts"] = words.tobytes(), counts.tobytes()
    out["hit_rows"] = ctx.fetch_hits()[0].tobytes()
    out["digest"] = ctx.result_digest(0, nblocks)
    for f in fields:
        out["values", f] = ctx.gather_values(f)[0]
    out["ts"] = ctx.gather_timestamps()[0].tobytes()
    for by in bys:
        out["hits", by] = ctx.hits_stats(STEP, 0, 0, by)
    out["facets"] = ctx.facets(fields + ["_time"])
    out["last"] = ctx.last_rows(25, fields)
    return out


def values_cells(hb, fields, blocks):
    """(block, field) cells of `blocks` that are values columns of one of `fields`, from the descriptors"""
    idx = [hb.field_names.index(f.encode()) for f in fields]
    n = 0
    for b in blocks:
        blk = hb.blocks[b]
        n += sum(1 for k in range(blk.ncols) if blk.cols[k].kind == 2 and blk.cols[k].field in idx)
    return n


def oracle_hit_blocks(oracle, blocks, of):
    """indexes of the blocks in which the oracle's filter selects a row"""
    return [i for i, blk in enumerate(blocks) if oracle.bitmap_rows(blk.search(of), blk.rows)]


def assert_lazy_counts(hb, info, fields, prog, hit_blocks):
    """stage_selected over the blocks with hits: every values cell of `fields` there is staged now or was before, and the cells of output fields
    (which the keep call never stages) are all staged now"""
    prog_fields = {f.decode() for f in prog.fields()}
    assert info["staged"] + info["already_staged"] == values_cells(hb, fields, hit_blocks)
    assert info["already_staged"] <= values_cells(hb, [f for f in fields if f in prog_fields], hit_blocks)


def keep_then_resident(env, hb, gf, fields, bys):
    oracle, vs, pu, ctx = env
    prog = vs.Program(gf)
    kw, kc, kst = ctx.scan_batch_keep(prog, hb)
    kw, kc = kw.copy(), kc.copy()
    hit_blocks = [b for b in range(hb.nblocks) if kc[b]]
    info = ctx.stage_selected(hb, fields)
    assert info["staged"] + info["already_staged"] == values_cells(hb, fields, hit_blocks), gf
    again = ctx.stage_selected(hb, fields)
    assert again["staged"] == 0 and again["already_staged"] == info["staged"] + info["already_staged"] and again["h2d_bytes"] == 0
    got = results(ctx, fields, bys, hb.nblocks)
    batch = ctx.upload(hb)
    ctx.scan_resident(prog, batch)
    want = results(ctx, fields, bys, hb.nblocks)
    batch.free()
    assert got.keys() == want.keys()
    for k in got:
        assert got[k] == want[k], (gf, k)
    sw, sc, sst = ctx.scan_batch(prog, hb)
    assert np.array_equal(sw, kw) and np.array_equal(sc, kc), gf
    for k in ACCOUNTING:
        assert getattr(kst, k) == getattr(sst, k), (gf, k)
    return info, hit_blocks


def mix_programs(vs, stamps):
    G = vs.Filter
    lo, hi = stamps[3][len(stamps[3]) // 2], stamps[15][len(stamps[15]) // 3]
    return [G.phrase("lvl", "error"), G.and_([G.phrase("msg", "row"), G.phrase("lvl", "warn")]), G.or_([G.phrase("lvl", "error"), G.exact("code", "205")]),
            G.not_(G.phrase("lvl", "info")), G.regexp("msg", "block 1[0-9] x"), G.time(lo, hi), G.not_(G.time(lo, hi)), G.eq_field("u16", "code"), G.noop()]


def test_differential_oracle_blocks(env, mix):
    oracle, vs, pu, ctx = env
    blocks, hb, stamps = mix
    for gf in mix_programs(vs, stamps):
        info, hit_blocks = keep_then_resident(env, hb, gf, MIX_FIELDS, MIX_BYS)
        if not vs.Program(gf).fields():   # no filter field: every values cell of a block with hits is staged here, nothing before
            assert info["already_staged"] == 0 and info["staged"] == values_cells(hb, MIX_FIELDS, hit_blocks)
            assert info["h2d_bytes"] > 0 and info["frames"] > 0


def test_differential_generated_ondisk(env, gen):
    oracle, vs, pu, ctx = env
    G = vs.Filter
    for gf in (G.phrase("_msg", "error"), G.noop(), G.regexp("_msg", "err.r"), G.not_(G.phrase("_msg", "error")), G.and_([G.phrase("_msg", "error"), G.phrase("level", "error")])):
        info, hit_blocks = keep_then_resident(env, gen, gf, GEN_FIELDS, GEN_BYS)
        prog_fields = [f.decode() for f in vs.Program(gf).fields()]
        if gf.desc.startswith("'_msg':'error'"):
            # the bloom filters rule out most blocks: their output columns never crossed PCIe
            assert hit_blocks == oracle_hit_blocks(oracle, gen.oracle_blocks, oracle.Filter.phrase("_msg", "error"))
            assert len(hit_blocks) < gen.nblocks
            assert info["staged"] == values_cells(gen, [f for f in GEN_FIELDS if f not in prog_fields], hit_blocks)


def test_against_restatements(env, mix):
    oracle, vs, pu, ctx = env
    blocks, hb, stamps = mix
    for of, gf in ((oracle.Filter.phrase("lvl", "error"), vs.Filter.phrase("lvl", "error")), (oracle.Filter.noop(), vs.Filter.noop())):
        prog = vs.Program(gf)
        ctx.scan_batch_keep(prog, hb)
        staged = ["lvl", "code", "msg", "u16"]
        assert_lazy_counts(hb, ctx.stage_selected(hb, staged), staged, prog, oracle_hit_blocks(oracle, blocks, of))
        for by in ((), (b"lvl",), (b"lvl", b"code")):
            assert ctx.hits_stats(STEP, 0, 0, by) == vlohits.hits_stats(blocks, of, STEP, 0, 0, list(by), info={})
        fields = ["lvl", "code", "u16", "_time", "cst"]
        want, rows, _ = facets_model(oracle, blocks, of, fields)
        assert ctx.facets(fields) == want


def test_only_needed_cells_are_staged_for_last_rows(env, mix, gen):
    """the two-call newest-rows flow: the rows chosen without fields, their distinct blocks staged, the same rows with their fields"""
    oracle, vs, pu, ctx = env
    for hb, fields, probe in ((mix[1], MIX_FIELDS, "lvl"), (gen, GEN_FIELDS, "_msg")):
        for gf in (vs.Filter.noop(), vs.Filter.phrase(probe, "error")):
            prog = vs.Program(gf)
            ctx.scan_batch_keep(prog, hb)
            for limit in (1, 7, 1000):
                first = ctx.last_rows(limit)
                chosen = sorted({b for _, b, _, _ in first})
                info = ctx.stage_selected(hb, fields, blocks=chosen)
                assert info["staged"] + info["already_staged"] == values_cells(hb, fields, chosen)
                second = ctx.last_rows(limit, fields)
                assert [r[:3] for r in second] == [r[:3] for r in first]   # deterministic selection, untouched scan result
            got = ctx.last_rows(1000, fields)
            batch = ctx.upload(hb)
            ctx.scan_resident(prog, batch)
            assert ctx.last_rows(1000, fields) == got
            batch.free()
    # with no filter field, the first stage_selected of a keep stages exactly the values cells of the returned rows' blocks
    hb = mix[1]
    ctx.scan_batch_keep(vs.Program(vs.Filter.noop()), hb)
    chosen = sorted({b for _, b, _, _ in ctx.last_rows(50)})
    assert ctx.stage_selected(hb, MIX_FIELDS, blocks=chosen)["staged"] == values_cells(hb, MIX_FIELDS, chosen)


def test_empty_field_list_and_empty_batch(env, mix):
    """`* | hits` and `_time:[a, b] | hits` without by-fields: no field at all; and a batch without blocks"""
    oracle, vs, pu, ctx = env
    blocks, hb, stamps = mix
    bare = vs.HostBlocks([], [dict(rows=b.rows, columns=[], timestamps=b.timestamps_block()) for b in blocks])
    lo, hi = stamps[3][len(stamps[3]) // 2], stamps[15][len(stamps[15]) // 3]
    for hbx in (bare, vs.HostBlocks(MIX_FIELDS, [])):
        for gf in (vs.Filter.noop(), vs.Filter.time(lo, hi)):
            prog = vs.Program(gf)
            kw, kc, kst = ctx.scan_batch_keep(prog, hbx)
            kw, kc = kw.copy(), kc.copy()
            def answers():
                return ctx.hits_stats(STEP), ctx.hits_stats(DAY_STEP), (ctx.last_rows(10) if hbx.nblocks else None)
            got = answers()
            sw, sc, sst = ctx.scan_batch(prog, hbx)
            assert np.array_equal(sw, kw) and np.array_equal(sc, kc), (gf, hbx.nblocks)
            for k in ACCOUNTING + ("staged_columns", "pruned_columns"):
                assert getattr(kst, k) == getattr(sst, k), (gf, k)
            batch = ctx.upload(hbx)
            ctx.scan_resident(prog, batch)
            assert got == answers(), (gf, hbx.nblocks)
            batch.free()
            assert (sum(c for _, _, c in got[0]) == 0) == (hbx.nblocks == 0 or not kc.any())


def test_stats_equal_scan_batch(env, mix, gen):
    """with the probe forced on and off, keep returns vlscan_scan_batch's counters (host->device bytes, launches and timings aside)"""
    import os
    oracle, vs, pu, ctx = env
    old = os.environ.get("VLSCAN_BLOOM_FIRST")
    try:
        for mode in ("0", "2"):
            os.environ["VLSCAN_BLOOM_FIRST"] = mode
            for hbx, gf in ((mix[1], vs.Filter.phrase("lvl", "error")), (gen, vs.Filter.phrase("_msg", "error")), (mix[1], vs.Filter.noop())):
                prog = vs.Program(gf)
                _, _, kst = ctx.scan_batch_keep(prog, hbx)
                _, _, sst = ctx.scan_batch(prog, hbx)
                for k in ACCOUNTING + ("staged_columns", "pruned_columns"):
                    assert getattr(kst, k) == getattr(sst, k), (mode, gf, k)
                if mode == "2" and prog.fields():
                    assert kst.pruned_columns > 0
    finally:
        if old is None:
            os.environ.pop("VLSCAN_BLOOM_FIRST", None)
        else:
            os.environ["VLSCAN_BLOOM_FIRST"] = old


def test_unstaged_reads_fail_cleanly(env, mix):
    oracle, vs, pu, ctx = env
    blocks, hb, stamps = mix
    prog = vs.Program(vs.Filter.noop())
    ctx.scan_batch_keep(prog, hb)
    with pytest.raises(vs.VlscanError, match="`msg`"):
        ctx.gather_values("msg")
    with pytest.raises(vs.VlscanError, match="`u16`"):
        ctx.hits_stats(STEP, 0, 0, ("u16",))
    with pytest.raises(vs.VlscanError, match="`f64`"):
        ctx.facets(["cst", "f64"])
    with pytest.raises(vs.VlscanError, match="`i64`"):
        ctx.last_rows(5, ["i64"])
    # const cells and timestamps are readable at once; the scan result is intact
    assert ctx.gather_values("cst")[0] == [b"same value"] * sum(b.rows for b in blocks)
    assert len(ctx.gather_timestamps()[0]) == sum(b.rows for b in blocks)
    ctx.stage_selected(hb, ["msg", "u16", "f64", "i64"])
    got = (ctx.gather_values("msg")[0], ctx.hits_stats(STEP, 0, 0, ("u16",)), ctx.facets(["cst", "f64"]), ctx.last_rows(5, ["i64"]))
    batch = ctx.upload(hb)
    ctx.scan_resident(prog, batch)
    assert got == (ctx.gather_values("msg")[0], ctx.hits_stats(STEP, 0, 0, ("u16",)), ctx.facets(["cst", "f64"]), ctx.last_rows(5, ["i64"]))
    batch.free()


def test_argument_errors(env, mix):
    oracle, vs, pu, ctx = env
    blocks, hb, stamps = mix
    fresh = vs.Ctx(0)
    with pytest.raises(vs.VlscanError, match="no kept scan"):
        fresh.stage_selected(hb, ["msg"])
    fresh.close()
    prog = vs.Program(vs.Filter.phrase("lvl", "error"))
    ctx.scan_batch_keep(prog, hb)
    with pytest.raises(vs.VlscanError, match="`nope`"):
        ctx.stage_selected(hb, ["msg", "nope"])
    with pytest.raises(vs.VlscanError, match="outside"):
        ctx.stage_selected(hb, ["msg"], blocks=[0, hb.nblocks])
    names = pu.field_names_of(blocks)
    fewer = vs.HostBlocks(names, [pu.oracle_block_to_desc(b) for b in blocks[:-1]])
    with pytest.raises(vs.VlscanError, match="differ"):
        ctx.stage_selected(fewer, ["msg"])
    other = [pu.oracle_block_to_desc(b) for b in blocks]
    other[2] = pu.oracle_block_to_desc(blocks[3])   # another block's columns in place of block 2
    with pytest.raises(vs.VlscanError, match="differ"):
        ctx.stage_selected(vs.HostBlocks(names, other), ["msg"], blocks=[2])
    decoded = pu.host_blocks_from_oracle(blocks, stage="decoded")   # same cells, another stage
    with pytest.raises(vs.VlscanError, match="differ"):
        ctx.stage_selected(decoded, ["msg"], blocks=[0])
    # decoded descriptors: lens items and data are checked each, not by their sum
    ddescs = [pu.oracle_block_to_desc(b, "decoded") for b in blocks]
    ctx.scan_batch_keep(prog, vs.HostBlocks(names, ddescs))
    shifted = [dict(d, columns=[dict(c) for c in d["columns"]]) for d in ddescs]
    col = next(c for c in shifted[1]["columns"] if c["field"] == b"msg" and c["kind"] == "values")
    col["lens_items"], col["data"] = col["lens_items"][:-1], col["data"] + b"x"
    with pytest.raises(vs.VlscanError, match="differ"):
        ctx.stage_selected(vs.HostBlocks(names, shifted), ["msg"], blocks=[1])
    assert ctx.stage_selected(vs.HostBlocks(names, ddescs), ["msg"], blocks=[1])["staged"] == 1
    ctx.scan_batch_keep(prog, hb)
    # none of this touched the kept result
    assert ctx.stage_selected(hb, ["msg"])["staged"] >= 0
    assert ctx.gather_values("msg")[0]
    # a later scan ends it
    ctx.scan_batch(prog, hb)
    with pytest.raises(vs.VlscanError, match="no scan result"):
        ctx.gather_values("msg")
    with pytest.raises(vs.VlscanError, match="no kept scan"):
        ctx.stage_selected(hb, ["msg"])
    ctx.scan_batch_keep(prog, hb)
    batch = ctx.upload(hb)
    ctx.scan_resident(prog, batch)
    with pytest.raises(vs.VlscanError, match="no kept scan"):
        ctx.stage_selected(hb, ["msg"])
    batch.free()


def test_repeated_keeps_reuse_device_memory(env, gen):
    oracle, vs, pu, ctx = env
    import torch
    torch.cuda.mem_get_info(0)   # the runtime's own context first
    c2 = vs.Ctx(0)
    prog = vs.Program(vs.Filter.phrase("_msg", "error"))
    free = []
    for _ in range(3):
        c2.scan_batch_keep(prog, gen)
        c2.stage_selected(gen, GEN_FIELDS)
        c2.last_rows(100, GEN_FIELDS)
        c2.facets(GEN_FIELDS)
        c2.sync()
        free.append(torch.cuda.mem_get_info(0)[0])
    c2.close()
    assert free[0] == free[1] == free[2], free
