"""GPU parity for the N newest selected rows (vlscan_last_rows, `/select/logsql/query?limit=N`; getLastNQueryResults
app/vlselect/logsql/logsql.go:1005-1080).  The expectation is brute force over the oracle: its bitmaps (Block.search), its timestamps decode and
the stored-value decode of test_gather_timestamps_and_values; the texts must also equal vlscan_gather_values at the same rows.  The blocks whose
timestamps were decoded must be exactly the model's (tests/last_rows_model.py)."""
import ctypes as C
import random

import pytest

import vlohits
from last_rows_model import I64_MIN, brute_force, gen_timestamps, model
from test_gpu_zzzzz_hits import nearest_delta, series, zstd_compress

pytestmark = pytest.mark.gpu

DAY = 86400 * 10 ** 9


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


def mixed_blocks(oracle, pu, seed, nblocks=20, scale=10 ** 9):
    """all six timestamp marshal types; blocks that overlap in time and share timestamps across blocks (a few common starting points, steps
    of 0 and 1); a field typed (uint8) in even blocks and stored as strings in odd ones; a field some blocks lack.
    -> oracle blocks, upload descriptors, timestamps per block"""
    rng = random.Random(seed)
    bases = [1_700_000_000_000_000_000 + k * 1000 for k in range(4)]
    blocks, descs, stamps = [], [], []
    for bi in range(nblocks):
        n = rng.choice([1, 64, 65, 300, 2100])
        ts = series(rng, ["const", "step", "jitter", "bursty"][bi % 4], n, scale)
        base = rng.choice(bases)
        ts = [v - ts[0] + base for v in ts]
        cols = {
            "msg": [b"row %d of block %d %s" % (i, bi, b"x" * (i % 40)) if i % 7 else b"" for i in range(n)],
            "u16": [b"%d" % (i * 37 % 60000) for i in range(n)],
            "f64": [b"%d.%d" % (i * 7 - 900, 1 + i % 97) for i in range(n)],
            "ip": [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)],
            "lvl": [[b"info", b"warn", b"error", b""][(i * 5 // 7) % 4] for i in range(n)],
            "cst": [b"same value"] * n,
            "code": [b"%d" % (200 + (i * 3) % 20) for i in range(n)] if bi % 2 == 0 else [b"x" if i == 0 else b"%d" % (200 + i % 20) for i in range(n)],
        }
        if bi % 3 == 2:
            del cols["ip"]
        blk = oracle.Block.from_columns(list(cols.items())).set_timestamps(ts)
        d = pu.oracle_block_to_desc(blk)
        if n >= 2 and bi % 5 == 3:     # NearestDelta (plain / ZSTD): the oracle's writer never picks it for sorted timestamps
            raw = nearest_delta(ts)
            d["timestamps"] = (raw, 6, ts[0], ts[-1]) if bi % 10 == 3 else (zstd_compress(raw), 4, ts[0], ts[-1])
        blocks.append(blk)
        descs.append(d)
        stamps.append(ts)
    return blocks, descs, stamps


def stored_texts(oracle, blocks):
    """what a reader of the stored blocks sees per field and row (test_gather_timestamps_and_values)"""
    out = []
    for blk in blocks:
        d = {name: [value] * blk.rows for name, value in blk.consts}
        for c in blk.columns:
            items = oracle.unmarshal_strings_block(c.values_block, blk.rows)
            d[c.name] = [c.dict[it[0]] if c.value_type == 2 else oracle.encoded_to_string(c.value_type, it) for it in items]
        out.append(d)
    return out


def expect(oracle, blocks, stamps, stored, flt, limit, floor, fields):
    """brute force over the oracle -> ([(ts, block, row, texts)], the model's decoded-block count)"""
    mblocks = []
    for blk, ts in zip(blocks, stamps):
        data, mt, mn, mx = blk.timestamps_block()
        dec = [int(v) for v in oracle.unmarshal_timestamps(data, mt, mn, blk.rows)]
        assert dec == ts
        mblocks.append((mn, mx, dec, [int(r) for r in oracle.bitmap_rows(blk.search(flt), blk.rows)]))
    rows = brute_force(mblocks, limit, floor)
    got_model, decoded = model(mblocks, limit, floor)
    assert got_model == rows
    want = [(t, bi, r, tuple(stored[bi].get(f.encode() or b"_msg", [b""] * blocks[bi].rows)[r] for f in fields)) for t, bi, r in rows]
    return want, decoded, sum(len(b[3]) for b in mblocks)


FIELD_SETS = [(), ("lvl",), ("msg", "code"), ("code", "ip", "f64"), ("nope",), ("cst", "u16")]


def test_differential_against_oracle(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = mixed_blocks(oracle, pu, 41)
    assert {d["timestamps"][1] for d in descs} == {1, 2, 3, 4, 5, 6}
    assert len({t for ts in stamps for t in ts}) < sum(len(ts) for ts in stamps)   # equal timestamps across blocks
    names = pu.field_names_of(blocks)
    batch = ctx.upload(vs.HostBlocks(names, descs))
    stored = stored_texts(oracle, blocks)
    allts = sorted(t for ts in stamps for t in ts)
    lo, hi = allts[len(allts) // 5], allts[len(allts) * 4 // 5]
    F, G = oracle.Filter, vs.Filter
    filters = [(F.noop(), G.noop()), (F.phrase("lvl", "error"), G.phrase("lvl", "error")), (F.time(lo, hi), G.time(lo, hi)),
               (F.not_(F.phrase("lvl", "warn")), G.not_(G.phrase("lvl", "warn"))), (F.phrase("msg", "absent"), G.phrase("msg", "absent"))]
    decoded_any = pruned_any = ties_any = 0
    sloped = sum(1 for ts in stamps if ts[0] != ts[-1])
    for k, (of, gf) in enumerate(filters):
        ctx.scan_resident(vs.Program(gf), batch)
        gathered = {f: ctx.gather_values(f, batch)[0] for f in ("lvl", "msg", "code", "ip", "f64", "nope", "cst", "u16")}
        _, hoffs = ctx.gather_timestamps(batch)
        hit_index = {}
        for bi in range(len(blocks)):   # (block, row) -> index of the hit in the gathers
            rows = [int(r) for r in oracle.bitmap_rows(blocks[bi].search(of), blocks[bi].rows)]
            for j, r in enumerate(rows):
                hit_index[(bi, r)] = int(hoffs[bi]) + j
        nsel = len(hit_index)
        for j, limit in enumerate((1, 7, 1000, nsel + 5)):
            for i, floor in enumerate((I64_MIN, lo, allts[len(allts) // 2] + 1, hi, allts[-1] + 1)):
                fields = FIELD_SETS[(k + j + i) % len(FIELD_SETS)]
                info = {}
                got = ctx.last_rows(limit, fields, None if floor == I64_MIN else floor, info=info)
                want, decoded, sel = expect(oracle, blocks, stamps, stored, of, limit, floor, fields)
                assert got == want, (k, limit, floor, fields)
                assert info["selected"] == sel and info["rows"] == len(want) and info["blocks_decoded"] == decoded, (k, limit, floor)
                assert info["value_bytes"] == sum(len(x) for w in want for x in w[3])
                for t, bi, r, texts in got:
                    assert texts == tuple(gathered[f][hit_index[(bi, r)]] for f in fields)
                decoded_any += decoded > 0
                pruned_any += 0 < decoded < sloped
                ties_any += len({t for t, _, _, _ in got}) < len(got)
    assert decoded_any and pruned_any and ties_any
    batch.free()


def gen_kw(vs, k, nb=40, rpb=2000):
    return dict(seed=20250718, total_rows=nb * rpb, rows_per_block=rpb, hot_block_permille=500, hit_row_permille=100,
                columns_mask=1 | 2 | vs.GEN_TIMESTAMPS | vs.gen_streams(k))


def generated_model(oracle, ocfg, batch_ctx, nb, flt, limit):
    ctx, vs, batch = batch_ctx
    words, counts = ctx.fetch(batch)
    per = vs.split_bitmaps(words, [ocfg.rows_per_block] * nb)
    mblocks = []
    for b in range(nb):
        ts = gen_timestamps(ocfg, b)
        rows = [int(r) for r in oracle.bitmap_rows(oracle.Block.generated(ocfg, b).search(flt), ocfg.rows_per_block)]
        assert rows == [int(r) for r in oracle.bitmap_rows(per[b].copy(), ocfg.rows_per_block)]
        mblocks.append((ts[0], ts[-1], ts, rows))
    return mblocks


def test_pruning_on_generated_data(env):
    """time-ordered blocks: only the newest ceil(N / R) blocks are decoded; S = 2^k interleaved blocks: every block with hits of the newest group"""
    oracle, vs, pu, ctx = env
    nb, rpb = 40, 2000
    for k, gf, of in ((0, vs.Filter.noop(), oracle.Filter.noop()), (0, vs.Filter.phrase("_msg", "error"), oracle.Filter.phrase("_msg", "error")),
                      (2, vs.Filter.noop(), oracle.Filter.noop()), (6, vs.Filter.noop(), oracle.Filter.noop())):
        every_row = gf.desc == vs.Filter.noop().desc
        kw = gen_kw(vs, k, nb, rpb)
        ocfg = oracle.GenConfig(**kw)
        batch = ctx.generate(vs.GenConfig(**kw), 0, nb)
        ctx.scan_resident(vs.Program(gf), batch)
        mblocks = generated_model(oracle, ocfg, (ctx, vs, batch), nb, of, 1000)
        for limit in (1, 1000, 4500):
            info = {}
            got = ctx.last_rows(limit, ("level",), info=info)
            want, decoded = model(mblocks, limit)
            assert want == brute_force(mblocks, limit)
            assert [(t, b, r) for t, b, r, _ in got] == want and info["blocks_decoded"] == decoded, (k, limit)
            if k == 0 and every_row:
                assert decoded == -(-limit // rpb)
            if k > 0:   # every row selected, the newest group holds more than `limit` rows
                s = 1 << k
                assert decoded == len(range((nb - 1) // s * s, nb)), (k, limit, decoded)
        batch.free()


def test_scan_result_untouched(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = mixed_blocks(oracle, pu, 5, nblocks=10)
    batch = ctx.upload(vs.HostBlocks(pu.field_names_of(blocks), descs))
    ctx.scan_resident(vs.Program(vs.Filter.phrase("lvl", "error")), batch)

    def snapshot():
        words, counts = ctx.fetch(batch)
        ts, offs = ctx.gather_timestamps(batch)
        return (words.tobytes(), counts.tobytes(), ts.tobytes(), offs.tobytes(), ctx.gather_values("msg", batch)[0], ctx.gather_values("code", batch)[0],
                ctx.hits_stats(10 ** 9, 0, 0, ("lvl", "code")))

    before = snapshot()
    first = ctx.last_rows(50, ("msg", "code"))
    with pytest.raises(vs.VlscanError):
        ctx.last_rows(5, ("_time",))
    ctx.last_rows(3, (), stamps[4][0])
    assert snapshot() == before
    assert ctx.last_rows(50, ("msg", "code")) == first
    batch.free()


def test_batch_halves_merge_to_the_whole(env):
    """Two halves of a batch, the second with the first's N-th newest timestamp as its floor; merged in (timestamp, half, block, row) order and
    cut to the last N they equal the whole batch's answer (the merge of INTEGRATION.md §3d)."""
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = mixed_blocks(oracle, pu, 9, nblocks=14)
    names = pu.field_names_of(blocks)
    half = 7
    for limit in (1, 7, 300, 100000):
        for gf in (vs.Filter.noop(), vs.Filter.phrase("lvl", "info")):
            merged, floor = [], None
            for h, part in enumerate((descs[:half], descs[half:])):
                batch = ctx.upload(vs.HostBlocks(names, part))
                ctx.scan_resident(vs.Program(gf), batch)
                res = ctx.last_rows(limit, ("msg",), floor)
                if h == 0 and len(res) == limit:
                    floor = res[0][0]
                merged += [(t, h, b, r, x) for t, b, r, x in res]
                batch.free()
            merged = sorted(merged)[-limit:]
            batch = ctx.upload(vs.HostBlocks(names, descs))
            ctx.scan_resident(vs.Program(gf), batch)
            whole = ctx.last_rows(limit, ("msg",))
            assert [(t, b + half * h, r, x) for t, h, b, r, x in merged] == whole, limit
            batch.free()


def test_error_paths_leave_the_ctx_usable(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = mixed_blocks(oracle, pu, 3, nblocks=6)
    names = pu.field_names_of(blocks)
    fresh = vs.Ctx(0)
    with pytest.raises(vs.VlscanError, match="no scan result"):
        fresh.last_rows(10)
    fresh.close()
    no_ts = ctx.upload(vs.HostBlocks(names, [{k: v for k, v in d.items() if k != "timestamps"} for d in descs]))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), no_ts)
    with pytest.raises(vs.VlscanError, match="timestamps"):
        ctx.last_rows(10, ("lvl",))
    no_ts.free()
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    want = ctx.last_rows(40, ("msg", "lvl"))
    assert len(want) == 40
    with pytest.raises(vs.VlscanError, match="_time"):
        ctx.last_rows(10, ("lvl", "_time"))
    with pytest.raises(vs.VlscanError, match="limit"):
        ctx.last_rows(0)
    assert ctx.last_rows(40, ("msg", "lvl")) == want
    # buffers too small: the call fails, writes nothing and reports the exact sizes it needs
    q, keep = vs.last_query(40, ["msg", "lvl"])
    info = (C.c_uint64 * 4)()
    rc = vs.lib().vlscan_last_rows(ctx.h, C.byref(q), None, None, None, C.c_uint64(0), None, C.c_uint64(0), None, info)
    nbytes = sum(len(x) for w in want for x in w[3])
    assert rc < 0 and list(info)[:3] == [40, nbytes, sum(d["rows"] for d in descs)]
    ts = (C.c_int64 * 40)(); b = (C.c_uint32 * 40)(); r = (C.c_uint32 * 40)(); o = (C.c_uint64 * 81)(*[7] * 81)
    rc = vs.lib().vlscan_last_rows(ctx.h, C.byref(q), ts, b, r, C.c_uint64(40), None, C.c_uint64(nbytes - 1), o, info)
    assert rc < 0 and info[1] == nbytes and list(o) == [7] * 81 and list(ts) == [0] * 40
    assert ctx.last_rows(40, ("msg", "lvl")) == want
    # a block whose decoded timestamps run past the maximum of its header
    bad = [dict(d) for d in descs]
    j = next(i for i, s in enumerate(stamps) if s[-1] - s[0] >= 2)   # still not flat with the lowered maximum
    data, mt, mn, mx = bad[j]["timestamps"]
    bad[j]["timestamps"] = (data, mt, mn, mx - 1)
    lying = ctx.upload(vs.HostBlocks(names, bad))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), lying)
    with pytest.raises(vs.VlscanError, match="header"):
        ctx.last_rows(10 ** 6)
    lying.free()
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    assert ctx.last_rows(40, ("msg", "lvl")) == want
    batch.free()


def test_generator_interleaved_timestamps(env):
    """columns_mask bits 12..16: S = 2^k interleaved blocks, byte-equal to the oracle's marshal of the interleaved series
    (last_rows_model.gen_timestamps); k = 0 is the series of vlohits.gen_timestamps, unchanged"""
    oracle, vs, pu, ctx = env
    nb, rpb = 9, 500
    for k in (0, 1, 3, 16):
        kw = gen_kw(vs, k, nb, rpb)
        kw["total_rows"] = nb * rpb - 100   # a shorter last block
        ocfg = oracle.GenConfig(**kw)
        batch = ctx.generate(vs.GenConfig(**kw), 0, nb)
        dl = ctx.download(batch)
        s = 1 << k
        for b in range(nb):
            blk = dl.blocks[b]
            series_ = gen_timestamps(ocfg, b)
            rows = min(rpb, kw["total_rows"] - b * rpb)
            assert series_ == [vs.GEN_T0 + ((b // s) * s * rpb + i * s + b % s) * vs.GEN_STEP for i in range(rows)]
            if k == 0:
                assert series_ == vlohits.gen_timestamps(ocfg, b) == [vs.GEN_T0 + (b * rpb + i) * vs.GEN_STEP for i in range(rows)]
            data, mt, first = oracle.marshal_timestamps(series_)
            assert (C.string_at(blk.timestamps, blk.timestamps_len), blk.ts_marshal_type, blk.min_timestamp, blk.max_timestamp) == (data, mt, first, series_[-1])
            assert mt == 2
        del dl
        batch.free()
    for bad in (vs.gen_streams(1), vs.gen_streams(17), 1 << 17):   # streams without bit 4, more than 2^16 streams, bits above 16
        kw = gen_kw(vs, 0, 1, 100)
        kw["columns_mask"] = 1 | (bad if bad == vs.gen_streams(1) else bad | vs.GEN_TIMESTAMPS)
        with pytest.raises(vs.VlscanError):
            ctx.generate(vs.GenConfig(**kw), 0, 1)
