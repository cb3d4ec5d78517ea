"""GPU parity for the hits aggregation, `stats by (_time:step offset off, f1, ...) count()` over the selected rows (vlscan_hits_stats;
app/vlselect/logsql/logsql.go:116-219, lib/logstorage/block_result.go:760-848), against the reference's own table (TestTruncateTimestamp)
and the CPU oracle (oracle/vlo_hits.h via oracle/vlohits.py: the oracle's bitmaps, its own timestamps decode, value decode and calendar).  Bar: equal groups, equal counts,
equal order; the blocks whose timestamps were decoded are exactly the multi-bucket blocks with hits."""
import ctypes as C
import json
import os
import random
from collections import Counter

import pytest

import vlohits

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DAY = 86400 * 10 ** 9


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


def varint(u):
    out = bytearray()
    while u >= 0x80:
        out.append(u & 0x7F | 0x80)
        u >>= 7
    out.append(u)
    return bytes(out)


def nearest_delta(ts):
    """MarshalTypeNearestDelta with precisionBits = 64: the zig-zag varints of the deltas (vm/lib/encoding/nearest_delta.go)"""
    out = b""
    for a, b in zip(ts, ts[1:]):
        d = (b - a) & ((1 << 64) - 1)
        d = d - (1 << 64) if d >> 63 else d
        out += varint(((d << 1) ^ (d >> 63)) & ((1 << 64) - 1))
    return out


def zstd_compress(data):
    z = C.CDLL("libzstd.so.1")
    z.ZSTD_compressBound.restype = C.c_size_t
    z.ZSTD_compress.restype = C.c_size_t
    cap = z.ZSTD_compressBound(C.c_size_t(len(data)))
    out = C.create_string_buffer(cap)
    n = z.ZSTD_compress(out, C.c_size_t(cap), data, C.c_size_t(len(data)), C.c_int(1))
    return out.raw[:n]


def series(rng, kind, n, scale):
    base = rng.choice([1_700_000_000_000_000_000, -5 * 10 ** 17, 1_704_067_199_000_000_000])
    if kind == "const":
        return [base] * n
    if kind == "step":
        d = rng.choice([1, 1000, scale])
        return [base + i * d for i in range(n)]
    t, out = base, []
    for _ in range(n):
        t += max(0, int(rng.gauss(scale, scale / 5))) if kind == "jitter" else rng.choice([0, 0, 0, 1, 7, scale * rng.randrange(1, 50)])
        out.append(t)
    return out


def run_both(env, blocks, descs, names, of, gf, step, offset, cal, by):
    oracle, vs, pu, ctx = env
    want_info, got_info = {}, {}
    want = vlohits.hits_stats(blocks, of, step, offset, cal, [b.encode() if isinstance(b, str) else b for b in by], info=want_info)
    got = ctx.hits_stats(step, offset, cal, by, info=got_info)
    assert got == want, (gf, step, offset, cal, by)
    assert got_info["rows"] == want_info["rows"] == sum(c for _, _, c in want)
    assert got_info["blocks_decoded"] == want_info["blocks_decoded"], (step, offset, cal)
    return got, got_info


def test_reference_table_on_device(env):
    """TestTruncateTimestamp through the kernels: a one-row block (its single bucket, no decode) and a row selected out of a two-row block
    that spans two buckets (decoded)."""
    oracle, vs, pu, ctx = env
    cases = json.load(open(os.path.join(HERE, "golden", "bucket_cases.json")))
    for c in cases:
        ts = c["ts_ns"]
        later = ts + (400 if c["calendar"] == vs.BUCKET_YEAR else 40) * DAY
        one = oracle.Block.from_columns([("x", [b"a"])]).set_timestamps([ts])
        two = oracle.Block.from_columns([("x", [b"a", b"b"])]).set_timestamps([ts, later])
        for blk, flt in ((one, vs.Filter.noop()), (two, vs.Filter.time(ts, ts))):
            batch = ctx.upload(pu.host_blocks_from_oracle([blk]))
            ctx.scan_resident(vs.Program(flt), batch)
            info = {}
            assert ctx.hits_stats(c["step_ns"], c["offset_ns"], c["calendar"], info=info) == [(c["want_ns"], (), 1)], c
            assert info["blocks_decoded"] == (0 if blk is one else 1)
            batch.free()


def block_mix(env, seed, nblocks=10, scale=10 ** 12):
    """the block mix of test_gather_timestamps_and_values plus a field stored typed in some blocks and as strings in others, and
    timestamps columns in all six marshal types"""
    oracle, vs, pu, ctx = env
    rng = random.Random(seed)
    blocks, descs, stamps, t0 = [], [], [], 1_700_000_000_000_000_000
    for bi in range(nblocks):
        n = rng.choice([1, 64, 65, 300, 2100])
        ts = series(rng, ["const", "step", "jitter", "bursty"][bi % 4], n, scale)
        ts = [v - ts[0] + t0 for v in ts]
        t0 = ts[-1] + rng.choice([1, scale, 40 * DAY])
        cols = {
            "msg": [b"row %d of block %d %s" % (i, bi, b"x" * (i % 40)) if i % 7 else b"" for i in range(n)],
            "u16": [b"%d" % (i * 37 % 60000) for i in range(n)],
            "i64": [b"%d" % ((i - n // 2) * 987654321) for i in range(n)],
            "f64": [b"%d.%d" % (i * 7 - 900, 1 + i % 97) for i in range(n)],
            "ip": [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)],
            "ts": [b"2024-03-%02dT12:%02d:%02d.%03dZ" % (1 + i % 28, i % 60, (i * 7) % 60, i % 1000) for i in range(n)],
            "lvl": [[b"info", b"warn", b"error", b""][(i * 5 // 7) % 4] for i in range(n)],
            "cst": [b"same value"] * n,
            # typed (uint8) in even blocks, strings in odd ones ("x" is no number): equal texts must meet in one group
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


def test_differential_against_oracle(env):
    oracle, vs, pu, ctx = env
    blocks, descs, stamps = block_mix(env, 31, nblocks=20)
    seen = {d["timestamps"][1] for d in descs}
    assert seen == {1, 2, 3, 4, 5, 6}, seen
    names = pu.field_names_of(blocks)
    batch = ctx.upload(vs.HostBlocks(names, descs))
    u8 = [c.value_type for b in blocks[::2] for c in b.columns if c.name == b"code"]
    st = [c.value_type for b in blocks[1::2] for c in b.columns if c.name == b"code"]
    assert set(u8) == {3} and set(st) == {1}, (u8, st)
    F, G = oracle.Filter, vs.Filter
    lo, hi = stamps[3][len(stamps[3]) // 2], stamps[15][len(stamps[15]) // 3]
    filters = [(F.noop(), G.noop()), (F.phrase("lvl", "error"), G.phrase("lvl", "error")), (F.time(lo, hi), G.time(lo, hi)), (F.phrase("msg", "absent"), G.phrase("msg", "absent"))]
    steps = [(1, 0, 0), (1000, 7, 0), (10 ** 6, -3 * 10 ** 5, 0), (10 ** 9, 0, 0), (3600 * 10 ** 9, 1800 * 10 ** 9, 0), (DAY, -2 * 3600 * 10 ** 9, 0),
             (7 * DAY, 0, vs.BUCKET_WEEK), (7 * DAY, 3 * 3600 * 10 ** 9, vs.BUCKET_WEEK), (0, 0, vs.BUCKET_MONTH), (0, -4 * 3600 * 10 ** 9, vs.BUCKET_MONTH),
             (0, 0, vs.BUCKET_YEAR), (0, 4 * 3600 * 10 ** 9, vs.BUCKET_YEAR), (10 ** 18, 0, 0), (-5, 0, 0)]
    bys = [(), ("lvl",), ("code",), ("lvl", "code"), ("msg",), ("f64", "ip", "cst"), ("u16", "i64", "ts"), ("nope", "lvl")]
    decoded_any = fast_any = groups_any = 0
    for k, (of, gf) in enumerate(filters):
        ctx.scan_resident(vs.Program(gf), batch)
        for j, (step, off, cal) in enumerate(steps):
            for by in (bys if j % 3 == k % 3 else bys[:4]):
                got, info = run_both(env, blocks, descs, names, of, gf, step, off, cal, by)
                decoded_any += info["blocks_decoded"] > 0
                fast_any += info["blocks_decoded"] < len(blocks)
                groups_any += len(got) > 1
        if k == 0:   # "200" stored as uint8 and as a string: one group
            got = ctx.hits_stats(10 ** 18, 0, 0, ("code",))
            assert [k for _, k, _ in got].count((b"205",)) == 1
    assert decoded_any and fast_any and groups_any
    batch.free()


def test_halves_add_up(env):
    oracle, vs, pu, ctx = env
    blocks, descs, _ = block_mix(env, 7, nblocks=12)
    names = pu.field_names_of(blocks)
    args = (3600 * 10 ** 9, 0, 0, ("lvl", "code"))
    total = Counter()
    for part in (descs[:6], descs[6:]):
        batch = ctx.upload(vs.HostBlocks(names, part))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        for b, keys, c in ctx.hits_stats(*args):
            total[(b, keys)] += c
        batch.free()
    batch = ctx.upload(vs.HostBlocks(names, descs))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    whole = ctx.hits_stats(*args)
    assert sorted(total.items()) == [((b, k), c) for b, k, c in whole]
    batch.free()


def test_many_distinct_keys_grow_the_table(env):
    """200 000 distinct strings: the table starts at 16 Ki slots and has to grow; every key still gets its exact count"""
    oracle, vs, pu, ctx = env
    blocks, t = [], 1_700_000_000_000_000_000
    for bi in range(100):
        n = 2000
        ts = [t + i * 10 ** 6 for i in range(n)]
        t = ts[-1] + 10 ** 6
        keys = [b"key-%06d" % ((bi * n + i) * 7919 % 200_000) for i in range(n)]
        blocks.append(oracle.Block.from_columns([("k", keys), ("m", [b"m%d" % (i % 3) for i in range(n)])]).set_timestamps(ts))
    batch = ctx.upload(pu.host_blocks_from_oracle(blocks))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
    for step, by in ((3600 * 10 ** 9, ("k",)), (10 ** 9, ("k", "m"))):
        info = {}
        got = ctx.hits_stats(step, 0, 0, by, info=info)
        want = vlohits.hits_stats(blocks, oracle.Filter.noop(), step, 0, 0, [b.encode() for b in by])
        assert got == want
        assert info["groups"] == len(want) >= 200_000
    batch.free()


def test_error_paths_leave_the_ctx_usable(env):
    oracle, vs, pu, ctx = env
    blocks, descs, _ = block_mix(env, 3, nblocks=4)
    names = pu.field_names_of(blocks)

    def good():
        batch = ctx.upload(vs.HostBlocks(names, descs))
        ctx.scan_resident(vs.Program(vs.Filter.noop()), batch)
        run_both(env, blocks, descs, names, oracle.Filter.noop(), None, 10 ** 9, 0, 0, ("lvl",))
        return batch

    fresh = vs.Ctx(0)
    with pytest.raises(vs.VlscanError, match="no scan result"):
        fresh.hits_stats(10 ** 9)
    fresh.close()
    no_ts = ctx.upload(vs.HostBlocks(names, [{k: v for k, v in d.items() if k != "timestamps"} for d in descs]))
    ctx.scan_resident(vs.Program(vs.Filter.noop()), no_ts)
    with pytest.raises(vs.VlscanError, match="timestamps"):
        ctx.hits_stats(10 ** 9, by=("lvl",))
    no_ts.free()
    batch = good()
    with pytest.raises(vs.VlscanError, match="_time"):
        ctx.hits_stats(10 ** 9, by=("_time",))
    # buffers too small: the call fails and reports the sizes it needs
    want = ctx.hits_stats(10 ** 6, 0, 0, ("msg",))
    q, keep = vs.hits_query(10 ** 6, 0, 0, ["msg"])
    info = (C.c_uint64 * 4)()
    rc = vs.lib().vlscan_hits_stats(ctx.h, C.byref(q), None, None, C.c_uint64(0), None, C.c_uint64(0), None, info)
    assert rc < 0 and info[0] == len(want) and info[1] == sum(len(k[0]) for _, k, _ in want) and info[2] == sum(c for _, _, c in want)
    b = (C.c_int64 * len(want))(); c = (C.c_uint64 * len(want))(); o = (C.c_uint64 * (len(want) + 1))()
    rc = vs.lib().vlscan_hits_stats(ctx.h, C.byref(q), b, c, C.c_uint64(len(want)), None, C.c_uint64(0), o, info)
    assert rc < 0 and info[1] > 0
    assert ctx.hits_stats(10 ** 6, 0, 0, ("msg",)) == want
    batch.free()
    good().free()


def test_generator_timestamps(env):
    """columns_mask bit 4: a DeltaConst timestamps column per block, byte-equal to the oracle's marshal of the same series"""
    oracle, vs, pu, ctx = env
    kw = dict(seed=20250718, total_rows=8 * 2000, rows_per_block=2000, hot_block_permille=500, hit_row_permille=100, columns_mask=1 | 2 | vs.GEN_TIMESTAMPS)
    ocfg, gcfg = oracle.GenConfig(**kw), vs.GenConfig(**kw)
    batch = ctx.generate(gcfg, 0, 8)
    dl = ctx.download(batch)
    oblocks = [oracle.Block.generated(ocfg, b).set_timestamps(vlohits.gen_timestamps(ocfg, b)) for b in range(8)]
    for b in range(8):
        blk = dl.blocks[b]
        series = [vs.GEN_T0 + (b * 2000 + i) * vs.GEN_STEP for i in range(2000)]
        assert series == vlohits.gen_timestamps(ocfg, b)
        data, mt, first = oracle.marshal_timestamps(series)
        assert (C.string_at(blk.timestamps, blk.timestamps_len), blk.ts_marshal_type, blk.min_timestamp, blk.max_timestamp) == (data, mt, first, series[-1])
        assert mt == 2 and oblocks[b].timestamps_block() == (data, mt, first, series[-1])
    del dl
    for gf, of in ((vs.Filter.phrase("_msg", "error"), oracle.Filter.phrase("_msg", "error")), (vs.Filter.noop(), oracle.Filter.noop())):
        ctx.scan_resident(vs.Program(gf), batch)
        for step, by in ((10 ** 9, ()), (3600 * 10 ** 9, ("level",))):
            info = {}
            got = ctx.hits_stats(step, 0, 0, by, info=info)
            want_info = {}
            assert got == vlohits.hits_stats(oblocks, of, step, 0, 0, [x.encode() for x in by], info=want_info)
            assert info["blocks_decoded"] == want_info["blocks_decoded"]
    # without bit 4 the generator's bytes are what they were
    kw["columns_mask"] = 1 | 2
    plain = ctx.generate(vs.GenConfig(**kw), 0, 8)
    a, b2 = ctx.download(plain), ctx.download(batch)
    assert all(a.blocks[i].ts_marshal_type == 0 for i in range(8))
    assert all(a.column(i, f) == b2.column(i, f) for i in range(8) for f in ("_msg", "level"))
    plain.free()
    batch.free()
