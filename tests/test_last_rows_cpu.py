"""CPU suite for the N newest selected rows (vlscan_last_rows, `/select/logsql/query?limit=N`, getLastNQueryResults
app/vlselect/logsql/logsql.go:1005-1080): the executable model of the device algorithm (block threshold from the headers, weighted radix select,
exact top N with the tie rule, floor) against brute-force sorting, and the ABI: struct layout, argument checks, loud failure without a device."""
import ctypes as C
import random

from last_rows_model import I64_MAX, I64_MIN, brute_force, model, radix_select
from victorialogs_b200 import scan as vs


def random_blocks(rng):
    regime = rng.randrange(5)
    if regime == 0:
        base = I64_MAX - rng.randrange(1000)          # top of int64
    elif regime == 1:
        base = I64_MIN + rng.randrange(1000)          # bottom of int64
    elif regime == 2:
        base = rng.randint(-50, 50)                   # around zero: the sign bit flips inside the data
    else:
        base = 1_700_000_000_000_000_000
    blocks = []
    for _ in range(rng.randint(0, 8)):
        n = rng.randint(1, 24)
        t = base + rng.randint(-20, 20)
        kind = rng.randrange(4)
        ts = []
        for _ in range(n):
            if kind == 1:
                t += rng.choice([0, 0, 1, 3])             # many equal timestamps
            elif kind == 2:
                t += rng.randrange(10)
            elif kind == 3:
                t += rng.choice([0, 1, 1000])
            ts.append(t)                                  # kind 0: a const block
        ts = [min(max(v, I64_MIN), I64_MAX) for v in ts]
        ts.sort()
        p = rng.choice([0.0, 0.3, 1.0, rng.random()])
        sel = [r for r in range(n) if rng.random() < p]
        blocks.append((ts[0], ts[-1], ts, sel))
    return blocks


def test_model_against_brute_force():
    rng = random.Random(2024)
    seen = set()
    for case in range(12_000):
        blocks = random_blocks(rng)
        stamps = [t for b in blocks for t in b[2]] or [0]
        fk = rng.randrange(5)
        floor = I64_MIN if fk == 0 else rng.choice(stamps) + (fk - 3 if fk > 1 else 0)   # at, just above / below a row, or none
        floor = min(max(floor, I64_MIN), I64_MAX)
        nsel = sum(len(b[3]) for b in blocks)
        limit = rng.choice([1, 2, 3, 7, nsel, nsel + 1, 1000, rng.randint(1, nsel + 3)]) or 1
        got, decoded = model(blocks, limit, floor)
        assert got == brute_force(blocks, limit, floor), (case, blocks, limit, floor)
        # decoded: exactly the blocks with hits that are not flat and whose maximum reaches T_lo
        sel = radix_select([(b[0], len(b[3])) for b in blocks if b[3] and b[0] >= floor], limit)
        t_lo = floor if sel is None else sel[0]
        assert decoded == sum(1 for b in blocks if b[3] and b[0] != b[1] and b[1] >= t_lo)
        assert all(blocks[bi][1] >= t_lo for _, bi, _ in got)
        seen.add((len(got) == limit, len(got) < limit, floor > I64_MIN, any(b[0] == b[1] for b in blocks if b[3])))
    assert len(seen) >= 8, seen


def test_radix_select_both_ends_and_weights():
    keys = [(I64_MIN, 3), (I64_MAX, 2), (-1, 1), (0, 4), (I64_MAX - 1, 1)]
    assert radix_select(keys, 1) == (I64_MAX, 1)
    assert radix_select(keys, 2) == (I64_MAX, 2)
    assert radix_select(keys, 3) == (I64_MAX - 1, 1)
    assert radix_select(keys, 5) == (0, 2)
    assert radix_select(keys, 8) == (-1, 1)
    assert radix_select(keys, 11) == (I64_MIN, 3)
    assert radix_select(keys, 12) is None
    assert radix_select([(5, 0)], 1) is None


def test_pruning_count_of_the_model():
    """time-ordered blocks of R rows, all selected: the newest ceil(N / R) blocks are decoded; interleaved blocks: all of them"""
    R = 100
    ordered = [(b * R, b * R + R - 1, list(range(b * R, b * R + R)), list(range(R))) for b in range(20)]
    for limit, want in ((1, 1), (100, 1), (101, 2), (250, 3), (2000, 20), (5000, 20)):
        got, decoded = model(ordered, limit)
        assert got == brute_force(ordered, limit) and decoded == want, (limit, decoded)
    S = 8
    inter = [(b, (R - 1) * S + b, [i * S + b for i in range(R)], list(range(R))) for b in range(S)]
    got, decoded = model(inter, 10)
    assert got == brute_force(inter, 10) and decoded == S
    flat = [(7, 7, [7] * R, list(range(R))) for _ in range(4)]
    got, decoded = model(flat, 150)
    assert got == brute_force(flat, 150) and decoded == 0
    assert got[0] == (7, 2, 50)   # ties: the later blocks and rows win


def test_last_query_layout():
    # include/vlscan.h, x86-64 SysV: u64, i64, u32 (+ 4 bytes padding), two pointers
    assert C.sizeof(vs.LastQuery) == 8 + 8 + 8 + 8 + 8
    assert vs.LastQuery.limit.offset == 0 and vs.LastQuery.min_timestamp.offset == 8 and vs.LastQuery.nfields.offset == 16
    assert vs.LastQuery.field_names.offset == 24 and vs.LastQuery.field_name_lens.offset == 32
    q, keep = vs.last_query(5, ["level"])
    assert (q.limit, q.min_timestamp, q.nfields) == (5, I64_MIN, 1)


def _call_without_ctx(limit, fields, info_init=7):
    q, keep = vs.last_query(limit, fields, 123)
    info = (C.c_uint64 * 4)(*[info_init] * 4)
    ts = (C.c_int64 * 4)(); b = (C.c_uint32 * 4)(); r = (C.c_uint32 * 4)(); o = (C.c_uint64 * 32)(); vb = C.create_string_buffer(64)
    rc = vs.lib().vlscan_last_rows(None, C.byref(q), ts, b, r, C.c_uint64(4), vb, C.c_uint64(64), o, info)
    return rc, vs.lib().vlscan_last_error(None).decode(), list(info)


def test_last_rows_fails_loudly_without_a_device():
    rc, err, info = _call_without_ctx(10, ["level", ""])
    assert rc != 0 and "CUDA device" in err
    assert info == [0, 0, 0, 0]


def test_last_rows_rejects_bad_queries():
    rc, err, _ = _call_without_ctx(0, [])
    assert rc < 0 and "limit" in err
    rc, err, _ = _call_without_ctx(3, ["level", "_time"])
    assert rc < 0 and "_time" in err
    assert vs.lib().vlscan_last_rows(None, None, None, None, None, C.c_uint64(0), None, C.c_uint64(0), None, None) < 0
    assert "query" in vs.lib().vlscan_last_error(None).decode()


def test_generator_streams_bits():
    assert vs.gen_streams(0) == 0 and vs.gen_streams(16) == 16 << 12 and vs.GEN_STREAMS_SHIFT == 12


def test_interleaved_generator_series():
    """the model's restatement of the generator's timestamps: k = 0 is the series vlohits restates; k > 0 keeps every block DeltaConst with
    delta S ms, and the S blocks of a group overlap in time while groups do not"""
    import vlohits
    from last_rows_model import GEN_STEP, GEN_T0, gen_timestamps
    assert (GEN_T0, GEN_STEP) == (vs.GEN_T0, vs.GEN_STEP)

    class Cfg:
        rows_per_block, total_rows = 100, 1250
    for k in (0, 2, 4):
        cfg = Cfg()
        cfg.columns_mask = 1 | vs.GEN_TIMESTAMPS | vs.gen_streams(k)
        s = 1 << k
        series = [gen_timestamps(cfg, b) for b in range(13)]
        if k == 0:
            assert series == [vlohits.gen_timestamps(cfg, b) for b in range(13)]
        assert all(len(t) == (100 if b < 12 else 50) for b, t in enumerate(series))
        assert all(t[i + 1] - t[i] == s * GEN_STEP for t in series for i in range(len(t) - 1))
        for g in range(0, 12 // s * s, s):   # a full group covers S * R consecutive milliseconds, one row each
            assert sorted(x for b in range(g, g + s) for x in series[b]) == [GEN_T0 + (g * 100 + i) * GEN_STEP for i in range(s * 100)]
        groups = [range(g, min(g + s, 13)) for g in range(0, 13, s)]
        for a, b in zip(groups, groups[1:]):
            assert max(series[x][-1] for x in a) < min(series[x][0] for x in b)
