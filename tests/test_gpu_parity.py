"""GPU parity tests: the CUDA path (through the C ABI, vlscan_scan_batch / vlscan_scan_resident) against the CPU oracle.

Bar: bit-exact row bitmaps and match counts (integer / byte work; no tolerance).  Fixtures: every
testFilterMatchForColumns(...) table of the reference's filter_{phrase,prefix,exact,in,regexp,not,and,or}_test.go
(tests/golden/), seeded random differential cases, generated vlogsgenerator-shaped blocks, and the edge cases the
reference tests cover (empty / single-row / const / dict / numeric / ragged / invalid UTF-8)."""
import numpy as np
import pytest

from golden_util import load_filter_cases, build_filter, and_or_cases

pytestmark = pytest.mark.gpu

CASES = load_filter_cases()


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


def check(env, columns_or_blocks, spec_or_pair, stage="ondisk"):
    oracle, vs, pu, ctx = env
    blocks = columns_or_blocks if isinstance(columns_or_blocks[0], oracle.Block) else [oracle.Block.from_columns(columns_or_blocks)]
    of, gf = spec_or_pair
    want = [oracle.bitmap_rows(b.search(of), b.rows) for b in blocks]
    got, counts, st = pu.gpu_rows(ctx, gf, blocks, stage)
    assert got == want, (gf, [c.name for c in blocks[0].columns])
    assert [int(c) for c in counts] == [len(w) for w in want]
    assert st.rows == sum(b.rows for b in blocks) and st.rows_matched == sum(len(w) for w in want)
    return want, st


def test_reference_filter_tables_on_gpu(env):
    """388 cases of filter_{phrase,prefix,exact,in,regexp,not}_test.go, on-disk stage (ZSTD decoded by the host stager)."""
    oracle, vs, pu, ctx = env
    for c in CASES:
        b = oracle.Block.from_columns(c["columns"])
        of, gf = build_filter(oracle.Filter, c["filter"]), build_filter(vs.Filter, c["filter"])
        got, counts, st = pu.gpu_rows(ctx, gf, [b])
        assert got[0] == c["expected"], (c["src"], c["filter"])
        assert int(counts[0]) == len(c["expected"])


def test_reference_filter_tables_decoded_stage(env):
    oracle, vs, pu, ctx = env
    for c in CASES[::7]:
        b = oracle.Block.from_columns(c["columns"])
        gf = build_filter(vs.Filter, c["filter"])
        got, counts, st = pu.gpu_rows(ctx, gf, [b], stage="decoded")
        assert got[0] == c["expected"], (c["src"], c["filter"])


def test_reference_and_or_tables_on_gpu(env):
    oracle, vs, pu, ctx = env
    for (q, cols, of, want), (_, _, gf, _) in zip(and_or_cases(oracle.Filter), and_or_cases(vs.Filter)):
        b = oracle.Block.from_columns(cols)
        got, counts, st = pu.gpu_rows(ctx, gf, [b])
        assert got[0] == want, q


def test_many_blocks_one_batch_and_resident_path(env):
    """All golden blocks of one filter kind in ONE batch; resident scan == end-to-end scan; hit offsets == set bits."""
    oracle, vs, pu, ctx = env
    blocks = [oracle.Block.from_columns(c["columns"]) for c in CASES[:120]]
    of, gf = oracle.Filter.phrase("foo", "abc"), vs.Filter.phrase("foo", "abc")
    want = [oracle.bitmap_rows(b.search(of), b.rows) for b in blocks]
    got, counts, st = pu.gpu_rows(ctx, gf, blocks)
    assert got == want
    hb = pu.host_blocks_from_oracle(blocks)
    batch = ctx.upload(hb)
    prog = vs.Program(gf)
    st2 = ctx.scan_resident(prog, batch)
    words, cnt = ctx.fetch()
    per = vs.split_bitmaps(words, [b.rows for b in blocks])
    assert [oracle.bitmap_rows(np.ascontiguousarray(w), b.rows) for w, b in zip(per, blocks)] == want
    assert st2.rows_matched == sum(len(w) for w in want) and st2.gpu_launches > 0
    hits, offs = ctx.fetch_hits()
    flat = [r for w in want for r in w]
    assert [int(h) for h in hits] == flat
    assert [int(offs[i + 1] - offs[i]) for i in range(len(blocks))] == [len(w) for w in want]
    batch.free()


def _rand_text(rng, n, alphabet):
    return "".join(rng.choice(alphabet, n))


def test_random_differential_strings(env):
    """Seeded random rows (ASCII, Cyrillic, CJK, invalid UTF-8, empty rows) x phrase / prefix / exact / in / regexp needles."""
    oracle, vs, pu, ctx = env
    rng = np.random.default_rng(20250718)
    words = ["error", "errors", "timeout", "GET", "conn", "refused", "foo", "bar", "a", "ab", "abc", "теСТ", "тест", "日本", "x_y", "12", "3.4", "_"]
    seps = [" ", "  ", ",", ".", "-", "/", ":", "=", "(", ")", "\n", "é", "€"]
    def row():
        k = int(rng.integers(0, 9))
        s = "".join(str(rng.choice(words)) + str(rng.choice(seps)) for _ in range(k)).encode()
        if rng.random() < 0.15:
            pos = int(rng.integers(0, len(s) + 1))
            s = s[:pos] + bytes([int(rng.integers(0x80, 0x100))]) + s[pos:]   # invalid / truncated UTF-8
        if rng.random() < 0.1:
            s = s[:int(rng.integers(0, len(s) + 1))]
        return s
    for trial in range(6):
        nrows = int(rng.choice([1, 2, 63, 64, 65, 700, 3000]))
        vals = [row() for _ in range(nrows)]
        if len(set(vals)) <= 8:
            vals += [b"pad %d" % i for i in range(9)]
        cols = [("f", vals), ("id", [b"%d" % i for i in range(len(vals))])]
        blk = oracle.Block.from_columns(cols)
        assert any(c.name == b"f" and c.value_type == 1 for c in blk.columns)
        needles = ["error", "err", "a", "ab", "GET", "теСТ", "ес", "日本", "x_y", "_", "12", "3.4", ".", " ", "", "conn", "é", "error,", "-foo", "o b", "refused)"]
        for nd in needles:
            for kind in ("phrase", "prefix", "exact"):
                check(env, [blk], (getattr(oracle.Filter, kind)("f", nd), getattr(vs.Filter, kind)("f", nd)))
        check(env, [blk], (oracle.Filter.in_("f", ["error ", "abc", "", vals[0]]), vs.Filter.in_("f", ["error ", "abc", "", vals[0]])))
        for rx in ["err.*out", "conn.*refused", "foo|bar", "^error", "refused.$", "(?i)ERROR", "a+b", "[0-9]+\\.[0-9]", "GET.+", ".+GET.+", "error.", "x_y$", "^$",
                   "тест|日本", "\\bfoo\\b", "o\\b", "e(rr|xx)or", "(foo|bar) (foo|bar)", "t.m.o", ".*", ".+", "", "foo.*", "[^a-z ]{3}"]:
            check(env, [blk], (oracle.Filter.regexp("f", rx), vs.Filter.regexp("f", rx)))


def test_numeric_and_special_columns(env):
    oracle, vs, pu, ctx = env
    blk = oracle.Block.from_columns(pu.numeric_and_special_columns())
    vts = {c.name: c.value_type for c in blk.columns}
    assert (vts[b"u8"], vts[b"u16"], vts[b"u32"], vts[b"u64"], vts[b"i64"], vts[b"ip"], vts[b"ts"], vts[b"lvl"]) == (3, 4, 5, 6, 10, 8, 9, 2)
    F, G = oracle.Filter, vs.Filter
    probes = [
        ("phrase", "u8", "7"), ("phrase", "u8", "199"), ("phrase", "u8", "300"), ("phrase", "u8", "07"), ("exact", "u16", "37"), ("exact", "u16", "x"),
        ("phrase", "u32", "104729"), ("phrase", "u64", "5000000000"), ("exact", "i64", "-987654321"), ("phrase", "i64", "0"), ("phrase", "i64", "-0"),
        ("prefix", "u8", "1"), ("prefix", "u8", ""), ("prefix", "u16", "37"), ("prefix", "u32", "1047"), ("prefix", "u64", "12345"), ("prefix", "i64", "-"), ("prefix", "i64", "-98"),
        ("prefix", "i64", "98"), ("phrase", "ip", "10.1.7.49"), ("phrase", "ip", "10.1"), ("phrase", "ip", "1"), ("prefix", "ip", "10.2"), ("prefix", "ip", "7"),
        ("exact", "ip", "10.0.0.0"), ("phrase", "ts", "2024-03-05T12:04:28.004Z"), ("phrase", "ts", "2024-03-05"), ("prefix", "ts", "2024-03-1"), ("phrase", "ts", "12"),
        ("phrase", "lvl", "error"), ("phrase", "lvl", "ERROR"), ("prefix", "lvl", "e"), ("exact", "lvl", "warn"), ("phrase", "lvl", "nope"),
        ("phrase", "cst", "same"), ("phrase", "cst", "other"), ("prefix", "cst", "va"), ("exact", "cst", "same value"),
        ("phrase", "missing", ""), ("phrase", "missing", "x"), ("prefix", "missing", ""), ("exact", "missing", ""),
        ("phrase", "msg", "status"), ("phrase", "msg", "203"), ("prefix", "msg", "20"), ("exact", "msg", "row 7 has status 202"),
    ]
    for kind, field, arg in probes:
        check(env, [blk], (getattr(F, kind)(field, arg), getattr(G, kind)(field, arg)))
    for field, rx in [("u8", "^1.$"), ("u16", "37"), ("ip", "^10\\.1\\."), ("ts", "T12:0[0-3]"), ("lvl", "(?i)error"), ("cst", "val"), ("missing", "^$"), ("missing", "x"), ("i64", "^-")]:
        check(env, [blk], (F.regexp(field, rx), G.regexp(field, rx)))
    for field, vals in [("u8", ["7", "8", "x", "256"]), ("u16", ["37", "74"]), ("i64", ["-987654321", "0"]), ("ip", ["10.1.7.49", "1.1.1.1"]), ("lvl", ["warn", "ERROR"]),
                        ("cst", ["same value"]), ("cst", ["other"]), ("missing", ["", "a"]), ("missing", ["a"]), ("msg", ["row 7 has status 202", "row 8 has status 203"]),
                        ("u8", []), ("ts", ["2024-03-05T12:04:28.004Z"])]:
        check(env, [blk], (F.in_(field, vals), G.in_(field, vals)))
    # combinators across column kinds
    # float64 column: phrase / prefix / regexp go through the per-row float -> shortest text formatting on the device
    fblk = oracle.Block.from_columns(pu.float64_columns())
    assert {c.name: c.value_type for c in fblk.columns}[b"f"] == 7
    for kind, arg in [("phrase", "123"), ("phrase", "-123"), ("phrase", "123.5"), ("phrase", "125"), ("phrase", "."), ("phrase", "-"), ("phrase", "0"), ("phrase", "56"), ("phrase", "9007199254740991"),
                      ("phrase", "00000015"), ("phrase", "0.00000015"), ("phrase", "12.50"), ("phrase", "12.5"), ("prefix", "12"), ("prefix", "-1"), ("prefix", "0.0"), ("prefix", "."), ("prefix", "-"),
                      ("prefix", "e"), ("prefix", "900719"), ("prefix", "5"), ("prefix", ""), ("exact", "9007199254740991"), ("exact", "123456789.125"), ("exact", "-0.000123"), ("exact", "12.50"),
                      ("exact", "12.5"), ("exact", "nope")]:
        check(env, [fblk], (getattr(F, kind)("f", arg), getattr(G, kind)("f", arg)))
    for rx in ["^-", "\\.5$", "^90+7", "^0\\.0+15$", "^[0-9]+\\.125$", "e", "^-?[0-9]+$", "^-?[0-9]+\\.[0-9]{2}$"]:
        check(env, [fblk], (F.regexp("f", rx), G.regexp("f", rx)))
    check(env, [fblk], (F.in_("f", ["125", "-0.000123", "7"]), G.in_("f", ["125", "-0.000123", "7"])))
    tree_o = F.and_([F.phrase("msg", "status"), F.or_([F.phrase("lvl", "error"), F.in_("u8", ["7", "9"])]), F.not_(F.prefix("ip", "10.2"))])
    tree_g = G.and_([G.phrase("msg", "status"), G.or_([G.phrase("lvl", "error"), G.in_("u8", ["7", "9"])]), G.not_(G.prefix("ip", "10.2"))])
    check(env, [blk], (tree_o, tree_g))


def test_block_shape_edge_cases(env):
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    shapes = {
        "single row": [("f", [b"only error row"]), ("g", [b"x"])],
        "two equal-length rows (const lens)": [("f", [b"error aa", b"bb error"]), ("g", [b"1", b"2"])],
        "rows of length 0 and 1": [("f", [b"", b"a", b"", b"b", b"error", b"", b"c", b"d", b"e", b"f"]), ("g", [b"%d" % i for i in range(10)])],
        "long rows (u16 lens)": [("f", [b"x" * 300 + b" error " + b"y" * i for i in range(12)]), ("g", [b"%d" % i for i in range(12)])],
        "very long row (u32 lens)": [("f", [b"z" * 70000 + b" error", b"short", b"error"] + [b"r%d" % i for i in range(9)]), ("g", [b"%d" % i for i in range(12)])],
        "64k rows": [("f", [b"row %d %s" % (i, b"error" if i % 97 == 0 else b"fine") for i in range(65536)])],
        "hit at the very end of the data": [("f", [b"aaa %d" % i for i in range(20)] + [b"tail error"])],
        "needle straddles a row boundary": [("f", [b"xx err", b"or yy", b"error", b"er", b"ror"] + [b"q%d" % i for i in range(8)])],
    }
    for name, cols in shapes.items():
        for kind, arg in [("phrase", "error"), ("prefix", "err"), ("exact", "error"), ("phrase", ""), ("prefix", ""), ("regexp", "err.*"), ("regexp", "^error$"), ("regexp", "r.w")]:
            check(env, cols, (getattr(F, kind)("f", arg), getattr(G, kind)("f", arg)))
    # an empty batch and a batch whose filter references no column at all
    hb = vs.HostBlocks([b"_msg"], [])
    words, counts, st = ctx.scan_batch(vs.Program(G.phrase("_msg", "x")), hb)
    assert len(words) == 0 and st.rows == 0
    check(env, shapes["single row"], (F.noop(), G.noop()))


def test_needles_all_lengths_alignments_and_tile_boundaries(env):
    """The substring scan looks at aligned 4-byte words only (k_substr_scan: per start alignment one (mask, pattern) pair, full masks from
    7 bytes on): needles of every length 1..17, every byte alignment of an occurrence, occurrences at row starts / ends, overlapping
    occurrences, occurrences straddling the 4 KiB / 16 KiB / 64 KiB work-item boundaries; phrase, prefix, and the regexp shapes that use the
    scan (literal prefix + suffix automaton, `PREFIX.*LITERAL` scanned by its longer literal)."""
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    rng = np.random.default_rng(7)
    for needle in [b"t", b"ti", b"GET", b"conn", b"error", b"timeou", b"timeout", b"timeouts", b"abcdefghi", b"aaaaaaaa", b"aaa", b"conn refused", b"0123456789abcdef0"]:
        rows = []
        for a in range(40):
            pad = b"." * a
            rows += [pad + needle, pad + needle + b" tail", pad + b"x" + needle, pad + needle + b"x", pad + b" " + needle + b" ", needle[:-1] + pad, needle + needle, needle[:3] + needle,
                     b"xq " + pad + needle, needle + pad + b" xq", b"xq" + needle, b"x" + pad + b"q" + needle]
        # long filler rows so that occurrences land on every kind of tile boundary: several 64 KiB tiles of data
        filler = [bytes(rng.integers(97, 123, int(rng.integers(50, 200)), dtype=np.uint8)) for _ in range(2500)]
        vals = []
        for i, f in enumerate(filler):
            vals.append(f)
            if i % 7 == 0:
                vals.append(rows[(i // 7) % len(rows)])
        cols = [("f", vals)]
        blk = oracle.Block.from_columns(cols)
        _, data = oracle.decode_values_block(blk.columns[0].values_block)
        assert len(data) > 200 * 1024
        for kind in ("phrase", "prefix"):
            check(env, [blk], (getattr(F, kind)("f", needle), getattr(G, kind)("f", needle)))
        for expr in (needle.decode() + ".*", needle.decode() + ".+tail", "xq.*" + needle.decode(), needle.decode() + ".*xq", needle.decode() + "[ x]+t"):
            check(env, [blk], (F.regexp("f", expr), G.regexp("f", expr)))


def test_dense_candidates_and_ragged_lens(env):
    """Every lane of a warp holds candidates at once: half of the rows match, rows of 0..600 bytes (u16 lens items), empty rows between
    them, and a block of equally long rows (const lens item).  Same bits as the per-row reference loop."""
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    rng = np.random.default_rng(11)
    words = [b"timeout", b"timeouts", b"error", b"conn 10.0.0.7 refused", b"connection refuse", b"GET /api", b"message", b"terror"]
    def row(maxlen):
        parts = []
        for _ in range(int(rng.integers(0, 6))):
            parts.append(words[int(rng.integers(0, len(words)))] if rng.random() < 0.5 else bytes(rng.integers(97, 123, int(rng.integers(1, maxlen)), dtype=np.uint8)))
        return b" ".join(parts)
    ragged = [row(12) if i % 5 else b"" for i in range(6000)]          # short rows: the per-row matcher
    ragged2 = [row(60) if i % 5 else b"" for i in range(6000)]         # the substring scan, empty rows in between
    wide = [row(150) for _ in range(3000)]
    assert max(len(v) for v in wide) > 255
    fixed = [(b"timeout " if i % 2 else b"timeouts") + b"%056d" % i for i in range(5000)]   # 64 bytes each: const lens item, scanned
    # every 16-byte vector of a 64 KiB tile holds a candidate word: more candidate vectors than the scan's queue takes (the tile is re-scanned in place)
    sat = [(b"timeout " * 8 if i % 3 else b"timeouts" * 8) + b"%d" % i for i in range(4000)]
    blocks = [oracle.Block.from_columns([("f", ragged), ("k", [b"%d" % i for i in range(len(ragged))])]),
              oracle.Block.from_columns([("f", ragged2), ("k", [b"%d" % i for i in range(len(ragged2))])]),
              oracle.Block.from_columns([("f", wide), ("k", [b"%d" % i for i in range(len(wide))])]),
              oracle.Block.from_columns([("f", fixed), ("k", [b"%d" % i for i in range(len(fixed))])]),
              oracle.Block.from_columns([("f", sat), ("k", [b"%d" % i for i in range(len(sat))])])]
    for kind, arg in [("phrase", "timeout"), ("phrase", "error"), ("prefix", "time"), ("phrase", "GET"), ("phrase", "t"), ("regexp", "conn.*refused"), ("regexp", "timeout.*error"),
                      ("regexp", "e.*timeouts"), ("regexp", "error [a-z]+ t")]:
        for stage in ("ondisk", "decoded"):
            check(env, blocks, (getattr(F, kind)("f", arg), getattr(G, kind)("f", arg)), stage)


def test_tile_boundary_occurrences(env):
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    # an occurrence placed exactly across each boundary kind inside one huge row set
    base = b"q" * 100
    for boundary in (4096, 16384, 65536, 65536 + 4096):
        for shift in range(-9, 3):
            vals, total = [], 0
            while total + 101 < boundary + shift - 50:
                vals.append(base)
                total += 100
            vals.append(b"-" * (boundary + shift - total) + b"timeout here")
            vals += [base] * 20
            blk = oracle.Block.from_columns([("f", vals), ("g", [b"%d" % i for i in range(len(vals))])])
            check(env, [blk], (F.phrase("f", "timeout"), G.phrase("f", "timeout")))


def test_malformed_blocks_are_rejected(env):
    """Corrupt inputs return an error (the Go side turns it into logger.Panicf FATAL) instead of undefined behaviour."""
    oracle, vs, pu, ctx = env
    blk = oracle.Block.from_columns([("f", [b"row %d" % i for i in range(100)])])
    d = pu.oracle_block_to_desc(blk, "decoded")
    prog = vs.Program(vs.Filter.phrase("f", "row"))
    bad = dict(d, columns=[dict(d["columns"][0], lens_items=d["columns"][0]["lens_items"][:-1])])
    with pytest.raises(vs.VlscanError):
        ctx.scan_batch(prog, vs.HostBlocks([b"f"], [bad]))
    bad = dict(d, columns=[dict(d["columns"][0], data=d["columns"][0]["data"][:-3])])   # lens do not add up to the data length
    with pytest.raises(vs.VlscanError):
        ctx.scan_batch(prog, vs.HostBlocks([b"f"], [bad]))
    bad = dict(d, columns=[dict(d["columns"][0], bloom=b"\x00" * 7)])
    with pytest.raises(vs.VlscanError):
        ctx.scan_batch(prog, vs.HostBlocks([b"f"], [bad]))
    d2 = pu.oracle_block_to_desc(blk, "ondisk")
    bad = dict(d2, columns=[dict(d2["columns"][0], values_block=d2["columns"][0]["values_block"][:-5])])
    with pytest.raises(vs.VlscanError):
        ctx.scan_batch(prog, vs.HostBlocks([b"f"], [bad]))
    # the context stays usable afterwards
    got, counts, st = pu.gpu_rows(ctx, vs.Filter.phrase("f", "row"), [blk])
    assert len(got[0]) == 100


def test_block_result_style_inputs(env):
    """pipeFilter / applyToBlockResult shape (lib/logstorage/pipe_filter.go:73-97): already-decoded columns, no bloom filters,
    no meaningful min/max.  An empty bloom matches everything (bloomfilter.go:175-177) and the widest min/max never prune, so the
    same predicates must yield the same bits as the blockSearch path."""
    oracle, vs, pu, ctx = env
    n = 200
    cols = [("u16", [b"%d" % (i * 37 % 60000) for i in range(n)]), ("i64", [b"%d" % ((i - 100) * 987654321) for i in range(n)]),
            ("ip", [b"10.%d.%d.%d" % (i % 3, i % 251, (i * 7) % 256) for i in range(n)]), ("lvl", [[b"info", b"warn", b"error"][i % 3] for i in range(n)]),
            ("msg", [b"row %d has status %d" % (i, 200 + i % 5) for i in range(n)])]
    blk = oracle.Block.from_columns(cols)
    d = pu.oracle_block_to_desc(blk, "decoded")
    widest = {4: (0, 2**16 - 1), 10: (2**63, 2**63 - 1), 8: (0, 2**32 - 1)}
    for c in d["columns"]:
        c["bloom"] = b""
        if c.get("value_type") in widest:
            c["min_value"], c["max_value"] = widest[c["value_type"]]
    hb = vs.HostBlocks(pu.field_names_of([blk]), [d])
    F, G = oracle.Filter, vs.Filter
    for kind, field, arg in [("phrase", "u16", "37"), ("exact", "i64", "-987654321"), ("prefix", "ip", "10.2"), ("phrase", "lvl", "error"), ("phrase", "msg", "203"),
                             ("prefix", "msg", "sta"), ("regexp", "msg", "row 1.* 20[12]"), ("phrase", "msg", "absent")]:
        want = oracle.bitmap_rows(blk.search(getattr(F, kind)(field, arg)), blk.rows)
        words, counts, st = ctx.scan_batch(vs.Program(getattr(G, kind)(field, arg)), hb)
        assert oracle.bitmap_rows(np.ascontiguousarray(words), blk.rows) == want, (kind, field, arg)
    # float64 column holding values the values encoder never emits (exponent range, subnormals, -0, Inf, NaN): the per-row text must
    # still be strconv.AppendFloat(f,'f',-1,64).  Expected bits: the same predicate over a string column of those texts.
    import struct, random
    rng = random.Random(5)
    bits = [0, 1 << 63, 1, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0x0010000000000000, 0x000FFFFFFFFFFFFF]
    bits += [struct.unpack(">Q", struct.pack(">d", float(s)))[0] for s in ("1e21", "1e22", "1.5e-7", "5e-324", "123456.789", "-2.5e300", "3e-310", "1e23", "9.5e15")]
    bits += [rng.getrandbits(64) for _ in range(181)]
    texts = [oracle.encoded_to_string(7, struct.pack(">Q", b)) for b in bits]
    sblk = oracle.Block.from_columns([("f", texts), ("k", [b"k%d" % i for i in range(len(bits))])])
    assert {c.name: c.value_type for c in sblk.columns}[b"f"] == 1
    tmpl = oracle.Block.from_columns([("f", [b"%d.5" % i for i in range(len(bits))])])   # same row count: borrow its lens block (all 8)
    fd = pu.oracle_block_to_desc(tmpl, "decoded")
    fc = fd["columns"][0]
    assert fc["value_type"] == 7 and len(fc["data"]) == 8 * len(bits)
    fc.update(min_value=0xFFF0000000000000, max_value=0x7FF0000000000000, bloom=b"", data=b"".join(struct.pack(">Q", b) for b in bits))
    fhb = vs.HostBlocks([b"f"], [fd])
    for kind, arg in [("phrase", "-"), ("phrase", "."), ("phrase", "0"), ("phrase", "100000"), ("phrase", "5"), ("prefix", "1797693134862315"), ("prefix", "0.0000"),
                      ("prefix", "-"), ("prefix", "."), ("prefix", "e"), ("regexp", "0{200}"), ("regexp", "^-?0\\.0{300}"), ("regexp", "Inf|NaN"), ("regexp", "^\\+Inf$"), ("regexp", "^-0$"),
                      ("regexp", "^[0-9]+$"), ("regexp", "^-?[0-9]*\\.?[0-9]*$")]:
        want = oracle.bitmap_rows(sblk.search(getattr(F, kind)("f", arg)), sblk.rows)
        words, counts, st = ctx.scan_batch(vs.Program(getattr(G, kind)("f", arg)), fhb)
        assert oracle.bitmap_rows(np.ascontiguousarray(words), sblk.rows) == want, (kind, arg)
