"""GPU parity of the regexp leaf on every device strategy (`regex_strategy`, csrc/vl_program.h): every row, the substring scan in its
SCAN_CONTAINS / SCAN_RX_DOTPLUS / SCAN_RX_TAIL / SCAN_RX_SUFFIX modes, and the per-row matcher `regex_match`.  The device (through
parity_util.gpu_rows: staged in one go and bloom-first) against the oracle's Block.search, whose regexp engine is a rune-level Pike VM.
Bar: bit-exact row bitmaps and counts.  Expressions and blocks come from tests/regexp_gen.py; `scan_kernel_bytes` shows which
strategy ran: > 0 when the substring scan streamed a block, 0 when every block went per row or matched whole."""
import re

import pytest

import regexp_gen as rg

pytestmark = pytest.mark.gpu

PER_FAMILY = 12
STAGES = ("ondisk", "decoded")


@pytest.fixture(scope="module")
def env(oracle):
    from victorialogs_b200 import scan as vs
    import parity_util as pu
    ctx = vs.Ctx(0)
    yield oracle, vs, pu, ctx
    ctx.close()


@pytest.fixture(scope="module")
def corpus():
    return rg.family_corpus(seed=1, per_family=PER_FAMILY)


def _blocks(oracle, row_sets, first_id=0):
    out, i = [], first_id
    for rows in row_sets:
        out.append(oracle.Block.from_columns([("f", rows), ("id", [b"%d" % (i + k) for k in range(len(rows))])]))
        i += len(rows)
    return out


@pytest.fixture(scope="module")
def long_blocks(oracle):
    blocks = _blocks(oracle, [rg.long_rows(s) for s in (101, 102, 103)])
    for b in blocks:
        _, data = oracle.decode_values_block(b.columns[0].values_block)
        assert len(data) > 2 * 65536 and len(data) > 100 * b.rows   # several 64 KiB tiles, rows well above VL_SHORT_ROW_BYTES
    return blocks


@pytest.fixture(scope="module")
def short_blocks(oracle):
    blocks = _blocks(oracle, [rg.short_rows(s) for s in (201, 202)])
    for b in blocks:
        _, data = oracle.decode_values_block(b.columns[0].values_block)
        assert len(data) < 48 * b.rows
    return blocks


def check(env, blocks, of, gf, stage="ondisk", want=None):
    """device == oracle on every block; -> (oracle rows, stats of the one-go call)"""
    oracle, vs, pu, ctx = env
    if want is None:
        want = [oracle.bitmap_rows(b.search(of), b.rows) for b in blocks]
    got, counts, st = pu.gpu_rows(ctx, gf, blocks, stage)
    assert got == want, (gf, stage)
    assert [int(c) for c in counts] == [len(w) for w in want]
    assert st.rows_matched == sum(len(w) for w in want)
    return want, st


def check_rx(env, blocks, rx, stages=("ondisk",), field="f"):
    oracle, vs, pu, ctx = env
    want, out = None, []
    for stage in stages:
        want, st = check(env, blocks, oracle.Filter.regexp(field, rx), vs.Filter.regexp(field, rx), stage, want)
        out.append(st.scan_kernel_bytes)
    return want, out


def test_families_on_long_rows(env, corpus, long_blocks):
    """Every family on long-row blocks, on-disk and decoded stage: the scan families stream the blocks through the substring scan
    (scan_kernel_bytes > 0), the per-row and every-row families do not."""
    counts = {}
    for name, exprs in corpus.items():
        path = rg.FAMILIES[name][1]
        for rx in exprs:
            want, scanned = check_rx(env, long_blocks, rx, STAGES)
            if path == "scan":
                assert all(b > 0 for b in scanned), (name, rx, scanned)
            else:
                assert scanned == [0, 0], (name, rx, scanned)
            if path == "all":
                assert want == [list(range(b.rows)) for b in long_blocks], rx
        counts[name] = len(exprs) * len(STAGES)
    print("long rows, (expression, stage) comparisons per family:", counts)


def test_families_per_row(env, corpus, long_blocks, short_blocks):
    """The same expressions where the scan strategies fall back to the per-row matcher: short-row blocks (VL_SHORT_ROW_BYTES), and
    the long-row blocks behind an AND whose first child, an in() on the id column, leaves fewer than 1/16 of each block's rows."""
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    ids = [b"%d" % i for i in range(0, sum(b.rows for b in long_blocks), 20)]   # every 20th row, the planted rows among them
    counts = {}
    for name, exprs in corpus.items():
        for rx in exprs:
            _, scanned = check_rx(env, short_blocks, rx)
            assert scanned == [0], (name, rx)
            want, st = check(env, long_blocks, F.and_([F.in_("id", ids), F.regexp("f", rx)]), G.and_([G.in_("id", ids), G.regexp("f", rx)]))
            assert st.scan_kernel_bytes == 0, (name, rx)
        counts[name] = 2 * len(exprs)
    print("per row, (expression, block set) comparisons per family:", counts)


def test_utf8_at_row_ends(env, corpus):
    """Rows that end inside a multi-byte sequence next to rows that begin with its continuation bytes, short (per row) and padded
    (the scan): classes and `.` that would match the joined rune, `\\b` after a non-ASCII rune; the phrase and prefix boundary rules
    read the neighbouring rune with the same decoder."""
    oracle, vs, pu, ctx = env
    F, G = oracle.Filter, vs.Filter
    sets = {"short": _blocks(oracle, [rg.utf8_edge_rows(301), rg.utf8_edge_rows(302)]),
            "padded": _blocks(oracle, [rg.utf8_edge_rows(303, pad=60), rg.utf8_edge_rows(304, pad=60)])}
    fixed = ["日本.", "本.$", ".語", "[日語]", "[^a-z]$", "^[^a-z]", "日本\\b", "é\\b", "\\b語", "[\\x{80}-\\x{10FFFF}]$", "^.\\x{FFFD}", "\\x{FFFD}", "日本.+",
             "ab.{1}$", "err.?$", "t\\B", "conn[^ ]$", "foo\\W", "ed(?:.)\\z", "(?i)é", "(?i)ТЕСТ.", "error.*語", "x.*日", "😀", "^\\x{1F600}", "é.*$"]
    exprs = fixed + [rx for v in corpus.values() for rx in v[:4]]
    for blocks in sets.values():
        for rx in exprs:
            check_rx(env, blocks, rx, STAGES)
        for needle in ["日本", "日", "語", "é", "ed", "t", "conn", "x", "error", "тест", "😀", "ab"]:
            for kind in ("phrase", "prefix"):
                check(env, blocks, getattr(F, kind)("f", needle), getattr(G, kind)("f", needle))
    print("utf-8 row ends: %d expressions x %d block sets x %d stages" % (len(exprs), len(sets), len(STAGES)))


def test_every_column_kind(env, corpus):
    """A sample of every family on dict, const and missing columns and on the typed columns (the regexp runs over the row's text)."""
    oracle, vs, pu, ctx = env
    blk = oracle.Block.from_columns(pu.numeric_and_special_columns())
    fblk = oracle.Block.from_columns(pu.float64_columns())
    typed = ["1.+", "10\\.1.*5", "2024.*Z", "T1.*:0", "-9.*1", "12(3|4)", ".+0.+", "^-?[0-9]+$", "[0-9]\\.[0-9]", "(?i)t", "5$", "0\\b", "1\\B", "^1.$",
             "9.*0", "err.+", "val.*e", "E.*R", "(?i)error.", "\\.", ".*0.*", "same.+", "s.+ e", "2.*5", "[^0-9]"]
    exprs = typed + [rx for v in corpus.values() for rx in v[:3]]
    for rx in exprs:
        for field in ("u8", "u16", "u32", "u64", "i64", "ip", "ts", "lvl", "cst", "missing", "msg"):
            check_rx(env, [blk], rx, field=field)
        check_rx(env, [fblk], rx)
    print("column kinds: %d expressions x 12 columns" % len(exprs))


def test_random_expressions(env, long_blocks, short_blocks):
    """320 expressions from regexp_gen.gen, half of them behind a literal prefix from the vocabulary, on long and short rows."""
    exprs = rg.random_corpus(seed=5, n=320)
    scanned = 0
    for rx in exprs:
        _, s = check_rx(env, long_blocks, rx)
        scanned += s[0] > 0
        check_rx(env, short_blocks, rx)
    assert scanned > 50
    print("random: %d expressions x 2 block sets, %d of them scanned on long rows" % (len(exprs), scanned))


_ASSERTIONS = re.compile(r"\\[bBAz]|[$^]")
_BARE_FLAGS = re.compile(r"\(\?[a-zA-Z-]+\)")
_PY_CLASS = {"\\d": "[0-9]", "\\D": "[^0-9]", "\\w": "[0-9A-Za-z_]", "\\W": "[^0-9A-Za-z_]", "\\s": "[\\t\\n\\f\\r ]", "\\S": "[^\\t\\n\\f\\r ]",
             "[[:alpha:]]": "[A-Za-z]"}


def python_pattern(oracle, rx):
    """the expression in Python's `re` when regexutil's prefix / suffix split cannot change its language, else None: no assertions
    (`\\b \\B ^ $ \\A \\z`), not a lone `.` behind the prefix (it loses DotNL), no substrDotPlus (its first-occurrence rule),
    `(?i)` only on ASCII, flag groups only at the start (Python takes no mid-pattern `(?i)`).  Go's `\\d \\w \\s` are ASCII; `.`
    matches `\\n` because regexutil turns DotNL on."""
    if _ASSERTIONS.search(rx) or "\\x{" in rx or "(?-s" in rx or "(?m" in rx or any(m.start() > 0 for m in _BARE_FLAGS.finditer(rx)):
        return None
    if "(?i" in rx and not rx.isascii():
        return None
    d = oracle.regex_describe(rx)
    if d["substrDotPlus"] or rx[len(d["prefix"]):].replace("(?:", "").replace("(", "").replace(")", "") in (".", ".{1}"):
        return None
    py = rx
    for k, v in _PY_CLASS.items():
        py = py.replace(k, v)
    return re.compile(py, re.DOTALL)


def test_python_re_reference(env, corpus, long_blocks, short_blocks):
    """A third reference where the prefix / suffix split cannot change the language: Python's `re` on the rows decoded with
    surrogateescape (one character per invalid byte, as Go's decoder yields one U+FFFD per invalid byte).  Catches what the oracle and
    the product, which share the analysis of regexutil.Regex, get wrong the same way."""
    oracle, vs, pu, ctx = env
    exprs = [rx for v in corpus.values() for rx in v] + rg.random_corpus(seed=5, n=320)
    texts_long = [[v.decode("utf-8", "surrogateescape") for v in rg.long_rows(s)] for s in (101, 102, 103)]
    texts_short = [[v.decode("utf-8", "surrogateescape") for v in rg.short_rows(s)] for s in (201, 202)]
    compared = 0
    for rx in exprs:
        cre = python_pattern(oracle, rx)
        if cre is None:
            continue
        for blocks, tx in ((long_blocks, texts_long), (short_blocks, texts_short)):
            want, _ = check_rx(env, blocks, rx)
            assert want == [[i for i, s in enumerate(rows) if cre.search(s)] for rows in tx], (rx, cre.pattern)
        compared += 1
    assert compared > 150
    print("python re: %d expressions x 2 block sets" % compared)


def test_bloom_tokens_of_case_folded_literals(env):
    """A `(?i)` literal is not a bloom token (GetLiterals skips FoldCase literals, regexutil.go:141-149): a block whose rows hold the
    words only in another case keeps its matching rows."""
    oracle, vs, pu, ctx = env
    rows = [b"error TIMEOUT refused now %d" % i if i % 3 else b"GET /API/V1 x conn %d" % i for i in range(600)]
    blocks = _blocks(oracle, [rows, [r.lower() for r in rows]])
    for rx in ["error (?i)timeout refused", "error (?i:timeout) refused", "GET /(?i)api/v1 x", "x (?i)CONN \\d", "now (?i)%d" % 7, "(?i)error timeout refused"]:
        assert oracle.Filter.regexp("f", rx).tokens() == vs.Program(vs.Filter.regexp("f", rx)).leaf_tokens(0), rx
        for stage in STAGES:
            want, _ = check_rx(env, blocks, rx, (stage,))
            assert want[0], rx

