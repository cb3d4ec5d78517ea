"""Seeded regexp expressions and string blocks for the regexp leaf's tests (tests only).

`gen` draws random expressions of the supported syntax.  The family builders put a literal PREFIX from the block vocabulary in
front of a SUFFIX aimed at one of the device strategies `regex_strategy` (csrc/vl_program.h) picks, and check with the oracle's
`regex_describe` that regexutil's prefix / suffix analysis sees the shape the family is named for.  The block builders lay the
vocabulary out as long rows (the substring scan), short rows (the per-row matcher) and rows cut inside UTF-8 sequences."""
import random

import vloracle

ATOMS = ["a", "b", "c", "x", "é", "й", "日", ".", "\\d", "\\w", "\\s", "\\W", "\\D", "[a-c]", "[^a-c]", "[0-9x]", "[[:alpha:]]", "\\.", "\\b", "\\B", "^", "$",
         "\\A", "\\z", " ", "_", "0", "-", "foo", "bar", "(?i)q", "\\x41", "[é-я]"]


def gen(rng, depth=0):
    """a random expression over ATOMS; parentheses may be left open (`expr` closes them)"""
    k = rng.randrange(10)
    if depth > 3 or k < 4:
        return rng.choice(ATOMS)
    if k == 4:
        return gen(rng, depth + 1) + gen(rng, depth + 1)
    if k == 5:
        return "(" + gen(rng, depth + 1) + "|" + gen(rng, depth + 1) + ")"
    if k == 6:
        return "(?:" + gen(rng, depth + 1) + ")" + rng.choice(["*", "+", "?", "{2}", "{1,3}", "{0,2}", "*?", "{2,}"])
    if k == 7:
        return "(" + gen(rng, depth + 1) + ")" + rng.choice(["*", "+", "?"])
    if k == 8:
        return rng.choice([".*", ".+"]) + gen(rng, depth + 1) + rng.choice(["", ".*", ".+"])
    return rng.choice(["(?i)", "(?s)", "(?m)", "(?-s)", "(?i:", "("]) + gen(rng, depth + 1)


def expr(rng):
    rx = gen(rng)
    return rx + ")" * max(0, rx.count("(") - rx.count(")"))


def is_valid(rx):
    try:
        vloracle.regex_match(rx, b"")
        return True
    except RuntimeError:
        return False


# ---- block vocabulary ----------------------------------------------------------------------------------------------------------
PREFIXES = ["conn", "timeout", "ab", "GET /", "error", "тест", "日本", "x_y"]
TAILS = ["refused", "err", "error", "ed", "foo", "ошибка", "語", "t"]
WORDS = PREFIXES + TAILS + ["connection", "conn refused", "timeouts", "terror", "GET /404", "GET /api/v1", "foobar", "foo bar baz", "bar", "baz",
                            "abab", "errored", "Error", "ERROR", "ТЕСТ", "日本語", "12", "3.45", "500", "x", "é", "q"]
SEPS = [" ", " ", " ", "", ",", ".", "-", "/", ":", "=", "(", ")", "\n", "\t", "é", "€", "  "]


def _text(rng, nbytes):
    out = []
    n = 0
    while n < nbytes:
        r = rng.random()
        if r < 0.6:
            w = rng.choice(WORDS)
        elif r < 0.9:
            w = "".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randrange(1, 12)))
        else:
            w = "".join(rng.choice("0123456789") for _ in range(rng.randrange(1, 5)))
        w = (w + rng.choice(SEPS)).encode()
        if rng.random() < 0.02:
            w += bytes([rng.randrange(0x80, 0x100)])   # invalid / truncated UTF-8
        out.append(w)
        n += len(w)
    return b"".join(out)


def _cut(rng, stream, mean, spread):
    """cut a byte stream into rows at arbitrary byte offsets (inside words and multi-byte runes, so that occurrences straddle rows
    and rows end in the middle of a literal); about 3 % of the rows are empty"""
    rows, i = [], 0
    while i < len(stream):
        if rng.random() < 0.03:
            rows.append(b"")
            continue
        n = max(1, int(rng.gauss(mean, spread)))
        rows.append(stream[i:i + n])
        i += n
    return rows


def long_rows(seed, nrows=1500):
    """rows of about 130 bytes (well above VL_SHORT_ROW_BYTES): a block of ~190 KiB, several 64 KiB scan tiles.  Besides the cut
    stream, every 5th row is planted: several prefix occurrences of which only a later one is followed by what the suffix wants,
    the tail before and after the prefix, the prefix at the row end, `\\n` between prefix and tail."""
    rng = random.Random(seed)
    rows = _cut(rng, _text(rng, nrows * 130), 130, 60)[:nrows]
    for i in range(0, len(rows), 5):
        p, t = rng.choice(PREFIXES), rng.choice(TAILS)
        sep = rng.choice([" ", "", "\n", " x\n", "  ", "é"])
        shape = rng.randrange(7)
        planted = [p + "x " + p + sep + t,                # retry: the first occurrence does not verify
                   t + " " + p,                           # tail only before the prefix
                   p + sep + t + " " + p,                 # tail after, then the prefix at the row end
                   p + "\n" + t,                          # newline between prefix and tail
                   p + p + sep + t + sep + t,
                   "x" * rng.randrange(0, 40) + p,        # the prefix ends the row
                   t + sep + p + sep + t + " 404 " + p + "0 " + p + "/404"][shape].encode()
        rows[i] = (rows[i][:rng.randrange(0, 100)] + planted)[-300:] if rng.random() < 0.5 else planted + rows[i][:rng.randrange(0, 100)]
    return rows


def short_rows(seed, nrows=3000):
    """rows of about 22 bytes: under VL_SHORT_ROW_BYTES on average, so the scan strategies fall back to the per-row matcher"""
    rng = random.Random(seed)
    return _cut(rng, _text(rng, nrows * 22), 22, 12)[:nrows]


def utf8_edge_rows(seed, pad=0):
    """rows that end in a truncated multi-byte sequence followed by rows that begin with the continuation bytes (the decoder reads an
    invalid byte as U+FFFD of width 1 and never looks past the row), next to the literals the families use.  `pad` filler bytes in
    front of every row make the rows long enough for the substring scan."""
    rng = random.Random(seed)
    cuts = ["日".encode(), "語".encode(), "é".encode(), "й".encode(), "€".encode(), "😀".encode()]
    rows = []
    for _ in range(400):
        full = rng.choice(cuts)
        k = rng.randrange(1, len(full))
        p, t = rng.choice(PREFIXES).encode(), rng.choice(TAILS).encode()
        left = b"-" * pad + rng.choice([p, t, p + b" " + t, b"x", b"", p + b"x", t + p])
        right = rng.choice([p, t, b" " + t, b"x", b"", b"q" + p, t + b" " + p])
        rows.append(left + full[:k])
        rows.append(full[k:] + right + b"-" * pad)
        if rng.random() < 0.3:
            rows.append(b"-" * pad + full + right)
        if rng.random() < 0.3:
            rows.append(left + b"\xff" + right)
    return rows


# ---- families ------------------------------------------------------------------------------------------------------------------
DESCRIBED = ("prefix", "isOnlyPrefix", "isSuffixDotStar", "isSuffixDotPlus", "substrDotStar", "substrDotPlus")


def _want(prefix="", only=False, dot_star=False, dot_plus=False, substr_star="", substr_plus=""):
    return {"prefix": prefix, "isOnlyPrefix": str(int(only)), "isSuffixDotStar": str(int(dot_star)), "isSuffixDotPlus": str(int(dot_plus)),
            "substrDotStar": substr_star, "substrDotPlus": substr_plus}


def _general_suffix(rng, p):
    fixed = [" [a-z]+ t", "/[0-9]{3}\\b", "(bar|baz)", "(refused|ed)", " ?(?:x|ed)+", "[^ ]*err", "\\s+\\S", "[a-z]{2,}\\.", "(?:.*)(ed|err)x?",
             ".{3}t", "[[:alpha:]]+ [0-9]", ".*(?:foo|t)\\b"]
    for _ in range(100):
        sub = rng.choice(fixed) if rng.random() < 0.5 else expr(rng)
        rx = p + sub
        if is_valid(rx):
            d = vloracle.regex_describe(rx)
            if d["prefix"] == p and all(d[k] in ("", "0") for k in DESCRIBED[1:]):
                return rx, _want(p)
    raise AssertionError("no general suffix for %r" % p)


def _fam_all(rng):
    return rng.choice([".*", "", "(?:)", "(?s).*", ".*.*", "(.*)", "(?:.*)", "(?:)(?:)", "()", ".*(?:)", "(?s:.*)", "(?m).*", ".*?", "(?i).*"]), _want(only=True)


def _fam_only_prefix(rng):
    p = rng.choice(PREFIXES + ["conn refused", "GET /404"])
    rx = rng.choice([p, p + ".*", "(?:" + p + ")", "(" + p + ")", p + ".*.*"])
    return rx, _want(p, only=True)


def _fam_substr_dot_star(rng):
    # `.*LIT.*`: SimplifyRegex drops the dots at both ends (regexutil.go:161-176), leaving the or-value LIT and no prefix
    t = rng.choice(TAILS + PREFIXES)
    return rng.choice([".*%s.*", "(?s).*%s.*", ".*%s"]) % t, _want()


def _fam_dot_plus(rng):
    p = rng.choice(PREFIXES)
    return rng.choice([p + ".+", p + ".+.*", p + "(?s:.+)"]), _want(p, dot_plus=True)


def _fam_tail_longer(rng):
    p = rng.choice(["ab", "x", "t", "er", "é"])
    t = rng.choice([w for w in TAILS + PREFIXES if len(w.encode()) > len(p.encode())])
    return rng.choice(["%s.*%s", "%s.*%s.*", "%s(?s:.*)%s"]) % (p, t), _want(p)


def _fam_tail_shorter(rng):
    p = rng.choice(["timeout", "conn", "error", "тест", "日本"])
    t = rng.choice([w for w in TAILS + ["t", "x", "e"] if len(w.encode()) <= len(p.encode())])
    return rng.choice(["%s.*%s", "%s.*%s.*"]) % (p, t), _want(p)


def _fam_general(rng):
    return _general_suffix(rng, rng.choice(PREFIXES))


def _fam_substr_dot_plus(rng):
    t = rng.choice(TAILS)
    if rng.random() < 0.5:
        return ".+%s.+" % t, _want(substr_plus=t)
    p = rng.choice(PREFIXES)
    return "%s.+%s.+" % (p, t), _want(p, substr_plus=t)


def _fam_no_prefix(rng):
    fixed = ["(?i)error", "\\bfoo\\b", "^$", "[0-9]+\\.[0-9]", "(?i)тест", "[a-z]+ed\\b", "^conn", "\\Aerror", "(conn|GET) ", "\\d{3}",
             "[^a-z ]{3}", "(?i)GET /", "e(rr|xx)or", "^[^ ]+$", ".+", ".+t", "\\Btest"]
    for _ in range(100):
        rx = rng.choice(fixed) if rng.random() < 0.5 else rng.choice(["[a-z]", "\\w", "(?i)e", "(x|y)", "\\b"]) + expr(rng)
        if is_valid(rx):
            d = vloracle.regex_describe(rx)
            if d["prefix"] == "" and d["isOnlyPrefix"] == "0" and d["isSuffixDotStar"] == "0" and d["substrDotPlus"] == "":
                return rx, {k: d[k] for k in DESCRIBED}
    raise AssertionError("no expression without a prefix")


def _fam_newline(rng):
    # the suffix stops at `\n`: neither the tail-literal nor the `.+` shortcut may be taken.  A lone `.` suffix loses DotNL
    # through the textual `(?s:.)` -> `.` replacement (regexutil.go:229)
    p, t = rng.choice(PREFIXES), rng.choice(TAILS)
    rx = rng.choice(["(?-s)%s.*%s" % (p, t), "%s." % p, "(?-s)%s.+" % p, "%s(?-s:.*)%s" % (p, t), "(?-s)%s.*%s.*" % (p, t), "%s.%s" % (p, t)])
    return rx, _want(p)


def _fam_folded(rng):
    # a `(?i)` literal between plain words: GetLiterals skips FoldCase literals (regexutil.go:141-149), so it yields no bloom token
    p, a, b = rng.choice(["error", "GET", "conn", "x_y"]), rng.choice(["timeout", "api", "refused", "bar"]), rng.choice(["refused", "err", "baz", "v1"])
    k = rng.randrange(3)
    rx = ["%s (?i)%s %s" % (p, a, b), "%s (?i:%s) %s" % (p, a, b), "%s %s(?i)%s %s" % (p, b, a, b)][k]
    return rx, _want([p + " ", p + " ", p + " " + b][k])


def _fam_end(rng):
    p = rng.choice(PREFIXES + TAILS)
    return rng.choice([p + "$", p + "\\z", p + "\\b", p + "\\B", p + " x*", p + "(?:x|)"]), None


def _fam_end_checked(rng):
    for _ in range(100):
        rx, _ = _fam_end(rng)
        p = vloracle.regex_describe(rx)["prefix"]
        if p:
            return rx, _want(p)
    raise AssertionError("no end-of-remainder expression")


# name -> (builder, where the leaf runs on long-row string blocks: "all" = STR_ALL, "scan" = the substring scan, "row" = per row)
FAMILIES = {
    "all_rows": (_fam_all, "all"),
    "only_prefix": (_fam_only_prefix, "scan"),
    "substr_dot_star": (_fam_substr_dot_star, "row"),
    "prefix_dot_plus": (_fam_dot_plus, "scan"),
    "prefix_dot_star_longer_tail": (_fam_tail_longer, "scan"),
    "prefix_dot_star_shorter_tail": (_fam_tail_shorter, "scan"),
    "prefix_general_suffix": (_fam_general, "scan"),
    "substr_dot_plus": (_fam_substr_dot_plus, "row"),
    "no_literal_prefix": (_fam_no_prefix, "row"),
    "newline_sensitive": (_fam_newline, "scan"),
    "end_of_remainder": (_fam_end_checked, "scan"),
    "case_folded_literal": (_fam_folded, "scan"),
}


def family(name, rng, n):
    """n distinct expressions of one family, each checked against the oracle's regexutil analysis"""
    build, _ = FAMILIES[name]
    out = []
    for _ in range(50 * n):
        if len(out) == n:
            break
        rx, want = build(rng)
        if rx in out:
            continue
        d = vloracle.regex_describe(rx)
        got = {k: d[k] for k in DESCRIBED}
        assert got == want, ("family %s drifted" % name, rx, got, want)
        out.append(rx)
    assert len(out) == n, ("family %s has fewer than %d expressions" % (name, n), out)
    return out


def family_corpus(seed=1, per_family=12):
    """{family: [expressions]} with the same expressions for the same seed"""
    rng = random.Random(seed)
    return {name: family(name, rng, per_family) for name in FAMILIES}


def random_corpus(seed, n, vocab_prefix_share=0.5):
    """n valid expressions from `gen`, a literal prefix from the vocabulary in front of about half of them"""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        rx = expr(rng)
        if rng.random() < vocab_prefix_share:
            rx = rng.choice(PREFIXES) + rx
        if is_valid(rx):
            out.append(rx)
    return out
