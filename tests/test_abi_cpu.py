"""CPU suite for the product's host side: the C-ABI library loads and exports every symbol include/vlscan.h declares,
the host-side program compiler derives the same tokens as the reference filters, and computing calls fail loudly
without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from golden_util import load_filter_cases, build_filter, and_or_cases
from victorialogs_b200 import scan as vs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "vlscan.h")).read()
    declared = sorted(set(re.findall(r"\b(vlscan_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 25
    L = vs.lib()
    for name in declared:
        assert hasattr(L, name), "libvlscan.so does not export %s" % name
    assert sorted(declared) == sorted(vs.EXPORTS)


def test_header_is_plain_c_and_links(tmp_path):
    # cgo compiles include/vlscan.h as C: it has to parse as strict C99, and a C translation unit that takes the address of every
    # declared entry point has to link against libvlscan.so with no C++ runtime on the command line
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "vlscan.h")).read()
    declared = sorted(set(re.findall(r"\b(vlscan_[a-z0-9_]+)\s*\(", hdr)))
    src = tmp_path / "abi_check.c"
    src.write_text("#include <stddef.h>\n#include <stdint.h>\n#include \"vlscan.h\"\n"
                   "typedef void (*fn)(void);\nfn table[] = {\n"
                   + "".join("  (fn)%s,\n" % n for n in declared) + "};\n"
                   "int main(void) { return (int)(sizeof table / sizeof table[0]) == 0; }\n")
    libdir = os.path.dirname(vs.lib()._name)
    out = tmp_path / "abi_check"
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic",
                        "-I", os.path.join(ROOT, "include"), str(src), "-o", str(out),
                        "-L", libdir, "-l:libvlscan.so", "-Wl,--unresolved-symbols=ignore-in-shared-libs"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_struct_layouts_match_header():
    # sizes asserted against the C layout rules of include/vlscan.h (x86-64 SysV)
    assert C.sizeof(vs.CColumn) == 4 + 4 + 8 + 8 + 8 * 12
    assert C.sizeof(vs.CBlock) == 24 + 8 + 8 + 8 + 8   # + timestamps pointer, length, minTimestamp, maxTimestamp
    assert C.sizeof(vs.CStats) == 8 * 16   # + staged_columns, pruned_columns
    assert C.sizeof(vs.GenConfig) == 32


def test_program_tokens_match_oracle(oracle):
    """getTokens() of phrase / prefix / exact / regexp leaves (tokenizeStrings, getTokensSkipLast, skipFirstLastToken)."""
    seen = 0
    for c in load_filter_cases():
        spec = c["filter"]
        if spec["kind"] in ("not", "in"):
            continue
        want = build_filter(oracle.Filter, spec).tokens()
        got = vs.Program(build_filter(vs.Filter, spec)).leaf_tokens(0)
        assert got == want, spec
        seen += 1
    assert seen > 250


PRODUCT_NEXT_KINDS = ("exact_prefix", "len_range", "string_range", "ipv4_range", "value_type", "any_case_phrase", "any_case_prefix", "sequence", "contains_all", "contains_any", "eq_field", "le_field", "range")


def test_next_filter_kinds_compile_and_tokens(oracle):
    """The filters of SURVEY §8(f) rank 3 that libvlscan compiles: every reference-table filter builds; the tokens of the kinds that feed the
    AND / OR bloom pre-pass (exact_prefix: getTokensSkipLast, seq(): the tokens of all phrases) equal the oracle's; the kinds not built yet are
    rejected, not guessed."""
    seen = {}
    for c in load_filter_cases("filter_cases_next.json"):
        spec = c["filter"]
        k = spec["kind"]
        if k not in PRODUCT_NEXT_KINDS:
            continue
        p = vs.Program(build_filter(vs.Filter, spec))
        want_fields = [bytes.fromhex(spec["field"]) or b"_msg"]
        if k in ("eq_field", "le_field") and (bytes.fromhex(spec["arg"]) or b"_msg") not in want_fields:
            want_fields.append(bytes.fromhex(spec["arg"]) or b"_msg")
        assert p.fields() == want_fields
        if k in ("exact_prefix", "sequence"):
            want = build_filter(oracle.Filter, spec).tokens()
            if k == "sequence" and not [v for v in spec["values"] if v]:
                want = []   # a sequence without phrases compiles to a no-op node: there is no leaf to ask
            try:
                got = p.leaf_tokens(0)
            except IndexError:
                got = []
            assert got == want, spec
        else:
            try:
                assert p.leaf_tokens(0) == []
            except IndexError:
                pass        # compiled to a no-op (contains_all of nothing, contains_any with an empty value)
        seen[k] = seen.get(k, 0) + 1
    assert seen == {"exact_prefix": 62, "len_range": 30, "string_range": 48, "ipv4_range": 24, "value_type": 35, "any_case_phrase": 107, "any_case_prefix": 114, "sequence": 103,
                    "contains_all": 104, "contains_any": 88, "eq_field": 78, "le_field": 139, "range": 62}
    with pytest.raises(vs.VlscanError):
        vs.Program(vs.Filter(bytes([vs.F_IPV4_RANGE, 1, ord("f")]) + bytes([0x80, 0x80, 0x80, 0x80, 0x10, 0]), "ipv4 bound > 32 bits"))
    for kind in (23, 24, 200):
        with pytest.raises(vs.VlscanError):
            vs.Program(vs.Filter(bytes([kind, 1, ord("f"), 1, ord("x")]), "kind not built yet"))
    # AND: exact_prefix contributes its tokens to the per-field bloom pre-pass (filter_and.go:141-143)
    vs.Program(vs.Filter.and_([vs.Filter.exact_prefix("m", "foo bar"), vs.Filter.len_range("m", 1, 5), vs.Filter.not_(vs.Filter.value_type("m", "dict"))]))


def test_value_predicates_match_oracle(oracle):
    """vl::range_predicate - the function the row kernels call for kinds 9..12, here in its host build - against the oracle's
    matchExactPrefix / matchLenRange / matchStringRange / matchIPv4Range on seeded random values (ASCII, UTF-8, invalid bytes,
    IPv4-looking strings incl. the two-character quirk of tryParseDateUint64)."""
    import random
    rng = random.Random(20250923)
    O = oracle.lib()
    O.vlo_eval_predicate.argtypes = [C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64]

    def rnd_string():
        kind = rng.randrange(6)
        if kind == 0:
            return bytes(rng.choice(b"ab 01.-") for _ in range(rng.randrange(0, 8)))
        if kind == 1:
            return "".join(rng.choice("aйц日🙂é ") for _ in range(rng.randrange(0, 6))).encode()
        if kind == 2:
            return bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 7)))
        if kind == 3:
            return b".".join(b"%d" % rng.choice([0, 1, 7, 10, 99, 127, 255, 256, 300]) for _ in range(rng.choice([3, 4, 4, 4, 5])))
        if kind == 4:
            return b".".join(bytes(rng.choice(b"0123456789:/a") for _ in range(rng.randrange(0, 4))) for _ in range(4))
        return b"%d" % rng.randrange(-10**6, 10**12)

    n = 0
    for _ in range(20000):
        s, a, b = rnd_string(), rnd_string(), rnd_string()
        lo, hi = sorted([rng.randrange(0, 9), rng.randrange(0, 9)])
        ip_lo, ip_hi = sorted([rng.getrandbits(32), rng.getrandbits(32)])
        for kind, a1, a2, x0, x1 in ((9, a, b"", 0, 0), (10, b"", b"", lo, hi), (11, a, b, 0, 0), (12, b"", b"", ip_lo, ip_hi), (12, b"", b"", 0, 0xFFFFFFFF)):
            want = O.vlo_eval_predicate(kind, s, len(s), a1, len(a1), a2, len(a2), x0, x1)
            assert want in (0, 1)
            assert vs.eval_predicate(kind, s, a1, a2, x0, x1) == bool(want), (kind, s, a1, a2, x0, x1)
            n += want
    assert n > 5000   # the sample is not vacuous
    with pytest.raises(ValueError):
        vs.eval_predicate(1, b"x")


def test_next_value_predicates_match_oracle(oracle):
    """The host builds of the predicates that are written for the device but not wired into the row kernels yet (csrc/vl_anycase.cuh):
    i(phrase) / i(prefix*) on a value that is lowercased on the fly - never materialised -, seq(), contains_all(), contains_any().
    Against the oracle, which lowercases into a buffer like the reference (stringsutil.AppendLowercase) and was pinned by the reference's
    tables (tests/test_oracle_next_filters.py)."""
    import random
    rng = random.Random(20250924)
    O = oracle.lib()
    O.vlo_eval_predicate.argtypes = [C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64]
    O.vlo_strings_to_lower.restype = C.c_int64

    def lower(b):
        out = C.create_string_buffer(4 * len(b) + 8)
        n = O.vlo_strings_to_lower(b, C.c_uint64(len(b)), out, C.c_uint64(len(out)))
        assert n >= 0
        return out.raw[:n]

    # letters whose lowercase has another byte length (İ -> i, Ⱥ -> ⱥ, K (Kelvin) -> k), cased and uncased scripts, digits, separators
    alphabet = ["a", "B", "c", "Z", "é", "É", "й", "Й", "ß", "İ", "Ⱥ", "ⱥ", "K", "Σ", "ς", "日", "🙂", "𐐀", "𐐨", "0", "7", "_", " ", ".", "-", ":", "/"]

    def rnd_text(lo=0, hi=10):
        k = rng.randrange(5)
        if k == 0:
            return bytes(rng.choice(b"abAB 01._-") for _ in range(rng.randrange(lo, hi)))
        if k == 1:
            return bytes(rng.getrandbits(8) for _ in range(rng.randrange(lo, hi)))
        s = "".join(rng.choice(alphabet) for _ in range(rng.randrange(lo, hi))).encode()
        if k == 2 and s:                                           # damage the encoding somewhere
            i = rng.randrange(len(s))
            s = s[:i] + bytes([rng.choice([0x80, 0xC3, 0xE2, 0xF0, 0xFF])]) + s[i + rng.randrange(0, 2):]
        return s

    def sub_of(s):
        if not s or rng.random() < 0.3:
            return rnd_text(0, 4)
        i = rng.randrange(len(s))
        return s[i:i + rng.randrange(1, 6)]

    def pack(phrases):
        out = b""
        for p in phrases:
            n, enc = len(p), bytearray()
            while n >= 0x80:
                enc.append((n & 0x7F) | 0x80)
                n >>= 7
            enc.append(n)
            out += bytes(enc) + p
        return out

    hits = {k: 0 for k in (14, 15, 16, 17, 18)}
    for _ in range(30000):
        s = rnd_text(0, 14)
        needle = lower(sub_of(s) if rng.random() < 0.7 else rnd_text(0, 5))
        for kind in (14, 15):
            want = O.vlo_eval_predicate(kind, s, len(s), needle, len(needle), b"", 0, 0, 0)
            assert want in (0, 1)
            assert vs.eval_predicate(kind, s, needle) == bool(want), (kind, s, needle)
            hits[kind] += want
        phrases = [sub_of(s) if rng.random() < 0.8 else b"" for _ in range(rng.randrange(0, 4))]
        packed = pack(phrases)
        for kind in (16, 17, 18):
            want = O.vlo_eval_predicate(kind, s, len(s), packed, len(packed), b"", 0, 0, 0)
            assert want in (0, 1)
            assert vs.eval_predicate(kind, s, packed) == bool(want), (kind, s, phrases)
            hits[kind] += want
    assert all(v > 2000 for v in hits.values()), hits
    # the byte-length check happens before lowercasing (filter_any_case_phrase.go:164-166): Ⱥ (2 bytes) lowercases to ⱥ (3 bytes)
    assert vs.eval_predicate(14, "Ⱥ".encode(), "ⱥ".encode()) is False and vs.eval_predicate(14, "ȺȺ".encode(), "ⱥ".encode()) is False
    assert vs.eval_predicate(14, "Ⱥ x".encode(), "ⱥ".encode()) is True
    assert vs.eval_predicate(14, "İstanbul".encode(), b"istanbul") is True and vs.eval_predicate(15, "X İSTANBUL".encode(), b"ist") is True
    assert vs.eval_predicate(14, b"FOO\xffBAR", b"bar") is False and vs.eval_predicate(14, b"FOO\xff BAR", b"bar") is True     # an invalid byte counts as a token char


def test_and_or_prepass_tokens_match_oracle(oracle):
    """The bloom pre-pass of AND / OR nodes prunes whole blocks, so wrong tokens there would be false negatives: the per-field tokens the
    program compiler merges (union under AND incl. the common tokens of nested ORs, intersection under OR incl. nested ANDs) against the
    oracle's getCommonTokensForAndFilters / getCommonTokensForOrFilters on the reference's AND / OR tables and on random trees."""
    import random
    rng = random.Random(13)
    O = oracle.lib()
    O.vlo_filter_prepass_tokens.restype = C.c_int64
    L = vs.lib()
    L.vlscan_program_prepass_tokens.restype = C.c_int64

    def dump_oracle(f):
        buf = C.create_string_buffer(1 << 20)
        n = O.vlo_filter_prepass_tokens(f.h, buf, C.c_uint64(1 << 20))
        assert n >= 0
        return buf.raw[:n]

    def dump_product(f):
        p = vs.Program(f)
        buf = C.create_string_buffer(1 << 20)
        n = L.vlscan_program_prepass_tokens(p.h, buf, C.c_size_t(1 << 20))
        assert n >= 0
        return buf.raw[:n]

    def canon(d):      # field order inside a node is not part of the contract; token order inside a field is (hash order is irrelevant, the set is not)
        out = []
        for line in d.split(b"\n")[:-1]:
            parts = line.split(b"\t")
            out.append((parts[0], sorted((p.split(b"\x1f")[0].replace(b"_msg", b"") or b"", tuple(sorted(p.split(b"\x1f")[1:]))) for p in parts[1:])))
        return out

    words = ["error", "timeout", "GET", "a b", "foo_bar", "x-y z", "conn refused", "é", "", "10.0.0.1", "a", "b"]
    fields = ["_msg", "level", "path"]

    def leaf(F):
        k = rng.randrange(7)
        f, w = rng.choice(fields), rng.choice(words)
        if k == 0:
            return F.phrase(f, w)
        if k == 1:
            return F.prefix(f, w)
        if k == 2:
            return F.exact(f, w)
        if k == 3:
            return F.regexp(f, rng.choice(["conn.*refused", "foo", "a+b", "err(or)? 5", ".*x.*"]))
        if k == 4:
            return F.in_(f, [rng.choice(words) for _ in range(rng.randrange(1, 4))])
        if k == 5:
            return F.exact_prefix(f, w)
        return F.noop()

    def tree(F, depth=0):
        k = rng.randrange(6)
        if depth >= 3 or k <= 1:
            return leaf(F)
        if k == 2:
            return F.not_(tree(F, depth + 1))
        kids = [tree(F, depth + 1) for _ in range(rng.randrange(1, 5))]
        return F.and_(kids) if k in (3, 4) else F.or_(kids)

    compared = 0
    for (q, cols, pf, want), (_, _, of, _) in zip(and_or_cases(vs.Filter), and_or_cases(oracle.Filter)):
        assert canon(dump_product(pf)) == canon(dump_oracle(of)), q
        compared += 1
    for trial in range(600):
        state = rng.getstate()
        pf = tree(vs.Filter)
        rng.setstate(state)
        of = tree(oracle.Filter)
        a, b = canon(dump_product(pf)), canon(dump_oracle(of))
        assert a == b, (trial, pf, a, b)
        compared += len(a)
    assert compared > 600


def test_in_probe_hashes_match_oracle(oracle):
    """in(): the hashes probed in the bloom filter - common tokens of all values, then the remaining tokens of every value, a block
    being skipped when no value's set is contained (matchBloomFilterAnyTokenSet) - against the oracle, hash by hash."""
    import random
    import numpy as np
    rng = random.Random(17)
    O = oracle.lib()
    O.vlo_filter_in_hashes.restype = C.c_int64
    L = vs.lib()
    L.vlscan_program_in_hashes.restype = C.c_int64
    words = ["error", "timeout", "GET /api", "a b c", "foo_bar", "x-y z", "conn refused", "é ü", "", "10.0.0.1", "a", "b", "status 500", "status 502", "status"]

    def parse(a):
        a = [int(x) for x in a]
        nc = a[0]
        common, rest = sorted(a[1:1 + nc]), a[1 + nc:]
        if rest[0] == 2 ** 64 - 1:
            return common, None
        sets, i = [], 1
        for _ in range(rest[0]):
            n = rest[i]
            sets.append(tuple(sorted(rest[i + 1:i + 1 + n])))
            i += 1 + n
        assert i == len(rest)
        return common, sets

    for trial in range(400):
        vals = [rng.choice(words) + rng.choice(["", " x", " timeout"]) for _ in range(rng.choice([0, 1, 2, 3, 5, 9]))]
        if trial == 0:
            vals = ["v%d common" % i for i in range(1001)]          # above maxTokenSetsToInit
        pa = np.zeros(200000, dtype=np.uint64)
        oa = np.zeros(200000, dtype=np.uint64)
        p = vs.Program(vs.Filter.in_("f", vals))
        n1 = L.vlscan_program_in_hashes(p.h, C.c_uint32(0), pa.ctypes.data_as(C.c_void_p), C.c_size_t(len(pa)))
        f = oracle.Filter.in_("f", vals)
        n2 = O.vlo_filter_in_hashes(f.h, oa.ctypes.data_as(C.c_void_p), C.c_uint64(len(oa)))
        assert n1 > 0 and n2 > 0
        pc, ps = parse(pa[:n1])
        oc, os_ = parse(oa[:n2])
        assert pc == oc, vals
        if ps is None:
            assert len(os_) > 1000                                  # the oracle keeps them and skips them at probe time, like the reference
        else:
            assert ps == os_, vals
    assert L.vlscan_program_in_hashes(vs.Program(vs.Filter.phrase("f", "x")).h, C.c_uint32(0), pa.ctypes.data_as(C.c_void_p), C.c_size_t(8)) == -1
    # the typed value sets a numeric column is matched with (in_values.go:141-315)
    O.vlo_filter_in_typed.restype = C.c_int64
    L.vlscan_program_in_typed.restype = C.c_int64
    pool = ["0", "1", "255", "256", "65535", "65536", "4294967295", "4294967296", "18446744073709551615", "18446744073709551616", "-1", "-9223372036854775808", "007", "1_0",
            "1.5", "-0.25", "1.50", "9007199254740993", "10.0.0.1", "255.255.255.255", "256.1.1.1", "1.2.3", "2024-05-06T07:08:09.123Z", "2024-05-06 07:08:09.123Z", "abc", ""]
    nonempty = 0
    for trial in range(200):
        vals = [rng.choice(pool) for _ in range(rng.randrange(1, 9))]
        p, f = vs.Program(vs.Filter.in_("f", vals)), oracle.Filter.in_("f", vals)
        for vt in (vs.VT_UINT8, vs.VT_UINT16, vs.VT_UINT32, vs.VT_UINT64, vs.VT_INT64, vs.VT_FLOAT64, vs.VT_IPV4, vs.VT_ISO8601):
            n1 = L.vlscan_program_in_typed(p.h, C.c_uint32(0), C.c_int(vt), pa.ctypes.data_as(C.c_void_p), C.c_size_t(len(pa)))
            n2 = O.vlo_filter_in_typed(f.h, C.c_int(vt), oa.ctypes.data_as(C.c_void_p), C.c_uint64(len(oa)))
            assert n1 == n2 >= 0 and list(pa[:n1]) == list(oa[:n2]), (vals, vt)
            nonempty += n1 > 0
    assert nonempty > 300


def test_typed_needles_match_oracle(oracle):
    """How the program compiler reads a filter argument as a value of a typed column (the typed needles of phrase / exact / in() leaves)
    against the oracle's tryParseUint64 / Int64 / Float64 / IPv4 / TimestampISO8601, on seeded number-like strings."""
    import random
    import struct
    rng = random.Random(11)

    def text():
        k = rng.randrange(9)
        if k == 0:
            return str(rng.choice([0, 1, 7, 255, 256, 65535, 65536, 2 ** 32 - 1, 2 ** 32, 2 ** 53, 2 ** 53 + 1, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1, 2 ** 64]) + rng.randrange(-1, 2))
        if k == 1:
            return rng.choice(["", "-", "+", "-0", "00", "01", "1_000", "_1", "1_", "1__0", "0x10", "1e5", "1E5", " 1", "1 ", "٣"]) + rng.choice(["", "5"])
        if k == 2:
            return "%s%d.%s" % (rng.choice(["", "-"]), rng.randrange(0, 10 ** rng.randrange(1, 18)), "".join(rng.choice("0123456789") for _ in range(rng.randrange(0, 18))))
        if k == 3:
            return rng.choice([".5", "5.", "1.2.3", "-.5", "1._5", "1.5_0", "0.000000000000000000001", "123456789012345678901234567", "1234567890123456789012345678"])
        if k == 4:
            return ".".join(str(rng.choice([0, 1, 9, 10, 99, 100, 255, 256, 999, 1000])) for _ in range(rng.choice([3, 4, 4, 4, 5])))
        if k == 5:
            return ".".join(rng.choice(["1", "01", "001", "1a", ":9", "/1", "", "25", "255"]) for _ in range(4))
        if k == 6:
            return "%04d-%02d-%02dT%02d:%02d:%02d.%03dZ" % (rng.choice([1676, 1677, 1970, 2024, 2262, 2263]), rng.randrange(0, 14), rng.randrange(0, 33), rng.randrange(0, 26),
                                                          rng.randrange(0, 62), rng.randrange(0, 62), rng.randrange(0, 1000))
        if k == 7:
            base = "2024-05-06T07:08:09.123Z"
            i = rng.randrange(len(base))
            return base[:i] + rng.choice(["x", " ", "", "0", ":", "-"]) + base[i + 1:]
        return str(rng.randrange(-10 ** 19, 10 ** 19))

    hits = {}
    for _ in range(40000):
        s = text().encode()
        u, ok = oracle.try_parse_uint64(s)
        for vt in (vs.VT_UINT8, vs.VT_UINT64):
            assert vs.parse_typed(vt, s) == (u if ok else None), (vt, s)
        hits["u"] = hits.get("u", 0) + ok
        i, ok = oracle.try_parse_int64(s)
        assert vs.parse_typed(vs.VT_INT64, s) == ((i & (2 ** 64 - 1)) if ok else None), s
        hits["i"] = hits.get("i", 0) + ok
        f, ok = oracle.try_parse_float64(s)
        assert vs.parse_typed(vs.VT_FLOAT64, s) == (struct.unpack("<Q", struct.pack("<d", f))[0] if ok else None), s
        hits["f"] = hits.get("f", 0) + ok
        ip, ok = oracle.try_parse_ipv4(s)
        assert vs.parse_typed(vs.VT_IPV4, s) == (ip if ok else None), s
        hits["ip"] = hits.get("ip", 0) + ok
        t, ok = oracle.try_parse_iso8601(s)
        assert vs.parse_typed(vs.VT_ISO8601, s) == ((t & (2 ** 64 - 1)) if ok else None), s
        hits["ts"] = hits.get("ts", 0) + ok
    assert all(v > 500 for v in hits.values()), hits
    with pytest.raises(ValueError):
        vs.parse_typed(vs.VT_STRING, b"x")


def test_regexp_automaton_matches_oracle(oracle):
    """The compiled form of a regexp leaf - prefix / suffix split plus the rune-class DFA with delayed assertions, in its host mirror
    (what const and dict values are matched with; the kernels step the same tables) - against the oracle's Pike VM on random expressions
    of the supported syntax and random subjects (UTF-8, newlines, an invalid byte).  The leaf's bloom tokens (GetLiterals through
    skipFirstLastToken) must be the oracle's: one token too many drops blocks that hold matching rows.  The family expressions of
    tests/regexp_gen.py (the shapes each device strategy is chosen for) go through the same two checks."""
    import random
    import regexp_gen
    rng = random.Random(7)
    alphabet = ["a", "b", "c", "x", "A", "Q", "q", "é", "É", "й", "日", " ", "\n", "0", "9", "_", "-", ".", "foo", "bar"]
    compared = 0
    for _ in range(1500):
        rx = regexp_gen.expr(rng)
        valid = regexp_gen.is_valid(rx)
        if valid:
            assert vs.Program(vs.Filter.regexp("f", rx)).leaf_tokens(0) == oracle.Filter.regexp("f", rx).tokens(), rx
        for _ in range(10):
            s = "".join(rng.choice(alphabet) for _ in range(rng.randrange(0, 9))).encode()
            if rng.random() < 0.1:
                s += b"\xff"
            try:
                got = vs.eval_predicate(5, s, rx.encode())
            except ValueError:
                got = None
            if not valid:
                assert got is None, ("the oracle rejects it, the compiler accepts it", rx)
                break
            assert got is not None, ("the compiler rejects it", rx)
            assert got == oracle.regex_match(rx, s), (rx, s)
            compared += 1
    assert compared == 15000
    subjects = [b"", b"\n", b"\xff", b"\xe6\x97", "é".encode()] + [w.encode() for w in regexp_gen.WORDS] + regexp_gen.long_rows(3, 60) + regexp_gen.utf8_edge_rows(4)[:60]
    families = 0
    for name, exprs in regexp_gen.family_corpus().items():
        for rx in exprs:
            assert vs.Program(vs.Filter.regexp("f", rx)).leaf_tokens(0) == oracle.Filter.regexp("f", rx).tokens(), (name, rx)
            for s in subjects:
                assert vs.eval_predicate(5, s, rx.encode()) == oracle.regex_match(rx, s), (name, rx, s)
            families += 1
    assert families == 12 * len(regexp_gen.FAMILIES)


def test_host_entry_points_are_reentrant(oracle):
    """8 host threads at once through the entry points that need no device: the (itself multi-threaded) header walk, the program compiler,
    a malformed tree whose error text must stay on the calling thread, the regexp mirror.  (tests/test_gpu_zzz_workers.py does the same with
    one vlscan_ctx per thread on a device.)"""
    import threading
    from parity_util import oracle_block_to_desc, field_names_of
    cfg = oracle.GenConfig(seed=5, total_rows=3000 * 30, rows_per_block=3000, hot_block_permille=500, hit_row_permille=60, columns_mask=0b1111)
    blocks = [oracle.Block.generated(cfg, i) for i in range(30)]
    hb = vs.HostBlocks(field_names_of(blocks), [oracle_block_to_desc(b) for b in blocks] * 30)
    ref = vs.zstd_walk_digest(hb, 1)["digest"]
    F = vs.Filter
    trees = [F.and_([F.phrase("_msg", "timeout"), F.phrase("level", "error")]), F.regexp("_msg", "conn.*refused"), F.or_([F.in_("status", ["500", "503"]), F.prefix("path", "api")])]
    errors = []

    def worker(w):
        try:
            for r in range(12):
                if vs.zstd_walk_digest(hb, [0, 1, 4, 16][(r + w) % 4])["digest"] != ref:
                    errors.append("digest differs")
                for t in trees:
                    p = vs.Program(t)
                    p.fields()
                    p.leaf_tokens(0)
                try:
                    vs.Program(vs.Filter(bytes([200 + w]), "bad"))
                    errors.append("malformed tree accepted")
                except vs.VlscanError as e:
                    if ("unknown filter kind %d" % (200 + w)) not in str(e):
                        errors.append("error text of another thread: " + str(e))
                if not vs.eval_predicate(5, b"conn was refused", b"conn.*refused"):
                    errors.append("regexp mirror")
        except Exception as e:          # noqa: BLE001 - reported below
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(w,)) for w in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not errors, errors[:3]


def test_hostile_nesting_is_refused_not_crashed():
    """Recursion of the compilers is bounded: a filter tree deeper than 64 levels and a regexp with more than 1000 open parentheses are
    errors (Go's regexp refuses trees higher than 1000 too: ErrNestingDepth), not stack overflows.  Runs in a child so that a crash is a
    test failure, not the end of the test session."""
    import subprocess
    import sys
    import textwrap
    child = textwrap.dedent('''
        import sys
        sys.path.insert(0, %r)
        from victorialogs_b200 import scan as vs
        leaf = vs.Filter.phrase("a", "b").blob
        def tree(blob):
            try:
                vs.Program(vs.Filter(blob, "deep")); return "ok"
            except vs.VlscanError as e:
                return "nests too deeply" in str(e) and "deep"
        assert tree(bytes([8]) * 60 + leaf) == "ok"
        for n in (64, 5000, 99000):
            assert tree(bytes([8]) * n + leaf) == "deep", n
            assert tree((bytes([6, 2]) + leaf) * n + leaf) == "deep", n
        def rx(n, open_="("):
            try:
                vs.Program(vs.Filter.regexp("_msg", open_ * n + "a" + ")" * n)); return "ok"
            except vs.VlscanError as e:
                return "nests too deeply" in str(e) and "deep"
        assert rx(1000) == "ok" and rx(1000, "(?:") == "ok"
        for n in (1001, 400000):
            assert rx(n) == "deep" and rx(n, "(?:") == "deep" and rx(n, "(?i:") == "deep", n
        print("fine")
    ''')
    r = subprocess.run([sys.executable, "-c", child % ROOT], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "fine" in r.stdout, (r.returncode, r.stdout[-300:], r.stderr[-1500:])


def test_program_fields_and_errors():
    p = vs.Program(vs.Filter.and_([vs.Filter.phrase("", "GET"), vs.Filter.prefix("path", "api"), vs.Filter.in_("status", ["500", "502", "503"])]))
    assert p.fields() == [b"_msg", b"path", b"status"]
    for bad in ("foo(", "a**", "[z-a]", r"\pL+", "(?P<n", "x{2,1}"):
        with pytest.raises(vs.VlscanError):
            vs.Program(vs.Filter.regexp("f", bad))
    with pytest.raises(vs.VlscanError):   # malformed tree
        vs.Program(vs.Filter(bytes([vs.F_AND, 3, vs.F_NOOP]), "truncated"))
    with pytest.raises(vs.VlscanError):
        vs.Program(vs.Filter(bytes([42]), "unknown kind"))


def test_and_or_trees_compile():
    for q, cols, f, want in and_or_cases(vs.Filter):
        vs.Program(f)


def test_format_float64_matches_oracle_and_golden(oracle):
    # host build of the per-row float64 -> text routine of the scan kernels (marshalFloat64String, values_encoder.go:1397-1399)
    import json, random, struct
    here = os.path.dirname(os.path.abspath(__file__))
    table = json.load(open(os.path.join(here, "golden", "func_tables.json")))["TestMarshalFloat64String"]
    for f, want in table:   # values_encoder_test.go TestMarshalFloat64String
        bits = struct.unpack(">Q", struct.pack(">d", float(bytes.fromhex(f["hex"]) if "hex" in f else f["num"])))[0]
        assert vs.format_float64(bits) == bytes.fromhex(want["hex"])
    rng = random.Random(20240922)
    cases = [0, 1 << 63, 1, 0x7FEFFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0x0010000000000000, 0x000FFFFFFFFFFFFF]
    cases += [rng.getrandbits(64) for _ in range(20000)]
    cases += [rng.getrandbits(52) for _ in range(2000)]   # subnormals
    cases += [struct.unpack(">Q", struct.pack(">d", rng.randint(-10**9, 10**9) / 10 ** rng.randint(0, 9)))[0] for _ in range(20000)]
    cases += [struct.unpack(">Q", struct.pack(">d", float("%de%d" % (m, e))))[0] for e in range(-330, 310) for m in (1, 5, 9)]
    cases += [(e << 52) | m for e in range(0, 2047, 3) for m in (0, 1, (1 << 52) - 1)]
    for bits in cases:
        x = struct.unpack(">d", struct.pack(">Q", bits))[0]
        if x != x:
            assert vs.format_float64(bits) == b"NaN"
            continue
        assert vs.format_float64(bits) == oracle.encoded_to_string(7, struct.pack(">Q", bits)), hex(bits)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on CPU-only hosts")
    assert vs.device_count() == 0
    with pytest.raises(vs.VlscanError) as e:
        vs.Ctx(0)
    assert "no CUDA device" in str(e.value)


def test_token_rune_table_against_an_independent_unicode_database():
    """isTokenRune = unicode.IsLetter || unicode.IsDigit || '_' (tokenizer.go:142-148).  The product's and the oracle's range tables are both generated
    from CPython's unicodedata, so comparing them with each other cannot catch a generation error.  The `regex` module carries its own
    Unicode database (a newer version): on every code point assigned in Unicode 15.0 - Go 1.24's version - its \\p{L} / \\p{Nd} must agree
    with what the product's tokenizer does to the code point, and everything it adds on top must be unassigned in 15.0."""
    import unicodedata
    regex = pytest.importorskip("regex")
    if unicodedata.unidata_version != "15.0.0":
        pytest.skip("needs a Python with Unicode 15.0 tables to know which code points Go 1.24 has assigned")
    letter_or_digit = regex.compile(r"[\p{L}\p{Nd}]")
    cps = [cp for cp in range(0x110000) if not 0xD800 <= cp <= 0xDFFF]
    product = {}
    for i in range(0, len(cps), 1000):
        chunk = cps[i:i + 1000]
        text = " ".join("a" + chr(cp) + "b" for cp in chunk).encode("utf-8")
        tokens = set(vs.Program(vs.Filter.phrase("f", text)).leaf_tokens(0))
        for cp in chunk:
            product[cp] = ("a" + chr(cp) + "b").encode("utf-8") in tokens
    newer_only = 0
    for cp in cps:
        ch = chr(cp)
        independent = letter_or_digit.match(ch) is not None or ch == "_"
        if unicodedata.category(ch) == "Cn":          # unassigned in Unicode 15.0: never a token character for Go 1.24
            assert not product[cp], hex(cp)
            newer_only += independent
        else:
            assert product[cp] == independent, (hex(cp), unicodedata.category(ch), product[cp], independent)
    assert 1000 < newer_only < 20000                  # the other database really is a different (newer) one
