"""ctypes binding of the CPU oracle (oracle/liboracle.so).

TEST INFRASTRUCTURE ONLY: import this from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs, never from victorialogs_b200/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

VT_NAMES = {1: "string", 2: "dict", 3: "uint8", 4: "uint16", 5: "uint32", 6: "uint64", 7: "float64", 8: "ipv4", 9: "iso8601", 10: "int64"}


class GenConfig(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("total_rows", C.c_uint64), ("rows_per_block", C.c_uint32),
                ("hot_block_permille", C.c_uint32), ("hit_row_permille", C.c_uint32), ("columns_mask", C.c_uint32)]


class ColumnView(C.Structure):
    _fields_ = [("name", C.c_void_p), ("name_len", C.c_uint64), ("value_type", C.c_uint32), ("dict_len", C.c_uint32),
                ("min_value", C.c_uint64), ("max_value", C.c_uint64), ("dict_ptr", C.c_void_p * 8), ("dict_lens", C.c_uint64 * 8),
                ("values_block", C.c_void_p), ("values_block_len", C.c_uint64), ("bloom", C.c_void_p), ("bloom_len", C.c_uint64)]


def build():
    subprocess.check_call([os.path.join(_HERE, "build.sh")], stdout=subprocess.DEVNULL)


# the C++ restatements of the facets and stats pipes over this oracle's headers (test infrastructure next to the tests that bind them)
COMPANIONS = (("facets_oracle", "liboracle_facets.so"), ("stats_oracle", "liboracle_stats.so"))


def build_companions():
    """build the restatements a tree lacks (a test directory restored without its build products), as lib() builds liboracle.so; a
    read-only tree is left as it is"""
    tests = os.path.join(os.path.dirname(_HERE), "tests")
    for sub, so in COMPANIONS:
        script = os.path.join(tests, sub, "build.sh")
        if os.path.exists(script) and not os.path.exists(os.path.join(tests, sub, so)) and os.access(os.path.dirname(script), os.W_OK):
            subprocess.check_call([script], stdout=subprocess.DEVNULL)


def lib():
    global _LIB
    if _LIB is None:
        # VLORACLE_LIB: bench.py's CPU arm points this at oracle/_ref/liboracle_zstd157.so (same code linked against the reference's own
        # libzstd 1.5.7 static library) when that build exists; everything else uses the plain build
        path = os.environ.get("VLORACLE_LIB") or os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build()
        build_companions()
        L = C.CDLL(path)
        L.vlo_last_error.restype = C.c_char_p
        L.vlo_xxh64.restype = C.c_uint64
        for name in ("vlo_tokenize_strings", "vlo_tokenize_hashes", "vlo_bloom_marshal_tokens", "vlo_skip_first_last_token",
                     "vlo_regex_describe", "vlo_encoded_to_string", "vlo_marshal_strings_block", "vlo_filter_tokens"):
            getattr(L, name).restype = C.c_int64
        for name in ("vlo_block_build", "vlo_filter_phrase", "vlo_filter_prefix", "vlo_filter_exact", "vlo_filter_in", "vlo_filter_regexp",
                     "vlo_filter_noop", "vlo_filter_and", "vlo_filter_or", "vlo_filter_not", "vlo_gen_block",
                     "vlo_filter_exact_prefix", "vlo_filter_sequence", "vlo_filter_contains_all", "vlo_filter_contains_any", "vlo_filter_any_case_phrase", "vlo_filter_any_case_prefix", "vlo_filter_value_type", "vlo_filter_eq_field", "vlo_filter_range", "vlo_filter_le_field", "vlo_filter_time", "vlo_filter_day_range", "vlo_filter_week_range", "vlo_filter_len_range", "vlo_filter_string_range", "vlo_filter_ipv4_range"):
            getattr(L, name).restype = C.c_void_p
        L.vlo_parse_math_number.restype = C.c_double
        L.vlo_marshal_timestamps.restype = C.c_int64
        for name in ("vlo_block_rows", "vlo_block_ncolumns", "vlo_block_nconsts"):
            getattr(L, name).restype = C.c_uint64
        _LIB = L
    return _LIB


def _b(s):
    return s.encode("utf-8", "surrogateescape") if isinstance(s, str) else bytes(s)


def _pack(strings):
    bs = [_b(s) for s in strings]
    offs = np.zeros(len(bs) + 1, dtype=np.uint64)
    if bs:
        offs[1:] = np.cumsum([len(x) for x in bs], dtype=np.uint64)
    blob = b"".join(bs)
    return blob, offs


def _err():
    return RuntimeError(lib().vlo_last_error().decode())


def xxh64(data):
    data = _b(data)
    return lib().vlo_xxh64(data, C.c_uint64(len(data)))


def tokenize_strings(strings):
    blob, offs = _pack(strings)
    cap = len(blob) + len(strings) + 16
    out = C.create_string_buffer(cap)
    n = lib().vlo_tokenize_strings(blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(strings)), out, C.c_uint64(cap))
    assert n >= 0
    raw = out.raw[:n]
    return [t for t in raw.split(b"\n")] if n else []


def tokenize_hashes(strings):
    blob, offs = _pack(strings)
    cap = len(blob) + 16
    out = np.zeros(cap, dtype=np.uint64)
    n = lib().vlo_tokenize_hashes(blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(strings)), out.ctypes.data_as(C.c_void_p), C.c_uint64(cap))
    assert n >= 0
    return out[:n].copy()


def token_hashes(token):
    token = _b(token)
    out = np.zeros(6, dtype=np.uint64)
    lib().vlo_token_hashes(token, C.c_uint64(len(token)), out.ctypes.data_as(C.c_void_p))
    return out


def bloom_marshal_tokens(tokens):
    blob, offs = _pack(tokens)
    cap = len(tokens) * 2 + 64
    out = C.create_string_buffer(cap)
    n = lib().vlo_bloom_marshal_tokens(blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(tokens)), out, C.c_uint64(cap))
    assert n >= 0
    return out.raw[:n]


def bloom_contains_all(bloom, tokens):
    blob, offs = _pack(tokens)
    r = lib().vlo_bloom_contains_all_tokens(bloom, C.c_uint64(len(bloom)), blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(tokens)))
    assert r >= 0
    return bool(r)


def match_phrase(s, phrase):
    s, phrase = _b(s), _b(phrase)
    return bool(lib().vlo_match_phrase(s, C.c_uint64(len(s)), phrase, C.c_uint64(len(phrase))))


def match_prefix(s, prefix):
    s, prefix = _b(s), _b(prefix)
    return bool(lib().vlo_match_prefix(s, C.c_uint64(len(s)), prefix, C.c_uint64(len(prefix))))


def skip_first_last_token(s):
    s = _b(s)
    out = C.create_string_buffer(len(s) + 1)
    n = lib().vlo_skip_first_last_token(s, C.c_uint64(len(s)), out, C.c_uint64(len(s) + 1))
    return out.raw[:n]


def regex_match(expr, s):
    expr, s = _b(expr), _b(s)
    r = lib().vlo_regex_match(expr, C.c_uint64(len(expr)), s, C.c_uint64(len(s)))
    if r < 0:
        raise _err()
    return bool(r)


def regex_describe(expr):
    expr = _b(expr)
    out = C.create_string_buffer(65536)
    n = lib().vlo_regex_describe(expr, C.c_uint64(len(expr)), out, C.c_uint64(65536))
    if n < 0:
        raise _err()
    d = {}
    for line in out.raw[:n].decode("utf-8", "replace").split("\n"):
        k, _, v = line.partition("=")
        d[k] = v
    return d


def _parse(fn, ctype, s):
    s = _b(s)
    out = ctype()
    ok = fn(s, C.c_uint64(len(s)), C.byref(out))
    return (out.value, bool(ok))


def try_parse_uint64(s):
    return _parse(lib().vlo_try_parse_uint64, C.c_uint64, s)


def try_parse_int64(s):
    return _parse(lib().vlo_try_parse_int64, C.c_int64, s)


def try_parse_float64(s):
    return _parse(lib().vlo_try_parse_float64, C.c_double, s)


def try_parse_ipv4(s):
    return _parse(lib().vlo_try_parse_ipv4, C.c_uint32, s)


def try_parse_iso8601(s):
    return _parse(lib().vlo_try_parse_iso8601, C.c_int64, s)


def encoded_to_string(vt, v):
    out = C.create_string_buffer(512)
    n = lib().vlo_encoded_to_string(C.c_int(vt), v, C.c_uint64(len(v)), out, C.c_uint64(512))
    if n < 0:
        raise _err()
    return out.raw[:n]


def marshal_strings_block(strings):
    blob, offs = _pack(strings)
    cap = len(blob) + 9 * len(strings) + 1024
    out = C.create_string_buffer(cap)
    n = lib().vlo_marshal_strings_block(blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(strings)), out, C.c_uint64(cap))
    if n < 0:
        raise _err()
    return out.raw[:n]


def decode_values_block(src, cap=None):
    """-> (lens_items bytes, data bytes): the post-ZSTD stage of a values block."""
    cap = cap or (64 << 20)
    lens = C.create_string_buffer(cap)
    data = C.create_string_buffer(cap)
    ll, dl = C.c_uint64(cap), C.c_uint64(cap)
    if lib().vlo_decode_values_block(src, C.c_uint64(len(src)), lens, C.byref(ll), data, C.byref(dl)):
        raise _err()
    return lens.raw[:ll.value], data.raw[:dl.value]


def unmarshal_strings_block(src, items, cap=None):
    cap = cap or (64 << 20)
    out = C.create_string_buffer(cap)
    offs = np.zeros(items + 1, dtype=np.uint64)
    if lib().vlo_unmarshal_strings_block(src, C.c_uint64(len(src)), C.c_uint64(items), out, C.c_uint64(cap), offs.ctypes.data_as(C.c_void_p)):
        raise _err()
    raw = out.raw
    return [raw[int(offs[i]):int(offs[i + 1])] for i in range(items)]


class Column:
    __slots__ = ("name", "value_type", "min_value", "max_value", "dict", "values_block", "bloom")


class Block:
    """An encoded block as the reference writer would produce it (one column = header fields + values block + bloom)."""

    def __init__(self, handle):
        assert handle, _err()
        self.h = C.c_void_p(handle)
        L = lib()
        self.rows = L.vlo_block_rows(self.h)
        self.columns = []
        for i in range(L.vlo_block_ncolumns(self.h)):
            v = ColumnView()
            L.vlo_block_column(self.h, C.c_uint64(i), C.byref(v))
            c = Column()
            c.name = C.string_at(v.name, v.name_len)
            c.value_type = v.value_type
            c.min_value, c.max_value = v.min_value, v.max_value
            c.dict = [C.string_at(v.dict_ptr[k], v.dict_lens[k]) for k in range(v.dict_len)]
            c.values_block = C.string_at(v.values_block, v.values_block_len)
            c.bloom = C.string_at(v.bloom, v.bloom_len)
            self.columns.append(c)
        self.consts = []
        for i in range(L.vlo_block_nconsts(self.h)):
            n, nl, val, vl = C.c_void_p(), C.c_uint64(), C.c_void_p(), C.c_uint64()
            L.vlo_block_const(self.h, C.c_uint64(i), C.byref(n), C.byref(nl), C.byref(val), C.byref(vl))
            self.consts.append((C.string_at(n, nl.value), C.string_at(val, vl.value)))

    def __del__(self):
        try:
            lib().vlo_block_free(self.h)
        except Exception:
            pass

    @staticmethod
    def from_columns(columns, rows=None):
        """columns: list of (name, [values...]) column-major, like `[]column{{name, values}}` in filter_test.go."""
        names = [c[0] for c in columns]
        if rows is None:
            rows = len(columns[0][1]) if columns else 0
        vals = []
        for _, v in columns:
            assert len(v) == rows
            vals.extend(v)
        nb, no = _pack(names)
        vb, vo = _pack(vals)
        h = lib().vlo_block_build(nb, no.ctypes.data_as(C.c_void_p), C.c_uint64(len(names)), vb, vo.ctypes.data_as(C.c_void_p), C.c_uint64(rows))
        if not h:
            raise _err()
        return Block(h)

    def set_timestamps(self, timestamps):
        """timestamps: sorted int64 nanoseconds, one per row (the block's _time column)."""
        a = np.asarray(timestamps, dtype=np.int64)
        if lib().vlo_block_set_timestamps(self.h, a.ctypes.data_as(C.c_void_p), C.c_uint64(len(a))):
            raise _err()
        return self

    def timestamps_block(self):
        """-> (encoded bytes, marshalType, minTimestamp, maxTimestamp): what timestamps.bin + the block header hold"""
        p, n, mt, mn, mx = C.c_void_p(), C.c_uint64(), C.c_int(), C.c_int64(), C.c_int64()
        if lib().vlo_block_timestamps(self.h, C.byref(p), C.byref(n), C.byref(mt), C.byref(mn), C.byref(mx)):
            raise ValueError("the block has no timestamps")
        return C.string_at(p, n.value), mt.value, mn.value, mx.value

    @staticmethod
    def generated(cfg, block_id):
        h = lib().vlo_gen_block(C.byref(cfg), C.c_uint64(block_id))
        if not h:
            raise _err()
        return Block(h)

    def search(self, flt, stats=None):
        words = np.zeros((self.rows + 63) // 64, dtype=np.uint64)
        st = stats.ctypes.data_as(C.c_void_p) if stats is not None else None
        if lib().vlo_block_search(self.h, flt.h, words.ctypes.data_as(C.c_void_p), st):
            raise _err()
        return words


def bitmap_rows(words, rows):
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:rows]
    return [int(i) for i in np.nonzero(bits)[0]]


class Filter:
    def __init__(self, handle, keep=()):
        if not handle:
            raise _err()
        self.h = C.c_void_p(handle)
        self._keep = keep

    def tokens(self):
        out = C.create_string_buffer(65536)
        n = lib().vlo_filter_tokens(self.h, out, C.c_uint64(65536))
        assert n >= 0
        return out.raw[:n].split(b"\n") if n else []

    @staticmethod
    def phrase(field, phrase):
        f, p = _b(field), _b(phrase)
        return Filter(lib().vlo_filter_phrase(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def prefix(field, prefix):
        f, p = _b(field), _b(prefix)
        return Filter(lib().vlo_filter_prefix(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def exact(field, value):
        f, p = _b(field), _b(value)
        return Filter(lib().vlo_filter_exact(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def in_(field, values):
        f = _b(field)
        blob, offs = _pack(values)
        return Filter(lib().vlo_filter_in(f, C.c_uint64(len(f)), blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(values))))

    @staticmethod
    def regexp(field, expr):
        f, p = _b(field), _b(expr)
        return Filter(lib().vlo_filter_regexp(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    # --- SURVEY §8(f) rank 3 filters (oracle side; pinned by the reference's filter_*_test.go tables) ---
    @staticmethod
    def exact_prefix(field, prefix):
        f, p = _b(field), _b(prefix)
        return Filter(lib().vlo_filter_exact_prefix(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def sequence(field, phrases):
        f = _b(field)
        blob, offs = _pack(phrases)
        return Filter(lib().vlo_filter_sequence(f, C.c_uint64(len(f)), blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(phrases))))

    @staticmethod
    def any_case_phrase(field, phrase):
        f, p = _b(field), _b(phrase)
        return Filter(lib().vlo_filter_any_case_phrase(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def any_case_prefix(field, prefix):
        f, p = _b(field), _b(prefix)
        return Filter(lib().vlo_filter_any_case_prefix(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def value_type(field, type_name):
        f, p = _b(field), _b(type_name)
        return Filter(lib().vlo_filter_value_type(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def range(field, min_value, max_value):
        f = _b(field)
        return Filter(lib().vlo_filter_range(f, C.c_uint64(len(f)), C.c_double(min_value), C.c_double(max_value)))

    @staticmethod
    def le_field(field, other_field, exclude_equal=False):
        f, p = _b(field), _b(other_field)
        return Filter(lib().vlo_filter_le_field(f, C.c_uint64(len(f)), p, C.c_uint64(len(p)), C.c_int(1 if exclude_equal else 0)))

    @staticmethod
    def day_range(start, end, offset=0):
        return Filter(lib().vlo_filter_day_range(C.c_int64(start), C.c_int64(end), C.c_int64(offset)))

    @staticmethod
    def week_range(start_day, end_day, offset=0):
        return Filter(lib().vlo_filter_week_range(C.c_int(start_day), C.c_int(end_day), C.c_int64(offset)))

    @staticmethod
    def time(min_timestamp, max_timestamp):
        return Filter(lib().vlo_filter_time(C.c_int64(min_timestamp), C.c_int64(max_timestamp)))

    @staticmethod
    def eq_field(field, other_field):
        f, p = _b(field), _b(other_field)
        return Filter(lib().vlo_filter_eq_field(f, C.c_uint64(len(f)), p, C.c_uint64(len(p))))

    @staticmethod
    def contains_all(field, values):
        f = _b(field)
        blob, offs = _pack(values)
        return Filter(lib().vlo_filter_contains_all(f, C.c_uint64(len(f)), blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(values))))

    @staticmethod
    def contains_any(field, values):
        f = _b(field)
        blob, offs = _pack(values)
        return Filter(lib().vlo_filter_contains_any(f, C.c_uint64(len(f)), blob, offs.ctypes.data_as(C.c_void_p), C.c_uint64(len(values))))

    @staticmethod
    def len_range(field, min_len, max_len):
        f = _b(field)
        return Filter(lib().vlo_filter_len_range(f, C.c_uint64(len(f)), C.c_uint64(min_len), C.c_uint64(max_len)))

    @staticmethod
    def string_range(field, min_value, max_value):
        f, a, b = _b(field), _b(min_value), _b(max_value)
        return Filter(lib().vlo_filter_string_range(f, C.c_uint64(len(f)), a, C.c_uint64(len(a)), b, C.c_uint64(len(b))))

    @staticmethod
    def ipv4_range(field, min_value, max_value):
        f = _b(field)
        return Filter(lib().vlo_filter_ipv4_range(f, C.c_uint64(len(f)), C.c_uint32(min_value), C.c_uint32(max_value)))

    @staticmethod
    def noop():
        return Filter(lib().vlo_filter_noop())

    @staticmethod
    def and_(filters):
        arr = (C.c_void_p * len(filters))(*[f.h for f in filters])
        return Filter(lib().vlo_filter_and(arr, C.c_uint64(len(filters))), keep=tuple(filters))

    @staticmethod
    def or_(filters):
        arr = (C.c_void_p * len(filters))(*[f.h for f in filters])
        return Filter(lib().vlo_filter_or(arr, C.c_uint64(len(filters))), keep=tuple(filters))

    @staticmethod
    def not_(f):
        return Filter(lib().vlo_filter_not(f.h), keep=(f,))


def marshal_timestamps(timestamps):
    """encoding.MarshalTimestamps(ts, 64) -> (bytes, marshalType, firstTimestamp)"""
    a = np.asarray(timestamps, dtype=np.int64)
    out = C.create_string_buffer(len(a) * 10 + 64)
    mt, first = C.c_int(), C.c_int64()
    n = lib().vlo_marshal_timestamps(a.ctypes.data_as(C.c_void_p), C.c_uint64(len(a)), out, C.c_uint64(len(out)), C.byref(mt), C.byref(first))
    if n < 0:
        raise _err()
    return out.raw[:n], mt.value, first.value


def unmarshal_timestamps(data, marshal_type, first, items):
    out = np.zeros(items, dtype=np.int64)
    if lib().vlo_unmarshal_timestamps(data, C.c_uint64(len(data)), C.c_int(marshal_type), C.c_int64(first), C.c_uint64(items), out.ctypes.data_as(C.c_void_p)):
        raise _err()
    return out


def gen_rows(cfg, block_id, column, cap=None):
    rows = min(cfg.rows_per_block, cfg.total_rows - block_id * cfg.rows_per_block)
    cap = cap or rows * 256 + 1024
    out = C.create_string_buffer(cap)
    offs = np.zeros(rows + 1, dtype=np.uint64)
    if lib().vlo_gen_rows(C.byref(cfg), C.c_uint64(block_id), C.c_int(column), out, C.c_uint64(cap), offs.ctypes.data_as(C.c_void_p)):
        raise _err()
    raw = out.raw
    return [raw[int(offs[i]):int(offs[i + 1])] for i in range(rows)]


def scan_generated(cfg, flt, block_lo, block_hi, threads, want_counts=False, passes=1, post_zstd=False, pin=False):
    """CPU baseline: multi-threaded blockSearch over generated blocks. -> dict(secs, stats, digest, matches, counts).
    post_zstd: values blocks are decompressed before the timed region (the input stage of the device-resident scan); pin: worker t -> CPU t."""
    secs = C.c_double()
    stats = np.zeros(6, dtype=np.uint64)
    dig, tot = C.c_uint64(), C.c_uint64()
    counts = np.zeros(block_hi - block_lo, dtype=np.uint32) if want_counts else None
    r = lib().vlo_scan_generated(C.byref(cfg), flt.h, C.c_uint64(block_lo), C.c_uint64(block_hi), C.c_int(threads), C.c_int(passes), C.byref(secs),
                                 stats.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p) if want_counts else None,
                                 C.byref(dig), C.byref(tot), C.c_int((1 if post_zstd else 0) | (2 if pin else 0)))
    if r:
        raise _err()
    return dict(secs=secs.value, passes=passes, stats=stats, digest=dig.value, matches=tot.value, counts=counts)


# ---- part files (oracle/vlo_part.h) --------------------------------------------------------------------------------------
BLOCK_HEADER_FIELDS = ("account_id", "project_id", "id_hi", "id_lo", "uncompressed_size_bytes", "rows_count", "ts_block_offset", "ts_block_size",
                       "min_timestamp", "max_timestamp", "ts_marshal_type", "columns_header_index_offset", "columns_header_index_size",
                       "columns_header_offset", "columns_header_size")
INDEX_BLOCK_HEADER_FIELDS = ("account_id", "project_id", "id_hi", "id_lo", "min_timestamp", "max_timestamp", "index_block_offset", "index_block_size")
COLUMN_HEADER_FIELDS = ("value_type", "min_value", "max_value", "values_offset", "values_size", "bloom_filter_offset", "bloom_filter_size")
PART_HEADER_FIELDS = ("FormatVersion", "CompressedSizeBytes", "UncompressedSizeBytes", "RowsCount", "BlocksCount", "MinTimestamp", "MaxTimestamp",
                      "BloomValuesShardsCount")
_SIGNED = {"min_timestamp", "max_timestamp", "MinTimestamp", "MaxTimestamp"}


def _to_u64s(fields, d):
    return np.array([int(d.get(k, 0)) & 0xFFFFFFFFFFFFFFFF for k in fields], dtype=np.uint64)


def _from_u64s(fields, a):
    out = {}
    for k, v in zip(fields, a):
        v = int(v)
        out[k] = v - (1 << 64) if k in _SIGNED and v >= 1 << 63 else v
    return out


def _i64(fn, *args):
    fn.restype = C.c_int64
    r = fn(*args)
    if r < 0:
        raise _err()
    return r


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def marshal_block_header(**f):
    out = C.create_string_buffer(256)
    a = _to_u64s(BLOCK_HEADER_FIELDS, f)
    n = _i64(lib().vlo_part_marshal_block_header, _ptr(a), out, C.c_uint64(256))
    return out.raw[:n]


def unmarshal_block_headers(data, format_version=3):
    data = bytes(data)
    cap = len(data) // 30 + 1
    out = np.zeros(cap * 15, dtype=np.uint64)
    n = _i64(lib().vlo_part_unmarshal_block_headers, data, C.c_uint64(len(data)), C.c_uint(format_version), _ptr(out), C.c_uint64(cap))
    return [_from_u64s(BLOCK_HEADER_FIELDS, out[15 * i:15 * i + 15]) for i in range(n)]


def marshal_index_block_header(**f):
    out = C.create_string_buffer(64)
    a = _to_u64s(INDEX_BLOCK_HEADER_FIELDS, f)
    n = _i64(lib().vlo_part_marshal_index_block_header, _ptr(a), out, C.c_uint64(64))
    return out.raw[:n]


def unmarshal_index_block_headers(data):
    data = bytes(data)
    cap = len(data) // 56 + 1
    out = np.zeros(cap * 8, dtype=np.uint64)
    n = _i64(lib().vlo_part_unmarshal_index_block_headers, data, C.c_uint64(len(data)), _ptr(out), C.c_uint64(cap))
    return [_from_u64s(INDEX_BLOCK_HEADER_FIELDS, out[8 * i:8 * i + 8]) for i in range(n)]


def marshal_column_header(dict_values=(), **f):
    out = C.create_string_buffer(4096)
    a = _to_u64s(COLUMN_HEADER_FIELDS, f)
    db, do = _pack(dict_values)
    n = _i64(lib().vlo_part_marshal_column_header, _ptr(a), db, _ptr(do), C.c_uint64(len(dict_values)), out, C.c_uint64(4096))
    return out.raw[:n]


def unmarshal_column_header(data, format_version=3):
    """-> (fields dict incl. 'dict', bytes consumed)"""
    data = bytes(data)
    f7 = np.zeros(7, dtype=np.uint64)
    dbuf = C.create_string_buffer(len(data) + 1)
    doffs = np.zeros(257, dtype=np.uint64)
    nd = C.c_uint64()
    used = _i64(lib().vlo_part_unmarshal_column_header, data, C.c_uint64(len(data)), C.c_uint(format_version), _ptr(f7), dbuf, C.c_uint64(len(data) + 1), _ptr(doffs), C.byref(nd))
    d = _from_u64s(COLUMN_HEADER_FIELDS, f7)
    d["dict"] = [dbuf.raw[int(doffs[i]):int(doffs[i + 1])] for i in range(nd.value)]
    return d, used


def marshal_columns_header_index(refs, const_refs):
    """refs / const_refs: lists of (columnNameID, offset)"""
    a = np.array([x for r in refs for x in r], dtype=np.uint64)
    b = np.array([x for r in const_refs for x in r], dtype=np.uint64)
    cap = 20 * (len(refs) + len(const_refs)) + 20
    out = C.create_string_buffer(cap)
    n = _i64(lib().vlo_part_marshal_columns_header_index, _ptr(a), C.c_uint64(len(refs)), _ptr(b), C.c_uint64(len(const_refs)), out, C.c_uint64(cap))
    return out.raw[:n]


def unmarshal_columns_header_index(data):
    data = bytes(data)
    cap = len(data) + 1
    a, b = np.zeros(2 * cap, dtype=np.uint64), np.zeros(2 * cap, dtype=np.uint64)
    na, nb = C.c_uint64(), C.c_uint64()
    if lib().vlo_part_unmarshal_columns_header_index(data, C.c_uint64(len(data)), _ptr(a), C.byref(na), _ptr(b), C.byref(nb), C.c_uint64(cap)):
        raise _err()
    return ([(int(a[2 * i]), int(a[2 * i + 1])) for i in range(na.value)], [(int(b[2 * i]), int(b[2 * i + 1])) for i in range(nb.value)])


def marshal_columns_header(columns, const_columns):
    """columns: list of (name, fields dict without dict values); const_columns: list of (name, value) -> (columnsHeader bytes, columnsHeaderIndex bytes)"""
    f = np.concatenate([_to_u64s(COLUMN_HEADER_FIELDS, c[1]) for c in columns]) if columns else np.zeros(0, dtype=np.uint64)
    nb, no = _pack([c[0] for c in columns] + [c[0] for c in const_columns])
    vb, vo = _pack([c[1] for c in const_columns])
    cap = 64 * len(columns) + sum(len(_b(c[1])) + 16 for c in const_columns) + 64
    out, idx = C.create_string_buffer(cap), C.create_string_buffer(cap)
    il = C.c_uint64()
    n = _i64(lib().vlo_part_marshal_columns_header, C.c_uint64(len(columns)), _ptr(f), nb, _ptr(no), C.c_uint64(len(const_columns)), vb, _ptr(vo),
             out, C.c_uint64(cap), idx, C.c_uint64(cap), C.byref(il))
    return out.raw[:n], idx.raw[:il.value]


def columns_header_roundtrip(csh, idx, names):
    """unmarshal + setColumnNames + marshal again -> (bytes identical?, resolved names: columns then const columns)"""
    csh, idx = bytes(csh), bytes(idx)
    nb, no = _pack(names)
    cap = sum(len(_b(x)) + 1 for x in names) * 4 + len(csh) * 260 + 64
    out = C.create_string_buffer(cap)
    ol = C.c_uint64()
    r = lib().vlo_part_columns_header_roundtrip(csh, C.c_uint64(len(csh)), idx, C.c_uint64(len(idx)), nb, _ptr(no), C.c_uint64(len(names)), out, C.c_uint64(cap), C.byref(ol))
    if r < 0:
        raise _err()
    return bool(r), out.raw[:ol.value].split(b"\0")[:-1]


def part_header_json(**f):
    out = C.create_string_buffer(512)
    a = _to_u64s(PART_HEADER_FIELDS, f)
    n = _i64(lib().vlo_part_header_json, _ptr(a), out, C.c_uint64(512))
    return out.raw[:n]


def part_header_parse(text):
    text = _b(text)
    f8 = np.zeros(8, dtype=np.uint64)
    if lib().vlo_part_header_parse(text, C.c_uint64(len(text)), _ptr(f8)):
        raise _err()
    return _from_u64s(PART_HEADER_FIELDS, f8)


class PartWriter:
    """blockStreamWriter for a file part: add blocks in (streamID, minTimestamp) order, then finalize() -> {file name: bytes}."""

    def __init__(self, max_index_block=0, max_shards=0):
        L = lib()
        L.vlo_part_writer_new.restype = C.c_void_p
        L.vlo_part_writer_nfiles.restype = C.c_uint64
        self.h = C.c_void_p(L.vlo_part_writer_new(C.c_uint64(max_index_block), C.c_uint64(max_shards)))
        self.header = None

    def __del__(self):
        try:
            lib().vlo_part_writer_free(self.h)
        except Exception:
            pass

    def add_block(self, stream_id, block, uncompressed_size=0):
        """stream_id: (accountID, projectID, hi, lo)"""
        sid = np.array(stream_id, dtype=np.uint64)
        if lib().vlo_part_writer_add_block(self.h, _ptr(sid), block.h, C.c_uint64(uncompressed_size)):
            raise _err()

    def finalize(self):
        L = lib()
        f8 = np.zeros(8, dtype=np.uint64)
        if L.vlo_part_writer_finalize(self.h, _ptr(f8)):
            raise _err()
        self.header = _from_u64s(PART_HEADER_FIELDS, f8)
        files = {}
        for i in range(L.vlo_part_writer_nfiles(self.h)):
            n, nl, d, dl = C.c_void_p(), C.c_uint64(), C.c_void_p(), C.c_uint64()
            L.vlo_part_writer_file(self.h, C.c_uint64(i), C.byref(n), C.byref(nl), C.byref(d), C.byref(dl))
            # ctypes.string_at takes a C int: a values file of a large part is longer than 2 GiB
            files[C.string_at(n, nl.value).decode()] = (C.c_char * dl.value).from_address(d.value).raw if dl.value else b""
        return files


def save_part(files, path):
    os.makedirs(path, exist_ok=False)      # fs.MustMkdirFailIfExist
    for name, data in files.items():
        with open(os.path.join(path, name), "wb") as f:
            f.write(data)


def load_part(path):
    return {name: open(os.path.join(path, name), "rb").read() for name in sorted(os.listdir(path))}


class PartReader:
    """part.mustOpenFilePart + the block access of blockSearch, over {file name: bytes}."""

    def __init__(self, files):
        L = lib()
        L.vlo_part_reader_open.restype = C.c_void_p
        L.vlo_part_reader_block.restype = C.c_void_p
        for name in ("vlo_part_reader_nindex", "vlo_part_reader_nblocks"):
            getattr(L, name).restype = C.c_uint64
        names = sorted(files)
        nb, no = _pack(names)
        db, do = _pack([files[k] for k in names])
        h = L.vlo_part_reader_open(nb, _ptr(no), db, _ptr(do), C.c_uint64(len(names)))
        if not h:
            raise _err()
        self.h = C.c_void_p(h)
        f8 = np.zeros(8, dtype=np.uint64)
        L.vlo_part_reader_header(self.h, _ptr(f8))
        self.header = _from_u64s(PART_HEADER_FIELDS, f8)
        self.nblocks = L.vlo_part_reader_nblocks(self.h)
        cap = sum(len(v) for v in files.values()) * 300 + 1024
        out = C.create_string_buffer(cap)
        n = _i64(L.vlo_part_reader_column_names, self.h, out, C.c_uint64(cap))
        self.column_names = out.raw[:n].split(b"\0")[:-1]

    def __del__(self):
        try:
            lib().vlo_part_reader_free(self.h)
        except Exception:
            pass

    def index_block_headers(self):
        L = lib()
        res = []
        for i in range(L.vlo_part_reader_nindex(self.h)):
            f8 = np.zeros(8, dtype=np.uint64)
            L.vlo_part_reader_index_header(self.h, C.c_uint64(i), _ptr(f8))
            res.append(_from_u64s(INDEX_BLOCK_HEADER_FIELDS, f8))
        return res

    def block_header(self, i):
        f = np.zeros(15, dtype=np.uint64)
        lib().vlo_part_reader_block_header(self.h, C.c_uint64(i), _ptr(f))
        return _from_u64s(BLOCK_HEADER_FIELDS, f)

    def block(self, i):
        h = lib().vlo_part_reader_block(self.h, C.c_uint64(i))
        if not h:
            raise _err()
        return Block(h)

    def column_header(self, i, name):
        """blockSearch.getColumnHeader -> fields dict or None"""
        name = _b(name)
        f7 = np.zeros(7, dtype=np.uint64)
        r = lib().vlo_part_reader_column_header(self.h, C.c_uint64(i), name, C.c_uint64(len(name)), _ptr(f7))
        if r < 0:
            raise _err()
        return _from_u64s(COLUMN_HEADER_FIELDS, f7) if r else None

    def const_value(self, i, name):
        name = _b(name)
        out = C.create_string_buffer(1 << 16)
        n = _i64(lib().vlo_part_reader_const_value, self.h, C.c_uint64(i), name, C.c_uint64(len(name)), out, C.c_uint64(1 << 16))
        return out.raw[:n]
