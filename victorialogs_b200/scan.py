"""ctypes host-side mirror of lib/logstorage's filter / blockSearch interface on top of libvlscan.so (include/vlscan.h).

The reference's host language is Go and there is no Go toolchain in this image, so the host side above the C ABI that a
Go maintainer would write (INTEGRATION.md shows the cgo stub) is mirrored here in Python with the same names and
argument meaning as the Go structs:

    filterPhrase{fieldName, phrase}      -> Filter.phrase(field, phrase)        lib/logstorage/filter_phrase.go:25-32
    filterPrefix{fieldName, prefix}      -> Filter.prefix(field, prefix)        filter_prefix.go:20-27
    filterExact{fieldName, value}        -> Filter.exact(field, value)          filter_exact.go:17-24
    filterIn{fieldName, values}          -> Filter.in_(field, values)           filter_in.go:14-18
    filterRegexp{fieldName, re}          -> Filter.regexp(field, expr)          filter_regexp.go:17-24
    filterAnd / filterOr / filterNot     -> Filter.and_ / or_ / not_            filter_and.go, filter_or.go, filter_not.go
    blockSearch.search(bsw, bm)          -> Ctx.scan_batch(program, blocks)     block_search.go:207-226

There is no CPU fallback: loading fails loudly when libvlscan.so is missing and every scan fails without a CUDA device.
"""
import ctypes as C
import math
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

F_NOOP, F_PHRASE, F_PREFIX, F_EXACT, F_IN, F_REGEXP, F_AND, F_OR, F_NOT = range(9)
F_EXACT_PREFIX, F_LEN_RANGE, F_STRING_RANGE, F_IPV4_RANGE, F_VALUE_TYPE = 9, 10, 11, 12, 13
F_ANY_CASE_PHRASE, F_ANY_CASE_PREFIX, F_SEQUENCE, F_CONTAINS_ALL, F_CONTAINS_ANY, F_EQ_FIELD, F_LE_FIELD, F_RANGE, F_TIME = 14, 15, 16, 17, 18, 19, 20, 21, 22
VT_STRING, VT_DICT, VT_UINT8, VT_UINT16, VT_UINT32, VT_UINT64, VT_FLOAT64, VT_IPV4, VT_ISO8601, VT_INT64 = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
COL_CONST, COL_VALUES = 1, 2
STAGE_ONDISK, STAGE_DECODED = 0, 1


class VlscanError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("vlscan error %d: %s" % (code, msg))
        self.code = code


class CColumn(C.Structure):
    _fields_ = [("field", C.c_uint32), ("kind", C.c_uint8), ("value_type", C.c_uint8), ("stage", C.c_uint8), ("dict_len", C.c_uint8),
                ("min_value", C.c_uint64), ("max_value", C.c_uint64),
                ("const_value", C.c_void_p), ("const_len", C.c_uint64),
                ("dict_blob", C.c_void_p), ("dict_offsets", C.c_void_p),
                ("values", C.c_void_p), ("values_len", C.c_uint64),
                ("lens_items", C.c_void_p), ("lens_items_len", C.c_uint64),
                ("data", C.c_void_p), ("data_len", C.c_uint64),
                ("bloom", C.c_void_p), ("bloom_len", C.c_uint64)]


class CBlock(C.Structure):
    _fields_ = [("rows", C.c_uint64), ("ncols", C.c_uint32), ("ts_marshal_type", C.c_uint32), ("cols", C.POINTER(CColumn)),
                ("timestamps", C.c_void_p), ("timestamps_len", C.c_uint64), ("min_timestamp", C.c_int64), ("max_timestamp", C.c_int64)]


class CStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("blocks", "rows", "rows_matched", "blocks_matched", "values_bytes", "bloom_probe_bytes", "bitmap_bytes",
                                          "columns_read", "gpu_launches", "h2d_bytes", "d2h_bytes")] + \
               [("gpu_ms", C.c_double), ("scan_kernel_ms", C.c_double), ("scan_kernel_bytes", C.c_uint64), ("staged_columns", C.c_uint64), ("pruned_columns", C.c_uint64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


BUCKET_PLAIN, BUCKET_WEEK, BUCKET_MONTH, BUCKET_YEAR = 0, 1, 2, 3
HITS_MAX_BY = 4
GEN_TIMESTAMPS = 1 << 4                   # vlscan_gen_config.columns_mask bit: a timestamps column per generated block
GEN_T0, GEN_STEP = 1700000000000000000, 1000000   # row i of a generated data set is at GEN_T0 + i * GEN_STEP nanoseconds
GEN_STREAMS_SHIFT = 12                    # columns_mask bits 12..16 = k (with GEN_TIMESTAMPS only): 2^k generated blocks interleave in time
I64_MIN = -(1 << 63)


def gen_streams(k):
    """columns_mask bits that interleave 2^k generated blocks in time (row i of block b at GEN_T0 + ((b // S) * S * R + i * S + b % S) * GEN_STEP)"""
    return k << GEN_STREAMS_SHIFT


class ByBucket(C.Structure):
    _fields_ = [("size", C.c_double), ("offset", C.c_double), ("calendar", C.c_uint32), ("enabled", C.c_uint32)]


class HitsQuery(C.Structure):
    _fields_ = [("step", C.c_int64), ("offset", C.c_int64), ("calendar", C.c_uint32), ("nby", C.c_uint32),
                ("by_names", C.POINTER(C.c_char_p)), ("by_name_lens", C.POINTER(C.c_size_t))]


class LastQuery(C.Structure):
    _fields_ = [("limit", C.c_uint64), ("min_timestamp", C.c_int64), ("nfields", C.c_uint32),
                ("field_names", C.POINTER(C.c_char_p)), ("field_name_lens", C.POINTER(C.c_size_t))]


class FacetsQuery(C.Structure):
    _fields_ = [("max_values_per_field", C.c_uint64), ("max_value_len", C.c_uint64), ("nfields", C.c_uint32),
                ("field_names", C.POINTER(C.c_char_p)), ("field_name_lens", C.POINTER(C.c_size_t))]


FACET_UINT64, FACET_NEGATIVE, FACET_STRING = 0, 1, 2
FACETS_DEFAULT_MAX_VALUES, FACETS_DEFAULT_MAX_VALUE_LEN = 1000, 128


class GenConfig(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("total_rows", C.c_uint64), ("rows_per_block", C.c_uint32), ("hot_block_permille", C.c_uint32),
                ("hit_row_permille", C.c_uint32), ("columns_mask", C.c_uint32)]


EXPORTS = ["vlscan_device_count", "vlscan_ctx_create", "vlscan_ctx_free", "vlscan_last_error", "vlscan_ctx_stream", "vlscan_ctx_sync",
           "vlscan_program_create", "vlscan_program_free", "vlscan_program_nfields", "vlscan_program_field", "vlscan_program_leaf_tokens", "vlscan_program_prepass_tokens", "vlscan_program_in_hashes", "vlscan_program_in_typed", "vlscan_format_float64", "vlscan_parse_math_number", "vlscan_parse_typed", "vlscan_eval_predicate",
           "vlscan_batch_upload", "vlscan_batch_free", "vlscan_batch_nblocks", "vlscan_batch_rows", "vlscan_batch_words", "vlscan_batch_device_bytes",
           "vlscan_batch_generate", "vlscan_batch_download", "vlscan_host_blocks_get", "vlscan_host_blocks_field", "vlscan_host_blocks_bytes",
           "vlscan_host_blocks_free", "vlscan_host_blocks_compress", "vlscan_zstd_decompress", "vlscan_zstd_inspect", "vlscan_zstd_walk_digest", "vlscan_part_open", "vlscan_part_free", "vlscan_part_header", "vlscan_part_nblocks", "vlscan_part_block_header", "vlscan_part_timestamps",
           "vlscan_part_ncolumn_names", "vlscan_part_column_name", "vlscan_part_blocks", "vlscan_host_blocks_source", "vlscan_scan_resident", "vlscan_last_scan_stats", "vlscan_fetch_results", "vlscan_fetch_hits", "vlscan_gather_timestamps", "vlscan_gather_values", "vlscan_hits_stats", "vlscan_hits_sums", "vlscan_hits_stats_bucketed", "vlscan_hits_sums_bucketed", "vlscan_hits_vmranges", "vlscan_vmrange_index", "vlscan_vmrange_text", "vlscan_truncate_timestamp", "vlscan_bucket_text", "vlscan_last_rows", "vlscan_facets", "vlscan_result_digest", "vlscan_totals_sum", "vlscan_result_device_ptrs", "vlscan_scan_batch",
           "vlscan_scan_batch_keep", "vlscan_stage_selected"]


def lib_path():
    return os.path.join(_HERE, "libvlscan.so")


def lib():
    global _LIB
    if _LIB is None:
        path = lib_path()
        if not os.path.exists(path):
            raise ImportError("libvlscan.so is missing (%s): build it with victorialogs_b200/build.sh; there is no fallback path" % path)
        L = C.CDLL(path)
        L.vlscan_ctx_create.restype = C.c_void_p
        L.vlscan_last_error.restype = C.c_char_p
        L.vlscan_last_error.argtypes = [C.c_void_p]
        L.vlscan_ctx_stream.restype = C.c_void_p
        L.vlscan_ctx_stream.argtypes = [C.c_void_p]
        L.vlscan_program_field.restype = C.c_void_p
        L.vlscan_host_blocks_field.restype = C.c_void_p
        L.vlscan_host_blocks_get.restype = C.POINTER(CBlock)
        L.vlscan_program_leaf_tokens.restype = C.c_int64
        for n in ("vlscan_batch_nblocks", "vlscan_batch_rows", "vlscan_batch_words", "vlscan_batch_device_bytes", "vlscan_host_blocks_bytes"):
            getattr(L, n).restype = C.c_uint64
            getattr(L, n).argtypes = [C.c_void_p]
        for n in ("vlscan_ctx_free", "vlscan_program_free", "vlscan_batch_free", "vlscan_host_blocks_free"):
            getattr(L, n).argtypes = [C.c_void_p]
            getattr(L, n).restype = None
        L.vlscan_truncate_timestamp.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_uint32]
        L.vlscan_truncate_timestamp.restype = C.c_int64
        L.vlscan_vmrange_index.argtypes = [C.c_double]
        L.vlscan_vmrange_text.argtypes = [C.c_uint32, C.c_char_p, C.c_size_t]
        L.vlscan_format_float64.argtypes = [C.c_uint64, C.c_char_p, C.c_size_t]
        L.vlscan_format_float64.restype = C.c_int
        _LIB = L
    return _LIB


def eval_predicate(kind, value, arg1=b"", arg2=b"", aux0=0, aux1=0):
    """Host build of the per-value predicate of filter kinds 9..12 (vlscan_eval_predicate)."""
    value, arg1, arg2 = _b(value), _b(arg1), _b(arg2)
    L = lib()
    L.vlscan_eval_predicate.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint64, C.c_uint64]
    r = L.vlscan_eval_predicate(kind, value, len(value), arg1, len(arg1), arg2, len(arg2), aux0, aux1)
    if r < 0:
        raise ValueError(kind)
    return bool(r)


def zstd_inspect(bytes_block):
    """Host-side walk of one bytes block (vlscan_zstd_inspect) -> dict(consumed, regenerated, blocks, compressed_blocks, sequences)."""
    out = (C.c_uint64 * 5)()
    rc = lib().vlscan_zstd_inspect(bytes_block, C.c_size_t(len(bytes_block)), out)
    if rc:
        raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
    return dict(consumed=out[0], regenerated=out[1], blocks=out[2], compressed_blocks=out[3], sequences=out[4])


def zstd_walk_digest(host_blocks, threads):
    """Host-side header walk over every on-disk column of a HostBlocks / DownloadedBlocks (vlscan_zstd_walk_digest)
    -> dict(digest=(4 ints), frames, blocks, groups, compressed_blocks, sequences, walk_seconds, lists_seconds)."""
    out = (C.c_uint64 * 12)()
    rc = lib().vlscan_zstd_walk_digest(host_blocks.blocks, C.c_uint64(host_blocks.nblocks), C.c_int(threads), out)
    if rc:
        raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
    return dict(digest=tuple(out[:4]), frames=out[4], blocks=out[5], groups=out[6], compressed_blocks=out[7], sequences=out[8],
                walk_seconds=out[9] * 1e-9, lists_seconds=out[10] * 1e-9)


def parse_typed(value_type, text):
    """vlscan_parse_typed -> the value as an unsigned 64-bit pattern, or None when the text is not a value of that type"""
    text = _b(text)
    out = C.c_uint64()
    r = lib().vlscan_parse_typed(C.c_int(value_type), text, C.c_size_t(len(text)), C.byref(out))
    if r < 0:
        raise ValueError(value_type)
    return out.value if r else None


def format_float64(bits):
    """Text of a float64 column value (IEEE bits) as the scan kernels format it; marshalFloat64String, values_encoder.go:1397."""
    buf = C.create_string_buffer(352)
    n = lib().vlscan_format_float64(C.c_uint64(bits), buf, C.c_size_t(352))
    if n < 0:
        raise ValueError(bits)
    return buf.raw[:n]


def truncate_timestamp(ts, step, offset=0, calendar=BUCKET_PLAIN):
    """The `_time` bucket of one timestamp (vlscan_truncate_timestamp: host build of the hits kernels' truncateTimestamp)."""
    return lib().vlscan_truncate_timestamp(ts, step, offset, calendar)


def _by_bucket(spec):
    """None (the by-field's plain text) or (size, offset, calendar) -> vlscan_by_bucket"""
    if spec is None:
        return ByBucket(0.0, 0.0, 0, 0)
    size, offset, calendar = spec
    return ByBucket(size, offset, calendar, 1)


def bucket_text(text, size, offset=0.0, calendar=BUCKET_PLAIN):
    """The bucketed text of one const, string or dict text (vlscan_bucket_text: host build of the hits kernels' getBucketedValue); ValueError
    for a bucket vlscan_hits_stats rejects"""
    text = _b(text)
    out = C.create_string_buffer(352)
    L = lib()
    L.vlscan_bucket_text.argtypes = [C.POINTER(ByBucket), C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    n = L.vlscan_bucket_text(C.byref(_by_bucket((size, offset, calendar))), text, len(text), out, 352)
    if n < 0:
        raise ValueError((size, offset, calendar))
    return out.raw[:n]


def hits_query(step, offset=0, calendar=BUCKET_PLAIN, by=()):
    """-> (vlscan_hits_query, objects that must stay alive while it is used)"""
    names = [_b(f) for f in by]
    arr = (C.c_char_p * max(len(names), 1))(*names)
    lens = (C.c_size_t * max(len(names), 1))(*[len(x) for x in names])
    return HitsQuery(step, offset, calendar, len(names), arr, lens), (arr, lens)


def by_buckets(buckets, nby):
    """the by_buckets argument of vlscan_hits_stats_bucketed / vlscan_hits_sums_bucketed: None (NULL), or one (size, offset, calendar) or None per
    by-field (`stats by (f:size offset off)`; calendar = BUCKET_WEEK / _MONTH / _YEAR for `f:week` ..., BUCKET_PLAIN otherwise)"""
    if buckets is None:
        return None
    if len(buckets) != nby:
        raise ValueError("one bucket (or None) per by-field")
    return (ByBucket * max(nby, 1))(*[_by_bucket(b) for b in buckets])


def last_query(limit, fields=(), min_timestamp=None):
    """-> (vlscan_last_query, objects that must stay alive while it is used); min_timestamp None = no floor"""
    names = [_b(f) for f in fields]
    arr = (C.c_char_p * max(len(names), 1))(*names)
    lens = (C.c_size_t * max(len(names), 1))(*[len(x) for x in names])
    floor = I64_MIN if min_timestamp is None else min_timestamp
    return LastQuery(limit, floor, len(names), arr, lens), (arr, lens)


def facets_query(fields, max_values_per_field=0, max_value_len=0):
    """-> (vlscan_facets_query, objects that must stay alive while it is used); 0 = the endpoint's default (1000 values, 128 bytes)"""
    names = [_b(f) for f in fields]
    arr = (C.c_char_p * max(len(names), 1))(*names)
    lens = (C.c_size_t * max(len(names), 1))(*[len(x) for x in names])
    return FacetsQuery(max_values_per_field, max_value_len, len(names), arr, lens), (arr, lens)


def facets_merge(states, limit=10, keep_const_fields=False, max_values_per_field=0):
    """The merge a caller runs over the per-batch states of Ctx.facets (pipeFacetsProcessor.flush, lib/logstorage/pipe_facets.go:338-420, with
    concurrency 1) -> [(field name, value text, hits)] ordered by field name bytewise, then by hits descending.

    states: [(state, selected rows)], state = {field: None (dropped) or [(class, text, hits)]} as Ctx.facets returns it, called with
    max_values_per_field (0 = default).  A field is dropped when a batch dropped it or when its merged entries outnumber max_values_per_field; a field whose single entry covers every selected row is skipped unless keep_const_fields; ties of hits go by text, then
    class (FACET_UINT64 < FACET_NEGATIVE < FACET_STRING)."""
    rows = sum(n for _, n in states)
    max_values = max_values_per_field or FACETS_DEFAULT_MAX_VALUES
    merged, dropped = {}, set()
    for st, _ in states:
        for field, entries in st.items():
            if entries is None:
                dropped.add(field)
                continue
            m = merged.setdefault(field, {})
            for cls, text, hits in entries:
                m[(cls, text)] = m.get((cls, text), 0) + hits
    out = []
    for field in sorted(merged.keys() - dropped):
        m = merged[field]
        if len(m) > max_values:
            continue
        if len(m) == 1 and next(iter(m.values())) == rows and not keep_const_fields:
            continue
        ents = sorted(m.items(), key=lambda kv: (-kv[1], kv[0][1], kv[0][0]))[:limit]
        out.extend((field, text, hits) for (cls, text), hits in ents)
    return out


def stats_merge(states):
    """The merge a caller runs over the per-batch states of Ctx.hits_sums (pipeStatsGroup.mergeState with statsSumProcessor.mergeState and
    statsAvgProcessor.mergeState, lib/logstorage/stats_sum.go, stats_avg.go) -> {(bucket, key texts): (rows, [(sum, count) per value field])}.

    states: lists of (bucket, keys, rows, [(sum, count)...]) as Ctx.hits_sums returns them.  Rows and counts add; a sum adds to another unless
    one of them is NaN (a group without numbers in that batch), which takes the other.  sum(f) of a group is then its sum (NaN: no numbers),
    avg(f) is sum / count (NaN when count is 0)."""
    out = {}
    for st in states:
        for bucket, keys, rows, vals in st:
            k = (bucket, keys)
            if k not in out:
                out[k] = (rows, list(vals))
                continue
            r0, v0 = out[k]
            out[k] = (r0 + rows, [(b if math.isnan(a) else a if math.isnan(b) else a + b, ca + cb) for (a, ca), (b, cb) in zip(v0, vals)])
    return out


VMRANGES = 488   # VLSCAN_VMRANGES: vmrange indexes 0 (lower) .. 487 (upper), in numeric order


def vmrange_index(v):
    """The vmrange index of one number as Histogram.Update files it (vlscan_vmrange_index: host build of the kernel's mapping); -1 for NaN
    and negative numbers, which it skips"""
    return lib().vlscan_vmrange_index(float(v))


def vmrange_text(index):
    """The vmrange text of index 0 .. VMRANGES - 1 ("0...1.000e-09", "1.000e-09...1.136e-09", ..., "1.000e+18...+Inf")"""
    out = C.create_string_buffer(64)
    n = lib().vlscan_vmrange_text(index, out, 64)
    if n < 0:
        raise ValueError(index)
    return out.raw[:n].decode()


def vmranges_merge(states):
    """The merge a caller runs over the per-batch states of Ctx.hits_vmranges (pipeStatsGroup.mergeState with
    statsHistogramProcessor.mergeState, lib/logstorage/stats_histogram.go) -> {(bucket, key texts): (rows, [{index: hits} per value field])}.
    Rows add, and so do the hits of each (value field, index)."""
    out = {}
    for st in states:
        for bucket, keys, rows, vals in st:
            k = (bucket, keys)
            r0, v0 = out.get(k, (0, [{} for _ in vals]))
            for m, add in zip(v0, vals):
                for i, h in add.items():
                    m[i] = m.get(i, 0) + h
            out[k] = (r0 + rows, v0)
    return out


def parse_math_number(s):
    """host build of the device's parseMathNumber (vlscan_parse_math_number) -> float (NaN when the value is no number)"""
    L = lib()
    L.vlscan_parse_math_number.restype = C.c_double
    s = _b(s)
    return L.vlscan_parse_math_number(s, C.c_size_t(len(s)))


def device_count():
    return lib().vlscan_device_count()


def _b(s):
    return s.encode("utf-8", "surrogateescape") if isinstance(s, str) else bytes(s)


def _row_texts(raw, offs, nrows, nf):
    """rows x fields texts packed into one blob: field f of row i is raw[offs[i * nf + f]:offs[i * nf + f + 1]] -> [tuple of nf bytes] per row"""
    return [tuple(raw[int(offs[i * nf + f]):int(offs[i * nf + f + 1])] for f in range(nf)) for i in range(nrows)]


def _varuint(n):
    out = bytearray()
    while n >= 0x80:
        out.append((n & 0x7F) | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


def _bytes(s):
    s = _b(s)
    return _varuint(len(s)) + s


class Filter:
    """A node of the filter tree; `blob` is its serialisation for vlscan_program_create (include/vlscan.h)."""

    def __init__(self, blob, desc):
        self.blob = blob
        self.desc = desc

    def __repr__(self):
        return self.desc

    @staticmethod
    def noop():
        return Filter(bytes([F_NOOP]), "*")

    @staticmethod
    def phrase(field, phrase):
        return Filter(bytes([F_PHRASE]) + _bytes(field) + _bytes(phrase), "%r:%r" % (field, phrase))

    @staticmethod
    def prefix(field, prefix):
        return Filter(bytes([F_PREFIX]) + _bytes(field) + _bytes(prefix), "%r:%r*" % (field, prefix))

    @staticmethod
    def exact(field, value):
        return Filter(bytes([F_EXACT]) + _bytes(field) + _bytes(value), "%r:=%r" % (field, value))

    @staticmethod
    def in_(field, values):
        values = list(values)
        return Filter(bytes([F_IN]) + _bytes(field) + _varuint(len(values)) + b"".join(_bytes(v) for v in values), "%r:in(%r)" % (field, values))

    @staticmethod
    def regexp(field, expr):
        return Filter(bytes([F_REGEXP]) + _bytes(field) + _bytes(expr), "%r:~%r" % (field, expr))

    @staticmethod
    def exact_prefix(field, prefix):       # &filterExactPrefix{fieldName, prefix}
        return Filter(bytes([F_EXACT_PREFIX]) + _bytes(field) + _bytes(prefix), "%r:=%r*" % (field, prefix))

    @staticmethod
    def len_range(field, min_len, max_len):   # &filterLenRange{fieldName, minLen, maxLen}
        return Filter(bytes([F_LEN_RANGE]) + _bytes(field) + _varuint(min_len) + _varuint(max_len), "%r:len_range(%d, %d)" % (field, min_len, max_len))

    @staticmethod
    def string_range(field, min_value, max_value):   # &filterStringRange{fieldName, minValue, maxValue}
        return Filter(bytes([F_STRING_RANGE]) + _bytes(field) + _bytes(min_value) + _bytes(max_value), "%r:string_range(%r, %r)" % (field, min_value, max_value))

    @staticmethod
    def ipv4_range(field, min_value, max_value):     # &filterIPv4Range{fieldName, minValue, maxValue}
        return Filter(bytes([F_IPV4_RANGE]) + _bytes(field) + _varuint(min_value) + _varuint(max_value), "%r:ipv4_range(%#x, %#x)" % (field, min_value, max_value))

    @staticmethod
    def value_type(field, type_name):      # &filterValueType{fieldName, valueType}
        return Filter(bytes([F_VALUE_TYPE]) + _bytes(field) + _bytes(type_name), "%r:value_type(%r)" % (field, type_name))

    @staticmethod
    def any_case_phrase(field, phrase):    # &filterAnyCasePhrase{fieldName, phrase}        `f:i(phrase)`
        return Filter(bytes([F_ANY_CASE_PHRASE]) + _bytes(field) + _bytes(phrase), "%r:i(%r)" % (field, phrase))

    @staticmethod
    def any_case_prefix(field, prefix):    # &filterAnyCasePrefix{fieldName, prefix}        `f:i(prefix*)`
        return Filter(bytes([F_ANY_CASE_PREFIX]) + _bytes(field) + _bytes(prefix), "%r:i(%r*)" % (field, prefix))

    @staticmethod
    def sequence(field, phrases):          # &filterSequence{fieldName, phrases}            `f:seq(a, b, ...)`
        phrases = list(phrases)
        return Filter(bytes([F_SEQUENCE]) + _bytes(field) + _varuint(len(phrases)) + b"".join(_bytes(v) for v in phrases), "%r:seq(%r)" % (field, phrases))

    @staticmethod
    def contains_all(field, values):       # &filterContainsAll{fieldName, values}          `f:contains_all(a, b, ...)`
        values = list(values)
        return Filter(bytes([F_CONTAINS_ALL]) + _bytes(field) + _varuint(len(values)) + b"".join(_bytes(v) for v in values), "%r:contains_all(%r)" % (field, values))

    @staticmethod
    def contains_any(field, values):       # &filterContainsAny{fieldName, values}          `f:contains_any(a, b, ...)`
        values = list(values)
        return Filter(bytes([F_CONTAINS_ANY]) + _bytes(field) + _varuint(len(values)) + b"".join(_bytes(v) for v in values), "%r:contains_any(%r)" % (field, values))

    @staticmethod
    def range(field, min_value, max_value):   # &filterRange{fieldName, minValue, maxValue}   `f:range[a, b]`, `f:>a` ... (float64 bounds, inclusive)
        import struct
        return Filter(bytes([F_RANGE]) + _bytes(field) + struct.pack("<dd", float(min_value), float(max_value)), "%r:range[%r, %r]" % (field, min_value, max_value))

    @staticmethod
    def eq_field(field, other_field):         # &filterEqField{fieldName, otherFieldName}    `f:eq_field(g)`
        return Filter(bytes([F_EQ_FIELD]) + _bytes(field) + _bytes(other_field), "%r:eq_field(%r)" % (field, other_field))

    @staticmethod
    def le_field(field, other_field, exclude_equal=False):   # &filterLeField{...}            `f:le_field(g)` / `f:lt_field(g)`
        return Filter(bytes([F_LE_FIELD]) + _bytes(field) + _bytes(other_field) + bytes([1 if exclude_equal else 0]), "%r:%s_field(%r)" % (field, "lt" if exclude_equal else "le", other_field))

    @staticmethod
    def time(min_timestamp, max_timestamp):   # &filterTime{minTimestamp, maxTimestamp}      `_time:[a, b]` (nanoseconds, inclusive)
        return Filter(bytes([F_TIME]) + int(min_timestamp).to_bytes(8, "little", signed=True) + int(max_timestamp).to_bytes(8, "little", signed=True), "_time:[%d, %d]" % (min_timestamp, max_timestamp))

    @staticmethod
    def and_(filters):
        return Filter(bytes([F_AND]) + _varuint(len(filters)) + b"".join(f.blob for f in filters), "(" + " AND ".join(f.desc for f in filters) + ")")

    @staticmethod
    def or_(filters):
        return Filter(bytes([F_OR]) + _varuint(len(filters)) + b"".join(f.blob for f in filters), "(" + " OR ".join(f.desc for f in filters) + ")")

    @staticmethod
    def not_(f):
        return Filter(bytes([F_NOT]) + f.blob, "!" + f.desc)


class Program:
    """Compiled filter tree (searchOptions.filter)."""

    def __init__(self, flt):
        self.h = C.c_void_p()
        rc = lib().vlscan_program_create(flt.blob, C.c_size_t(len(flt.blob)), C.byref(self.h))
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        self.filter = flt

    def fields(self):
        out = []
        for i in range(lib().vlscan_program_nfields(self.h)):
            ln = C.c_size_t()
            p = lib().vlscan_program_field(self.h, C.c_uint32(i), C.byref(ln))
            out.append(C.string_at(p, ln.value))
        return out

    def leaf_tokens(self, leaf):
        buf = C.create_string_buffer(1 << 16)
        n = lib().vlscan_program_leaf_tokens(self.h, C.c_uint32(leaf), buf, C.c_size_t(1 << 16))
        if n < 0:
            raise IndexError(leaf)
        return buf.raw[:n].split(b"\n") if n else []

    def __del__(self):
        try:
            if self.h:
                lib().vlscan_program_free(self.h)
        except Exception:
            pass


class HostBlocks:
    """A set of vlscan_block descriptors over host memory (what the Go shim would assemble per blockSearchWorkBatch)."""

    def __init__(self, field_names, blocks):
        """blocks: list of dict(rows=int, columns=[dict(field=name, kind='const'|'values', ...)])

        values columns: value_type, min_value, max_value, dict (list of bytes), bloom (bytes) and either
        values_block (bytes, on-disk stage) or lens_items + data (decoded stage).
        A block may carry its timestamps column: timestamps=(encoded bytes, marshalType, minTimestamp, maxTimestamp)."""
        self.field_names = [_b(f) for f in field_names]
        fidx = {f: i for i, f in enumerate(self.field_names)}
        self._keep = []
        ncols = sum(len(b["columns"]) for b in blocks)
        self.cols = (CColumn * max(ncols, 1))()
        self.blocks = (CBlock * max(len(blocks), 1))()
        self.nblocks = len(blocks)
        k = 0

        seen = {}

        def buf(data):
            data = bytes(data)
            hit = seen.get(id(data))       # the same bytes object described twice (repeated blocks) is staged once
            if hit is not None:
                return hit
            a = C.create_string_buffer(data, len(data)) if data else C.create_string_buffer(1)
            self._keep.append((a, data))
            seen[id(data)] = (C.cast(a, C.c_void_p), len(data))
            return seen[id(data)]

        for bi, blk in enumerate(blocks):
            first = k
            for col in blk["columns"]:
                c = self.cols[k]
                c.field = fidx[_b(col["field"])]
                if col["kind"] == "const":
                    c.kind = COL_CONST
                    c.const_value, c.const_len = buf(col["value"])
                else:
                    c.kind = COL_VALUES
                    c.value_type = col["value_type"]
                    c.min_value, c.max_value = col.get("min_value", 0), col.get("max_value", 0)
                    d = col.get("dict") or []
                    c.dict_len = len(d)
                    if d:
                        offs = np.zeros(len(d) + 1, dtype=np.uint32)
                        offs[1:] = np.cumsum([len(x) for x in d])
                        self._keep.append(offs)
                        c.dict_offsets = offs.ctypes.data
                        c.dict_blob, _ = buf(b"".join(d))
                    if "values_block" in col:
                        c.stage = STAGE_ONDISK
                        c.values, c.values_len = buf(col["values_block"])
                    else:
                        c.stage = STAGE_DECODED
                        c.lens_items, c.lens_items_len = buf(col["lens_items"])
                        c.data, c.data_len = buf(col["data"])
                    c.bloom, c.bloom_len = buf(col.get("bloom", b""))
                k += 1
            self.blocks[bi].rows = blk["rows"]
            if blk.get("timestamps") is not None:
                data, mt, mn, mx = blk["timestamps"]
                self.blocks[bi].timestamps, self.blocks[bi].timestamps_len = buf(data)
                self.blocks[bi].ts_marshal_type, self.blocks[bi].min_timestamp, self.blocks[bi].max_timestamp = mt, mn, mx
            self.blocks[bi].ncols = k - first
            self.blocks[bi].cols = C.cast(C.byref(self.cols, first * C.sizeof(CColumn)), C.POINTER(CColumn))
        self.rows = [b["rows"] for b in blocks]

    def name_arrays(self):
        names = (C.c_char_p * max(len(self.field_names), 1))(*self.field_names)
        lens = (C.c_size_t * max(len(self.field_names), 1))(*[len(f) for f in self.field_names])
        return names, lens


class DownloadedBlocks:
    """Host copy (pinned memory owned by the library) of a device-resident batch: vlscan_batch_download."""

    def __init__(self, ctx, batch, _handle=None):
        self.h = C.c_void_p()
        if _handle is not None:
            self.h = _handle
        else:
            ctx._check(lib().vlscan_batch_download(ctx.h, batch.h, C.byref(self.h)))
        nb, nf = C.c_uint64(), C.c_uint32()
        self.blocks = lib().vlscan_host_blocks_get(self.h, C.byref(nb), C.byref(nf))
        self.nblocks = nb.value
        self.field_names = []
        for i in range(nf.value):
            ln = C.c_size_t()
            p = lib().vlscan_host_blocks_field(self.h, C.c_uint32(i), C.byref(ln))
            self.field_names.append(C.string_at(p, ln.value))
        self.bytes = lib().vlscan_host_blocks_bytes(self.h)
        self.rows = [self.blocks[i].rows for i in range(self.nblocks)]

    def name_arrays(self):
        names = (C.c_char_p * max(len(self.field_names), 1))(*self.field_names)
        lens = (C.c_size_t * max(len(self.field_names), 1))(*[len(f) for f in self.field_names])
        return names, lens

    def column(self, block, field):
        """-> dict view of one column (bytes copied out) for tests"""
        blk = self.blocks[block]
        fi = self.field_names.index(_b(field))
        for k in range(blk.ncols):
            c = blk.cols[k]
            if c.field != fi:
                continue
            if c.kind == COL_CONST:
                return dict(kind="const", value=C.string_at(c.const_value, c.const_len))
            d = []
            if c.dict_len:
                offs = np.ctypeslib.as_array(C.cast(c.dict_offsets, C.POINTER(C.c_uint32)), (c.dict_len + 1,))
                blob = C.string_at(c.dict_blob, int(offs[-1]))
                d = [blob[int(offs[i]):int(offs[i + 1])] for i in range(c.dict_len)]
            out = dict(kind="values", value_type=c.value_type, min_value=c.min_value, max_value=c.max_value, dict=d, bloom=C.string_at(c.bloom, c.bloom_len))
            if c.stage == STAGE_ONDISK:
                out["values_block"] = C.string_at(c.values, c.values_len)
            else:
                out["lens_items"], out["data"] = C.string_at(c.lens_items, c.lens_items_len), C.string_at(c.data, c.data_len)
            return out
        return None

    def compress(self, threads=0):
        """Writer-side re-encoding into the on-disk stage (marshalBytesBlock, encoding.go:343-370): vlscan_host_blocks_compress."""
        h = C.c_void_p()
        rc = lib().vlscan_host_blocks_compress(self.h, C.c_int(threads), C.byref(h))
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        return DownloadedBlocks(None, None, _handle=h)

    def __del__(self):
        try:
            if self.h:
                lib().vlscan_host_blocks_free(self.h)
        except Exception:
            pass


INFLATE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t)
BLOCK_HEADER_FIELDS = ("account_id", "project_id", "id_hi", "id_lo", "uncompressed_size_bytes", "rows_count", "ts_block_offset", "ts_block_size",
                       "min_timestamp", "max_timestamp", "ts_marshal_type", "columns_header_index_offset", "columns_header_index_size",
                       "columns_header_offset", "columns_header_size")
PART_HEADER_FIELDS = ("FormatVersion", "CompressedSizeBytes", "UncompressedSizeBytes", "RowsCount", "BlocksCount", "MinTimestamp", "MaxTimestamp",
                      "BloomValuesShardsCount")


def _signed(v):
    return v - (1 << 64) if v >= 1 << 63 else v


class Part:
    """One part directory opened through vlscan_part_open (part.mustOpenFilePart, lib/logstorage/part.go:105-173).

    ctx: the device decoder inflates the part's metadata; inflate: a Python callable (frame bytes, regenerated size) -> bytes used instead
    (an embedding process with its own ZSTD)."""

    def __init__(self, path, ctx=None, inflate=None):
        L = lib()
        L.vlscan_part_nblocks.restype = C.c_uint64
        L.vlscan_part_nblocks.argtypes = [C.c_void_p]
        L.vlscan_part_ncolumn_names.restype = C.c_uint32
        L.vlscan_part_ncolumn_names.argtypes = [C.c_void_p]
        L.vlscan_part_column_name.restype = C.c_void_p
        L.vlscan_part_free.argtypes = [C.c_void_p]
        L.vlscan_part_free.restype = None
        L.vlscan_host_blocks_source.restype = C.POINTER(C.c_uint64)
        self._cb = None
        if inflate is not None:
            def cb(user, frame, n, dst, dn):
                try:
                    out = inflate(C.string_at(frame, n), dn)
                    if len(out) != dn:
                        return 1
                    C.memmove(dst, out, dn)
                    return 0
                except Exception:
                    return 2
            self._cb = INFLATE_FN(cb)
        self.h = C.c_void_p()
        rc = L.vlscan_part_open(ctx.h if ctx is not None else None, _b(path), self._cb if self._cb is not None else C.cast(None, INFLATE_FN), None, C.byref(self.h))
        if rc:
            raise VlscanError(rc, L.vlscan_last_error(ctx.h if ctx is not None else None).decode("utf-8", "replace"))
        out = (C.c_uint64 * 8)()
        L.vlscan_part_header(self.h, out)
        self.header = {k: (_signed(out[i]) if k in ("MinTimestamp", "MaxTimestamp") else out[i]) for i, k in enumerate(PART_HEADER_FIELDS)}
        self.nblocks = L.vlscan_part_nblocks(self.h)
        self.column_names = []
        for i in range(L.vlscan_part_ncolumn_names(self.h)):
            ln = C.c_size_t()
            p = L.vlscan_part_column_name(self.h, C.c_uint32(i), C.byref(ln))
            self.column_names.append(C.string_at(p, ln.value))

    def block_header(self, i):
        out = (C.c_uint64 * 15)()
        rc = lib().vlscan_part_block_header(self.h, C.c_uint64(i), out)
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        return {k: (_signed(out[j]) if k in ("min_timestamp", "max_timestamp") else out[j]) for j, k in enumerate(BLOCK_HEADER_FIELDS)}

    def timestamps(self, i):
        """-> the encoded timestamps block of block i (bytes of timestamps.bin); marshal type, first value and row count are in block_header(i)"""
        p, n = C.c_void_p(), C.c_uint64()
        rc = lib().vlscan_part_timestamps(self.h, C.c_uint64(i), C.byref(p), C.byref(n))
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        return C.string_at(p, n.value) if n.value else b""

    def blocks(self, fields, lo=0, hi=None, min_timestamp=-(1 << 63), max_timestamp=(1 << 63) - 1):
        """-> DownloadedBlocks-like descriptors (on-disk stage) of the blocks [lo, hi) overlapping the time range; .source = their indices in the part"""
        fields = [_b(f) for f in fields]
        names = (C.c_char_p * max(len(fields), 1))(*fields)
        lens = (C.c_size_t * max(len(fields), 1))(*[len(f) for f in fields])
        h = C.c_void_p()
        rc = lib().vlscan_part_blocks(self.h, names, lens, C.c_uint32(len(fields)), C.c_uint64(lo), C.c_uint64(self.nblocks if hi is None else hi),
                                      C.c_int64(min_timestamp), C.c_int64(max_timestamp), C.byref(h))
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        hb = DownloadedBlocks(None, None, _handle=h)
        n = C.c_uint64()
        p = lib().vlscan_host_blocks_source(h, C.byref(n))
        hb.source = [p[i] for i in range(n.value)]
        hb._part = self           # the descriptors point into the part's mapped files
        return hb

    def close(self):
        if self.h:
            lib().vlscan_part_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def search_part(ctx, part, flt, min_timestamp=-(1 << 63), max_timestamp=(1 << 63) - 1, batch_blocks=8192):
    """The block loop of Storage.search for one part (storage_search.go:1022-1063 below the partition level): blocks are pruned by their
    time range, the filter tree runs on the rest in batches of `batch_blocks` through vlscan_scan_batch.

    -> list of (block index in the part, bitmap words, match count, inside) for blocks with matches.  `inside` is False for a block that
    only partly overlaps [min_timestamp, max_timestamp]: its rows still need the per-row `_time` check (filterTime, filter_time.go:114-137),
    which this engine does not run yet (SURVEY §8(f) rank 4)."""
    prog = Program(flt)
    fields = prog.fields()
    hits = []
    for lo in range(0, part.nblocks, batch_blocks):
        hb = part.blocks(fields, lo, min(part.nblocks, lo + batch_blocks), min_timestamp, max_timestamp)
        if hb.nblocks == 0:
            continue
        words, counts, _ = ctx.scan_batch(prog, hb)
        for src, w, c in zip(hb.source, split_bitmaps(words, hb.rows), counts):
            if c:
                bh = part.block_header(src)
                hits.append((src, w.copy(), int(c), min_timestamp <= bh["min_timestamp"] and bh["max_timestamp"] <= max_timestamp))
    return hits


def totals_sum(ctxs):
    """{rows, rows_matched, blocks_matched, values_bytes} of the last scans of several contexts (one per GPU), summed: vlscan_totals_sum"""
    arr = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    out = (C.c_uint64 * 4)()
    rc = lib().vlscan_totals_sum(arr, C.c_int(len(ctxs)), out)
    if rc:
        raise VlscanError(rc, lib().vlscan_last_error(None).decode("utf-8", "replace"))
    return [int(x) for x in out]


class Batch:
    def __init__(self, h, ctx):
        self.h = h
        self.ctx = ctx
        L = lib()
        self.nblocks = L.vlscan_batch_nblocks(h)
        self.rows = L.vlscan_batch_rows(h)
        self.words = L.vlscan_batch_words(h)
        self.device_bytes = L.vlscan_batch_device_bytes(h)

    def free(self):
        if self.h:
            lib().vlscan_batch_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class KeptBatch:
    """Sizes of the batch a scan_batch_keep left on the device (the library owns it; nothing to free)."""

    def __init__(self, nblocks, rows, words):
        self.nblocks, self.rows, self.words = nblocks, rows, words


class Ctx:
    """Per search-worker context (device + stream); mirrors the per-goroutine blockSearch of storage_search.go:1041-1043."""

    def __init__(self, device=0):
        h = lib().vlscan_ctx_create(C.c_int(device))
        if not h:
            raise VlscanError(100, lib().vlscan_last_error(None).decode("utf-8", "replace"))
        self.h = C.c_void_p(h)

    def _check(self, rc):
        if rc:
            raise VlscanError(rc, lib().vlscan_last_error(self.h).decode("utf-8", "replace"))

    def _call_grown(self, call, caps, needed):
        """call(*caps) -> (rc, outputs).  A call that fails while needed() reports sizes above its caps runs once more with the caps grown
        to them.  -> the outputs of the last call; raises its error."""
        rc, out = call(*caps)
        want = [int(w) for w in needed()]
        if rc and any(w > c for w, c in zip(want, caps)):
            rc, out = call(*[max(c, w) for c, w in zip(caps, want)])
        self._check(rc)
        return out

    @property
    def stream(self):
        return lib().vlscan_ctx_stream(self.h)

    def sync(self):
        self._check(lib().vlscan_ctx_sync(self.h))

    def zstd_decompress(self, frames, sizes):
        """Decode independent ZSTD frames (bytes) on the device -> list of bytes; sizes = regenerated size of each frame."""
        n = len(frames)
        keep = [C.create_string_buffer(f, len(f)) if f else C.create_string_buffer(1) for f in frames]
        ptrs = (C.c_void_p * max(n, 1))(*[C.cast(k, C.c_void_p) for k in keep])
        lens = (C.c_size_t * max(n, 1))(*[len(f) for f in frames])
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum(np.asarray(sizes, dtype=np.uint64)) if n else 0
        total = int(offs[-1])
        dst = C.create_string_buffer(max(total, 1))
        self._check(lib().vlscan_zstd_decompress(self.h, C.c_uint32(n), ptrs, lens, dst, offs.ctypes.data_as(C.c_void_p)))
        raw = dst.raw
        return [raw[int(offs[i]):int(offs[i + 1])] for i in range(n)]

    def upload(self, host_blocks, stats=None):
        names, lens = host_blocks.name_arrays()
        out = C.c_void_p()
        self._check(lib().vlscan_batch_upload(self.h, names, lens, C.c_uint32(len(host_blocks.field_names)), host_blocks.blocks,
                                              C.c_uint64(host_blocks.nblocks), C.byref(out), C.byref(stats) if stats is not None else None))
        return Batch(out, self)

    def generate(self, cfg, block_lo, block_hi):
        out = C.c_void_p()
        self._check(lib().vlscan_batch_generate(self.h, C.byref(cfg), C.c_uint64(block_lo), C.c_uint64(block_hi), C.byref(out)))
        return Batch(out, self)

    def download(self, batch):
        return DownloadedBlocks(self, batch)

    def scan_resident(self, program, batch, want_stats=True):
        st = CStats() if want_stats else None
        self._check(lib().vlscan_scan_resident(self.h, program.h, batch.h, C.byref(st) if st is not None else None))
        self._last = batch
        return st

    def last_scan_stats(self):
        st = CStats()
        self._check(lib().vlscan_last_scan_stats(self.h, C.byref(st)))
        return st

    def fetch(self, batch=None, bitmaps=True, counts=True, stats=None):
        batch = batch or self._last
        words = np.zeros(max(batch.words, 1), dtype=np.uint64) if bitmaps else None
        cnt = np.zeros(max(batch.nblocks, 1), dtype=np.uint32) if counts else None
        self._check(lib().vlscan_fetch_results(self.h, words.ctypes.data_as(C.c_void_p) if bitmaps else None,
                                               cnt.ctypes.data_as(C.c_void_p) if counts else None, C.byref(stats) if stats is not None else None))
        return (words[:batch.words] if bitmaps else None), (cnt[:batch.nblocks] if counts else None)

    def fetch_hits(self, batch=None, cap=None):
        batch = batch or self._last
        cap = cap if cap is not None else max(int(batch.rows), 1)
        hits = np.zeros(cap, dtype=np.uint32)
        offs = np.zeros(batch.nblocks + 1, dtype=np.uint64)
        self._check(lib().vlscan_fetch_hits(self.h, hits.ctypes.data_as(C.c_void_p), C.c_uint64(cap), offs.ctypes.data_as(C.c_void_p)))
        return hits[:int(offs[-1])], offs

    def gather_timestamps(self, batch=None):
        """`_time` of the selected rows of the last scan, block after block (vlscan_gather_timestamps) -> (int64 array, hit offsets per block)"""
        batch = batch or self._last
        cap = max(int(batch.rows), 1)
        ts = np.zeros(cap, dtype=np.int64)
        offs = np.zeros(batch.nblocks + 1, dtype=np.uint64)
        self._check(lib().vlscan_gather_timestamps(self.h, ts.ctypes.data_as(C.c_void_p), C.c_uint64(cap), offs.ctypes.data_as(C.c_void_p)))
        return ts[:int(offs[-1])], offs

    def gather_values(self, field, batch=None):
        """the value of `field` in every selected row of the last scan as bytes (vlscan_gather_values) -> (list of bytes, hit offsets per block)"""
        batch = batch or self._last
        field = _b(field)
        hoffs = np.zeros(batch.nblocks + 1, dtype=np.uint64)
        nrows = max(int(batch.rows), 1)
        voffs = np.zeros(nrows + 1, dtype=np.uint64)
        total = C.c_uint64()

        def call(cap):
            out = np.zeros(cap, dtype=np.uint8)
            return lib().vlscan_gather_values(self.h, field, C.c_size_t(len(field)), out.ctypes.data_as(C.c_void_p), C.c_uint64(cap), voffs.ctypes.data_as(C.c_void_p),
                                              C.c_uint64(nrows), C.byref(total), hoffs.ctypes.data_as(C.c_void_p)), out
        out = self._call_grown(call, (1 << 16,), lambda: (total.value,))
        n = int(hoffs[-1])
        raw = out.tobytes()
        return [raw[int(voffs[i]):int(voffs[i + 1])] for i in range(n)], hoffs

    def hits_stats(self, step, offset=0, calendar=BUCKET_PLAIN, by=(), batch=None, info=None, buckets=None):
        """`stats by (_time:step offset off, by...) count()` over the selected rows of the last scan (vlscan_hits_stats)
        -> [(bucket, (key texts as bytes...), count)] sorted by bucket, then by the texts.  `info` (a dict) receives groups, key_bytes,
        rows (selected) and blocks_decoded (blocks whose timestamps had to be decoded).  buckets: as for by_buckets (not None: through
        vlscan_hits_stats_bucketed)."""
        batch = batch or getattr(self, "_last", None)
        q, keep = hits_query(step, offset, calendar, by)
        bks = by_buckets(buckets, len(by))
        nby = len(by)
        out_info = (C.c_uint64 * 4)()

        def call(cap_groups, cap_bytes):
            buckets = np.zeros(cap_groups, dtype=np.int64)
            counts = np.zeros(cap_groups, dtype=np.uint64)
            offs = np.zeros(cap_groups * nby + 1, dtype=np.uint64)
            kb = np.zeros(max(cap_bytes, 1), dtype=np.uint8)
            outs = (buckets.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), C.c_uint64(cap_groups), kb.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes),
                    offs.ctypes.data_as(C.c_void_p), out_info)
            if bks is None:
                rc = lib().vlscan_hits_stats(self.h, C.byref(q), *outs)
            else:
                rc = lib().vlscan_hits_stats_bucketed(self.h, C.byref(q), bks, *outs)
            return rc, (buckets, counts, offs, kb)
        buckets, counts, offs, kb = self._call_grown(call, (max(1, min(int(batch.rows) if batch else 0, 1 << 16)), 1 << 16), lambda: out_info[:2])
        if info is not None:
            info.update(groups=out_info[0], key_bytes=out_info[1], rows=out_info[2], blocks_decoded=out_info[3])
        keys = _row_texts(kb.tobytes(), offs, int(out_info[0]), nby)
        return [(int(buckets[g]), keys[g], int(counts[g])) for g in range(int(out_info[0]))]

    def hits_sums(self, step, offset=0, calendar=BUCKET_PLAIN, by=(), values=(), batch=None, info=None, buckets=None):
        """`stats by (_time:step offset off, by...) count(), sum(v), avg(v)...` over the selected rows of the last scan (vlscan_hits_sums)
        -> [(bucket, (key texts as bytes...), rows, [(sum, count) per value field])] in the order of hits_stats.  A sum is NaN when its count
        is 0.  `info` and buckets as for hits_stats."""
        batch = batch or getattr(self, "_last", None)
        q, keep = hits_query(step, offset, calendar, by)
        bks = by_buckets(buckets, len(by))
        vn = [_b(f) for f in values]
        varr = (C.c_char_p * max(len(vn), 1))(*vn)
        vlens = (C.c_size_t * max(len(vn), 1))(*[len(x) for x in vn])
        nby, nv = len(by), len(vn)
        out_info = (C.c_uint64 * 4)()

        def call(cap_groups, cap_bytes):
            buckets = np.zeros(cap_groups, dtype=np.int64)
            counts = np.zeros(cap_groups, dtype=np.uint64)
            sums = np.zeros(max(cap_groups * nv, 1), dtype=np.float64)
            vcounts = np.zeros(max(cap_groups * nv, 1), dtype=np.uint64)
            offs = np.zeros(cap_groups * nby + 1, dtype=np.uint64)
            kb = np.zeros(max(cap_bytes, 1), dtype=np.uint8)
            args = (varr, vlens, C.c_uint32(nv), buckets.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), sums.ctypes.data_as(C.c_void_p),
                    vcounts.ctypes.data_as(C.c_void_p), C.c_uint64(cap_groups), kb.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), offs.ctypes.data_as(C.c_void_p), out_info)
            if bks is None:
                rc = lib().vlscan_hits_sums(self.h, C.byref(q), *args)
            else:
                rc = lib().vlscan_hits_sums_bucketed(self.h, C.byref(q), bks, *args)
            return rc, (buckets, counts, sums, vcounts, offs, kb)
        buckets, counts, sums, vcounts, offs, kb = self._call_grown(call, (max(1, min(int(batch.rows) if batch else 0, 1 << 16)), 1 << 16), lambda: out_info[:2])
        if info is not None:
            info.update(groups=out_info[0], key_bytes=out_info[1], rows=out_info[2], blocks_decoded=out_info[3])
        G = int(out_info[0])
        keys = _row_texts(kb.tobytes(), offs, G, nby)
        return [(int(buckets[g]), keys[g], int(counts[g]), [(float(sums[g * nv + f]), int(vcounts[g * nv + f])) for f in range(nv)]) for g in range(G)]

    def hits_vmranges(self, step, offset=0, calendar=BUCKET_PLAIN, by=(), values=(), batch=None, info=None, buckets=None):
        """`stats by (_time:step offset off, by...) histogram(v)...` over the selected rows of the last scan (vlscan_hits_vmranges)
        -> [(bucket, (key texts as bytes...), rows, [{vmrange index: hits} per value field])] in the order of hits_stats; vmrange_text names
        an index.  `info` (a dict) receives what hits_stats gives, plus entries and header_cells (cells counted from their header alone);
        buckets as for hits_stats."""
        batch = batch or getattr(self, "_last", None)
        q, keep = hits_query(step, offset, calendar, by)
        bks = by_buckets(buckets, len(by))
        vn = [_b(f) for f in values]
        varr = (C.c_char_p * max(len(vn), 1))(*vn)
        vlens = (C.c_size_t * max(len(vn), 1))(*[len(x) for x in vn])
        nby, nv = len(by), len(vn)
        out_info = (C.c_uint64 * 6)()

        def call(cap_groups, cap_bytes, cap_entries):
            buckets = np.zeros(cap_groups, dtype=np.int64)
            counts = np.zeros(cap_groups, dtype=np.uint64)
            offs = np.zeros(cap_groups * nby + 1, dtype=np.uint64)
            kb = np.zeros(max(cap_bytes, 1), dtype=np.uint8)
            eoffs = np.zeros(cap_groups * nv + 1, dtype=np.uint64)
            ranges = np.zeros(max(cap_entries, 1), dtype=np.uint16)
            hits = np.zeros(max(cap_entries, 1), dtype=np.uint64)
            rc = lib().vlscan_hits_vmranges(self.h, C.byref(q), bks, varr, vlens, C.c_uint32(nv), buckets.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
                                            C.c_uint64(cap_groups), kb.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), offs.ctypes.data_as(C.c_void_p),
                                            eoffs.ctypes.data_as(C.c_void_p), ranges.ctypes.data_as(C.c_void_p), hits.ctypes.data_as(C.c_void_p), C.c_uint64(cap_entries), out_info)
            return rc, (buckets, counts, offs, kb, eoffs, ranges, hits)
        cap = max(1, min(int(batch.rows) if batch else 0, 1 << 16))
        buckets, counts, offs, kb, eoffs, ranges, hits = self._call_grown(call, (cap, 1 << 16, cap * max(nv, 1)), lambda: (out_info[0], out_info[1], out_info[4]))
        if info is not None:
            info.update(groups=out_info[0], key_bytes=out_info[1], rows=out_info[2], blocks_decoded=out_info[3], entries=out_info[4], header_cells=out_info[5])
        G = int(out_info[0])
        keys = _row_texts(kb.tobytes(), offs, G, nby)
        out = []
        for g in range(G):
            vals = []
            for f in range(nv):
                a, z = int(eoffs[g * nv + f]), int(eoffs[g * nv + f + 1])
                vals.append({int(ranges[e]): int(hits[e]) for e in range(a, z)})
            out.append((int(buckets[g]), keys[g], int(counts[g]), vals))
        return out

    def last_rows(self, limit, fields=(), min_timestamp=None, info=None):
        """The `limit` newest selected rows of the last scan with _time >= min_timestamp (vlscan_last_rows)
        -> [(timestamp, block, row, (field texts as bytes...))] ascending by (timestamp, block, row).  `info` (a dict) receives rows,
        value_bytes, selected (rows of the scan) and blocks_decoded (blocks whose timestamps had to be decoded)."""
        q, keep = last_query(limit, fields, min_timestamp)
        nf = len(fields)
        out_info = (C.c_uint64 * 4)()

        def call(cap_rows, cap_bytes):
            ts = np.zeros(cap_rows, dtype=np.int64)
            blocks = np.zeros(cap_rows, dtype=np.uint32)
            rows = np.zeros(cap_rows, dtype=np.uint32)
            offs = np.zeros(cap_rows * nf + 1, dtype=np.uint64)
            vb = np.zeros(max(cap_bytes, 1), dtype=np.uint8)
            rc = lib().vlscan_last_rows(self.h, C.byref(q), ts.ctypes.data_as(C.c_void_p), blocks.ctypes.data_as(C.c_void_p), rows.ctypes.data_as(C.c_void_p),
                                        C.c_uint64(cap_rows), vb.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes), offs.ctypes.data_as(C.c_void_p), out_info)
            return rc, (ts, blocks, rows, offs, vb)
        ts, blocks, rows, offs, vb = self._call_grown(call, (max(1, min(int(limit), 1 << 12)), 1 << 16), lambda: out_info[:2])
        if info is not None:
            info.update(rows=out_info[0], value_bytes=out_info[1], selected=out_info[2], blocks_decoded=out_info[3])
        texts = _row_texts(vb.tobytes(), offs, int(out_info[0]), nf)
        return [(int(ts[i]), int(blocks[i]), int(rows[i]), texts[i]) for i in range(int(out_info[0]))]

    def facets(self, fields, max_values_per_field=0, max_value_len=0, info=None):
        """The facets state of the selected rows of the last scan (vlscan_facets) -> {field: None when dropped, else [(class, text as bytes,
        hits)] by hits descending, then text, then class}; field keys are the names as given.
        `info` (a dict) receives entries, value_bytes, rows (selected) and blocks_decoded (blocks whose timestamps had to be decoded)."""
        q, keep = facets_query(fields, max_values_per_field, max_value_len)
        nf = len(fields)
        out_info = (C.c_uint64 * 4)()

        def call(cap_entries, cap_bytes):
            dropped = np.zeros(max(nf, 1), dtype=np.uint8)
            foffs = np.zeros(nf + 1, dtype=np.uint64)
            hits = np.zeros(cap_entries, dtype=np.uint64)
            cls = np.zeros(cap_entries, dtype=np.uint8)
            voffs = np.zeros(cap_entries + 1, dtype=np.uint64)
            vb = np.zeros(max(cap_bytes, 1), dtype=np.uint8)
            rc = lib().vlscan_facets(self.h, C.byref(q), dropped.ctypes.data_as(C.c_void_p), foffs.ctypes.data_as(C.c_void_p), hits.ctypes.data_as(C.c_void_p),
                                     cls.ctypes.data_as(C.c_void_p), C.c_uint64(cap_entries), vb.ctypes.data_as(C.c_void_p), C.c_uint64(cap_bytes),
                                     voffs.ctypes.data_as(C.c_void_p), out_info)
            return rc, (dropped, foffs, hits, cls, voffs, vb)
        dropped, foffs, hits, cls, voffs, vb = self._call_grown(call, (1 << 12, 1 << 16), lambda: out_info[:2])
        if info is not None:
            info.update(entries=out_info[0], value_bytes=out_info[1], rows=out_info[2], blocks_decoded=out_info[3])
        raw = vb.tobytes()
        state = {}
        for f, name in enumerate(fields):
            state[name] = None if dropped[f] else [(int(cls[e]), raw[int(voffs[e]):int(voffs[e + 1])], int(hits[e])) for e in range(int(foffs[f]), int(foffs[f + 1]))]
        return state

    def result_digest(self, block_lo, block_hi, key_base=0):
        """xor over blocks of XXH64(bitmap words) * (2 * (key_base + block) + 1) of the last scan, computed on the device (vlscan_result_digest)"""
        d = C.c_uint64()
        self._check(lib().vlscan_result_digest(self.h, C.c_uint64(block_lo), C.c_uint64(block_hi), C.c_uint64(key_base), C.byref(d)))
        return d.value

    def result_device_ptrs(self):
        a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._check(lib().vlscan_result_device_ptrs(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def scan_batch(self, program, host_blocks, out_words=None, out_counts=None):
        """End-to-end call on host buffers: upload + scan + fetch (vlscan_scan_batch). -> (words, counts, stats)"""
        names, lens = host_blocks.name_arrays()
        nwords = sum((r + 63) // 64 for r in host_blocks.rows)
        words = out_words if out_words is not None else np.zeros(max(nwords, 1), dtype=np.uint64)
        cnt = out_counts if out_counts is not None else np.zeros(max(host_blocks.nblocks, 1), dtype=np.uint32)
        st = CStats()
        self._check(lib().vlscan_scan_batch(self.h, program.h, names, lens, C.c_uint32(len(host_blocks.field_names)), host_blocks.blocks,
                                            C.c_uint64(host_blocks.nblocks), words.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), C.byref(st)))
        return words[:nwords], cnt[:host_blocks.nblocks], st

    def scan_batch_keep(self, program, host_blocks, out_words=None, out_counts=None):
        """vlscan_scan_batch whose batch stays on the device as the ctx's last result (vlscan_scan_batch_keep): the gather and aggregation
        calls then work on it, output fields of `host_blocks` the program does not reference are staged by stage_selected.
        -> (words, counts, stats).  `host_blocks` must stay alive and unchanged for stage_selected."""
        names, lens = host_blocks.name_arrays()
        nwords = sum((r + 63) // 64 for r in host_blocks.rows)
        words = out_words if out_words is not None else np.zeros(max(nwords, 1), dtype=np.uint64)
        cnt = out_counts if out_counts is not None else np.zeros(max(host_blocks.nblocks, 1), dtype=np.uint32)
        st = CStats()
        self._last = None
        self._check(lib().vlscan_scan_batch_keep(self.h, program.h, names, lens, C.c_uint32(len(host_blocks.field_names)), host_blocks.blocks,
                                                 C.c_uint64(host_blocks.nblocks), words.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), C.byref(st)))
        self._last = KeptBatch(host_blocks.nblocks, sum(host_blocks.rows), nwords)
        return words[:nwords], cnt[:host_blocks.nblocks], st

    def stage_selected(self, host_blocks, fields, blocks=None):
        """Stage the values of `fields` of the kept batch for the blocks with selected rows, or for the block indexes in `blocks`
        (vlscan_stage_selected).  host_blocks: the descriptors scan_batch_keep was given.
        -> dict(staged, already_staged, h2d_bytes, frames)"""
        names = [_b(f) for f in fields]
        arr = (C.c_char_p * max(len(names), 1))(*names)
        lens = (C.c_size_t * max(len(names), 1))(*[len(x) for x in names])
        lst = None if blocks is None else np.ascontiguousarray(np.asarray(list(blocks), dtype=np.uint32))
        out = (C.c_uint64 * 4)()
        self._check(lib().vlscan_stage_selected(self.h, host_blocks.blocks, C.c_uint64(host_blocks.nblocks), arr, lens, C.c_uint32(len(names)),
                                                lst.ctypes.data_as(C.c_void_p) if lst is not None else None, C.c_uint64(0 if lst is None else len(lst)), out))
        return dict(staged=out[0], already_staged=out[1], h2d_bytes=out[2], frames=out[3])

    def close(self):
        if self.h:
            lib().vlscan_ctx_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def split_bitmaps(words, rows_per_block):
    """packed words -> list of per-block word arrays"""
    out, off = [], 0
    for r in rows_per_block:
        n = (r + 63) // 64
        out.append(words[off:off + n])
        off += n
    return out
