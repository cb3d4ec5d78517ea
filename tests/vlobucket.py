"""ctypes binding of the C++ restatement of bucketed by-fields, `stats by (_time:step, f:size offset off, ...) count(), sum(v), avg(v)`
(tests/bucket_oracle/vlo_bucket.h, built into tests/bucket_oracle/liboracle_bucket.so by tests/bucket_oracle/build.sh), and of getBucketedValue.
Test infrastructure: the blocks are the descriptor dicts victorialogs_b200.scan.HostBlocks takes (values blocks in their on-disk form, with the
column headers' minimum and maximum), the selected rows are bitmap words the caller computed."""
import ctypes as C
import os
import struct

import vloracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
FIELD_ABSENT, FIELD_CONST, FIELD_VALUES = 0, 1, 2


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "bucket_oracle", "liboracle_bucket.so")
        if not os.path.exists(path):
            raise ImportError("tests/bucket_oracle/liboracle_bucket.so is missing: build it with tests/bucket_oracle/build.sh (__graft_entry__.build() does)")
        L = C.CDLL(path)
        L.vlob_last_error.restype = C.c_char_p
        L.vlob_bucket_text.restype = C.c_int64
        L.vlob_bucket_text.argtypes = [C.c_double, C.c_double, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64]
        L.vlob_new.restype = C.c_void_p
        L.vlob_new.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_uint32, C.c_uint32]
        L.vlob_free.argtypes = [C.c_void_p]
        L.vlob_free.restype = None
        L.vlob_bucket.argtypes = [C.c_void_p, C.c_uint32, C.c_double, C.c_double, C.c_int, C.c_int]
        L.vlob_field.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64]
        L.vlob_block.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64]
        L.vlob_result.restype = C.c_int64
        L.vlob_result.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        _LIB = L
    return _LIB


def _check(rc):
    if rc:
        raise RuntimeError(lib().vlob_last_error().decode())


def bucket_text(text, size, offset=0.0, calendar=0):
    """getBucketedValue(text) (lib/logstorage/block_result.go:1666-1764) -> bytes; ValueError for a bucket the engine turns down"""
    text = vloracle._b(text)
    out = C.create_string_buffer(1024)
    n = lib().vlob_bucket_text(size, offset, calendar, text, len(text), out, 1024)
    if n == -2:
        raise ValueError((size, offset, calendar))
    return out.raw[:n]


def stats(descs, words, step, offset, calendar, by, buckets, values=()):
    """the groups of the selected rows (words[i]: bitmap words of block i) of the HostBlocks descriptor dicts `descs` -> {(bucket, key texts):
    (rows, [(sum, count, sum |x|, integers only) per value field])}; buckets: one (size, offset, calendar) or None per by-field"""
    L = lib()
    names = [vloracle._b(n) or b"_msg" for n in list(by) + list(values)]
    h = L.vlob_new(step, offset, calendar, len(by), len(values))
    try:
        for f, b in enumerate(buckets):
            if b is not None:
                _check(L.vlob_bucket(h, f, b[0], b[1], b[2], 1))
        for d, w in zip(descs, words):
            cols = {vloracle._b(c["field"]) or b"_msg": c for c in d["columns"]}
            for f, name in enumerate(names):
                if (f >= len(by) and name == b"_time") or name not in cols:
                    continue
                c = cols[name]
                if c["kind"] == "const":
                    v = vloracle._b(c["value"])
                    _check(L.vlob_field(h, f, FIELD_CONST, 0, v, len(v), None, None, 0, 0, 0))
                else:
                    blob, offs = vloracle._pack(c.get("dict") or [])
                    vb = c["values_block"]
                    _check(L.vlob_field(h, f, FIELD_VALUES, c["value_type"], vb, len(vb), blob, offs.ctypes.data_as(C.c_void_p), len(c.get("dict") or []),
                                        c["min_value"], c["max_value"]))
            data, mt, mn, mx = d["timestamps"]
            _check(L.vlob_block(h, d["rows"], w.ctypes.data_as(C.c_void_p), data, len(data), mt, mn, mx))
        n = L.vlob_result(h, None, 0)
        buf = C.create_string_buffer(max(n, 1))
        L.vlob_result(h, buf, n)
        raw = buf.raw[:n]
    finally:
        L.vlob_free(h)
    out, p = {}, 8
    for _ in range(struct.unpack_from("<Q", raw, 0)[0]):
        bucket, rows = struct.unpack_from("<qQ", raw, p)
        p += 16
        keys = []
        for _ in by:
            ln = struct.unpack_from("<Q", raw, p)[0]
            keys.append(raw[p + 8:p + 8 + ln])
            p += 8 + ln
        vals = []
        for _ in values:
            s, c, a = struct.unpack_from("<dQd", raw, p)
            vals.append((s, c, a, bool(raw[p + 24])))
            p += 25
        out[(bucket, tuple(keys))] = (rows, vals)
    return out
