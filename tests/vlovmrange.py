"""ctypes binding of the C++ restatement of `stats by (_time:step, f:bucket, ...) histogram(v...)` (tests/vmrange_oracle/vlo_vmrange.h, built
into tests/vmrange_oracle/liboracle_vmrange.so by tests/vmrange_oracle/build.sh).  Test infrastructure: the blocks are the descriptor dicts
victorialogs_b200.scan.HostBlocks takes, the selected rows are bitmap words the caller computed."""
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
        path = os.path.join(_HERE, "vmrange_oracle", "liboracle_vmrange.so")
        script = os.path.join(_HERE, "vmrange_oracle", "build.sh")
        if not os.path.exists(path) and os.access(os.path.dirname(script), os.W_OK):
            import subprocess
            subprocess.check_call([script], stdout=subprocess.DEVNULL)
        if not os.path.exists(path):
            raise ImportError("tests/vmrange_oracle/liboracle_vmrange.so is missing: build it with tests/vmrange_oracle/build.sh (__graft_entry__.build() does)")
        L = C.CDLL(path)
        L.vlov_last_error.restype = C.c_char_p
        L.vlov_index.argtypes = [C.c_double]
        L.vlov_parse_number.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_double)]
        L.vlov_new.restype = C.c_void_p
        L.vlov_new.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_uint32, C.c_uint32]
        L.vlov_free.argtypes = [C.c_void_p]
        L.vlov_free.restype = None
        L.vlov_bucket.argtypes = [C.c_void_p, C.c_uint32, C.c_double, C.c_double, C.c_int, C.c_int]
        L.vlov_field.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64]
        L.vlov_block.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64]
        L.vlov_result.restype = C.c_int64
        L.vlov_result.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        _LIB = L
    return _LIB


def _check(rc):
    if rc:
        raise RuntimeError(lib().vlov_last_error().decode())


def index(v):
    """Histogram.Update's index of v from its formula (-1: skipped)"""
    return lib().vlov_index(v)


def parse_number(s):
    """the oracle's tryParseNumber -> (value, ok)"""
    s = vloracle._b(s)
    x = C.c_double()
    ok = lib().vlov_parse_number(s, len(s), C.byref(x))
    return x.value, bool(ok)


def vmranges(descs, words, step, offset, calendar, by, buckets, values):
    """the groups of the selected rows (words[i]: bitmap words of block i) of the HostBlocks descriptor dicts `descs` -> {(bucket, key texts):
    (rows, [{index: hits} per value field])}; buckets: None or one (size, offset, calendar) or None per by-field"""
    L = lib()
    buckets = buckets or [None] * len(by)
    names = [vloracle._b(n) or b"_msg" for n in list(by) + list(values)]
    h = L.vlov_new(step, offset, calendar, len(by), len(values))
    try:
        for f, b in enumerate(buckets):
            if b is not None:
                _check(L.vlov_bucket(h, f, b[0], b[1], b[2], 1))
        for d, w in zip(descs, words):
            cols = {vloracle._b(c["field"]) or b"_msg": c for c in d["columns"]}
            for f, name in enumerate(names):
                if (f >= len(by) and name == b"_time") or name not in cols:
                    continue
                c = cols[name]
                if c["kind"] == "const":
                    v = vloracle._b(c["value"])
                    _check(L.vlov_field(h, f, FIELD_CONST, 0, v, len(v), None, None, 0, 0, 0))
                else:
                    blob, offs = vloracle._pack(c.get("dict") or [])
                    vb = c["values_block"]
                    _check(L.vlov_field(h, f, FIELD_VALUES, c["value_type"], vb, len(vb), blob, offs.ctypes.data_as(C.c_void_p), len(c.get("dict") or []),
                                        c["min_value"], c["max_value"]))
            data, mt, mn, mx = d["timestamps"]
            _check(L.vlov_block(h, d["rows"], w.ctypes.data_as(C.c_void_p), data, len(data), mt, mn, mx))
        n = L.vlov_result(h, None, 0)
        buf = C.create_string_buffer(max(n, 1))
        L.vlov_result(h, buf, n)
        raw = buf.raw[:n]
    finally:
        L.vlov_free(h)
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
            ne = struct.unpack_from("<Q", raw, p)[0]
            p += 8
            m = {}
            for _ in range(ne):
                i, c = struct.unpack_from("<QQ", raw, p)
                m[i] = c
                p += 16
            vals.append(m)
        out[(bucket, tuple(keys))] = (rows, vals)
    return out
