"""ctypes binding of the C++ restatement of `stats by (_time:step offset off, f1, ...) count(), sum(v...), avg(v...)`
(tests/stats_oracle/vlo_stats.h, built into tests/stats_oracle/liboracle_stats.so by tests/stats_oracle/build.sh) over vloracle blocks, and of
the oracle's tryParseFloat64 / tryParseNumber.  Test infrastructure: the selected rows come from the oracle's own filter, the timestamps and
values are decoded from the blocks' stored bytes in C++."""
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
        path = os.path.join(_HERE, "stats_oracle", "liboracle_stats.so")
        if not os.path.exists(path):
            raise ImportError("tests/stats_oracle/liboracle_stats.so is missing: build it with tests/stats_oracle/build.sh (__graft_entry__.build() does)")
        L = C.CDLL(path)
        L.vlos_last_error.restype = C.c_char_p
        L.vlos_new.restype = C.c_void_p
        L.vlos_new.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_uint32, C.c_uint32]
        L.vlos_free.argtypes = [C.c_void_p]
        L.vlos_free.restype = None
        L.vlos_field.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint32]
        L.vlos_block.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64]
        L.vlos_result.restype = C.c_int64
        L.vlos_result.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        for n in ("vlos_try_parse_float64", "vlos_try_parse_number"):
            getattr(L, n).argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
        _LIB = L
    return _LIB


def _check(rc):
    if rc:
        raise RuntimeError(lib().vlos_last_error().decode())


def _parse(fn, s):
    out = C.c_double()
    ok = fn(s, len(s), C.byref(out))
    return out.value, bool(ok)


def try_parse_float64(s):
    """tryParseFloat64 (lib/logstorage/values_encoder.go:779) -> (float, ok)"""
    return _parse(lib().vlos_try_parse_float64, s)


def try_parse_number(s):
    """tryParseNumber (lib/logstorage/block_result.go:2710-2737) -> (float, ok)"""
    return _parse(lib().vlos_try_parse_number, s)


def stats(blocks, flt, step, offset, calendar, by, values):
    """the groups of the rows the oracle filter `flt` selects in the vloracle `blocks` -> {(bucket, key texts): (rows, [(sum, count, sum |x|,
    integers only) per value field])}"""
    L = lib()
    names = [n.encode() if isinstance(n, str) else n for n in list(by) + list(values)]
    h = L.vlos_new(step, offset, calendar, len(by), len(values))
    try:
        for blk in blocks:
            consts = dict(blk.consts)
            cols = {c.name: c for c in blk.columns}
            for f, name in enumerate(names):
                name = name or b"_msg"
                if f >= len(by) and name == b"_time":
                    continue
                if name in consts:
                    _check(L.vlos_field(h, f, FIELD_CONST, 0, consts[name], len(consts[name]), None, None, 0))
                elif name in cols:
                    c = cols[name]
                    blob, offs = vloracle._pack(c.dict)
                    _check(L.vlos_field(h, f, FIELD_VALUES, c.value_type, c.values_block, len(c.values_block), blob, offs.ctypes.data_as(C.c_void_p), len(c.dict)))
            words = blk.search(flt)
            data, mt, mn, mx = blk.timestamps_block()
            _check(L.vlos_block(h, blk.rows, words.ctypes.data_as(C.c_void_p), data, len(data), mt, mn, mx))
        n = L.vlos_result(h, None, 0)
        buf = C.create_string_buffer(max(n, 1))
        L.vlos_result(h, buf, n)
        raw = buf.raw[:n]
    finally:
        L.vlos_free(h)
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
