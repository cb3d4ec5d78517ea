"""ctypes binding of the C++ restatement of `| facets` (tests/facets_oracle/vlo_facets.h, built into tests/facets_oracle/liboracle_facets.so by
tests/facets_oracle/build.sh): one shard with concurrency 1 over vloracle blocks, its per-field state and its flush.  Test infrastructure: the
selected rows come from the oracle's own filter, and the values and timestamps are decoded from the blocks' stored bytes in C++."""
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
        path = os.path.join(_HERE, "facets_oracle", "liboracle_facets.so")
        if not os.path.exists(path):
            raise ImportError("tests/facets_oracle/liboracle_facets.so is missing: build it with tests/facets_oracle/build.sh (__graft_entry__.build() does)")
        L = C.CDLL(path)
        L.vlof_last_error.restype = C.c_char_p
        L.vlof_new.restype = C.c_void_p
        L.vlof_new.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32]
        L.vlof_free.argtypes = [C.c_void_p]
        L.vlof_free.restype = None
        L.vlof_name.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint64, C.c_int]
        L.vlof_field.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint32]
        L.vlof_block.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64]
        L.vlof_state.restype = C.c_int64
        L.vlof_state.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.vlof_flush.restype = C.c_int64
        L.vlof_flush.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64]
        _LIB = L
    return _LIB


def _check(rc):
    if rc:
        raise RuntimeError(lib().vlof_last_error().decode())


def _read(fn, *args):
    n = fn(*args, None, 0)
    out = C.create_string_buffer(max(n, 1))
    fn(*args, out, n)
    return out.raw[:n]


def facets(blocks, flt, fields, max_values=0, max_len=0, limit=None, keep_const_fields=False):
    """the facets shard over the rows the oracle filter `flt` selects in the vloracle `blocks`, for the field names `fields` ("" and "_msg"
    both name the message field, "_time" the timestamps) -> (state, selected rows, blocks decoded, flush rows or None).  state = {field: None
    when dropped, else [(class, text, hits)] by hits descending, then text, then class}; flush rows = [(field, text, hits)] when `limit` is given."""
    L = lib()
    h = L.vlof_new(max_values, max_len, len(fields))
    try:
        for f, name in enumerate(fields):
            _check(L.vlof_name(h, f, name.encode(), len(name.encode()), int(name == "_time")))
        for blk in blocks:
            consts = dict(blk.consts)
            cols = {c.name: c for c in blk.columns}
            for f, name in enumerate(fields):
                stored = [n for n in ((b"_msg", b"") if name in ("", "_msg") else (name.encode(),)) if n in consts or n in cols]
                if name == "_time" or not stored:
                    continue
                if stored[0] in consts:
                    v = consts[stored[0]]
                    _check(L.vlof_field(h, f, FIELD_CONST, 0, v, len(v), None, None, 0))
                else:
                    c = cols[stored[0]]
                    blob, offs = vloracle._pack(c.dict)
                    _check(L.vlof_field(h, f, FIELD_VALUES, c.value_type, c.values_block, len(c.values_block), blob, offs.ctypes.data_as(C.c_void_p), len(c.dict)))
            words = blk.search(flt)
            try:
                data, mt, mn, mx = blk.timestamps_block()
            except ValueError:
                data, mt, mn, mx = b"", 0, 0, 0
            _check(L.vlof_block(h, blk.rows, words.ctypes.data_as(C.c_void_p), data, len(data), mt, mn, mx))
        raw = _read(L.vlof_state, h)
        flushed = _read(L.vlof_flush, h, limit, int(keep_const_fields)) if limit is not None else None
    finally:
        L.vlof_free(h)
    rows, decoded = struct.unpack_from("<QQ", raw, 0)
    p, state = 16, {}
    for name in fields:
        dropped, n = raw[p], struct.unpack_from("<Q", raw, p + 1)[0]
        p += 9
        ents = []
        for _ in range(n):
            cls, hits, ln = raw[p], *struct.unpack_from("<QQ", raw, p + 1)
            ents.append((cls, raw[p + 17:p + 17 + ln], hits))
            p += 17 + ln
        state[name] = None if dropped else ents
    out = None
    if flushed is not None:
        out, q = [], 8
        for _ in range(struct.unpack_from("<Q", flushed, 0)[0]):
            parts = []
            for _k in range(2):
                ln = struct.unpack_from("<Q", flushed, q)[0]
                parts.append(flushed[q + 8:q + 8 + ln])
                q += 8 + ln
            out.append((parts[0].decode(), parts[1], struct.unpack_from("<Q", flushed, q)[0]))
            q += 8
    return state, rows, decoded, out
