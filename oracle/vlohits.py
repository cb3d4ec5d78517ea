"""ctypes binding of the CPU restatement of the hits aggregation (oracle/vlo_hits.h, built into oracle/liboracle_hits.so by
oracle/build_hits.sh): `stats by (_time:step offset off, f1, ...) count()` over vloracle blocks, and truncateTimestamp.

TEST INFRASTRUCTURE ONLY: import this from tests/ and tools/, never from victorialogs_b200/.  The selected rows come from the oracle's
own filter (vloracle.Block.search); the timestamps and by-field values are decoded here from the blocks' stored bytes.
"""
import ctypes as C
import os

import numpy as np

import vloracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

BUCKET_PLAIN, BUCKET_WEEK, BUCKET_MONTH, BUCKET_YEAR = 0, 1, 2, 3
FIELD_ABSENT, FIELD_CONST, FIELD_VALUES = 0, 1, 2
GEN_TIMESTAMPS = 1 << 4                             # vlscan_gen_config.columns_mask bit of the generator's timestamps column
GEN_T0, GEN_STEP = 1700000000000000000, 1000000     # row i of a generated data set is at GEN_T0 + i * GEN_STEP nanoseconds


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "liboracle_hits.so")
        if not os.path.exists(path):
            raise ImportError("oracle/liboracle_hits.so is missing: build it with oracle/build_hits.sh (__graft_entry__.build() does)")
        L = C.CDLL(path)
        L.vloh_last_error.restype = C.c_char_p
        L.vloh_truncate_timestamp.restype = C.c_int64
        L.vloh_truncate_timestamp.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int]
        L.vloh_new.restype = C.c_void_p
        L.vloh_new.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_uint32]
        L.vloh_free.argtypes = [C.c_void_p]
        L.vloh_free.restype = None
        L.vloh_field.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint32]
        L.vloh_block.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_int64]
        L.vloh_result.restype = C.c_int64
        L.vloh_result.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        _LIB = L
    return _LIB


def _check(rc):
    if rc:
        raise RuntimeError(lib().vloh_last_error().decode())


def truncate_timestamp(ts, step, offset=0, calendar=BUCKET_PLAIN):
    """truncateTimestamp (block_result.go:818-848): the `_time` bucket of one timestamp"""
    return lib().vloh_truncate_timestamp(ts, step, offset, calendar)


def gen_timestamps(cfg, block_id):
    """the timestamps of block `block_id` of a generated data set with GEN_TIMESTAMPS in columns_mask: one row every GEN_STEP from GEN_T0"""
    first = block_id * cfg.rows_per_block
    rows = min(cfg.rows_per_block, cfg.total_rows - first)
    return [GEN_T0 + (first + i) * GEN_STEP for i in range(rows)]


def _canonical(name):
    name = vloracle._b(name)
    return name or b"_msg"


def hits_stats(blocks, flt, step, offset=0, calendar=BUCKET_PLAIN, by=(), info=None):
    """`stats by (_time:step offset off, by...) count()` over the rows the oracle filter `flt` selects in the vloracle `blocks`
    -> [(bucket, (key texts...), count)] sorted by bucket, then by the texts.  `info` (a dict) receives rows and blocks_decoded
    (blocks with selected rows whose minimum and maximum timestamps fall into different buckets)."""
    L = lib()
    names = [_canonical(f) for f in by]
    h = L.vloh_new(step, offset, calendar, len(names))
    try:
        for blk in blocks:
            consts = dict(blk.consts)
            cols = {c.name: c for c in blk.columns}
            for f, name in enumerate(names):
                if name in consts:
                    _check(L.vloh_field(h, f, FIELD_CONST, 0, consts[name], len(consts[name]), None, None, 0))
                elif name in cols:
                    c = cols[name]
                    blob, offs = vloracle._pack(c.dict)
                    _check(L.vloh_field(h, f, FIELD_VALUES, c.value_type, c.values_block, len(c.values_block), blob, offs.ctypes.data_as(C.c_void_p), len(c.dict)))
            words = blk.search(flt)
            try:
                data, mt, mn, mx = blk.timestamps_block()
            except ValueError:
                data, mt, mn, mx = b"", 0, 0, 0
            _check(L.vloh_block(h, blk.rows, words.ctypes.data_as(C.c_void_p), data, len(data), mt, mn, mx))
        n = L.vloh_result(h, None, 0)
        out = C.create_string_buffer(max(n, 1))
        L.vloh_result(h, out, n)
    finally:
        L.vloh_free(h)
    raw = out.raw[:n]
    ngroups, rows, decoded = (int(x) for x in np.frombuffer(raw[:24], dtype=np.uint64))
    if info is not None:
        info.update(rows=rows, blocks_decoded=decoded)
    res, p = [], 24
    for _ in range(ngroups):
        bucket, count = int(np.frombuffer(raw[p:p + 8], dtype=np.int64)[0]), int(np.frombuffer(raw[p + 8:p + 16], dtype=np.uint64)[0])
        p += 16
        keys = []
        for _f in names:
            ln = int(np.frombuffer(raw[p:p + 8], dtype=np.uint64)[0])
            keys.append(raw[p + 8:p + 8 + ln])
            p += 8 + ln
        res.append((bucket, tuple(keys), count))
    return res
