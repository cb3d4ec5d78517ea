"""CPU suite for the field-name arguments of vlscan_hits_stats: a query with by-fields but no name array (or no length array) is an
argument error reported without a device, never a read through NULL."""
import ctypes as C

from victorialogs_b200 import scan as vs


def test_hits_stats_rejects_missing_by_names():
    for missing in ("by_names", "by_name_lens"):
        q, keep = vs.hits_query(10 ** 9, 0, vs.BUCKET_PLAIN, ["level"])
        setattr(q, missing, None)
        info = (C.c_uint64 * 4)(7, 7, 7, 7)
        rc = vs.lib().vlscan_hits_stats(None, C.byref(q), None, None, C.c_uint64(0), None, C.c_uint64(0), None, info)
        assert rc < 0 and "vlscan_hits_stats: field names missing" in vs.lib().vlscan_last_error(None).decode(), missing
        assert list(info) == [0, 0, 0, 0]


def test_hits_stats_accepts_no_by_names_without_by_fields():
    # nby == 0 with NULL arrays is a valid query: the call gets past the argument checks and fails only for the missing device
    q, keep = vs.hits_query(10 ** 9, 0, vs.BUCKET_PLAIN, [])
    q.by_names = None
    q.by_name_lens = None
    rc = vs.lib().vlscan_hits_stats(None, C.byref(q), None, None, C.c_uint64(0), None, C.c_uint64(0), None, None)
    assert rc != 0 and "CUDA device" in vs.lib().vlscan_last_error(None).decode()
