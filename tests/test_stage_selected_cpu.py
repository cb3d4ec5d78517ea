"""CPU suite for keeping an end-to-end scan on the device (vlscan_scan_batch_keep) and staging the pipes' columns for the blocks that need them
(vlscan_stage_selected): the symbols and their prototypes, the ctypes wrappers, the argument checks that need no device, and the loud failure
without one.  The checks against a kept batch (no kept scan, unknown field, block list range, descriptor mismatch) run on the GPU
(tests/test_gpu_zzzzzzzz_stage_selected.py)."""
import ctypes as C
import os
import re

import pytest

from victorialogs_b200 import scan as vs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def prototype(name):
    hdr = open(os.path.join(ROOT, "include", "vlscan.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_symbols_are_exported_and_mirrored():
    L = vs.lib()
    for n in ("vlscan_scan_batch_keep", "vlscan_stage_selected"):
        assert n in vs.EXPORTS
        assert hasattr(L, n)
    assert hasattr(vs.Ctx, "scan_batch_keep") and hasattr(vs.Ctx, "stage_selected")


def test_prototypes():
    # the keep call takes exactly the arguments of vlscan_scan_batch
    assert prototype("vlscan_scan_batch_keep") == prototype("vlscan_scan_batch")
    assert prototype("vlscan_stage_selected") == [
        "vlscan_ctx* ctx", "const vlscan_block* blocks", "uint64_t nblocks", "const char* const* field_names", "const size_t* field_name_lens",
        "uint32_t nfields", "const uint32_t* block_list", "uint64_t nlist", "uint64_t out_info[4]"]


def test_stats_layout_is_unchanged():
    # new counters travel in out_info: vlscan_stats keeps its 16 fields
    assert C.sizeof(vs.CStats) == 16 * 8
    assert [n for n, _ in vs.CStats._fields_][-2:] == ["staged_columns", "pruned_columns"]


def _stage(ctx, fields, block_list=None, nlist=None, names=True, blocks=None):
    names_b = [f.encode() for f in fields]
    arr = (C.c_char_p * max(len(names_b), 1))(*names_b)
    lens = (C.c_size_t * max(len(names_b), 1))(*[len(x) for x in names_b])
    info = (C.c_uint64 * 4)(*[7] * 4)
    lst = None if block_list is None else (C.c_uint32 * max(len(block_list), 1))(*block_list)
    n = nlist if nlist is not None else (0 if block_list is None else len(block_list))
    rc = vs.lib().vlscan_stage_selected(ctx, blocks, C.c_uint64(0), arr if names else None, lens if names else None, C.c_uint32(len(names_b)),
                                        lst, C.c_uint64(n), info)
    return rc, vs.lib().vlscan_last_error(ctx).decode(), list(info)


def test_stage_selected_argument_errors():
    for kw, word in ((dict(fields=[]), "at least one field"), (dict(fields=["a"], names=False), "field names missing"),
                     (dict(fields=["a"], nlist=3), "block list missing")):
        rc, err, info = _stage(None, **kw)
        assert rc < 0 and word in err, (kw, err)
        assert info == [7] * 4   # out_info is written on success only


def test_stage_selected_fails_loudly_without_a_device():
    rc, err, info = _stage(None, ["level", "_msg"])
    assert rc < 0 and "CUDA device" in err
    rc, err, info = _stage(None, ["level"], block_list=[0, 1])
    assert rc < 0 and "CUDA device" in err


def test_scan_batch_keep_fails_loudly_without_a_device():
    words = (C.c_uint64 * 4)(); counts = (C.c_uint32 * 4)()
    rc = vs.lib().vlscan_scan_batch_keep(None, None, None, None, C.c_uint32(0), None, C.c_uint64(0), words, counts, None)
    assert rc < 0 and "CUDA device" in vs.lib().vlscan_last_error(None).decode()


@pytest.mark.skipif(vs.lib().vlscan_device_count() > 0, reason="a CUDA device is present")
def test_no_ctx_without_a_device():
    with pytest.raises(vs.VlscanError):
        vs.Ctx(0)
