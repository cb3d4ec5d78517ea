"""The multi-threaded header walk of an upload (ZstdJob::add_values_blocks, victorialogs_b200/csrc/vl_zstd.cu) on the CPU.

Everything the walk hands to the device - frame table, ZSTD block table with scratch offsets and table slots, launch groups, work lists -
must not depend on the number of host threads.  vlscan_zstd_walk_digest hashes exactly that; the constants below were produced by the
single-threaded block-by-block walk whose output the GPU parity tests (tests/test_gpu_zstd.py, the bench's on-disk end-to-end check)
were run against, so an equal digest means the device sees byte-identical tables."""
import random

import pytest

from victorialogs_b200 import scan as vs
from parity_util import oracle_block_to_desc, field_names_of

# digests of the single-threaded walk (one thread, std::stable_sort) that the device decoder's parity suite was run against.
# "groups" was re-pinned when the launch-group limits became tapered (vl_zstd_job.h: a small first group, large ones, small ones
# over the last twelfth of the sequences - 3 groups for this data set; the frame digest, which does not depend on the cut, is unchanged);
# the device decoder's parity suite runs with those limits.
GOLDEN = {
    "small": (296292749011898157, 13177515279369892816, 15039143775152434337, 10484151172081120490),
    "groups": (17384690534920848810, 2494078724288951318, 166322921929518477, 3889144665088860614),
}


def dataset(oracle, name):
    if name == "small":        # 50 blocks x 300 rows, all generator columns: one launch group, multi-block frames absent
        rpb, nb, rep = 300, 50, 1
    else:                      # 60000 tiny blocks (many plain containers), shuffled: several launch groups
        rpb, nb, rep = 64, 200, 300
    cfg = oracle.GenConfig(seed=rpb, total_rows=rpb * nb, rows_per_block=rpb, hot_block_permille=500, hit_row_permille=60, columns_mask=0b1111)
    blocks = [oracle.Block.generated(cfg, i) for i in range(nb)]
    descs = [oracle_block_to_desc(b) for b in blocks] * rep
    random.Random(rpb).shuffle(descs)
    return blocks, descs


@pytest.mark.parametrize("name", ["small", "groups"])
def test_walk_is_independent_of_the_thread_count(oracle, name):
    blocks, descs = dataset(oracle, name)
    hb = vs.HostBlocks(field_names_of(blocks), descs)
    seen = {}
    for threads in (0, 1, 2, 5, 16, 64):
        r = vs.zstd_walk_digest(hb, threads)
        seen[threads] = r
        assert r["digest"] == GOLDEN[name], (name, threads)
    ncols = sum(1 for d in descs for c in d["columns"] if c["kind"] == "values")
    r = seen[16]
    assert r["frames"] == 2 * ncols and r["blocks"] >= r["frames"] and r["compressed_blocks"] <= r["blocks"]
    assert r["groups"] == (1 if name == "small" else 3)
    for k in ("frames", "blocks", "groups", "compressed_blocks", "sequences"):
        assert len({seen[t][k] for t in seen}) == 1, k


def test_walk_reports_the_first_malformed_block_like_the_sequential_walk(oracle):
    blocks, descs = dataset(oracle, "small")
    descs = descs * 40                                     # 2000 blocks: several shards even with the 256-blocks-per-thread floor
    names = field_names_of(blocks)
    rng = random.Random(2)

    def damage(kind, vb):
        if kind == "truncate":
            return vb[:-3]
        if kind == "tail":
            return vb + b"\x00"
        if kind == "type":
            return b"\x07" + vb[1:]
        if kind == "magic":                               # only meaningful for a ZSTD container
            i = vb.index(b"\x28\xb5\x2f\xfd")
            return vb[:i] + b"\x29" + vb[i + 1:]
        if kind == "empty":
            return b""
        raise AssertionError(kind)

    for trial in range(12):
        bad = sorted(rng.sample(range(len(descs)), 3))
        kinds = [rng.choice(["truncate", "tail", "type", "magic", "empty"]) for _ in bad]
        d2 = list(descs)
        for bi, kind in zip(bad, kinds):
            cols = [dict(c) for c in d2[bi]["columns"]]
            target = next(c for c in cols if c["kind"] == "values" and b"\x28\xb5\x2f\xfd" in c["values_block"])
            target["values_block"] = damage(kind, target["values_block"])
            d2[bi] = dict(d2[bi], columns=cols)
        hb = vs.HostBlocks(names, d2)
        msgs = []
        for threads in (0, 1, 7, 16):
            with pytest.raises(vs.VlscanError) as e:
                vs.zstd_walk_digest(hb, threads)
            msgs.append(str(e.value))
        assert len(set(msgs)) == 1, msgs
        # the ordinal in the message is that of the first damaged values block
        first = sum(1 for d in d2[:bad[0]] for c in d["columns"] if c["kind"] == "values")
        first += next(i for i, c in enumerate(c for c in d2[bad[0]]["columns"] if c["kind"] == "values") if c["values_block"] != [x for x in descs[bad[0]]["columns"] if x["kind"] == "values"][i]["values_block"])
        assert ("values block %d:" % first) in msgs[0], (msgs[0], first)


def test_walk_of_nothing(oracle):
    hb = vs.HostBlocks([b"_msg"], [])
    r0, r8 = vs.zstd_walk_digest(hb, 0), vs.zstd_walk_digest(hb, 8)
    assert r0["digest"] == r8["digest"] and r0["frames"] == r8["frames"] == 0 and r8["groups"] == 0
    # decoded-stage columns and const columns take no part in the walk
    blocks, _ = dataset(oracle, "small")
    descs = [oracle_block_to_desc(b, stage="decoded") for b in blocks[:3]]
    hb = vs.HostBlocks(field_names_of(blocks), descs)
    assert vs.zstd_walk_digest(hb, 4)["digest"] == r0["digest"]
