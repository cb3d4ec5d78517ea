"""Frames built from chosen sequences (tests/zstd_frames.py), checked without a GPU before the device decodes them
(tests/test_gpu_zzzzzzzzzzzzzzz_zstd_sequences.py):

* the plain LZ replay of every case equals libzstd's ZSTD_decompress of its frame, so a builder bug cannot pass silently;
* the plain-Python reader (tests/zstd_reader.py) finds in every compressed block exactly the sequences the case asked for, and every
  block libzstd stored raw or RLE holds exactly the requested bytes; the host walker (vlscan_zstd_inspect) counts the same blocks,
  compressed blocks and sequences;
* every case reaches the decoder edges it exists for: a coverage table counted from the frames' bytes (and from k_execute's geometry)
  must have every entry >= 1, so a libzstd choice that drops a feature fails here instead of silently thinning the GPU test;
* the reader agrees with libzstd's ordinary compressor's frames too (block sums, offsets within the frame);
* the executor cases also run through the CPU model of k_execute (tests/test_zstd_models_cpu.py) at its ring size and at 256 bytes."""
import collections
import functools

import pytest

import zstd_frames as zf
import zstd_reader as zr
from test_gpu_zstd import compress, corpus
from test_zstd_host_walk_cpu import container
from test_zstd_models_cpu import RING, execute_model, lz_reference

EXECUTOR_CASES = ("overlap_ring", "overlap_byte", "ring_edges", "ring_lo", "dependencies", "literal_shapes")


@functools.lru_cache(maxsize=None)
def cases():
    return {c.name: c for c in zf.all_cases()}


@functools.lru_cache(maxsize=None)
def read(name):
    c = cases()[name]
    return zr.read_frame(c.frame())


@functools.lru_cache(maxsize=None)
def geometry(name):
    return zr.execute_geometry(read(name)["blocks"])


def all_names():
    return list(cases())


CASE_NAMES = ["overlap_ring", "overlap_byte", "ring_edges", "ring_lo", "dependencies", "literal_shapes", "literal_kinds", "blocks_between",
              "repeat_offsets", "table_modes", "repeat_tables", "large_codes", "huffman", "nseq_1", "nseq_127", "nseq_128", "nseq_32511",
              "nseq_32512", "nseq_32513", "nseq_42000"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_case_frame_reader_and_walker(name):
    from victorialogs_b200 import scan as vs
    c = cases()[name]
    want = c.expected()
    frame = c.frame()
    assert zf.zstd_decompress(frame, len(want)) == want
    R = read(name)
    assert R["fcs"] == len(want)
    assert len(R["blocks"]) == len(c.blocks)
    for B, req in zip(R["blocks"], c.blocks):
        got = want[B["out_base"]:B["out_base"] + B["out_len"]]
        if B["type"] == zr.COMPRESSED:
            assert zr.requested_blocks([B])[0] == (req[0], req[1]), (name, B["index"])
        elif B["type"] == zr.RAW:
            assert frame[B["src"]:B["src"] + B["size"]] == got
        else:
            assert got == bytes([B["byte"]]) * B["size"]
        assert B["out_len"] == sum(ll + ml for ll, ml, _ in req[0]) + req[1]
    info = vs.zstd_inspect(container(frame))
    assert info["regenerated"] == len(want)
    assert info["blocks"] == len(R["blocks"])
    assert info["compressed_blocks"] == sum(B["type"] == zr.COMPRESSED for B in R["blocks"])
    assert info["sequences"] == sum(B.get("nseq", 0) for B in R["blocks"])


def case_coverage(name):
    """Counts of the decoder edges one case reaches, from its frame's bytes and k_execute's geometry."""
    n = collections.Counter()
    overlap = {"ring": set(), "byte": set()}
    lit_align = set()
    blocks = read(name)["blocks"]
    geo = geometry(name)
    # -- k_execute --
    for g in geo["groups"]:
        for O in (4095, 4096, 4097):
            n["group_O_%d" % O] += g["O"] == O
        n["dep_chain_32"] += g["depth"] == 32
        B = blocks[g["block"]]
        grp = B["seqs"][g["first"]:g["first"] + g["cnt"]]
        n["group_without_literals"] += g["cnt"] == 32 and all(q[0] == 0 for q in grp)
        n["literal_chunks_over_128"] += g["path"] == "ring" and sum((q[0] + 3) // 4 for q in grp) > 128
        if g["path"] == "ring":
            p = g["out_run"]
            for ll, ml, _, _ in grp:
                if ll < 10:
                    lit_align.add((ll, (p + 16) % 4))
                p += ll + ml
    run_chunks = collections.Counter()
    for m in geo["matches"]:
        B = blocks[m["block"]]
        ll, ml, ov, off = B["seqs"][m["seq"]]
        overlap[m["path"]].add((off, ml))
        n["dep_adjacent_ring"] += m["path"] == "ring" and m["dep"] >= 0 and m["dep"] == m["seq"] % 32 - 1
        n["dep_31_back"] += m["seq"] % 32 == 31 and m["dep"] == 0
        n["straddle_ring_lo"] += m["path"] == "ring" and m["straddle"]
        n["src_at_ring_lo"] += m["path"] == "ring" and m["sa"] == m["ring_lo"] and m["ring_lo"] > 0
        if m["dep"] < 0 and m["path"] == "ring":
            run_chunks[m["group"]] += (ml + 3) // 4
        for b0, back, below, how, held in m["chunks"]:
            for X in (4095, 4096, 4097):
                n["src_at_gend_minus_%d" % X] += back == X
            n["ring_src_stale_at_4097_4100"] += 4096 < back <= 4100 and not below and held is False          # `gend - sa <= Z_RING + 4` would read it
            n["ring_src_stale_below_ring_lo"] += below and back <= zr.RING and held is False      # without `sa >= ring_lo` it would be read
            n["src_in_raw_or_rle_block_near"] += how == "ring" and _block_of(blocks, m["sa"] + b0) in (zr.RAW, zr.RLE)
        n["src_in_raw_or_rle_block_far"] += m["gend_minus_sa"] > zr.RING and _block_of(blocks, m["sa"]) in (zr.RAW, zr.RLE)
    n["independent_run_over_128_chunks"] += any(v > 128 for v in run_chunks.values())
    # -- sequences, repeat offsets --
    prev_kind, prev_all_rep = None, 0
    for i, B in enumerate(blocks):
        if B["type"] != zr.COMPRESSED:
            prev_kind = ("raw", "rle")[B["type"]]
            continue
        nseq = B["nseq"]
        for v in (0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 0x7EFF, 0x7F00, 0x7F01):
            n["nseq_%d" % v] += nseq == v
        n["nseq_ge_42000"] += nseq >= 42000
        n["nseq_3byte"] += B["nseq_bytes"] == 3
        n["nseq_2byte"] += B["nseq_bytes"] == 2
        if nseq == 0:
            n["literal_only_block"] += 1
            prev_kind = "lits"
            continue
        for kind in ("ll", "of", "ml"):
            n["%s_mode_%s" % (kind, B["modes"][kind])] += 1
            back = B["repeat_back"].get(kind, 0)
            between = blocks[i - back + 1:i]
            if back >= 2 and all(x["type"] != zr.COMPRESSED or x["nseq"] == 0 for x in between):   # through blocks without sequences
                for k2 in {("raw", "rle", "lits")[x["type"] if x["type"] != zr.COMPRESSED else 2] for x in between}:
                    n["%s_mode_repeat_over_%s" % (kind, k2)] += 1
            f = B["fse"].get(kind)
            if f:
                n["fse_zero_repeat_flags"] += f["zero_repeat"] > 0
                n["fse_zero_repeat_flag_3"] += f["zero_repeat_3"] > 0
                n["fse_less_than_one"] += f["less_than_one"] > 0
        redo = min(B["clean_from"], nseq) if not B["rep_known"] else 0
        inherited = 0
        d = [zr.DIRTY] * 3 if not B["rep_known"] else None
        for j, (ll, ml, ov, off) in enumerate(B["seqs"]):
            if ov <= 3:
                n["rep_ov%d_%s" % (ov, "ll0" if ll == 0 else "ll")] += 1
            if j < redo and ov <= 3:
                n["rep_ov%d_%s_dirty" % (ov, "ll0" if ll == 0 else "ll")] += 1
            if d is not None:
                d, o = zr.update_rep(*d, ov, ll)
                if o == zr.DIRTY and inherited == j:
                    inherited += 1
            n["ll_code_35"] += ll >= 65536
            n["ml_code_52"] += ml >= 65539
            n["of_code_20"] += ov >= 1 << 20
            n["wide_sequences_back_to_back"] += j > 0 and min(B["bits"][j - 1], B["bits"][j]) >= 60
        if not B["rep_known"]:
            for v in (0, 1, 2, 3, 10):
                n["inherited_prefix_%d" % v] += inherited == v
        never_clean = not B["rep_known"] and B["clean_from"] > nseq
        n["never_clean_block"] += never_clean
        all_rep = not B["rep_known"] and all(q[2] <= 3 for q in B["seqs"])
        n["all_repeat_block"] += all_rep
        if all_rep and prev_kind in ("raw", "rle", "lits"):
            n["all_repeat_after_%s" % prev_kind] += 1
        prev_all_rep = prev_all_rep + 1 if all_rep else 0
        n["all_repeat_chain_2"] += prev_all_rep == 2
        n["all_repeat_chain_3"] += prev_all_rep == 3
        n["after_never_clean_uses_history"] += _prev_seq_block_never_clean(blocks, i) and B["seqs"][0][2] <= 3
        prev_kind = "seq"
    # -- literals --
    prev_huf_then_raw = False
    for B in blocks:
        if B["type"] == zr.RAW:
            n["raw_block"] += 1
            prev_huf_then_raw = True
            continue
        if B["type"] == zr.RLE:
            n["rle_block"] += 1
            continue
        lt, h = B["lit_type"], B["huf"]
        if B["nseq"]:
            n["lit_%s_read_by_matches" % ("raw", "rle", "huffman", "treeless")[lt]] += 1
        if h:
            n["huf_%d_stream" % B["streams"]] += 1
            n["huf_maxbits_le2"] += h["maxbits"] <= 2
            n["huf_maxbits_11"] += h["maxbits"] == 11
            if lt == zr.L_COMPRESSED:
                n["huf_weights_%s" % h["form"]] += 1
                n["huf_weights_direct_ge_64"] += h["form"] == "direct" and h["nsyms"] >= 64
            if B["streams"] == 4:
                n["huf_4stream_regen_mod4_%d" % (B["lit_regen"] % 4)] += 1
            n["treeless_after_raw_block"] += lt == zr.L_TREELESS and prev_huf_then_raw
        if lt == zr.L_COMPRESSED:
            prev_huf_then_raw = False
    # trailing literals read by the next block
    for i in range(len(blocks) - 1):
        B, N = blocks[i], blocks[i + 1]
        if B["type"] == zr.COMPRESSED and B["nseq"] and N["type"] == zr.COMPRESSED and N["nseq"]:
            t = B["lit_regen"] - sum(q[0] for q in B["seqs"])
            end = B["out_base"] + B["out_len"]
            p, reads = N["out_base"], False
            for ll, ml, _, off in N["seqs"]:
                p += ll
                reads |= end - t <= p - off < end
                p += ml
            for v in (0, 1, 4095, 4096, 4097):
                n["trailing_%d_then_read" % v] += t == v and (reads or v == 0)
    for path in ("ring", "byte"):
        missing = [(o, m) for o in zf.OVERLAP_OFFSETS for m in zf.OVERLAP_LENGTHS if (o, m) not in overlap[path]]
        n["overlap_all_combos_%s_path" % path] = int(not missing)
    n["literal_runs_0_9_every_alignment"] = int(all((ll, a) in lit_align for ll in range(10) for a in range(4)))
    return n


def coverage():
    """The coverage of all cases together."""
    n = collections.Counter()
    for name in all_names():
        n.update(case_coverage(name))
    return n


def _block_of(blocks, pos):
    for B in blocks:
        if B["out_base"] <= pos < B["out_base"] + B["out_len"]:
            return B["type"]
    return None


def _prev_seq_block_never_clean(blocks, i):
    for B in reversed(blocks[:i]):
        if B["type"] == zr.COMPRESSED and B["nseq"]:
            return not B["rep_known"] and B["clean_from"] > B["nseq"]
    return False


WANT = """group_O_4095 group_O_4096 group_O_4097 src_at_gend_minus_4095 src_at_gend_minus_4096 src_at_gend_minus_4097
ring_src_stale_at_4097_4100 ring_src_stale_below_ring_lo straddle_ring_lo src_at_ring_lo dep_chain_32 dep_adjacent_ring dep_31_back
independent_run_over_128_chunks literal_chunks_over_128 group_without_literals literal_runs_0_9_every_alignment
overlap_all_combos_ring_path overlap_all_combos_byte_path src_in_raw_or_rle_block_near src_in_raw_or_rle_block_far
trailing_0_then_read trailing_1_then_read trailing_4095_then_read trailing_4096_then_read trailing_4097_then_read
rep_ov1_ll rep_ov2_ll rep_ov3_ll rep_ov1_ll0 rep_ov2_ll0 rep_ov3_ll0 rep_ov1_ll0_dirty rep_ov2_ll0_dirty rep_ov3_ll0_dirty
rep_ov1_ll_dirty rep_ov2_ll_dirty rep_ov3_ll_dirty inherited_prefix_0 inherited_prefix_1 inherited_prefix_2 inherited_prefix_3
inherited_prefix_10 all_repeat_block all_repeat_chain_2 all_repeat_chain_3 all_repeat_after_raw all_repeat_after_rle all_repeat_after_lits
never_clean_block after_never_clean_uses_history
nseq_0 nseq_1 nseq_31 nseq_32 nseq_33 nseq_63 nseq_64 nseq_65 nseq_127 nseq_128 nseq_32511 nseq_32512 nseq_32513 nseq_ge_42000
nseq_2byte nseq_3byte literal_only_block raw_block rle_block
ll_mode_predef ll_mode_rle ll_mode_fse ll_mode_repeat of_mode_predef of_mode_rle of_mode_fse of_mode_repeat
ml_mode_predef ml_mode_rle ml_mode_fse ml_mode_repeat
ll_mode_repeat_over_raw ll_mode_repeat_over_rle ll_mode_repeat_over_lits of_mode_repeat_over_raw of_mode_repeat_over_rle
of_mode_repeat_over_lits ml_mode_repeat_over_raw ml_mode_repeat_over_rle ml_mode_repeat_over_lits
fse_zero_repeat_flags fse_less_than_one ll_code_35 ml_code_52 of_code_20 wide_sequences_back_to_back
lit_raw_read_by_matches lit_rle_read_by_matches lit_huffman_read_by_matches lit_treeless_read_by_matches
huf_1_stream huf_4_stream huf_maxbits_le2 huf_maxbits_11 huf_weights_direct huf_weights_direct_ge_64 huf_weights_fse
huf_4stream_regen_mod4_0 huf_4stream_regen_mod4_1 huf_4stream_regen_mod4_2 huf_4stream_regen_mod4_3 treeless_after_raw_block""".split()


def test_cases_reach_their_edges():
    n = coverage()
    missing = [k for k in WANT if n[k] < 1]
    assert not missing, "features no case reaches any more: %s\n%s" % (missing, dict(sorted(n.items())))


@pytest.mark.parametrize("name", CASE_NAMES)
def test_each_case_reaches_its_own_targets(name):
    """Every case reaches the edges it is named for by itself, not only with the help of other cases."""
    c = cases()[name]
    assert c.targets and set(c.targets) <= set(WANT), (name, sorted(set(c.targets) - set(WANT)))
    n = case_coverage(name)
    missing = [k for k in c.targets if n[k] < 1]
    assert not missing, "%s no longer reaches %s\n%s" % (name, missing, dict(sorted(n.items())))


@pytest.mark.parametrize("level", [1, 3, 19])
def test_reader_on_libzstd_corpus(level):
    for name, data in corpus().items():
        if level == 19 and len(data) > 400_000:
            continue
        R = zr.read_frame(compress(data, level))
        assert R["fcs"] == len(data), name
        total = 0
        for B in R["blocks"]:
            if B["type"] == zr.COMPRESSED:
                p = total
                for ll, ml, ov, off in B["seqs"]:
                    p += ll
                    assert 1 <= off <= p, (name, level, B["index"])
                    p += ml
                assert sum(q[0] for q in B["seqs"]) <= B["lit_regen"]
                assert B["out_len"] == B["lit_regen"] + sum(q[1] for q in B["seqs"])
            total += B["out_len"]
        assert total == len(data), (name, level)


@pytest.mark.parametrize("name", EXECUTOR_CASES)
def test_executor_model_on_cases(name):
    """Each block of the executor cases through execute_model (its groups restart at the block, as k_execute's do)."""
    c = cases()[name]
    want = c.expected()
    lp = 0
    at = 0
    for seqs, tail in c.blocks:
        nl = sum(q[0] for q in seqs) + tail
        size = nl + sum(q[1] for q in seqs)
        reach = max([off - (sum(q[0] + q[1] for q in seqs[:i]) + seqs[i][0]) for i, (_, _, off) in enumerate(seqs)] + [0])
        keep = min(at, max(reach, 0) + 64)
        prefix = want[at - keep:at]
        lits = bytes(c.lits[lp:lp + nl])
        ref = lz_reference(lits, seqs, prefix)
        assert ref[keep:] == want[at:at + size]
        for ring in (RING, 256):
            assert execute_model(lits, seqs, prefix, ring_size=ring)[keep:] == want[at:at + size], (name, at, ring)
        lp += nl
        at += size
