"""The device ZSTD decoder (victorialogs_b200/csrc/vl_zstd.cuh) on frames built from chosen sequences (tests/zstd_frames.py): the
executor's ring and group edges, every overlap width on both copy paths, dependency chains, repeat offsets across blocks, the
sequence-section encodings and the Huffman table shapes.  tests/test_zstd_sequences_cpu.py proves, without a GPU, that each case
reaches the edges it is named for; here every case must decode byte-exact against the plain LZ replay:

* all cases in one call, and every case alone;
* every case at all 16 output phases (the flush split at 16-byte arena boundaries, the ring's 4-byte word reads) and at a spread of
  compressed-byte phases mod 256 (the sequence ring's origin, the Huffman decoder's 8-byte word reads), set by filler frames in front;
* a few thousand small crafted frames in one launch next to one block of 42 000 sequences, so lanes of one sequence CTA and one Huffman
  CTA hold blocks of very different sizes.

A mismatch names the first wrong byte's block, group, sequence, whether it is a literal or a match byte, the copy path k_execute took
and the source's distance from the group's end (tests/zstd_reader.py), so a failure points at the rule that broke."""
import functools

import pytest

import zstd_frames as zf
import zstd_reader as zr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cx():
    from victorialogs_b200 import scan as vs
    return vs.Ctx(0)


@functools.lru_cache(maxsize=None)
def cases():
    return zf.all_cases()


def where_wrong(case, got):
    want = case.expected()
    if len(got) != len(want):
        return "%s: %d bytes instead of %d" % (case.name, len(got), len(want))
    pos = next(i for i in range(len(want)) if got[i] != want[i])
    blocks = zr.read_frame(case.frame())["blocks"]
    nbad = sum(1 for i in range(pos, len(want)) if got[i] != want[i])
    return "%s: first wrong byte at %d of %d (%d wrong, got 0x%02x want 0x%02x): %s" % (
        case.name, pos, len(want), nbad, got[pos], want[pos], zr.locate(blocks, zr.execute_geometry(blocks), pos))


def check(case, got, what=""):
    if got != case.expected():
        pytest.fail(what + where_wrong(case, got))


def test_all_cases_in_one_call(cx):
    cs = cases()
    got = cx.zstd_decompress([c.frame() for c in cs], [len(c.expected()) for c in cs])
    for c, g in zip(cs, got):
        check(c, g)


def test_every_case_alone(cx):
    for c in cases():
        check(c, cx.zstd_decompress([c.frame()], [len(c.expected())])[0], "alone: ")


def test_every_output_phase_and_a_spread_of_source_phases(cx):
    items, who = [], []
    for k, c in enumerate(cases()):
        big = len(c.expected()) > 500_000
        phases = [((37 * d + 11 * k) % 256, d) for d in range(16)]
        phases += [((16 * s + 5 * k + 1) % 256, (3 * s + k) % 16) for s in range(16)]
        for cp, op in phases[:16] if big else phases:      # a 2 MB case: every output phase once, 16 source phases
            items.append((c.frame(), len(c.expected()), cp, op))
            who.append((c, cp, op))
    frames, sizes, where = zf.placed(items)
    got = cx.zstd_decompress(frames, sizes)
    comp_at, out_at = [0], [0]
    for f, n in zip(frames, sizes):
        comp_at.append(comp_at[-1] + len(f)); out_at.append(out_at[-1] + n)
    for (c, cp, op), i in zip(who, where):
        assert (512 + comp_at[i]) % 256 == cp and (16 + out_at[i]) % 16 == op    # where vlscan_zstd_decompress puts frame i
        check(c, got[i], "compressed phase %d, output phase %d: " % (cp, op))


def test_small_frames_next_to_a_huge_block(cx):
    small = zf.small_frames(3000)
    huge = next(c for c in cases() if c.name == "nseq_42000")
    cs = small[:1500] + [huge] + small[1500:]
    got = cx.zstd_decompress([c.frame() for c in cs], [len(c.expected()) for c in cs])
    for c, g in zip(cs, got):
        check(c, g)
