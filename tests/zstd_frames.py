"""ZSTD frames built from chosen sequences, for the device decoder's tests (tests/test_zstd_sequences_cpu.py,
tests/test_gpu_zzzzzzzzzzzzzzz_zstd_sequences.py).

libzstd's ordinary compressor decides which sequences, table modes and block shapes a frame holds, so a suite that only compresses
corpora cannot say which of the decoder's edges it reaches.  Here the test chooses every literal length, match length, offset and block
boundary and hands them to libzstd's `ZSTD_compressSequences` with explicit block delimiters; libzstd still picks the literal and table
encodings, so the frames are what the writer library produces.  `lz_replay` is the plain reference of what such a frame regenerates.

A `Case` is a list of blocks, each a list of sequences `(literal length, match length, offset)` and a count of trailing literals, plus
the literal bytes of the whole frame.  The builders below make one family of cases each; every case names the features it exists for,
and tests/zstd_reader.py proves from the frame's bytes that it reached them."""
import ctypes as C
import random

P_LEVEL, P_WINDOW_LOG, P_MIN_MATCH, P_CONTENT_SIZE = 100, 101, 105, 200
P_LITERAL_MODE, P_BLOCK_DELIMITERS, P_VALIDATE, P_REPCODES = 1002, 1008, 1009, 1016
LIT_AUTO, LIT_HUFFMAN, LIT_RAW = 0, 1, 2
BLOCK_MAX = 128 << 10
RING = 4096                     # k_execute's per-warp ring (Z_RING)


class ZSeq(C.Structure):
    _fields_ = [("offset", C.c_uint), ("litLength", C.c_uint), ("matchLength", C.c_uint), ("rep", C.c_uint)]


_Z = None


def zlib():
    """libzstd.so.1 with the sequence API; 1.5.5 is the first release whose ZSTD_compressSequences resolves repeat codes on request."""
    global _Z
    if _Z is None:
        z = C.CDLL("libzstd.so.1")
        z.ZSTD_versionNumber.restype = C.c_uint
        v = z.ZSTD_versionNumber()
        if v < 10505:
            raise RuntimeError("libzstd.so.1 is %d.%d.%d; frames built from sequences need 1.5.5 or later" % (v // 10000, v // 100 % 100, v % 100))
        z.ZSTD_compressBound.restype = C.c_size_t
        z.ZSTD_compressBound.argtypes = [C.c_size_t]
        z.ZSTD_compress.restype = C.c_size_t
        z.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        z.ZSTD_decompress.restype = C.c_size_t
        z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        z.ZSTD_createCCtx.restype = C.c_void_p
        z.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        z.ZSTD_CCtx_setParameter.restype = C.c_size_t
        z.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
        z.ZSTD_compressSequences.restype = C.c_size_t
        z.ZSTD_compressSequences.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        z.ZSTD_isError.restype = C.c_uint
        z.ZSTD_isError.argtypes = [C.c_size_t]
        z.ZSTD_getErrorName.restype = C.c_char_p
        z.ZSTD_getErrorName.argtypes = [C.c_size_t]
        _Z = z
    return _Z


def lz_replay(lits, blocks):
    """The reference: literal runs and matches in order, byte by byte (a match may overlap its own output)."""
    out = bytearray()
    lp = 0
    for seqs, tail in blocks:
        for ll, ml, off in seqs:
            out += lits[lp:lp + ll]
            lp += ll
            assert 1 <= off <= len(out), (off, len(out))
            if off >= ml:
                out += out[len(out) - off:len(out) - off + ml]
            else:
                for _ in range(ml):
                    out.append(out[len(out) - off])
        out += lits[lp:lp + tail]
        lp += tail
    assert lp == len(lits)
    return bytes(out)


def zstd_decompress(frame, size):
    z = zlib()
    dst = C.create_string_buffer(max(size, 1))
    n = z.ZSTD_decompress(dst, size, frame, len(frame))
    assert not z.ZSTD_isError(n), z.ZSTD_getErrorName(n)
    assert n == size
    return dst.raw[:size]


def zstd_compress(data, level=1):
    z = zlib()
    cap = z.ZSTD_compressBound(len(data))
    dst = C.create_string_buffer(max(cap, 64))
    n = z.ZSTD_compress(dst, cap, data, len(data), level)
    assert not z.ZSTD_isError(n)
    return dst.raw[:n]


# ---- literal alphabets ------------------------------------------------------------------------------------------------------------------
def alpha_symbols(k, base=0x41):
    """k equally likely symbols (k <= 16: Huffman literals with small tables; 2..4 symbols: maxbits <= 2)."""
    return lambda rng, n: bytes(base + rng.randrange(k) for _ in range(n))


def alpha_random(rng, n):         # incompressible: raw literals, raw blocks
    return rng.randbytes(n)


def alpha_skewed(rng, n):         # all 256 symbols, geometric: FSE-compressed Huffman weights, maxbits 11
    return bytes(min(255, int(rng.expovariate(0.045))) for _ in range(n))


def alpha_weighted(k, seed):      # symbols 0..k-1 with uneven random weights: Huffman tables of many code lengths
    w = [random.Random(seed * 1000 + i).randrange(1, 60) for i in range(k)]
    return lambda rng, n: bytes(rng.choices(range(k), w, k=n))


def alpha_balanced(k):
    """symbols 0..k-1 (k a power of two) equally often in every run of a multiple of k bytes: every code has the same length, the
    weight list is one repeated value, which libzstd does not FSE-compress (direct weights, k - 1 of them)"""
    def gen(rng, n):
        assert n % k == 0
        out = bytearray()
        for _ in range(n // k):
            perm = list(range(k))
            rng.shuffle(perm)
            out += bytes(perm)
        return bytes(out)
    return gen


def alpha_const(byte):            # one symbol: RLE literals
    return lambda rng, n: bytes([byte]) * n


class Case:
    """A frame described by its blocks.  `seq` / `tail` / `end_block` append to the open block; the builder tracks the output position
    and the repeat-offset history exactly as a decoder would see it (RFC 8878 3.1.1.5, with libzstd's choice of repeat codes), so a family
    can ask for a repeat code by naming the offset the history holds."""

    def __init__(self, name, seed, targets=(), level=3, lit_mode=LIT_AUTO, window_log=None, alpha=None):
        self.name, self.targets, self.level, self.lit_mode, self.window_log = name, tuple(targets), level, lit_mode, window_log
        self.rng = random.Random(seed)
        self.alpha = alpha or alpha_symbols(16)
        self.blocks = []
        self.lits = bytearray()
        self.pos = 0
        self.rep = [1, 4, 8]
        self._seqs, self._tail, self._size = [], 0, 0
        self._frame = None

    # -- building --
    def _lit(self, n, alpha):
        self.lits += (alpha or self.alpha)(self.rng, n)

    def seq(self, ll, ml, off, alpha=None):
        assert self._tail == 0, "trailing literals end a block"
        assert ml >= 3 and off >= 1
        self._lit(ll, alpha)
        self.pos += ll
        assert off <= self.pos, (self.name, off, self.pos)
        self.pos += ml
        self._size += ll + ml
        self._seqs.append((ll, ml, off))
        r1, r2, r3 = self.rep                   # libzstd's repeat-code choice (ZSTD_finalizeOffBase), then the decoder's history update
        if ll and off == r1:
            pass                                # repeat code 1: the history stays
        elif off == r2:
            self.rep = [r2, r1, r3]             # r2 moves to the front
        else:
            self.rep = [off, r1, r2]            # r3, r1 - 1 or a new offset: pushed in front
        return self

    def tail(self, n, alpha=None):
        self._lit(n, alpha)
        self.pos += n
        self._size += n
        self._tail += n
        return self

    def end_block(self):
        assert 0 < self._size <= BLOCK_MAX, (self.name, self._size)
        self.blocks.append((self._seqs, self._tail))
        self._seqs, self._tail, self._size = [], 0, 0
        return self

    def block_bytes(self):
        return self._size

    def raw_block(self, n):
        """A block of incompressible literals and no sequences: libzstd stores it raw, and the history stays what it was."""
        assert not self._seqs and not self._tail
        return self.tail(n, alpha_random).end_block()

    def rle_block(self, n, byte=0x5A):
        """One literal and a match of offset 1: libzstd stores the block as an RLE block (it does so for short sequence lists only)."""
        assert not self._seqs and not self._tail
        hist = list(self.rep)
        self.seq(1, n - 1, 1, alpha_const(byte)).end_block()
        self.rep = hist                          # a block stored as RLE does not touch the history
        return self

    # -- the frame --
    def expected(self):
        assert not self._seqs and not self._tail, "open block"
        return lz_replay(bytes(self.lits), self.blocks)

    def frame(self):
        if self._frame is None:
            self._frame = compress_sequences(self.blocks, self.expected(), self.level, self.lit_mode, self.window_log)
        return self._frame


def compress_sequences(blocks, data, level=3, lit_mode=LIT_AUTO, window_log=None):
    z = zlib()
    arr = []
    for seqs, tail in blocks:
        arr += [(off, ll, ml) for ll, ml, off in seqs]
        arr.append((0, tail, 0))                # block delimiter: the block's trailing literals
    sq = (ZSeq * len(arr))(*[ZSeq(o, l, m, 0) for o, l, m in arr])
    cctx = z.ZSTD_createCCtx()
    try:
        params = [(P_LEVEL, level), (P_CONTENT_SIZE, 1), (P_MIN_MATCH, 3), (P_BLOCK_DELIMITERS, 1), (P_VALIDATE, 1), (P_REPCODES, 1),
                  (P_LITERAL_MODE, lit_mode)]
        if window_log:
            params.append((P_WINDOW_LOG, window_log))
        for k, v in params:
            r = z.ZSTD_CCtx_setParameter(cctx, k, v)
            assert not z.ZSTD_isError(r), (k, z.ZSTD_getErrorName(r))
        cap = z.ZSTD_compressBound(len(data)) + 1024
        dst = C.create_string_buffer(cap)
        n = z.ZSTD_compressSequences(cctx, dst, cap, sq, len(arr), data, len(data))
        assert not z.ZSTD_isError(n), z.ZSTD_getErrorName(n)
        return dst.raw[:n]
    finally:
        z.ZSTD_freeCCtx(cctx)


# ---- placement: compressed-byte phase mod 256, output phase mod 16 ----------------------------------------------------------------------
# vlscan_zstd_decompress packs the frames back to back behind 512 bytes of headroom and writes frame i at 16 + dst_offsets[i], so the
# bytes in front of a frame alone decide where its compressed bytes (sequence-ring origin, Huffman word reads) and its output (flush
# split, ring word reads) fall.  Fillers: k empty frames (9 bytes, no output) and one frame of n random bytes (stored raw).
_FILL = {}


def _filler(n):
    if n not in _FILL:
        _FILL[n] = zstd_compress(random.Random(n).randbytes(n), 1)
    return _FILL[n]


def fillers(comp_at, out_at, comp_phase, out_phase):
    """Frames that move a frame from (comp_at, out_at) bytes behind the start to the given phases; -> list of (frame, size)."""
    e = len(_filler(0))
    for m in range(16):
        n = (out_phase - out_at) % 16 + 16 * m
        c = comp_at + (len(_filler(n)) if n else 0)
        for k in range(256):
            if (c + k * e) % 256 == comp_phase % 256:
                return [(_filler(0), 0)] * k + ([(_filler(n), n)] if n else [])
    raise AssertionError("no filler reaches phase %d/%d" % (comp_phase, out_phase))


def placed(items):
    """items: (frame, size, comp_phase or None, out_phase or None) -> frames, sizes, index of every item in them."""
    frames, sizes, where = [], [], []
    c = o = 0
    for fr, sz, cp, op in items:
        if cp is not None or op is not None:
            for f, s in fillers(c, o, c if cp is None else cp, o if op is None else op):
                frames.append(f); sizes.append(s); c += len(f); o += s
        where.append(len(frames))
        frames.append(fr); sizes.append(sz); c += len(fr); o += sz
    return frames, sizes, where


# ---- the families -------------------------------------------------------------------------------------------------------------------------
def _prefix(c, n=9000):
    """A first block that gives later matches something to reach back into (offsets up to n)."""
    c.seq(64, 8, 7)
    while c.pos < n:
        c.seq(c.rng.randrange(1, 40), c.rng.randrange(3, 30), c.rng.randrange(1, min(c.pos, 3000)))
    return c.end_block()


class Grouper:
    """Lays out groups of exactly 32 sequences (k_execute's unit; groups restart at every block), padding a group with short matches
    and cutting blocks between groups."""

    def __init__(self, c, block_limit=60000):
        self.c, self.limit = c, block_limit

    def group(self, seqs, pad=(0, 4, 16), alpha=None):
        c = self.c
        need = sum(ll + ml for ll, ml, _ in seqs) + pad[0] * 32 + pad[1] * 32
        if c.block_bytes() and c.block_bytes() + need > self.limit:
            c.end_block()
        for ll, ml, off in seqs:
            c.seq(ll, ml, off, alpha)
        for _ in range(32 - len(seqs)):
            c.seq(pad[0], pad[1], pad[2], alpha)

    def close(self):
        if self.c.block_bytes():
            self.c.end_block()


OVERLAP_OFFSETS = list(range(1, 65)) + [127, 128, 255, 256, 4095, 4096, 4097]
OVERLAP_LENGTHS = [3, 4, 5, 7, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000]


def case_overlap(ring_path):
    """Every offset x match length, on the ring path (group output < 4096) or on the byte path (a 4096-byte literal run in the group)."""
    name = "overlap_ring" if ring_path else "overlap_byte"
    c = Case(name, 101 if ring_path else 102, targets=("overlap_all_combos_ring_path" if ring_path else "overlap_all_combos_byte_path",))
    _prefix(c, 9000)
    G = Grouper(c, 100000)
    combos = [(off, ml) for off in OVERLAP_OFFSETS for ml in OVERLAP_LENGTHS]
    c.rng.shuffle(combos)
    i = 0
    while i < len(combos):
        grp, o = [], 0
        if not ring_path:
            grp.append((4096, 3, 4097)); o = 4099
        while i < len(combos) and len(grp) < 30:
            off, ml = combos[i]
            ll = c.rng.choice([0, 1, 2, 3, 5])
            if ring_path and o + ll + ml + 200 >= RING:
                break
            grp.append((ll, ml, off)); o += ll + ml; i += 1
        G.group(grp)
    G.close()
    return c


def case_ring_edges():
    """Groups whose output is 4095 / 4096 / 4097 bytes, and sources 4093..4101 bytes behind the group's end, each next to a last
    sequence whose match is 3 bytes long, so the 4 bytes in front of the group's end are a literal and a source just out of the ring's
    reach shares its slot with a byte the group has already written."""
    c = Case("ring_edges", 103, targets=("group_O_4095", "group_O_4096", "group_O_4097", "src_at_gend_minus_4095",
                                                "src_at_gend_minus_4096", "src_at_gend_minus_4097", "ring_src_stale_at_4097_4100"))
    _prefix(c, 12000)
    G = Grouper(c, 60000)
    for O in (4090, 4094, 4095, 4096, 4097, 4098, 4200):
        # 31 sequences of 4 + 16 bytes and one that makes the output O
        rest = O - 31 * 20
        G.group([(4, 16, 1000 + 7 * k) for k in range(31)] + [(rest - 8, 8, 5000)])
    for X in range(4092, 4102):
        for ml_a in (3, 4, 5, 8, 9, 64):
            for ll_b in (1, 2, 4):
                # A reads X bytes behind the group's end; B = (ll_b literals, 3-byte match) closes the group
                fill = [(2, 12, 900 + k) for k in range(30)]
                tail_len = ml_a + ll_b + 3
                off_a = X - tail_len
                G.group(fill + [(3, ml_a, off_a), (ll_b, 3, 20)], pad=(0, 4, 16))
    G.close()
    return c


def case_ring_lo():
    """Small groups right after an oversized group (byte path, ring_lo moves to its end): sources below ring_lo whose ring slot the
    oversized group overwrote (a match written after a literal 4096 bytes further on), at ring_lo, and straddling it."""
    c = Case("ring_lo", 104, targets=("straddle_ring_lo", "src_at_ring_lo", "ring_src_stale_below_ring_lo"))
    _prefix(c, 9000)
    G = Grouper(c, 60000)
    for trial in range(12):
        big_ll = 4300 + 97 * trial
        # oversized group: an early match (300 bytes), then a literal run that reaches 4096 bytes past it
        G.group([(10, 300, 40 + trial), (big_ll, 3, 17)] + [(1, 4, 9)] * 30)
        # the next group starts at ring_lo = the oversized group's end; sources reach back into the literal run
        d = 30 * 5                                  # bytes the first group's padding wrote after the literal run
        reach = [d + 3 + 40, d + 3 + 200, d + 3 + big_ll - 4096 + 150, 1200 + 13 * trial]
        seqs = []
        o = 0
        for k, back in enumerate(reach):
            seqs.append((2, 9, back + o + 2)); o += 11
        seqs.append((0, 24, o + 8))                  # straddles ring_lo: starts 8 bytes below it
        o += 24
        seqs.append((1, 5, o + 1))                   # exactly at ring_lo
        o += 6
        seqs.append((0, 40, o + 20))                 # straddles with a longer source
        G.group(seqs)
    G.close()
    return c


def case_dependencies():
    """A 32-deep chain, alternating dependent / independent matches, a dependency 31 slots back, sources over two destinations, and
    more than 128 chunks in one run."""
    c = Case("dependencies", 105, targets=("dep_chain_32", "dep_adjacent_ring", "dep_31_back", "independent_run_over_128_chunks",
                                                 "literal_chunks_over_128"))
    _prefix(c, 9000)
    G = Grouper(c, 60000)
    for m in (3, 4, 5, 8, 13, 40):
        G.group([(0, m, m)] * 32)                                        # each match reads the previous one's destination
        G.group([(1, m, m + 1)] * 32)
    G.group([(2, 6, 8) if k % 2 else (2, 6, 3000 + k) for k in range(32)])   # alternating
    s = [(3, 7, 2500 + k) for k in range(31)]
    G.group(s + [(0, 7, sum(a + b for a, b, _ in s[1:]) + 7)])           # the last match reads the first one's destination
    G.group([(2, 10, 6), (0, 10, 14), (0, 12, 16), (1, 20, 27)] * 8)     # sources over two earlier destinations
    G.group([(1, 20, 3000 + 5 * k) for k in range(32)])                  # 32 x 5 = 160 chunks in one independent run
    G.group([(20, 20, 3000 + 5 * k) for k in range(32)])                 # and 160 literal chunks
    G.close()
    return c


def case_literal_shapes():
    """Groups without literals, literal runs of 0..9 bytes at every alignment, trailing literals of 0, 1, 4095, 4096, 4097 bytes read
    by the next block's matches."""
    c = Case("literal_shapes", 106, targets=("group_without_literals", "literal_runs_0_9_every_alignment", "trailing_0_then_read",
                                                   "trailing_1_then_read", "trailing_4095_then_read", "trailing_4096_then_read",
                                                   "trailing_4097_then_read"))
    _prefix(c, 9000)
    G = Grouper(c, 60000)
    G.group([(0, 5 + k % 7, 30 + k) for k in range(32)])
    for a in range(16):
        G.group([((a + k) % 10, 3 + (a * k) % 6, 11 + k) for k in range(32)])
    G.close()
    for t in (0, 1, 4095, 4096, 4097):
        c.seq(5, 20, 100).seq(3, 40, 2000)
        if t:
            c.tail(t)
        c.end_block()
        c.seq(0, 16, max(1, t // 2)).seq(2, 30, t + 40).seq(1, 8, t + 60).end_block()
    return c


def case_literal_kinds():
    """Raw, RLE, Huffman 1-stream and 4-stream and treeless literals, each read by matches."""
    c = Case("literal_kinds", 107, targets=("lit_raw_read_by_matches", "lit_rle_read_by_matches",
                                                  "lit_huffman_read_by_matches", "lit_treeless_read_by_matches", "huf_1_stream",
                                                  "huf_4_stream"), level=19)
    _prefix(c, 9000)
    for i, n in enumerate((100, 200, 1000, 3000)):           # Huffman over a new alphabet each time, 1 stream below 256 literals
        for k in range(8):
            c.seq(n // 8, 20, 50 + k, alpha_symbols(8 + i, base=0x61 + 8 * i))
        c.seq(0, 30, n // 2).end_block()
    for k in range(16):                                      # raw literals
        c.seq(60, 12, 200 + k, alpha_random)
    c.seq(0, 40, 300).end_block()
    for k in range(16):                                      # RLE literals
        c.seq(40, 10, 100 + k, alpha_const(0x33))
    c.seq(0, 40, 300).end_block()
    for b in range(3):                                       # the same alphabet again: treeless literals
        for k in range(20):
            c.seq(60, 10, 90 + k, alpha_symbols(16))
        c.seq(2, 50, 700).end_block()
    return c


def case_blocks_between():
    """Raw and RLE blocks between compressed blocks, read by near (< 4096) and far matches; 1..65 sequences per block; a literal-only
    block between blocks with sequences."""
    c = Case("blocks_between", 108, targets=("raw_block", "rle_block", "literal_only_block", "src_in_raw_or_rle_block_near",
                                                    "src_in_raw_or_rle_block_far", "nseq_1", "nseq_31", "nseq_32", "nseq_33",
                                                    "nseq_63", "nseq_64", "nseq_65"))
    _prefix(c, 9000)
    for n in (1, 31, 32, 33, 63, 64, 65):
        c.raw_block(700 + n)
        for k in range(n):
            c.seq(1 + k % 3, 60 if n == 1 else 12 + k % 11, 10 + (k * 37) % 600 if k % 2 else 6000 + k)
        c.end_block()
        c.rle_block(500 + n)
        c.seq(0, 30, 100).seq(3, 30, 480).seq(2, 20, 7000).end_block()
        c.tail(300 + n, alpha_symbols(8)).end_block()         # literal-only block
        c.seq(1, 9, 350).seq(0, 12, 2000).end_block()
    return c


def case_repeat_offsets():
    """Every repeat code x (ll == 0, ll > 0), history permutations, dirty prefixes of 0, 1, 2, 3 and 10 sequences at a block start,
    blocks made only of repeat codes (alone and in chains of two and three), with raw, RLE and literal-only blocks in between."""
    c = Case("repeat_offsets", 109, targets=(
        "rep_ov1_ll", "rep_ov2_ll", "rep_ov3_ll", "rep_ov1_ll0", "rep_ov2_ll0", "rep_ov3_ll0", "rep_ov1_ll0_dirty", "rep_ov2_ll0_dirty",
        "rep_ov3_ll0_dirty", "rep_ov1_ll_dirty", "rep_ov2_ll_dirty", "rep_ov3_ll_dirty", "inherited_prefix_0", "inherited_prefix_1",
        "inherited_prefix_2", "inherited_prefix_3", "inherited_prefix_10", "all_repeat_block", "all_repeat_chain_2", "all_repeat_chain_3",
        "all_repeat_after_raw", "all_repeat_after_rle", "all_repeat_after_lits", "never_clean_block", "after_never_clean_uses_history"))
    _prefix(c, 9000)

    def set_history(a, b, d):
        c.seq(2, 6, d).seq(2, 6, b).seq(2, 6, a)              # history = (a, b, d)

    def rep_code(k, ll):
        """the offset that makes a repeat code: k = 1, 2, 3 with ll > 0 -> r1, r2, r3; with ll == 0 -> r2, r3, r1 - 1"""
        r1, r2, r3 = c.rep
        return (r1, r2, r3)[k - 1] if ll else (r2, r3, r1 - 1)[k - 1]

    # inside a block (history known)
    set_history(300, 500, 700)
    for k in (1, 2, 3):
        for ll in (0, 3):
            c.seq(ll, 7, rep_code(k, ll))
    c.end_block()
    # at block starts: dirty prefixes
    for prefix_len in (0, 1, 2, 3, 10):
        for ll0 in (0, 1):
            set_history(310 + prefix_len, 520, 730 + ll0)
            c.end_block()
            for j in range(prefix_len):
                ll = 0 if (j + ll0) % 2 == 0 else 2
                c.seq(ll, 5, rep_code(1 + (j % 3), ll))
            c.seq(1, 6, 1111 + prefix_len).seq(0, 6, 222).seq(3, 6, 333).seq(0, 5, c.rep[1]).end_block()
    # blocks made only of repeat codes, chains of 1..3, things in between
    for between in (None, "raw", "rle", "lits"):
        for chain in (1, 2, 3):
            set_history(600 + chain, 800, 990)
            c.end_block()
            for b in range(chain):
                if between == "raw":
                    c.raw_block(300)
                elif between == "rle":
                    c.rle_block(400)
                elif between == "lits":
                    c.tail(200, alpha_symbols(4)).end_block()
                for j in range(6):
                    ll = (j + b) % 2
                    c.seq(ll * 3, 4 + j, rep_code(1 + (j + b) % 3, ll * 3))
                c.end_block()
            c.seq(0, 9, rep_code(1, 0)).seq(2, 9, rep_code(3, 2)).seq(0, 9, rep_code(3, 0)).seq(1, 9, 4321).end_block()
    return c


def case_nseq(n):
    """One block of n sequences (3-byte matches): Number_of_Sequences in its 1-, 2- and 3-byte forms."""
    t = ("nseq_%d" % n,) if n < 42000 else ("nseq_ge_42000",)
    t += ("nseq_2byte",) if 128 <= n < 0x7F00 else ("nseq_3byte",) if n >= 0x7F00 else ()
    c = Case("nseq_%d" % n, 110 + n, targets=t, alpha=alpha_symbols(4))
    c.seq(16, 3, 7).end_block() if n > 1000 else c.tail(64).end_block()
    if n == 1:
        return c.seq(0, 200, 9).end_block()
    rng = c.rng
    for k in range(n):
        c.seq(0 if n > 30000 else k % 2, 3, rng.choice((1, 2, 3, 5, 9, 12)))
    return c.end_block()


def case_table_modes():
    """LL / OF / ML tables in predefined, RLE and FSE mode, with raw and literal-only blocks between the FSE blocks; sparse code
    sets (zero-repeat flags)."""
    c = Case("table_modes", 111, targets=("ll_mode_predef", "of_mode_predef", "ml_mode_predef", "ll_mode_rle", "of_mode_rle",
                                          "ml_mode_rle", "ll_mode_fse", "of_mode_fse", "ml_mode_fse", "fse_zero_repeat_flags"))
    _prefix(c, 9000)
    rng = c.rng
    # few sequences: predefined tables
    c.seq(1, 40, 5).seq(2, 50, 17).end_block()
    # one code per field: RLE tables
    for k in range(60):
        c.seq(5, 6, 61 + k)                                  # offset code 6 for all of them, none a repeat
    c.end_block()
    # FSE tables with fresh statistics each time, with blocks without sequences in between
    def fse_block(sparse=False):
        for k in range(150 if sparse else 400):
            if sparse:
                c.seq(rng.choice((0, 40)), rng.choice((3, 600)), rng.choice((61, 4000)))
            else:
                c.seq(rng.randrange(0, 14), rng.randrange(3, 40), rng.randrange(1, 2000))
        c.end_block()
    fse_block()
    fse_block()
    c.tail(300, alpha_symbols(6)).end_block()
    fse_block()
    c.raw_block(500)
    c.tail(300, alpha_symbols(6)).end_block()
    fse_block()
    fse_block(sparse=True)
    fse_block(sparse=True)
    return c


def case_repeat_tables():
    """Repeat-mode tables that point two or more blocks back through blocks without sequences: the same 20 sequences in a block that
    describes its tables and again after literal-only, raw and RLE blocks (one and two of them in between)."""
    c = Case("repeat_tables", 114, targets=tuple("%s_mode_repeat_over_%s" % (k, b) for k in ("ll", "of", "ml") for b in ("raw", "rle", "lits")),
             level=19)
    _prefix(c, 9000)

    def same_block(same):
        for ll, ml, off in same:
            c.seq(ll, ml, off)
        c.end_block()

    for p, between in enumerate(("lits", "raw", "rle", "lits2", "raw2", "rle2")):
        # 300 sequences over a few codes per field, different for every pair: FSE tables, then the same statistics repeated
        r = c.rng
        lls, mls, offs = r.sample(range(0, 40), 4), r.sample(range(3, 60), 4), r.sample(range(16, 4000), 6)
        same = [(r.choice(lls), r.choice(mls), r.choice(offs)) for _ in range(300)]
        same_block(same)
        for _ in range(2 if between.endswith("2") else 1):
            if between.startswith("lits"):
                c.tail(300, alpha_symbols(6)).end_block()
            elif between.startswith("raw"):
                c.raw_block(500)
            else:
                c.rle_block(400)
        same_block(same)
    return c


def case_large_codes():
    """The largest codes: literal runs >= 65536 (LL 35), matches >= 65539 (ML 52), offsets >= 2^20 (OF 20, windowLog 21), and
    consecutive sequences with wide fields (long literal runs, long matches, far offsets)."""
    c = Case("large_codes", 112, targets=("ll_code_35", "ml_code_52", "of_code_20", "wide_sequences_back_to_back"), window_log=21)
    c.tail(120000, alpha_symbols(16)).end_block()
    c.seq(70000, 50000, 69000).end_block()                     # LL 35
    c.seq(10, 70000, 30000).seq(5, 40000, 65000).end_block()  # ML 52
    while c.pos < (1 << 20) + 200000:
        c.tail(100000, alpha_symbols(16)).end_block()
    for b in range(6):                                        # far offsets, wide literal and match fields, several per block
        for k in range(8):
            c.seq(4100 + 513 * k, 5000 + 997 * k, (1 << 20) + 20011 * k + 1000 * b)
        c.end_block()
    for b in range(4):                                        # sequences of ~48 bits of extra fields each, back to back
        for k in range(4):
            c.seq((8192, 16384)[k % 2] + 97 * b + 7 * k, (16387, 8195)[k % 2] + 89 * b + 5 * k, ((1 << 20) + 12345 * b + 999 * k, (1 << 19) + 777 * k)[k // 2])
        c.end_block()
    return c


def case_huffman():
    """Literal alphabets of 2, 3 and 4 symbols (tables of fewer than 8 entries), 64 balanced symbols (63 direct weights), 10..128 symbols of uneven weight and 256 skewed symbols (FSE weights, maxbits up to 11), 4-stream sizes of every residue
    mod 4, and treeless literals across a raw block."""
    c = Case("huffman", 113, targets=("huf_maxbits_le2", "huf_maxbits_11", "huf_weights_direct", "huf_weights_direct_ge_64",
                                      "huf_weights_fse", "huf_4stream_regen_mod4_0", "huf_4stream_regen_mod4_1", "huf_4stream_regen_mod4_2",
                                      "huf_4stream_regen_mod4_3", "treeless_after_raw_block"), level=19, lit_mode=LIT_HUFFMAN)
    c.tail(64, alpha_symbols(16)).end_block()
    for k in (2, 3, 4):
        for base in (0, 0x70):
            for n in (300, 1001):
                for j in range(10):
                    c.seq(n // 10, 6, 30 + j, alpha_symbols(k, base))
                c.tail(n % 10, alpha_symbols(k, base)).end_block()
    for k in (10, 30, 60, 100, 128):
        for j in range(30):
            c.seq(40, 6, 30 + j, alpha_weighted(k, k))
        c.end_block()
    for k in (40, 100, 128):
        for j in range(10):
            c.seq(300, 6, 30 + j, alpha_symbols(k, base=0))
        c.end_block()
    for k in (64,):
        for j in range(10):
            c.seq(2 * k, 6, 30 + j, alpha_balanced(k))
        c.end_block()
    for n in (4000, 4001, 4002, 4003, 20000):
        for j in range(10):
            c.seq(n // 10, 8, 100 + j, alpha_skewed)
        c.tail(n % 10, alpha_skewed).end_block()
    for r in range(4):                                       # 4 streams: literal counts = 0..3 mod 4
        for j in range(8):
            c.seq(100, 10, 50 + j, alpha_symbols(20))
        c.tail(r + 4, alpha_symbols(20)).end_block()
    for j in range(8):                                       # a table, a raw block, then the same alphabet again
        c.seq(100, 10, 50 + j, alpha_symbols(12))
    c.end_block()
    c.raw_block(400)
    for b in range(2):
        for j in range(8):
            c.seq(100, 10, 50 + j, alpha_symbols(12))
        c.end_block()
    return c


def all_cases():
    return [case_overlap(True), case_overlap(False), case_ring_edges(), case_ring_lo(), case_dependencies(), case_literal_shapes(),
            case_literal_kinds(), case_blocks_between(), case_repeat_offsets(), case_table_modes(), case_repeat_tables(), case_large_codes(), case_huffman()] + \
        [case_nseq(n) for n in (1, 127, 128, 0x7EFF, 0x7F00, 0x7F01, 42000)]


def small_frames(n, seed=7):
    """Many small crafted frames (a few dozen sequences each, every literal kind) for one launch next to one huge block."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        c = Case("small_%d" % i, seed * 100003 + i, alpha=(alpha_symbols(rng.choice((2, 4, 16, 60))), alpha_random, alpha_const(7))[i % 3])
        c.tail(rng.randrange(8, 200)).end_block() if i % 4 else c.seq(20, 5, 3).end_block()
        for b in range(rng.randrange(1, 3)):
            for k in range(rng.randrange(1, 70)):
                c.seq(rng.randrange(0, 12), rng.randrange(3, 40), rng.randrange(1, min(c.pos, 3000) + 1))
            c.end_block()
        out.append(c)
    return out
