"""A plain-Python ZSTD frame reader (RFC 8878) down to the sequences, independent of the device kernels and of the host walker
(victorialogs_b200/csrc/vl_zstd_walk.h), and a model of where k_execute (victorialogs_b200/csrc/vl_zstd.cuh) puts every byte.

`read_frame` parses the frame and block headers, the literals section header (and, for Huffman literals, the weights: direct or
FSE-compressed, which give maxbits), the sequences header, the FSE table descriptions (predefined, RLE, FSE, repeat) and the sequence
bitstream, with the repeat-offset history carried across blocks.  Huffman streams are not decoded.

`execute_geometry` repeats k_execute's grouping over the blocks `read_frame` returns: groups of 32 sequences restarting at every block,
the group output O, its end gend, every match's `dep`, which copy path runs, where each 4-byte chunk's source lies relative to gend and
to ring_lo, and - by replaying the order in which the kernel writes its ring - whether the ring still holds each source byte.  Those
last facts tell a test whether a case can tell a correct validity rule from a slightly wrong one."""

RAW, RLE, COMPRESSED = 0, 1, 2
L_RAW, L_RLE, L_COMPRESSED, L_TREELESS = 0, 1, 2, 3
RING = 4096
DIRTY = 0xFFFFFFFF

LL_BASE = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096,
           8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_DEFAULT = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_DEFAULT = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_DEFAULT = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5


class ReadError(Exception):
    pass


# ---- bit readers ----------------------------------------------------------------------------------------------------------------------
class Fwd:
    def __init__(self, b):
        self.b, self.pos = b, 0

    def read(self, n):
        lo = self.pos >> 3
        v = int.from_bytes(self.b[lo:lo + 8], "little") >> (self.pos & 7)
        self.pos += n
        return v & ((1 << n) - 1)


class Back:
    """A backward bitstream: starts below the end mark, reads towards the start; bits in front of the stream read as zero."""

    def __init__(self, b):
        if not b or not b[-1]:
            raise ReadError("backward bitstream without an end mark")
        self.b = b
        self.pos = len(b) * 8 - (8 - (b[-1].bit_length() - 1))

    def read(self, n):
        if n == 0:
            return 0
        self.pos -= n
        lo = max(self.pos, 0)
        v = int.from_bytes(self.b[lo >> 3:((self.pos + n + 7) >> 3)], "little") >> (lo & 7)
        v &= (1 << (self.pos + n - lo)) - 1
        return v << (lo - self.pos)


# ---- FSE ------------------------------------------------------------------------------------------------------------------------------
def read_counts(b, max_al, max_sym):
    """FSE table description (RFC 8878 4.1.1) -> (normalized counts, accuracy log, bytes used, facts)"""
    r = Fwd(b)
    al = 5 + r.read(4)
    if al > max_al:
        raise ReadError("accuracy log too large")
    remaining = (1 << al) + 1
    threshold = 1 << al
    nbits = al + 1
    norm, prev0 = [], False
    facts = dict(zero_repeat=0, zero_repeat_3=0, less_than_one=0)
    while remaining > 1:
        if prev0:
            while True:
                rep = r.read(2)
                norm += [0] * rep
                facts["zero_repeat"] += 1
                if rep != 3:
                    break
                facts["zero_repeat_3"] += 1
        mx = (2 * threshold - 1) - remaining
        low = r.read(nbits - 1)
        if low < mx:
            count = low
        else:
            r.pos -= nbits - 1
            count = r.read(nbits)
            if count >= threshold:
                count -= mx
        count -= 1
        remaining -= abs(count)
        norm.append(count)
        facts["less_than_one"] += count == -1
        prev0 = count == 0
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    if remaining != 1 or len(norm) > max_sym + 1:
        raise ReadError("bad FSE table description")
    return norm, al, (r.pos + 7) >> 3, facts


def build_table(norm, al):
    """normalized counts -> decoding table [(symbol, nbits, baseline)] (RFC 8878 4.1.1)"""
    size = 1 << al
    sym = [None] * size
    high = size - 1
    nxt = {}
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
            nxt[s] = 1
    step = (size >> 1) + (size >> 3) + 3
    pos = 0
    for s, c in enumerate(norm):
        if c <= 0:
            continue
        nxt[s] = c
        for _ in range(c):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    if pos != 0:
        raise ReadError("FSE spread did not return to 0")
    tab = []
    for i in range(size):
        s = sym[i]
        x = nxt[s]
        nxt[s] += 1
        nb = al - (x.bit_length() - 1)
        tab.append((s, nb, (x << nb) - size))
    return tab


PREDEF = {"ll": (build_table(LL_DEFAULT, 6), 6), "ml": (build_table(ML_DEFAULT, 6), 6), "of": (build_table(OF_DEFAULT, 5), 5)}


# ---- Huffman tree description: weights -> maxbits (RFC 8878 4.2.1) -----------------------------------------------------------------------
def read_huffman_weights(b):
    hb = b[0]
    if hb >= 128:
        nw = hb - 127
        desc = 1 + (nw + 1) // 2
        w = [(b[1 + i // 2] >> 4) if i % 2 == 0 else (b[1 + i // 2] & 15) for i in range(nw)]
        form = "direct"
    else:
        desc = 1 + hb
        norm, al, used, _ = read_counts(b[1:1 + hb], 6, 255)
        tab = build_table(norm, al)
        r = Back(b[1 + used:1 + hb])
        s1, s2 = r.read(al), r.read(al)
        w = []
        while True:                                      # two interleaved states until the stream runs dry
            e = tab[s1]; w.append(e[0]); s1 = e[2] + r.read(e[1])
            if r.pos < 0:
                w.append(tab[s2][0]); break
            e = tab[s2]; w.append(e[0]); s2 = e[2] + r.read(e[1])
            if r.pos < 0:
                w.append(tab[s1][0]); break
            if len(w) > 255:
                raise ReadError("too many Huffman weights")
        form = "fse"
    total = sum(1 << (x - 1) for x in w if x)
    if not total or max(w) > 11:
        raise ReadError("bad Huffman weights")
    maxbits = total.bit_length()
    left = (1 << maxbits) - total
    if left & (left - 1):
        raise ReadError("Huffman weights do not complete a tree")
    w.append(left.bit_length())
    return dict(form=form, desc=desc, maxbits=maxbits, nsyms=sum(1 for x in w if x))


# ---- frames -----------------------------------------------------------------------------------------------------------------------------
def le(b, n):
    return int.from_bytes(b[:n], "little")


def read_frame(f):
    """One ZSTD frame -> dict(fcs, window, blocks=[...]).  Every block: type, size, out_base, out_len; compressed blocks also lit_type,
    streams, lit_regen, lit_comp, huf (maxbits, form, nsyms or None), nseq, nseq_bytes, modes (ll, of, ml: 'predef' | 'rle' | 'fse' |
    'repeat'), repeat_back (how many blocks back each repeat-mode table was described), fse facts, seqs = [(ll, ml, ov, offset)],
    bits = [bits each sequence took], rep_known, ndirty / clean_from (as k_seq_decode counts them), rep_in (the history it starts with)."""
    if le(f, 4) != 0xFD2FB528:
        raise ReadError("not a ZSTD frame")
    fhd = f[4]
    fcs_flag, single, did_flag = fhd >> 6, (fhd >> 5) & 1, fhd & 3
    pos = 5
    window = None
    if not single:
        wd = f[pos]; pos += 1
        wlog = 10 + (wd >> 3)
        window = (1 << wlog) + ((1 << wlog) >> 3) * (wd & 7)
    pos += (0, 1, 2, 4)[did_flag]
    fsz = (1 if single else 0, 2, 4, 8)[fcs_flag]
    fcs = le(f[pos:], fsz) + (256 if fsz == 2 else 0)
    pos += fsz
    if single:
        window = fcs
    blocks = []
    out = 0
    rep = [1, 4, 8]
    huf_prev = None
    tables = {"ll": None, "of": None, "ml": None}         # last table of each kind: (table, al, index of the block that described it)
    seen_seq = False
    while True:
        h = le(f[pos:], 3); pos += 3
        last, btype, bsize = h & 1, (h >> 1) & 3, h >> 3
        B = dict(index=len(blocks), type=btype, size=bsize, out_base=out, src=pos)
        if btype == RAW:
            B["out_len"] = bsize; pos += bsize
        elif btype == RLE:
            B["out_len"] = bsize; B["byte"] = f[pos]; pos += 1
        elif btype == COMPRESSED:
            B["rep_known"] = not seen_seq
            rep = read_compressed(f[pos:pos + bsize], B, rep, tables, huf_prev)
            if B["lit_type"] == L_COMPRESSED:
                huf_prev = B["huf"]
            if B["nseq"]:
                seen_seq = True
            pos += bsize
        else:
            raise ReadError("reserved block type")
        out += B["out_len"]
        blocks.append(B)
        if last:
            break
    if fhd & 4:
        pos += 4
    if pos != len(f) or out != fcs:
        raise ReadError("frame size mismatch")
    return dict(fcs=fcs, window=window, blocks=blocks)


def read_compressed(b, B, rep, tables, huf_prev):
    lt, sf = b[0] & 3, (b[0] >> 2) & 3
    if lt in (L_RAW, L_RLE):
        hl = (1, 2, 1, 3)[sf]
        regen = {1: b[0] >> 3, 2: le(b, 2) >> 4, 3: le(b, 3) >> 4}[hl]
        comp, streams = (regen if lt == L_RAW else 1), 0
    else:
        hl = (3, 3, 4, 5)[sf]
        v = le(b, hl)
        bits = (10, 10, 14, 18)[sf]
        regen, comp = (v >> 4) & ((1 << bits) - 1), v >> (4 + bits)
        streams = 1 if sf == 0 else 4
    B.update(lit_type=lt, streams=streams, lit_regen=regen, lit_comp=comp, lit_hdr=hl, huf=None)
    if lt == L_COMPRESSED:
        B["huf"] = read_huffman_weights(b[hl:hl + comp])
    elif lt == L_TREELESS:
        if huf_prev is None:
            raise ReadError("treeless literals without a table")
        B["huf"] = dict(huf_prev, form="treeless")
    q = hl + comp
    n0 = b[q]
    if n0 < 128:
        nseq, nb = n0, 1
    elif n0 < 255:
        nseq, nb = ((n0 - 128) << 8) + b[q + 1], 2
    else:
        nseq, nb = b[q + 1] + (b[q + 2] << 8) + 0x7F00, 3
    q += nb
    B.update(nseq=nseq, nseq_bytes=nb, seqs=[], bits=[], modes=None, repeat_back={}, fse={}, rep_in=list(rep))
    if nseq == 0:
        B["out_len"] = regen
        B.update(ndirty=0, clean_from=0)
        if q != len(b):
            raise ReadError("bytes after an empty sequences section")
        return rep
    m = b[q]; q += 1
    names = {0: "predef", 1: "rle", 2: "fse", 3: "repeat"}
    B["modes"] = dict(ll=names[m >> 6], of=names[(m >> 4) & 3], ml=names[(m >> 2) & 3])
    cur = {}
    for kind, max_al, max_sym in (("ll", 9, 35), ("of", 8, 31), ("ml", 9, 52)):
        mode = B["modes"][kind]
        if mode == "predef":
            tab, al = PREDEF[kind]; cur[kind] = (tab, al, B["index"])
        elif mode == "rle":
            cur[kind] = ([(b[q], 0, 0)], 0, B["index"]); q += 1
        elif mode == "fse":
            norm, al, used, facts = read_counts(b[q:], max_al, max_sym)
            B["fse"][kind] = dict(facts, nsyms=sum(1 for c in norm if c), al=al)
            cur[kind] = (build_table(norm, al), al, B["index"]); q += used
        else:
            if tables[kind] is None:
                raise ReadError("repeat mode without a table")
            cur[kind] = tables[kind]
            B["repeat_back"][kind] = B["index"] - tables[kind][2]
        tables[kind] = cur[kind]
    r = Back(b[q:])
    (llt, llal, _), (oft, ofal, _), (mlt, mlal, _) = cur["ll"], cur["of"], cur["ml"]
    sl, so, sm = r.read(llal), r.read(ofal), r.read(mlal)
    r1, r2, r3 = rep
    d1, d2, d3 = (1, 4, 8) if B["rep_known"] else (DIRTY, DIRTY, DIRTY)    # k_seq_decode's view: unknown history is DIRTY
    ndirty = 0
    sum_ll = sum_ml = 0
    for i in range(nseq):
        p0 = r.pos
        oc, mc, lc = oft[so][0], mlt[sm][0], llt[sl][0]
        ov = (1 << oc) + r.read(oc)
        ml = ML_BASE[mc] + r.read(ML_BITS[mc])
        ll = LL_BASE[lc] + r.read(LL_BITS[lc])
        if i + 1 < nseq:
            e = llt[sl]; sl = e[2] + r.read(e[1])
            e = mlt[sm]; sm = e[2] + r.read(e[1])
            e = oft[so]; so = e[2] + r.read(e[1])
        (r1, r2, r3), off = update_rep(r1, r2, r3, ov, ll)
        (d1, d2, d3), _ = update_rep(d1, d2, d3, ov, ll)
        ndirty += DIRTY in (d1, d2, d3)
        B["seqs"].append((ll, ml, ov, off))
        B["bits"].append(p0 - r.pos)
        sum_ll += ll; sum_ml += ml
    if r.pos != 0:
        raise ReadError("sequence bitstream not consumed exactly (%d bits left)" % r.pos)
    if sum_ll > regen:
        raise ReadError("literal lengths exceed the literals")
    B.update(out_len=regen + sum_ml, ndirty=ndirty, clean_from=0 if B["rep_known"] else ndirty + 1)
    return [r1, r2, r3]


def update_rep(r1, r2, r3, ov, ll):
    """RFC 8878 3.1.1.5 (DIRTY stays DIRTY: r1 - 1 of an unknown offset is unknown)"""
    if ov > 3:
        o = ov - 3
        return (o, r1, r2), o
    idx = ov + (ll == 0)
    if idx == 1:
        return (r1, r2, r3), r1
    if idx == 2:
        return (r2, r1, r3), r2
    o = r3 if idx == 3 else (DIRTY if r1 == DIRTY else r1 - 1)
    return (o, r1, r2), o


def requested_blocks(blocks):
    """The reader's blocks as (sequences [(ll, ml, offset)], trailing literals) - the form a Case is written in."""
    out = []
    for B in blocks:
        if B["type"] != COMPRESSED:
            out.append(None)
            continue
        s = [(ll, ml, off) for ll, ml, _, off in B["seqs"]]
        out.append((s, B["lit_regen"] - sum(x[0] for x in s)))
    return out


# ---- k_execute's geometry ------------------------------------------------------------------------------------------------------------------
def _probe(keys, cnt, x):
    """number of leading entries of an ascending list that are < x, by k_execute's 5 probes (only the first cnt entries count)"""
    lo = 0
    for s in (16, 8, 4, 2, 1):
        i = lo + s - 1
        if i < cnt and keys[i & 31] < x:
            lo += s
    return lo


def execute_geometry(blocks, ring=RING):
    """k_execute over one frame's blocks (read_frame) -> dict(groups=[...], matches=[...]).

    groups: (block, first sequence, cnt, out_run, O, gend, ring_lo before, path 'ring' | 'byte', max dependency depth).
    matches: dict(block, seq, group, path, amd, sa, gend_minus_sa, dep, depth, ring_lo, straddle, chunks) where chunks lists, for
    the ring path, (b0, gend - source, source below ring_lo, the kernel's source: 'ring' | 'hbm' | 'bytes', the ring holds the source)."""
    R = ring
    owner = [-1] * R                         # frame position each ring slot holds (replayed in the kernel's store order)
    groups, matches = [], []
    ring_lo = 0

    def store(p):
        owner[p & (R - 1)] = p

    for bi, B in enumerate(blocks):
        base = B["out_base"]
        if B["type"] != COMPRESSED:
            for p in range(base, base + B["out_len"]):
                store(p)
            continue
        seqs = B["seqs"]
        out_run = base
        for g in range(0, len(seqs), 32):
            grp = seqs[g:g + 32]
            cnt = len(grp)
            O = sum(q[0] + q[1] for q in grp)
            gend = out_run + O
            amd, o_start, acc = [], [], 0
            for ll, ml, _, _ in grp:
                o_start.append(acc)
                amd.append(out_run + acc + ll)
                acc += ll + ml
            dep, depth = [], []
            for j, (ll, ml, _, off) in enumerate(grp):
                s = amd[j] - off
                e = s + min(ml, off)
                lo = _probe(amd, cnt, e)
                d = lo - 1 if lo > 0 and amd[lo - 1] + grp[lo - 1][1] > s else -1
                dep.append(d)
                depth.append(depth[d] + 1 if d >= 0 else 1)
            path = "ring" if O < R else "byte"
            groups.append(dict(block=bi, first=g, cnt=cnt, out_run=out_run, O=O, gend=gend, ring_lo=ring_lo, path=path, depth=max(depth)))
            for j, (ll, ml, _, off) in enumerate(grp):              # literal runs first
                for p in range(out_run + o_start[j], out_run + o_start[j] + ll):
                    store(p)
            info = []
            for j, (ll, ml, _, off) in enumerate(grp):
                sa = amd[j] - off
                info.append(dict(block=bi, seq=g + j, group=len(groups) - 1, path=path, amd=amd[j], sa=sa, gend_minus_sa=gend - sa,
                                 dep=dep[j], depth=depth[j], ring_lo=ring_lo, straddle=sa < ring_lo < sa + min(ml, off), chunks=[]))
            cur = 0
            while cur < cnt:                                         # runs of matches that are ready together (the ballot)
                n = 0
                while cur + n < cnt and dep[cur + n] < cur:
                    n += 1
                n = max(n, 1)
                if path == "ring":
                    chunks = [(j, b0) for j in range(cur, cur + n) for b0 in range(0, grp[j][1], 4)]
                    for c0 in range(0, len(chunks), 128):            # loads of up to 128 chunks, then their stores
                        step = chunks[c0:c0 + 128]
                        for j, b0 in step:
                            ml, off = grp[j][1], grp[j][3]
                            nb = min(4, ml - b0)
                            sa = amd[j] - off + b0
                            if off >= ml and sa >= ring_lo and gend - sa <= R:
                                how = "ring"
                            elif off >= ml and sa + nb <= out_run:
                                how = "hbm"
                            else:
                                how = "bytes"
                            held = all(owner[(sa + t) & (R - 1)] == sa + t for t in range(nb)) if off >= ml else None
                            info[j]["chunks"].append((b0, gend - sa, sa < ring_lo, how, held))
                        for j, b0 in step:
                            for t in range(min(4, grp[j][1] - b0)):
                                store(amd[j] + b0 + t)
                else:
                    for j in range(cur, cur + n):
                        for k in range(grp[j][1]):
                            store(amd[j] + k)
                cur += n
            if path == "byte":
                ring_lo = gend
            matches += info
            out_run = gend
        for p in range(out_run, base + B["out_len"]):             # trailing literals
            store(p)
    return dict(groups=groups, matches=matches)


def locate(blocks, geo, pos):
    """Where frame position `pos` comes from: block, group, sequence, literal or match, copy path, gend - sa."""
    for bi, B in enumerate(blocks):
        if not (B["out_base"] <= pos < B["out_base"] + B["out_len"]):
            continue
        if B["type"] != COMPRESSED:
            return "block %d (%s block), byte %d" % (bi, ("raw", "rle")[B["type"]], pos - B["out_base"])
        p = B["out_base"]
        for i, (ll, ml, ov, off) in enumerate(B["seqs"]):
            if pos < p + ll:
                return "block %d, group %d, sequence %d: literal byte %d of %d (literals %s)" % (bi, i // 32, i, pos - p, ll, ("raw", "rle", "huffman", "treeless")[B["lit_type"]])
            p += ll
            if pos < p + ml:
                m = next(x for x in geo["matches"] if x["block"] == bi and x["seq"] == i)
                g = geo["groups"][m["group"]]
                return ("block %d, group %d (O=%d, %s path, ring_lo=%d), sequence %d: match byte %d of %d, offset %d (ov %d), gend - sa = %d, "
                        "dep %d, depth %d, straddles ring_lo: %s" % (bi, i // 32, g["O"], g["path"], g["ring_lo"], i, pos - p, ml, off, ov,
                                                                     m["gend_minus_sa"], m["dep"], m["depth"], m["straddle"]))
            p += ml
        return "block %d: trailing literal byte %d" % (bi, pos - p)
    return "past the frame"
