// ZSTD frame decoding on the device (RFC 8878) for values blocks staged in their on-disk form.
//
// The reference decompresses every bytes block of a values block with libzstd on a CPU core before it can look at a row
// (unmarshalBytesBlock, lib/logstorage/encoding.go:372-426 -> encoding.DecompressZSTD, lib/encoding/compress.go:24-32).
// Here the compressed frames are copied to HBM as they are and decoded there, so the host->device link carries the compressed
// bytes only.  The format leaves three kinds of parallelism, and each phase below is shaped after one of them:
//
//   k_huf_build     one warp  per Huffman tree description   (weights -> 2^maxbits-entry decoding table)
//   k_huf_decode    one LANE  per Huffman stream             (4 independent backward bitstreams per block; tables staged in shared memory)
//   k_fse_build     one lane  per compressed block           (LL / OF / ML table descriptions -> decoding tables)
//   k_seq_decode    one lane  per compressed block           (the FSE-interleaved sequence bitstream is strictly serial inside a block;
//                                                             tables staged in shared memory, repeat offsets resolved on the fly)
//   k_seq_resolve   one lane  per frame                      (block output bases; replays the few sequences whose repeat offsets depended
//                                                             on the previous block)
//   k_execute       one warp  per frame                      (literal runs as one flat copy, matches in dependency order)
//
// Tables that a later block may reuse (Treeless literals, Repeat_Mode) live in per-block slots in HBM; the host resolves which
// slot a block reads while it walks the block headers (it needs those for the layout anyway).  DESIGN.md §3.5 has the full picture.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vl_zstd_types.h"

namespace vl {
namespace zs {

struct ZView {
    const uint8_t* src;        // compressed staging buffer
    uint8_t* arena;
    const ZFrame* frames; const ZBlock* blocks; ZBlockState* bstate;
    uint16_t* huf_tab; uint8_t* fse_tab; ZSlotState* huf_state; ZSlotState* fse_state;
    const uint8_t* predef;     // one slot: predefined LL / ML / OF tables (accuracy 6 / 6 / 5)
    uint8_t* lits; uint4* seqs;
    unsigned int* frame_err;   // per frame: first error code
    unsigned long long* status;   // [0] = max error code, [1] = a failing frame + 1
};

static __device__ __forceinline__ void zfail(const ZView& V, uint32_t frame, unsigned code) {
    atomicCAS(&V.frame_err[frame], 0u, code);
    atomicMax(&V.status[0], (unsigned long long)code);
    atomicMax(&V.status[1], (unsigned long long)frame + 1);
}

// ---- bit readers ------------------------------------------------------------------------------------------------------------------
static __device__ __forceinline__ uint64_t ldu64(const uint8_t* p) {   // little-endian 8 bytes at any address (two aligned loads)
    uintptr_t a = (uintptr_t)p & ~(uintptr_t)7; uint32_t sh = (uint32_t)((uintptr_t)p & 7) * 8;
    uint64_t lo = *(const uint64_t*)a;
    if (!sh) return lo;
    uint64_t hi = *(const uint64_t*)(a + 8);
    return (lo >> sh) | (hi << (64 - sh));
}
// The 64 bits just below bit `pos` of a backward bitstream, top aligned (bit pos-1 -> bit 63); bits before the start read as zero.
static __device__ __forceinline__ uint64_t peek64(const uint8_t* base, int64_t pos) {
    if (pos >= 64) { int junk = (int)((-pos) & 7); return ldu64(base + ((pos + 7) >> 3) - 8) << junk; }
    if (pos <= 0) return 0;
    uint64_t v = 0; int nb = (int)((pos + 7) >> 3);
    for (int i = 0; i < nb; i++) v |= (uint64_t)base[i] << (8 * i);
    return v << (64 - pos);
}
struct BackReader {
    const uint8_t* base; int64_t pos; uint64_t w; int avail;
    __device__ __forceinline__ bool init(const uint8_t* p, uint32_t len) {   // false: empty stream or missing end mark
        base = p; w = 0; avail = 0; pos = 0;
        if (!len) return false;
        uint32_t last = p[len - 1];
        if (!last) return false;
        pos = (int64_t)len * 8 - (int64_t)(__clz(last) - 23);   // padding = 8 - highest set bit index; __clz counts from bit 31
        return true;
    }
    __device__ __forceinline__ uint32_t read(int n) {   // n <= 32
        if (n == 0) return 0;
        if (n > avail) { w = peek64(base, pos); avail = 57; }
        uint32_t v = (uint32_t)(w >> (64 - n)); w <<= n; avail -= n; pos -= n;
        return v;
    }
};
struct FwdReader {
    const uint8_t* base; uint32_t len; uint32_t pos;
    __device__ __forceinline__ uint32_t read(int n) { uint32_t v = (uint32_t)(ldu64(base + (pos >> 3)) >> (pos & 7)) & ((1u << n) - 1); pos += n; return v; }
    __device__ __forceinline__ bool overrun() const { return ((pos + 7) >> 3) > len; }
};
static __device__ __forceinline__ int hibit(uint32_t v) { return 31 - __clz(v); }

// ---- FSE table description -> normalized counts (RFC 8878 4.1.1) ---------------------------------------------------------------------
// returns the number of bytes consumed, 0 on corruption
static __device__ uint32_t fse_read_counts(const uint8_t* p, uint32_t len, int max_al, int max_syms, int16_t* freq, int* nsyms, int* al_out) {
    FwdReader r{p, len, 0};
    if (len < 1) return 0;
    int al = 5 + (int)r.read(4);
    if (al > max_al) return 0;
    int remaining = 1 << al, s = 0;
    while (remaining > 0 && s < max_syms) {
        if (r.overrun()) return 0;
        int bits = hibit((uint32_t)remaining + 1) + 1;
        int val = (int)r.read(bits);
        int lower = (1 << (bits - 1)) - 1;
        int thr = (1 << bits) - 1 - (remaining + 1);
        if ((val & lower) < thr) { r.pos -= 1; val &= lower; }
        else if (val > lower) val -= thr;
        int proba = val - 1;
        remaining -= proba < 0 ? -proba : proba;
        freq[s++] = (int16_t)proba;
        if (proba == 0) {
            int rep = (int)r.read(2);
            for (;;) {
                for (int i = 0; i < rep && s < max_syms; i++) freq[s++] = 0;
                if (rep != 3) break;
                if (r.overrun()) return 0;
                rep = (int)r.read(2);
            }
        }
    }
    if (remaining != 0 || r.overrun()) return 0;
    *nsyms = s; *al_out = al;
    return (r.pos + 7) >> 3;
}

// normalized counts -> decoding table: entry = symbol | nbits << 8 | baseline << 16   (RFC 8878 4.1.1, "from normalized distribution to decoding tables")
// `next` is scratch of nsyms entries.  The table itself is the only other storage: the spread pass leaves the symbol in each cell.
static __device__ bool fse_build_table(uint32_t* tab, int al, const int16_t* freq, int nsyms, uint16_t* next) {
    const int size = 1 << al, mask = size - 1;
    int high = size;
    for (int s = 0; s < nsyms; s++) if (freq[s] == -1) { tab[--high] = (uint32_t)s; next[s] = 1; }
    const int step = (size >> 1) + (size >> 3) + 3;
    int pos = 0;
    for (int s = 0; s < nsyms; s++) {
        if (freq[s] <= 0) continue;
        next[s] = (uint16_t)freq[s];
        for (int i = 0; i < freq[s]; i++) { tab[pos] = (uint32_t)s; do { pos = (pos + step) & mask; } while (pos >= high); }
    }
    if (pos != 0) return false;
    for (int i = 0; i < size; i++) {
        uint32_t s = tab[i]; uint32_t nx = next[s]++;
        int nb = al - hibit(nx);
        uint32_t base = (nx << nb) - (uint32_t)size;
        tab[i] = s | ((uint32_t)nb << 8) | (base << 16);
    }
    return true;
}

// sequence decoding tables in the compact slot layout (see Z_FSE_SLOT_BYTES)
static __device__ bool fse_build_seq_table(uint16_t* trans, uint8_t* sym, int al, const int16_t* freq, int nsyms, uint16_t* next) {
    const int size = 1 << al, mask = size - 1;
    int high = size;
    for (int s = 0; s < nsyms; s++) if (freq[s] == -1) { sym[--high] = (uint8_t)s; next[s] = 1; }
    const int step = (size >> 1) + (size >> 3) + 3;
    int pos = 0;
    for (int s = 0; s < nsyms; s++) {
        if (freq[s] <= 0) continue;
        next[s] = (uint16_t)freq[s];
        for (int i = 0; i < freq[s]; i++) { sym[pos] = (uint8_t)s; do { pos = (pos + step) & mask; } while (pos >= high); }
    }
    if (pos != 0) return false;
    for (int i = 0; i < size; i++) {
        uint32_t nx = next[sym[i]]++;
        int nb = al - hibit(nx);
        trans[i] = (uint16_t)(((nx << nb) - (uint32_t)size) | ((uint32_t)nb << 12));
    }
    return true;
}

// predefined distributions (RFC 8878 3.1.1.3.2.2)
static __device__ const int16_t Z_LL_DEFAULT[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
static __device__ const int16_t Z_ML_DEFAULT[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
static __device__ const int16_t Z_OF_DEFAULT[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
// literal-length / match-length codes: baseline and number of extra bits (RFC 8878 3.1.1.3.2.1.1)
static __device__ const uint32_t Z_LL_BASE[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
static __device__ const uint8_t Z_LL_BITS[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
static __device__ const uint32_t Z_ML_BASE[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
static __device__ const uint8_t Z_ML_BITS[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

static __global__ void k_zstd_predef(uint8_t* predef) {
    if (threadIdx.x || blockIdx.x) return;
    int16_t f[53]; uint16_t nx[53];
    uint16_t* tr = (uint16_t*)predef; uint8_t* sy = predef + 2 * Z_FSE_ENTRIES;
    for (int i = 0; i < 36; i++) f[i] = Z_LL_DEFAULT[i];
    fse_build_seq_table(tr + Z_FSE_LL, sy + Z_FSE_LL, 6, f, 36, nx);
    for (int i = 0; i < 53; i++) f[i] = Z_ML_DEFAULT[i];
    fse_build_seq_table(tr + Z_FSE_ML, sy + Z_FSE_ML, 6, f, 53, nx);
    for (int i = 0; i < 29; i++) f[i] = Z_OF_DEFAULT[i];
    fse_build_seq_table(tr + Z_FSE_OF, sy + Z_FSE_OF, 5, f, 29, nx);
}

// ---- Huffman tree description -> decoding table (RFC 8878 4.2.1); one warp per description ------------------------------------------
// table entry = symbol | nbits << 8
static __global__ void __launch_bounds__(128) k_huf_build(ZView V, const uint32_t* __restrict__ list, uint32_t n) {
    __shared__ uint8_t s_w[4][256];
    __shared__ uint16_t s_start[4][256];
    __shared__ int s_meta[4][4];   // nweights, maxbits, ok
    const uint32_t wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t item = blockIdx.x * 4 + wi;
    if (item >= n) return;
    const uint32_t bi = list[item];
    const ZBlock& B = V.blocks[bi];
    const uint8_t* p = V.src + B.src + B.lit_hdr;
    const uint32_t avail = B.lit_comp;
    uint8_t* w = s_w[wi];
    if (lane == 0) {
        int ok = 1, nw = 0; uint32_t desc = 0;
        if (avail < 1) ok = 0;
        else {
            uint32_t hb = p[0];
            if (hb >= 128) {   // direct representation: 4 bits per weight
                nw = (int)hb - 127; desc = 1 + (uint32_t)(nw + 1) / 2;
                if (desc > avail) ok = 0;
                else for (int i = 0; i < nw; i++) { uint8_t b = p[1 + i / 2]; w[i] = (i & 1) ? (b & 15) : (b >> 4); }
            } else {           // FSE compressed weights: two interleaved states until the bitstream runs dry
                desc = 1 + hb;
                int16_t freq[256]; uint16_t nx[256]; __align__(4) uint32_t tab[64];
                int ns = 0, al = 0;
                uint32_t used = (hb == 0 || desc > avail) ? 0 : fse_read_counts(p + 1, hb, 6, 256, freq, &ns, &al);
                if (!used || used >= hb || !fse_build_table(tab, al, freq, ns, nx)) ok = 0;
                else {
                    BackReader r;
                    if (!r.init(p + 1 + used, hb - used)) ok = 0;
                    else {
                        uint32_t s1 = r.read(al), s2 = r.read(al);
                        for (;;) {   // at most 255 weights are listed; the last one is implied
                            if (nw >= 254) { ok = 0; break; }
                            uint32_t e1 = tab[s1]; w[nw++] = (uint8_t)e1; s1 = (e1 >> 16) + r.read((e1 >> 8) & 0xFF);
                            if (r.pos < 0) { w[nw++] = (uint8_t)tab[s2]; break; }
                            if (nw >= 254) { ok = 0; break; }
                            uint32_t e2 = tab[s2]; w[nw++] = (uint8_t)e2; s2 = (e2 >> 16) + r.read((e2 >> 8) & 0xFF);
                            if (r.pos < 0) { w[nw++] = (uint8_t)tab[s1]; break; }
                        }
                    }
                }
            }
        }
        int maxbits = 0;
        if (ok) {
            uint32_t sum = 0;
            for (int i = 0; i < nw; i++) { if (w[i] > 11) { ok = 0; break; } if (w[i]) sum += 1u << (w[i] - 1); }
            if (ok && sum == 0) ok = 0;
            if (ok) {
                maxbits = hibit(sum) + 1;
                uint32_t left = (1u << maxbits) - sum;
                if (maxbits > 11 || (left & (left - 1)) != 0) ok = 0;
                else { w[nw++] = (uint8_t)(hibit(left) + 1); }
            }
        }
        if (ok) {   // first table cell of every symbol: cells are handed out by increasing weight, then by symbol value
            uint32_t cnt[13]; for (int i = 0; i < 13; i++) cnt[i] = 0;
            for (int i = 0; i < nw; i++) cnt[w[i]]++;
            uint32_t nxt[13]; uint32_t acc = 0;
            for (int k = 1; k <= maxbits; k++) { nxt[k] = acc; acc += cnt[k] << (k - 1); }
            for (int i = 0; i < nw; i++) if (w[i]) { s_start[wi][i] = (uint16_t)nxt[w[i]]; nxt[w[i]] += 1u << (w[i] - 1); }
        }
        s_meta[wi][0] = nw; s_meta[wi][1] = maxbits; s_meta[wi][2] = ok;
        V.bstate[bi].huf_desc_len = desc;
    }
    __syncwarp();
    if (!s_meta[wi][2]) { if (lane == 0) zfail(V, B.frame, ZERR_HUF_DESC); return; }
    const int nw = s_meta[wi][0], maxbits = s_meta[wi][1];
    uint16_t* tab = V.huf_tab + (size_t)B.huf_own * Z_HUF_TABLE;
    for (int s = (int)lane; s < nw; s += 32) {
        uint32_t ww = w[s];
        if (!ww) continue;
        uint32_t len = 1u << (ww - 1), st = s_start[wi][s];
        uint16_t e = (uint16_t)(s | ((maxbits + 1 - ww) << 8));
        for (uint32_t k = 0; k < len; k++) tab[st + k] = e;
    }
    if (lane == 0) V.huf_state[B.huf_own].huf_maxbits = (uint8_t)maxbits;
}

// ---- Huffman streams; one lane per stream (RFC 8878 4.2.2) --------------------------------------------------------------------------
// A CTA takes Z_HUF_CTA_BLOCKS blocks (4 lanes each) and first copies their decoding tables into shared memory: with the tables in
// HBM every symbol costs a 32-byte sector from L2 for a 2-byte entry and the kernel runs at the L2's sector rate; in shared memory
// the per-symbol chain is one ~30-cycle lookup.  Dynamic shared memory: Z_HUF_CTA_BLOCKS * 2^11 entries * 2 bytes.
// Round 2: the bitstream is no longer pulled through a per-lane line buffer in shared memory (22 instructions per symbol, all of them on the one
// dependent chain a lane has).  A lane now reloads a 64-bit container straight from the staging buffer - the 8 bytes that end at its bit
// cursor, >= 57 fresh bits - and cuts four symbols out of it: lookup, shift count += code length.  ~10 instructions per symbol, and the
// shared memory the line buffers took holds the tables of 16 more blocks per CTA (56 instead of 40).
static const uint32_t Z_HUF_CTA_BLOCKS = 56;
static __global__ void __launch_bounds__(Z_HUF_CTA_BLOCKS * 4) k_huf_decode(ZView V, const uint32_t* __restrict__ list, uint32_t n) {
    extern __shared__ uint16_t s_tab[];
    const uint32_t local = threadIdx.x >> 2, k = threadIdx.x & 3;
    const uint32_t first = blockIdx.x * Z_HUF_CTA_BLOCKS;
    const uint32_t here = min(Z_HUF_CTA_BLOCKS, n - first);
    for (uint32_t it = 0; it < here; it++) {   // stage the tables: 2^maxbits entries each, 16 bytes per thread and step
        const ZBlock& Bt = V.blocks[list[first + it]];
        const uint32_t entries = 1u << V.huf_state[Bt.huf_slot].huf_maxbits;
        const uint4* g = (const uint4*)(V.huf_tab + (size_t)Bt.huf_slot * Z_HUF_TABLE);
        uint4* d = (uint4*)(s_tab + (size_t)it * Z_HUF_TABLE);
        for (uint32_t e = threadIdx.x; e < entries / 8; e += blockDim.x) d[e] = g[e];
        if (entries < 8 && threadIdx.x == 0) d[0] = g[0];
    }
    __syncthreads();
    if (local >= here) return;
    const uint32_t bi = list[first + local];
    const ZBlock& B = V.blocks[bi];
    if (V.frame_err[B.frame]) return;
    if (B.lit_streams == 1 && k) return;
    const uint32_t maxbits = V.huf_state[B.huf_slot].huf_maxbits;
    const uint16_t* tab = s_tab + (size_t)local * Z_HUF_TABLE;
    const uint32_t desc = B.lit_type == ZL_COMPRESSED ? V.bstate[bi].huf_desc_len : 0;
    if (maxbits == 0 || desc > B.lit_comp) { zfail(V, B.frame, ZERR_HUF_STREAM); return; }
    const uint8_t* s = V.src + B.src + B.lit_hdr + desc;
    uint32_t total = B.lit_comp - desc, len, nout;
    uint8_t* out = V.lits + B.lit_off;
    if (B.lit_streams == 1) { len = total; nout = B.lit_regen; }
    else {
        if (total < 6) { if (!k) zfail(V, B.frame, ZERR_HUF_STREAM); return; }
        uint32_t s1 = s[0] | (s[1] << 8), s2 = s[2] | (s[3] << 8), s3 = s[4] | (s[5] << 8);
        if ((uint64_t)6 + s1 + s2 + s3 > total) { if (!k) zfail(V, B.frame, ZERR_HUF_STREAM); return; }
        uint32_t seg = (B.lit_regen + 3) / 4;
        if (3 * seg > B.lit_regen) { if (!k) zfail(V, B.frame, ZERR_HUF_STREAM); return; }
        uint32_t off = 6 + (k > 0 ? s1 : 0) + (k > 1 ? s2 : 0) + (k > 2 ? s3 : 0);
        len = k == 0 ? s1 : k == 1 ? s2 : k == 2 ? s3 : total - 6 - s1 - s2 - s3;
        s += off; out += (size_t)k * seg; nout = k < 3 ? seg : B.lit_regen - 3 * seg;
    }
    // backward bitstream: `pos` unread bits; peek64(s, pos) = the 64 bits just below the cursor, top aligned (>= 57 of them real while pos >= 64,
    // zeros in front of the stream)
    if (!len || !s[len - 1]) { zfail(V, B.frame, ZERR_HUF_STREAM); return; }
    int64_t pos = (int64_t)len * 8 - (int64_t)(__clz((uint32_t)s[len - 1]) - 23);   // the end mark and the padding above it are not part of the stream
    const int sh = 64 - (int)maxbits;
    uint32_t i = 0;
    // head: byte stores until the output is 8-byte aligned
    while (i < nout && (((uintptr_t)(out + i)) & 7) && pos >= 0) { const uint32_t e = tab[peek64(s, pos) >> sh]; pos -= (int64_t)(e >> 8); out[i++] = (uint8_t)e; }
    // body: 8 symbols per 64-bit store, two containers of 4 symbols (<= 44 bits).  The container is cut out of a register window over
    // ALIGNED 8-byte words of the stream - hi:lo hold the cursor, n1 and n2 are the two words below, requested 128+ bits (>= 12 symbols)
    // before they are needed - so no load sits on the symbol chain (round 2; before, every container was an exposed L1/L2 round trip:
    // 10.8 long-scoreboard stall cycles per issued instruction in ncu).
    if (nout - i >= 8 && pos >= 128) {
        const uint64_t* org = (const uint64_t*)((uintptr_t)s & ~(uintptr_t)7);
        const uint32_t s0 = (uint32_t)((uintptr_t)s & 7) * 8;
        uint32_t ab = s0 + (uint32_t)pos;            // bit index (relative to org) one past the first unread bit; streams are < 2^20 bytes
        uint32_t k = (ab - 1) >> 6;
        // words below the stream are staging-buffer headroom or the bytes in front of the stream: loaded, never used
        uint64_t hi = org[k], lo = org[(int32_t)k - 1], n1 = org[(int32_t)k - 2], n2 = org[(int32_t)k - 3];
        const uint32_t sh32 = 32 - maxbits;
        while (nout - i >= 8 && ab - s0 >= 128) {   // 8 symbols consume <= 88 bits: the cursor never passes the start of the stream in here
            uint64_t acc = 0;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const uint32_t sft = (0u - ab) & 63u;   // unused bits at the top of hi
                const bool up = sft < 32;
                const uint32_t a = up ? (uint32_t)(hi >> 32) : (uint32_t)hi, b = up ? (uint32_t)hi : (uint32_t)(lo >> 32), c = up ? (uint32_t)(lo >> 32) : (uint32_t)lo;
                uint32_t ch = __funnelshift_l(b, a, sft), cl = __funnelshift_l(c, b, sft);   // the 64 bits below the cursor, top aligned
                uint32_t used = 0;
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const uint32_t e = tab[ch >> sh32];
                    const uint32_t nb = e >> 8;       // 1..11
                    ch = __funnelshift_l(cl, ch, nb); cl <<= nb;
                    used += nb;
                    acc |= (uint64_t)(e & 0xFF) << (8 * (4 * half + q));
                }
                ab -= used;
                const uint32_t k2 = (ab - 1) >> 6;
                if (k2 != k) { hi = lo; lo = n1; n1 = n2; n2 = org[(int32_t)k2 - 3]; k = k2; }
            }
            *(uint64_t*)(out + i) = acc; i += 8;
        }
        pos = (int64_t)ab - (int64_t)s0;
    }
    while (i < nout && pos >= 0) { const uint32_t e = tab[peek64(s, pos) >> sh]; pos -= (int64_t)(e >> 8); out[i++] = (uint8_t)e; }
    if (i != nout || pos != 0) zfail(V, B.frame, ZERR_HUF_STREAM);
}

// ---- sequence section: table descriptions; one lane per block (RFC 8878 3.1.1.3.2.1) ---------------------------------------------------
static __global__ void __launch_bounds__(64) k_fse_build(ZView V, const uint32_t* __restrict__ list, uint32_t n) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t bi = list[t];
    const ZBlock& B = V.blocks[bi];
    const uint8_t* p = V.src + B.src;
    uint32_t off = B.seq_hdr + 1;   // first byte after Symbol_Compression_Modes
    bool ok = off <= B.size && (B.modes & 3) == 0;
    int16_t freq[53]; uint16_t nx[53];
    ZSlotState st{0, 0, 0, 0};
    for (int k = 0; k < 3 && ok; k++) {   // order in the stream: literal lengths, offsets, match lengths
        int mode = k == 0 ? (B.modes >> 6) & 3 : k == 1 ? (B.modes >> 4) & 3 : (B.modes >> 2) & 3;
        int max_al = k == 1 ? 8 : 9, max_syms = k == 0 ? 36 : k == 1 ? 32 : 53;
        uint32_t toff = k == 0 ? Z_FSE_LL : k == 1 ? Z_FSE_OF : Z_FSE_ML;
        int al = 0;
        if (mode == 1) {        // RLE_Mode: one symbol, zero bits per state update
            if (off + 1 > B.size) { ok = false; break; }
            uint32_t sym = p[off++];
            if ((int)sym >= max_syms) { ok = false; break; }
            uint8_t* slot = V.fse_tab + (size_t)B.fse_own * Z_FSE_SLOT_BYTES;
            ((uint16_t*)slot)[toff] = 0; slot[2 * Z_FSE_ENTRIES + toff] = (uint8_t)sym;
        } else if (mode == 2) { // FSE_Compressed_Mode
            int ns = 0;
            uint32_t used = off < B.size ? fse_read_counts(p + off, B.size - off, max_al, max_syms, freq, &ns, &al) : 0;
            uint8_t* slot = V.fse_tab + (size_t)B.fse_own * Z_FSE_SLOT_BYTES;
            if (!used || !fse_build_seq_table((uint16_t*)slot + toff, slot + 2 * Z_FSE_ENTRIES + toff, al, freq, ns, nx)) { ok = false; break; }
            off += used;
        } else continue;        // Predefined_Mode / Repeat_Mode: nothing stored in the block
        if (k == 0) st.ll_al = (uint8_t)al; else if (k == 1) st.of_al = (uint8_t)al; else st.ml_al = (uint8_t)al;
    }
    if (!ok || off > B.size) { zfail(V, B.frame, ZERR_FSE_DESC); return; }
    if (B.fse_own != Z_PREDEF) V.fse_state[B.fse_own] = st;
    V.bstate[bi].seq_bits_off = off;
}

// ---- sequence bitstream -> (literal length, match length, offset); one lane per block (RFC 8878 3.1.1.3.2.1.2 / 3.1.1.4) ------------------
// Every sequence is three table lookups whose results decide where the next three happen: a chain of dependent steps per block.  With the
// tables in HBM (10 KB per block, far more than L2 over all blocks in flight) each link costs a DRAM round trip; so a CTA stages the tables
// of Z_SEQ_CTA_LANES blocks (3840 bytes each) in shared memory and its lanes run their chains against those.  Shared memory caps an SM at 56
// chains = two warps, so nothing hides latency and the kernel's time is (instructions per sequence) x (issue-to-issue latency): round 1's loop
// was 277 SASS instructions per sequence (six independent field extractions out of a 192-bit register window, a refill loop with cp.async
// line management inside it).  Round 2 rewrote the loop around a cheaper window:
//   * the stream lives in a 256-byte ring per lane in shared memory, topped up by at most ONE predicated 16-byte cp.async per sequence (a
//     sequence consumes at most 89 bits = 11.1 bytes, so one chunk per step always keeps up); `cp.async.wait_group 3` guarantees that what
//     the reader touches (it stays 160 bytes ahead) has landed - no data-dependent branch, no loop;
//   * per sequence FOUR aligned ring words are loaded and funnel-shifted into a 96-bit left-aligned window c2:c1:c0; the three value fields
//     (offset bits | match-length bits + literal-length bits, <= 31 + 32) and the three state updates (<= 26 bits, cut as ONE field and split
//     with bfe) come out of it with one funnel shift each; the position is a single 32-bit bit index relative to a 256-byte aligned origin;
//   * errors are sticky bits checked once after the loop; the last sequence (no state update) is peeled off.
// (Round 2 also tried FOUR lanes per block - one FSE state per lane of a quad, widths exchanged by shuffles, 7 warps per SM: byte-exact, but
// slower; the shuffles put ~90 instructions on every sequence of every quad.)
static const uint32_t Z_SEQ_CTA_LANES = 56;
static const uint32_t Z_LINEBUF = 272;    // bytes of shared memory per lane: the 256-byte ring + a 16-byte skew against bank conflicts
static const uint32_t Z_SEQ_LEAD = 160;   // the ring is kept filled this many bytes below the reader
static __device__ __forceinline__ uint32_t lds_u32(uint32_t sa) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(sa)); return v; }
static __device__ __forceinline__ uint32_t bfe_u32(uint32_t a, uint32_t pos, uint32_t len) { uint32_t d; asm("bfe.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(pos), "r"(len)); return d; }
static __device__ __forceinline__ uint32_t top_bits(uint32_t x, uint32_t n) { return __funnelshift_rc(x, 0u, 32u - n); }   // n = 0..32 highest bits of x
struct SeqLane {
    // stream
    const uint8_t* gorg;      // 256-byte aligned origin in the staging buffer, below the stream
    uint32_t ring;            // shared-memory address of the lane's ring; byte a of the origin space lives at ring + (a & 255)
    uint32_t p;               // bit index (origin space) one past the first unread bit
    uint32_t fc;              // 16-byte chunks >= fc have been requested
    // tables
    const uint16_t* tr; const uint8_t* sy; const uint32_t* llv; const uint32_t* mlv;
    // chain state
    uint32_t sl, so, sm, r1, r2, r3, ndirty, sum_ll, sum_ml, sticky;
    uint4* out;
    __device__ __forceinline__ void fetch_chunk() {
        fc--;
        const uint32_t sa = ring + ((fc & 15u) << 4);
        const uint8_t* g = gorg + (size_t)fc * 16;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(g) : "memory");
    }
    __device__ __forceinline__ void window(uint32_t& c2, uint32_t& c1, uint32_t& c0) const {
        const uint32_t k = (p - 1u) >> 5, s = (0u - p) & 31u;
        const uint32_t w3 = lds_u32(ring + ((k << 2) & 252u)), w2 = lds_u32(ring + (((k - 1u) << 2) & 252u));
        const uint32_t w1 = lds_u32(ring + (((k - 2u) << 2) & 252u)), w0 = lds_u32(ring + (((k - 3u) << 2) & 252u));
        c2 = __funnelshift_l(w2, w3, s); c1 = __funnelshift_l(w1, w2, s); c0 = __funnelshift_l(w0, w1, s);
    }
    template <bool LAST>
    __device__ __forceinline__ void step() {
        const uint32_t tl = tr[sl], to = tr[so], tm = tr[sm];
        const uint32_t oc = sy[so], vl = llv[sy[sl]], vm = mlv[sy[sm]];
        // keep the ring ahead of the reader: one chunk per step is enough in the worst case
        if (p < fc * 128u + Z_SEQ_LEAD * 8u && fc > 0) fetch_chunk();
        asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 3;" ::: "memory");
        uint32_t c2, c1, c0;
        window(c2, c1, c0);
        // bit layout of one sequence, top down: offset bits, match-length bits, literal-length bits, then (unless it is the last sequence)
        // the LL, ML, OF state updates
        const uint32_t nL = vl >> 24, nM = vm >> 24, n2 = nM + nL;
        const uint32_t ov = (1u << oc) + top_bits(c2, oc);
        const uint32_t v2 = top_bits(__funnelshift_l(c1, c2, oc), n2);   // oc <= 31
        const uint32_t ml = (vm & 0xFFFFFFu) + (v2 >> nL), ll = (vl & 0xFFFFFFu) + bfe_u32(v2, 0, nL);
        const uint32_t o3 = oc + n2;                                     // <= 63
        if (!LAST) {
            const uint32_t bL = tl >> 12, bM = tm >> 12, bO = to >> 12, n3 = bL + bM + bO;   // <= 26
            const bool up = o3 < 32;
            const uint32_t v3 = top_bits(__funnelshift_l(up ? c1 : c0, up ? c2 : c1, o3), n3);
            sl = Z_FSE_LL + (tl & 0xFFFu) + (v3 >> (bM + bO));
            sm = Z_FSE_ML + (tm & 0xFFFu) + bfe_u32(v3, bO, bM);
            so = Z_FSE_OF + (to & 0xFFFu) + bfe_u32(v3, 0, bO);
            p -= o3 + n3;
        } else p -= o3;
        // repeat offsets (RFC 8878 3.1.1.5), resolved on the fly; unknown ones are DIRTY = 0xFFFFFFFF (real offsets stay below 2^31)
        uint32_t o;
        if (ov > 3) { o = ov - 3; r3 = r2; r2 = r1; r1 = o; }
        else {
            const uint32_t idx = ov + (ll == 0 ? 1 : 0);
            if (idx == 1) o = r1;
            else {
                o = idx == 2 ? r2 : idx == 3 ? r3 : (r1 == 0xFFFFFFFFu ? r1 : r1 - 1);
                if (idx != 2) r3 = r2;
                r2 = r1; r1 = o;
            }
        }
        ndirty += (r1 | r2 | r3) >> 31;   // once the three are known they stay known: the dirty steps form a prefix
        *out++ = make_uint4(ll, ml, o, ov);
        sum_ll += ll; sum_ml += ml;       // each term < 2^18: a sum that passes 2^31 sets a sticky bit before it can wrap
        sticky |= p | sum_ll | sum_ml;
    }
};
static __global__ void __launch_bounds__(64) k_seq_decode(ZView V, const uint32_t* __restrict__ list, uint32_t n) {
    extern __shared__ __align__(16) uint8_t s_fse[];
    __shared__ uint32_t s_llv[36], s_mlv[53];   // code -> value baseline | extra bits << 24
    const uint32_t first = blockIdx.x * Z_SEQ_CTA_LANES;
    const uint32_t here = min(Z_SEQ_CTA_LANES, n - first);
    if (threadIdx.x < 36) s_llv[threadIdx.x] = Z_LL_BASE[threadIdx.x] | ((uint32_t)Z_LL_BITS[threadIdx.x] << 24);
    if (threadIdx.x < 53) s_mlv[threadIdx.x] = Z_ML_BASE[threadIdx.x] | ((uint32_t)Z_ML_BITS[threadIdx.x] << 24);
    for (uint32_t it = 0; it < here; it++) {   // slot layout == shared layout: 240 chunks of 16 bytes, each from the slot its table lives in
        const ZBlock& Bt = V.blocks[list[first + it]];
        const uint4* src_ll = (const uint4*)(Bt.ll_slot == Z_PREDEF ? V.predef : V.fse_tab + (size_t)Bt.ll_slot * Z_FSE_SLOT_BYTES);
        const uint4* src_ml = (const uint4*)(Bt.ml_slot == Z_PREDEF ? V.predef : V.fse_tab + (size_t)Bt.ml_slot * Z_FSE_SLOT_BYTES);
        const uint4* src_of = (const uint4*)(Bt.of_slot == Z_PREDEF ? V.predef : V.fse_tab + (size_t)Bt.of_slot * Z_FSE_SLOT_BYTES);
        uint4* d = (uint4*)(s_fse + (size_t)it * Z_FSE_SLOT_BYTES);
        for (uint32_t c = threadIdx.x; c < Z_FSE_SLOT_BYTES / 16; c += blockDim.x) {
            // trans: LL chunks 0..63, ML 64..127, OF 128..159; sym: LL 160..191, ML 192..223, OF 224..239
            const uint4* src = c < 64 ? src_ll : c < 128 ? src_ml : c < 160 ? src_of : c < 192 ? src_ll : c < 224 ? src_ml : src_of;
            d[c] = src[c];
        }
    }
    __syncthreads();
    if (threadIdx.x >= here) return;
    const uint32_t bi = list[first + threadIdx.x];
    const ZBlock& B = V.blocks[bi];
    if (V.frame_err[B.frame]) return;
    const uint32_t off = V.bstate[bi].seq_bits_off;
    const int ll_al = B.ll_slot == Z_PREDEF ? 6 : V.fse_state[B.ll_slot].ll_al;
    const int of_al = B.of_slot == Z_PREDEF ? 5 : V.fse_state[B.of_slot].of_al;
    const int ml_al = B.ml_slot == Z_PREDEF ? 6 : V.fse_state[B.ml_slot].ml_al;
    if (off >= B.size) { zfail(V, B.frame, ZERR_SEQ_STREAM); return; }
    const uint64_t st = B.src + off;           // first byte of the bitstream; it ends with the block
    const uint32_t len = B.size - off;
    const uint32_t last = V.src[st + len - 1];
    if (!last) { zfail(V, B.frame, ZERR_SEQ_STREAM); return; }   // the end mark is missing
    SeqLane L;
    const uint64_t org = (st & ~255ull) - 256;   // the staging buffer keeps 512 bytes of headroom in front of the first stream
    const uint32_t s0 = (uint32_t)(st - org) * 8;
    L.gorg = V.src + org;
    L.ring = (uint32_t)__cvta_generic_to_shared(s_fse + (size_t)Z_SEQ_CTA_LANES * Z_FSE_SLOT_BYTES + (size_t)threadIdx.x * Z_LINEBUF);
    L.p = s0 + len * 8 - (uint32_t)(__clz(last) - 23);   // the end mark and the padding above it are not part of the stream
    L.fc = ((L.p - 1u) >> 7) + 1u;                       // p >= s0 >= 2048: at least 16 chunks lie below
#pragma unroll
    for (int q = 0; q < 12; q++) L.fetch_chunk();
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    L.tr = (const uint16_t*)(s_fse + (size_t)threadIdx.x * Z_FSE_SLOT_BYTES);
    L.sy = s_fse + (size_t)threadIdx.x * Z_FSE_SLOT_BYTES + 2 * Z_FSE_ENTRIES;
    L.llv = s_llv; L.mlv = s_mlv;
    {   // initial states: LL, OF, ML (<= 9 + 8 + 9 bits)
        uint32_t c2, c1, c0;
        L.window(c2, c1, c0);
        L.sl = Z_FSE_LL + top_bits(c2, ll_al);
        L.so = Z_FSE_OF + top_bits(__funnelshift_l(c1, c2, ll_al), of_al);
        L.sm = Z_FSE_ML + top_bits(__funnelshift_l(c1, c2, ll_al + of_al), ml_al);
        L.p -= ll_al + of_al + ml_al;
        (void)c0;
    }
    // Repeat offsets are resolved on the fly.  A block that follows other blocks with sequences does not know the three offsets it starts
    // with: they are tracked as DIRTY until real offsets have pushed them out of the history, and k_seq_resolve redoes only that prefix of
    // the block once the predecessor's final history is known.
    const uint32_t DIRTY = 0xFFFFFFFFu;
    L.r1 = B.rep_known ? 1 : DIRTY; L.r2 = B.rep_known ? 4 : DIRTY; L.r3 = B.rep_known ? 8 : DIRTY;
    L.ndirty = 0; L.sum_ll = 0; L.sum_ml = 0; L.sticky = L.p;
    L.out = V.seqs + B.seq_base;
    const uint32_t nseq = B.nseq;
    for (uint32_t i = 0; i + 1 < nseq; i++) L.step<false>();
    if (nseq) L.step<true>();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // sticky bit 31: the position ran below the origin (wrapped) or a sum left the range of any valid block
    if ((L.sticky >> 31) || L.p != s0 || L.sum_ll > B.lit_regen) { zfail(V, B.frame, ZERR_SEQ_STREAM); return; }
    ZBlockState& S = V.bstate[bi];
    S.out_len = B.lit_regen + L.sum_ml;
    S.clean_from = B.rep_known ? 0 : L.ndirty + 1;   // first step after which all three offsets were known; nseq + 1: never
    S.rep[0] = L.r1; S.rep[1] = L.r2; S.rep[2] = L.r3;
}

// ---- block output bases + the repeat offsets k_seq_decode could not know; one lane per frame (RFC 8878 3.1.1.5) ---------------------------
static __global__ void __launch_bounds__(64) k_seq_resolve(ZView V, uint32_t frame_lo, uint32_t nframes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nframes) return;
    const uint32_t f = frame_lo + t;
    if (V.frame_err[f]) return;
    const ZFrame& F = V.frames[f];
    uint64_t out = 0;
    uint32_t r1 = 1, r2 = 4, r3 = 8;
    for (uint32_t bi = F.blk_lo; bi < F.blk_hi; bi++) {
        const ZBlock& B = V.blocks[bi];
        ZBlockState& S = V.bstate[bi];
        S.out_base = (uint32_t)out;
        if (B.type != ZB_COMPRESSED) { out += B.size; S.out_len = B.size; continue; }
        if (!B.nseq) { S.out_len = B.lit_regen; out += B.lit_regen; }
        else {
            uint4* __restrict__ sq = V.seqs + B.seq_base;
            const uint32_t redo = min(S.clean_from, B.nseq);
            for (uint32_t i = 0; i < redo; i++) {
                uint4 q = sq[i];
                uint32_t ll = q.x, ov = q.w, o;
                if (ov > 3) { o = ov - 3; r3 = r2; r2 = r1; r1 = o; }
                else {
                    uint32_t idx = ov + (ll == 0 ? 1 : 0);
                    if (idx == 1) o = r1;
                    else {
                        o = idx == 2 ? r2 : idx == 3 ? r3 : r1 - 1;
                        if (idx != 2) r3 = r2;
                        r2 = r1; r1 = o;
                    }
                }
                sq[i].z = o;
            }
            if (S.clean_from <= B.nseq) { r1 = S.rep[0]; r2 = S.rep[1]; r3 = S.rep[2]; }
            out += S.out_len;
        }
        if (out > F.fcs) { zfail(V, f, ZERR_SIZE); return; }
    }
    if (out != F.fcs) zfail(V, f, ZERR_SIZE);
}

// ---- sequence execution; one warp per frame (RFC 8878 3.1.1.4) -------------------------------------------------------------------------------
// A frame is a serial chain of groups of 32 sequences (lane j holds sequence j).  Prefix sums give every literal run and every match its
// place; a match must wait only for the matches whose destination its source overlaps: `dep` is the index of the last such match inside
// the group (destinations are disjoint and ascending: 5 shuffle probes), and a run of consecutive matches with dep < (first match of the run)
// is copied as one flat, warp-wide copy.
//
// Round 2.  ncu on the round-1 kernel (one BYTE per lane per step, straight to HBM, mirrored in a shared-memory ring) showed 34 warp
// instructions per sequence: zstd level 3 turns log lines into ~13 sequences per row of 4 literal bytes + a 5-byte match, so the 5-probe
// owner search, four shuffles and the address arithmetic (incl. an integer modulo for overlapping matches that almost never occur) were paid
// per byte.  Now
//   * the unit of work is a CHUNK of up to 4 bytes of one literal run or one match (prefix sums over chunk counts; one owner search per
//     chunk): an unaligned 32-bit load (two aligned words + a funnel shift) instead of four byte loads, the modulo only in the branch that
//     needs it;
//   * the group is assembled in the ring only (byte stores to shared memory), then flushed to HBM with aligned 16-byte stores: the ring is
//     indexed by the output ADDRESS modulo its size, so 16-byte chunks of the ring are 16-byte chunks of the arena;
//   * the next group's sequence records are loaded while the current group is executed.
// Groups that span the ring or more (a literal run of kilobytes) take the byte-per-lane path of round 1, which also stayed the reference for
// tests/test_zstd_models_cpu.py.  (Two other round-2 variants were byte-exact but slower: every lane copying its own sequence - a memory
// wavefront per lane per byte -, and far matches batched beside the literals - they were already in long runs.)
static const uint32_t Z_RING = 4096;
static const uint32_t Z_EXEC_WARPS = 4;
static __device__ __forceinline__ uint32_t ldu32(const uint8_t* p) {   // little-endian 4 bytes at any address: two aligned loads, up to 7 bytes of slack touched
    const uintptr_t a = (uintptr_t)p & ~(uintptr_t)3;
    const uint32_t lo = *(const uint32_t*)a, hi = *(const uint32_t*)(a + 4);
    return __funnelshift_r(lo, hi, (uint32_t)((uintptr_t)p & 3) * 8);
}
static __global__ void __launch_bounds__(128) k_execute(ZView V, const uint32_t* __restrict__ order, uint32_t nframes) {
    __shared__ __align__(16) uint8_t s_ring[Z_EXEC_WARPS][Z_RING];
    const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wid >= nframes) return;
    const uint32_t f = order[wid];
    if (V.frame_err[f]) return;
    const ZFrame& F = V.frames[f];
    uint8_t* dst = V.arena + F.dst;
    uint8_t* ring = s_ring[threadIdx.x >> 5];
    const uint32_t abase = (uint32_t)(uintptr_t)dst;   // ring slot of frame position p = (address of dst + p) & (Z_RING - 1)
#define VL_RIDX(p) ((abase + (p)) & (Z_RING - 1))
#define VL_RING(p) ring[VL_RIDX(p)]
    uint32_t ring_lo = 0;   // frame position from which the ring content can be trusted
    for (uint32_t bi = F.blk_lo; bi < F.blk_hi; bi++) {
        const ZBlock& B = V.blocks[bi];
        const uint32_t blk_base = V.bstate[bi].out_base;   // position of the block inside the frame
        const uint8_t* p = V.src + B.src;
        if (B.type == ZB_RAW) { for (uint32_t k = lane; k < B.size; k += 32) { uint8_t v = p[k]; dst[blk_base + k] = v; VL_RING(blk_base + k) = v; } __syncwarp(); continue; }
        if (B.type == ZB_RLE) { uint8_t v = p[0]; for (uint32_t k = lane; k < B.size; k += 32) { dst[blk_base + k] = v; VL_RING(blk_base + k) = v; } __syncwarp(); continue; }
        const uint8_t* lit = B.lit_type == ZL_RAW ? p + B.lit_hdr : V.lits + B.lit_off;
        const bool lit_rle = B.lit_type == ZL_RLE;
        const uint8_t rle_byte = lit_rle ? p[B.lit_hdr] : 0;
        const uint4* __restrict__ sq = V.seqs + B.seq_base;
        uint32_t lit_run = 0, out_run = blk_base;   // out_run: frame position where the group starts
        uint4 qn = lane < B.nseq ? sq[lane] : make_uint4(0, 0, 0, 0);
        for (uint32_t g = 0; g < B.nseq; g += 32) {
            const uint4 q = qn;
            qn = g + 32 + lane < B.nseq ? sq[g + 32 + lane] : make_uint4(0, 0, 0, 0);   // the next group's records travel while this group is executed
            uint32_t il = q.x, io = q.x + q.y;   // inclusive prefix sums over the 32 sequences of the group
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t a = __shfl_up_sync(0xffffffffu, il, d), b = __shfl_up_sync(0xffffffffu, io, d); if ((int)lane >= d) { il += a; io += b; } }
            const uint32_t lit_start = il - q.x;            // literal offset of this lane's sequence inside the group
            const uint32_t o_start = io - q.x - q.y;        // output offset of this lane's literals inside the group
            const uint32_t T = __shfl_sync(0xffffffffu, il, 31), O = __shfl_sync(0xffffffffu, io, 31);
            const uint32_t gend = out_run + O;              // frame position one past the group
            const uint32_t cnt = min(32u, B.nseq - g);
            const uint32_t ml = q.y, off = q.z, amd = out_run + o_start + q.x;   // amd: frame position of the match destination
            if (__any_sync(0xffffffffu, lane < cnt && (off == 0 || off > amd))) { if (lane == 0) zfail(V, f, ZERR_OFFSET); return; }
            // dep: the last match of the group whose destination [amd_i, amd_i + ml_i) overlaps this match's source [s, e); destinations are
            // disjoint and ascending, so that is the last one starting below e, if it reaches beyond s
            const uint32_t s_src = amd - off, e_src = s_src + min(ml, off);
            int dep = -1;
            {
                uint32_t lo = 0;   // number of matches i with amd_i < e_src (all of them precede this lane: e_src <= amd)
#pragma unroll
                for (int s = 16; s; s >>= 1) { uint32_t v = __shfl_sync(0xffffffffu, amd, (lo + s - 1) & 31); if ((lo + s - 1) < cnt && v < e_src) lo += s; }
                const uint32_t ci = (lo - 1) & 31;
                const uint32_t ca = __shfl_sync(0xffffffffu, amd, ci), cm = __shfl_sync(0xffffffffu, ml, ci);
                if (lo > 0 && ca + cm > s_src) dep = (int)lo - 1;
            }
            if (O < Z_RING) {
                // ---- chunks of up to 4 bytes, assembled in the ring, flushed with 16-byte stores --------------------------------------------
                // Positions of one group never share a ring slot (O < Z_RING), and a source position sa with gend - sa <= Z_RING cannot have
                // been overwritten by anything of this group; older sources are in front of the group, i.e. flushed, and come from HBM.
                uint32_t cl = (q.x + 3) >> 2, cm = (ml + 3) >> 2;   // inclusive prefix sums of the chunk counts of literal runs / matches
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { uint32_t a = __shfl_up_sync(0xffffffffu, cl, d), b = __shfl_up_sync(0xffffffffu, cm, d); if ((int)lane >= d) { cl += a; cm += b; } }
                const uint32_t CL = __shfl_sync(0xffffffffu, cl, 31);
                const uint32_t pk = lit_start | (o_start << 16);   // both < Z_RING = 2^12
                const uint8_t* lsrc = lit + lit_run;
                for (uint32_t c0 = 0; c0 < CL; c0 += 128) {   // four steps of 32 chunks: all loads first, then all stores
                    uint32_t w[4], at[4], nb[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        nb[u] = 0; w[u] = 0; at[u] = 0;
                        if (c0 + 32 * u >= CL) continue;   // warp-uniform
                        const uint32_t c = c0 + 32 * u + lane;
                        uint32_t lo = 0;   // smallest j with cl[j] > c
#pragma unroll
                        for (int s = 16; s; s >>= 1) { uint32_t x = __shfl_sync(0xffffffffu, cl, (lo + s - 1) & 31); if (x <= c) lo += s; }
                        const uint32_t jc = __shfl_sync(0xffffffffu, cl, lo & 31), jl = __shfl_sync(0xffffffffu, q.x, lo & 31), jp = __shfl_sync(0xffffffffu, pk, lo & 31);
                        if (c < CL) {
                            const uint32_t b0 = (c - (jc - ((jl + 3) >> 2))) * 4;   // first byte of the chunk inside its literal run
                            nb[u] = min(4u, jl - b0);
                            w[u] = lit_rle ? rle_byte * 0x01010101u : ldu32(lsrc + (jp & 0xFFFF) + b0);
                            at[u] = out_run + (jp >> 16) + b0;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
#pragma unroll
                        for (int t = 0; t < 4; t++) if ((uint32_t)t < nb[u]) VL_RING(at[u] + t) = (uint8_t)(w[u] >> (8 * t));
                    }
                }
                __syncwarp();
                uint32_t cur = 0;
                while (cur < cnt) {
                    const uint32_t ready = __ballot_sync(0xffffffffu, lane >= cur && lane < cnt && dep < (int)cur) >> cur;   // bit 0 = match `cur`, always set
                    const uint32_t n = ready == 0xffffffffu ? 32u : max((uint32_t)__ffs((int)~ready) - 1u, 1u);
                    const uint32_t hi = cur + n;
                    const uint32_t c_lo = cur ? __shfl_sync(0xffffffffu, cm, cur - 1) : 0u, C = __shfl_sync(0xffffffffu, cm, hi - 1) - c_lo;
                    for (uint32_t c0 = 0; c0 < C; c0 += 128) {
                        uint32_t w[4], at[4], nb[4];
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            nb[u] = 0; w[u] = 0; at[u] = 0;
                            if (c0 + 32 * u >= C) continue;   // warp-uniform
                            const uint32_t c = c_lo + c0 + 32 * u + lane;
                            uint32_t lo = 0;   // smallest j with cm[j] > c
#pragma unroll
                            for (int s = 16; s; s >>= 1) { uint32_t x = __shfl_sync(0xffffffffu, cm, (lo + s - 1) & 31); if (x <= c) lo += s; }
                            const uint32_t jc = __shfl_sync(0xffffffffu, cm, lo & 31), jm = __shfl_sync(0xffffffffu, ml, lo & 31);
                            const uint32_t jf = __shfl_sync(0xffffffffu, off, lo & 31), jd = __shfl_sync(0xffffffffu, amd, lo & 31);
                            if (c0 + 32 * u + lane < C) {
                                const uint32_t b0 = (c - (jc - ((jm + 3) >> 2))) * 4;   // first byte of the chunk inside its match
                                nb[u] = min(4u, jm - b0);
                                at[u] = jd + b0;
                                const uint32_t sa = jd - jf + b0;
                                if (jf >= jm && sa >= ring_lo && gend - sa <= Z_RING) {   // no overlap, first byte in the ring: so are the others
                                    const uint32_t i0 = VL_RIDX(sa), a0 = i0 & ~3u;
                                    w[u] = __funnelshift_r(*(const uint32_t*)(ring + a0), *(const uint32_t*)(ring + ((a0 + 4) & (Z_RING - 1))), (i0 & 3) * 8);
                                } else if (jf >= jm && sa + nb[u] <= out_run) {           // no overlap, wholly in front of the group: flushed
                                    w[u] = ldu32(dst + sa);
                                } else {
                                    // byte by byte: a match that repeats its own output (byte kk comes from the first `offset` bytes, all in front of
                                    // it), or a source that starts in front of what the ring holds and runs into it
                                    for (uint32_t t = 0; t < nb[u]; t++) {
                                        const uint32_t sb = jd - jf + (jf >= jm ? b0 + t : (b0 + t) % jf);
                                        const uint32_t v = (sb >= ring_lo && gend - sb <= Z_RING) ? VL_RING(sb) : dst[sb];
                                        w[u] |= v << (8 * t);
                                    }
                                }
                            }
                        }
#pragma unroll
                        for (int u = 0; u < 4; u++) {
#pragma unroll
                            for (int t = 0; t < 4; t++) if ((uint32_t)t < nb[u]) VL_RING(at[u] + t) = (uint8_t)(w[u] >> (8 * t));
                        }
                    }
                    __syncwarp();
                    cur = hi;
                }
                // flush [out_run, gend): bytes up to the first 16-byte boundary of the arena, aligned 16-byte chunks, the bytes behind the last one
                {
                    const uintptr_t a0 = (uintptr_t)dst + out_run, a1 = (uintptr_t)dst + gend;
                    const uintptr_t h0 = (a0 + 15) & ~(uintptr_t)15, h1 = a1 & ~(uintptr_t)15;
                    if (h0 <= h1) {
                        if (lane < h0 - a0) *(uint8_t*)(a0 + lane) = ring[(a0 + lane) & (Z_RING - 1)];
                        for (uintptr_t c = h0 + 16 * lane; c < h1; c += 512) *(uint4*)c = *(const uint4*)(ring + (c & (Z_RING - 1)));
                        if (lane < a1 - h1) *(uint8_t*)(h1 + lane) = ring[(h1 + lane) & (Z_RING - 1)];
                    } else if (lane < O) *(uint8_t*)(a0 + lane) = ring[(a0 + lane) & (Z_RING - 1)];   // the group lies inside one 16-byte chunk
                }
                __syncwarp();
            } else {
                // ---- a group that spans the ring or more: one byte per lane per step, straight to HBM (round 1's path) ----------------------
                // Stores are not in position order inside a group (all literals first), so the ring cannot be trusted below the end of
                // such a group: sources come from HBM, and ring_lo moves to gend.
                for (uint32_t k0 = 0; k0 < T; k0 += 32) {
                    uint32_t k = k0 + lane;
                    uint32_t lo = 0;   // smallest j with il[j] > k, by 5 shuffle probes
#pragma unroll
                    for (int s = 16; s; s >>= 1) { uint32_t v = __shfl_sync(0xffffffffu, il, (lo + s - 1) & 31); if (v <= k) lo += s; }
                    uint32_t js = __shfl_sync(0xffffffffu, lit_start, lo & 31), jo = __shfl_sync(0xffffffffu, o_start, lo & 31);
                    if (k < T) { uint8_t v = lit_rle ? rle_byte : lit[lit_run + k]; uint32_t at = out_run + jo + (k - js); dst[at] = v; VL_RING(at) = v; }
                }
                __syncwarp();
                const uint32_t im = io - il;   // inclusive prefix sum of the match lengths
                uint32_t cur = 0;
                while (cur < cnt) {
                    const uint32_t ready = __ballot_sync(0xffffffffu, lane >= cur && lane < cnt && dep < (int)cur) >> cur;
                    const uint32_t n = ready == 0xffffffffu ? 32u : max((uint32_t)__ffs((int)~ready) - 1u, 1u);
                    const uint32_t hi = cur + n;
                    const uint32_t im_lo = cur ? __shfl_sync(0xffffffffu, im, cur - 1) : 0u, M = __shfl_sync(0xffffffffu, im, hi - 1) - im_lo;
                    for (uint32_t k0 = 0; k0 < M; k0 += 32) {
                        const uint32_t k = im_lo + k0 + lane;   // position in the group's concatenated match bytes
                        uint32_t lo = 0;                         // smallest j with im[j] > k
#pragma unroll
                        for (int s = 16; s; s >>= 1) { uint32_t v = __shfl_sync(0xffffffffu, im, (lo + s - 1) & 31); if (v <= k) lo += s; }
                        const uint32_t jm = __shfl_sync(0xffffffffu, ml, lo & 31), jo = __shfl_sync(0xffffffffu, off, lo & 31);
                        const uint32_t jd = __shfl_sync(0xffffffffu, amd, lo & 31), je = __shfl_sync(0xffffffffu, im, lo & 31);
                        if (k0 + lane < M) {
                            const uint32_t kk = k - (je - jm);   // byte index inside match `lo`
                            const uint32_t sa = jd - jo + (jo >= jm ? kk : kk % jo);   // frame position of the source byte
                            const uint8_t v = dst[sa];
                            dst[jd + kk] = v; VL_RING(jd + kk) = v;
                        }
                    }
                    __syncwarp();
                    cur = hi;
                }
                ring_lo = gend;
            }
            lit_run += T; out_run += O;
        }
        // literals after the last sequence
        const uint32_t rest = B.lit_regen - lit_run;
        for (uint32_t k = lane; k < rest; k += 32) { uint8_t v = lit_rle ? rle_byte : lit[lit_run + k]; dst[out_run + k] = v; VL_RING(out_run + k) = v; }
        __syncwarp();
    }
#undef VL_RING
#undef VL_RIDX
}

}  // namespace zs
}  // namespace vl
