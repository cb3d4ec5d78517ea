// CUDA kernels of the block-scan engine (sm_90a).  HBM-bound byte / bitmap work: coalesced 16-byte vector loads,
// warp ballots / shuffles, no tensor cores.  Each kernel names the reference code it replaces.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vl_hd.cuh"
#include "vl_anycase.cuh"
#include "vl_mathnum.cuh"
#include "vl_types.h"

namespace vl {

struct DevProgram {
    const DevLeaf* leaves; const DevPrepass* prepass; const DevRegex* regexes;
    const uint8_t* blob; const uint64_t* u64s; const uint32_t* u32s;
};

// stats slots (device u64 array)
enum { ST_VALUES_BYTES = 0, ST_BLOOM_BYTES, ST_COLUMNS_READ, ST_BITMAP_BYTES, ST_ROWS_MATCHED, ST_BLOCKS_MATCHED, ST_ERROR, ST_SCAN_BYTES, ST_COUNT };
// atomicMax keeps the largest code: the numbers rank the errors (4 and 5 are unused)
enum { ERR_NONE = 0, ERR_LENS_MISMATCH = 1, ERR_DICT_INDEX = 2, ERR_BAD_WIDTH = 3, ERR_NO_TIMESTAMPS = 6, ERR_BAD_TIMESTAMPS = 7, ERR_VALUES_ABSENT = 8,
       ERR_TS_HEADER = 9 };   // decoded timestamps outside the [min, max] of their block header (k_last_rows)

struct BatchView {
    const uint8_t* arena;         // values payloads: lens items, data, encoded timestamps (lens_off, data_off, DevTimestamps.off)
    const uint8_t* hdr;           // header payloads: bloom filters, const values, dict tables (bloom_off, meta_off).  The same buffer as `arena`
                                  // unless the batch was staged bloom-first (vlscan_scan_batch): then it is the phase-1 buffer
    const DevColumn* cols;        // [nblocks * nfields]
    const uint32_t* blk_rows;     // [nblocks]
    const uint64_t* blk_word_off; // [nblocks + 1]
    const uint32_t* word_block;   // [nwords] owning block of each bitmap word
    const DevTimestamps* ts;      // [nblocks] or NULL when the batch was staged without timestamps
    uint32_t nblocks, nfields;
    uint64_t nwords;
};

static __device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
#define VL_SHORT_ROW_BYTES 48u   /* average row length below which a string block is matched per row instead of row-agnostically */
static __device__ __forceinline__ uint32_t width_of_vt(uint32_t vt) {
    switch (vt) { case VT_DICT: case VT_UINT8: return 1; case VT_UINT16: return 2; case VT_UINT32: case VT_IPV4: return 4; case VT_UINT64: case VT_FLOAT64: case VT_ISO8601: case VT_INT64: return 8; }
    return 0;
}
static __device__ __forceinline__ uint64_t lens_stored_bytes(const DevColumn& c, uint32_t rows) {
    return 1 + (c.lens_type < 4 ? ((uint64_t)rows << c.lens_type) : (1ull << (c.lens_type - 4)));
}
// a values cell whose rows are found through k_lens_offsets: per-row lens items, and not every row the whole payload (encoding.go:113-120)
static __device__ __forceinline__ bool cell_needs_offsets(const DevColumn& c) { return c.kind == COL_VALUES && c.lens_type < 4 && !c.data_const; }
// length of row r (unmarshalUint64Items lib/logstorage/encoding.go:246-336)
static __device__ __forceinline__ uint32_t row_len(const DevColumn& c, const uint8_t* lens, uint32_t r) {
    switch (c.lens_type) {
    case 0: return lens[r];
    case 1: return ld_be16(lens + 2 * (uint64_t)r);
    case 2: return ld_be32(lens + 4 * (uint64_t)r);
    case 3: return (uint32_t)ld_be64(lens + 8 * (uint64_t)r);
    default: return c.lens_const;
    }
}
static __device__ __forceinline__ uint64_t load_fixed_be(const uint8_t* p, uint32_t w) {
    switch (w) { case 1: return p[0]; case 2: return ld_be16(p); case 4: return ld_be32(p); default: return ld_be64(p); }
}
static __device__ __forceinline__ int64_t unzigzag64(uint64_t u) { return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); }

// ---- regex on device (regexutil.Regex.MatchString, regex.go:86-212) -----------------------------------------------------------
static __device__ __forceinline__ uint32_t rx_class(const DevRegex& R, const uint8_t* blob, int32_t r) {
    if (r < 128) return blob[R.ascii_off + r];
    const int32_t* b = (const int32_t*)(blob + R.bounds_off);
    int lo = 0, hi = (int)R.nclasses - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (b[mid] <= r) lo = mid; else hi = mid - 1; }
    return (uint32_t)lo;
}
static __device__ bool dfa_run(const DevRegex& R, const uint8_t* blob, const uint8_t* s, uint32_t n) {
    const uint16_t* T = (const uint16_t*)(blob + R.trans_off);
    uint32_t st = 0;
    for (uint32_t i = 0; i < n;) {
        int w; int32_t r = s[i];
        if (r < 0x80) w = 1; else r = decode_rune(s + i, n - i, &w);
        i += w;
        uint32_t e = T[st * R.nclasses + rx_class(R, blob, r)];
        if (e & 0x8000) return true;
        st = e & 0x7FFF;
        if (st == 0x7FFF) return false;
    }
    return blob[R.accept_off + st] != 0;
}
static __device__ bool regex_match(const DevRegex& R, const uint8_t* blob, const uint8_t* s, uint32_t n) {
    const uint8_t* pre = blob + R.prefix_off; uint32_t pl = R.prefix_len;
    const uint8_t* sub = blob + R.sub_off; uint32_t sl = R.sub_len;
    if (R.only_prefix) return pl == 0 || find_bytes(s, n, pre, pl, 0) >= 0;
    if (pl == 0) {
        if (R.dot_star) return true;
        if (R.dot_plus) return n > 0;
        if (R.sub_kind == 1) return find_bytes(s, n, sub, sl, 0) >= 0;
        if (R.sub_kind == 2) { int k = find_bytes(s, n, sub, sl, 0); return k > 0 && (uint32_t)k + sl < n; }
        return dfa_run(R, blob, s, n);
    }
    int k = find_bytes(s, n, pre, pl, 0);
    if (k < 0) return false;
    uint32_t rem = (uint32_t)k + pl;
    if (R.dot_star) return true;
    if (R.dot_plus) return n > rem;
    if (R.sub_kind == 1) return find_bytes(s + rem, n - rem, sub, sl, 0) >= 0;
    if (R.sub_kind == 2) { int m = find_bytes(s + rem, n - rem, sub, sl, 0); return m > 0 && (uint32_t)m + sl < n - rem; }
    if (R.tail_len) return find_bytes(s + rem, n - rem, blob + R.tail_off, R.tail_len, 0) >= 0;   // `.*LIT` after the first prefix occurrence
    for (;;) {
        if (dfa_run(R, blob, s + rem, n - rem)) return true;
        k = find_bytes(s, n, pre, pl, (uint32_t)k + 1);
        if (k < 0) return false;
        rem = (uint32_t)k + pl;
    }
}

// in(): is the string one of the values (filter_in.go:187-200 for string columns / const / dict)
static __device__ bool in_contains_string(const DevLeaf& L, const uint8_t* blob, const uint8_t* s, uint32_t n) {
    const uint32_t* offs = (const uint32_t*)(blob + L.in_offs_off);
    const uint8_t* base = blob + L.in_blob_off;
    for (uint32_t i = 0; i < L.in_count; i++) { uint32_t a = offs[i], b = offs[i + 1]; if (b - a == n && bytes_equal(base + a, n, s, n)) return true; }
    return false;
}
static __device__ __forceinline__ bool in_contains_typed(const DevLeaf& L, const uint64_t* u64s, uint32_t vt, uint64_t v) {
    const uint64_t* set = u64s + L.in_typed_off[vt];
    int lo = 0, hi = (int)L.in_typed_cnt[vt] - 1;
    while (lo <= hi) { int mid = (lo + hi) >> 1; uint64_t x = set[mid]; if (x == v) return true; if (x < v) lo = mid + 1; else hi = mid - 1; }
    return false;
}

// generic string predicate of a leaf: the closure passed to visitValues / applied to const + dict values
static __device__ bool leaf_match_string(const DevProgram& P, const DevLeaf& L, const uint8_t* s, uint32_t n) {
    const uint8_t* nd = P.blob + L.needle_off;
    switch (L.kind) {
    case F_PHRASE: return match_phrase(s, n, nd, L.needle_len);
    case F_PREFIX: return match_prefix(s, n, nd, L.needle_len);
    case F_EXACT: return bytes_equal(s, n, nd, L.needle_len);
    case F_IN: return in_contains_string(L, P.blob, s, n);
    case F_REGEXP: return regex_match(P.regexes[L.regex], P.blob, s, n);
    case F_EXACT_PREFIX: case F_LEN_RANGE: case F_STRING_RANGE: case F_IPV4_RANGE:   // matchExactPrefix / matchLenRange / matchStringRange / matchIPv4Range
        return range_predicate(L.kind, s, n, nd, L.needle_len, P.blob + L.needle2_off, L.needle2_len, L.aux0, L.aux1);
    case F_VALUE_TYPE: return false;   // decided from the column header alone (k_plan_leaf)
    case F_ANY_CASE_PHRASE: return any_case_match(s, n, nd, L.needle_len, false);   // matchAnyCasePhrase: needle = the lower-cased phrase
    case F_ANY_CASE_PREFIX: return any_case_match(s, n, nd, L.needle_len, true);
    case F_SEQUENCE: return match_sequence(s, n, PhraseList{P.blob + L.list_off, L.list_len});
    case F_CONTAINS_ALL: return match_all_phrases(s, n, PhraseList{P.blob + L.list_off, L.list_len});
    case F_CONTAINS_ANY: return match_any_phrase(s, n, PhraseList{P.blob + L.list_off, L.list_len});
    case F_RANGE: {   // matchRange filter_range.go:352-355: the value as parseMathNumber reads it; NaN is outside every range
        const double f = mn::parse_math_number(s, n);
        return f >= __longlong_as_double((long long)L.rng_fmin) && f <= __longlong_as_double((long long)L.rng_fmax);
    }
    }
    return true;
}
// The text of a typed value (number, IPv4, timestamp) against the leaf.  i(...) leaves run the plain phrase / prefix matcher here, with the
// lower-cased needle and, on iso8601 columns, the upper-cased one ("T", "Z"): filter_any_case_phrase.go:103-126, filter_any_case_prefix.go:106-129.
static __device__ bool leaf_match_typed_text(const DevProgram& P, const DevLeaf& L, uint32_t vt, const uint8_t* s, uint32_t n) {
    if (L.kind == F_ANY_CASE_PHRASE || L.kind == F_ANY_CASE_PREFIX) {
        const uint8_t* nd = P.blob + (vt == VT_ISO8601 ? L.needle2_off : L.needle_off); const uint32_t nl = vt == VT_ISO8601 ? L.needle2_len : L.needle_len;
        return L.kind == F_ANY_CASE_PHRASE ? match_phrase(s, n, nd, nl) : match_prefix(s, n, nd, nl);
    }
    return leaf_match_string(P, L, s, n);
}

// numeric value -> string (toUint8String .. toTimestampISO8601String, filter_prefix.go:365-408, filter_phrase.go:310-346)
static __device__ int encoded_to_string(uint32_t vt, uint64_t raw, uint8_t* buf) {
    switch (vt) {
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: return fmt_u64(buf, raw);
    case VT_INT64: return fmt_i64(buf, unzigzag64(raw));
    case VT_IPV4: return fmt_ipv4(buf, (uint32_t)raw);
    case VT_ISO8601: return fmt_iso8601(buf, (int64_t)raw);
    }
    return -1;   // float64 takes leaf_match_f64 (its text can be 300+ bytes long)
}

// float64 value -> shortest decimal text -> string matcher (toFloat64String, filter_phrase.go:304-308; matchFloat64ByPrefix,
// filter_prefix.go:224-252; matchFloat64ByRegex filter_regexp.go).  Kept out of line: the 352-byte text buffer must not
// grow the frame of the common integer path.
static __device__ __noinline__ bool leaf_match_f64(const DevProgram& P, const DevLeaf& L, uint64_t raw) {
    uint8_t buf[VL_FMT_F64_MAX];
    int n = fmt_f64(buf, raw);
    return leaf_match_typed_text(P, L, VT_FLOAT64, buf, (uint32_t)n);
}

// ---- bloom probe, warp wide (bloomFilter.containsAll, lib/logstorage/bloomfilter.go:173-191) -----------------------------------
// All 32 lanes call with identical arguments; lanes split the probe hashes; result is uniform.
static __device__ bool bloom_contains_all_warp(const uint8_t* bloom_be, uint32_t nwords, const uint64_t* hashes, uint32_t nh) {
    if (nwords == 0) return true;
    uint64_t maxbits = (uint64_t)nwords * 64;
    bool ok = true;
    for (uint32_t i = lane_id(); i < nh; i += 32) {
        uint64_t idx = hashes[i] % maxbits;
        uint64_t w = ld_be64(bloom_be + (idx >> 6) * 8);   // words are stored big-endian (bloomfilter.go:49-55)
        if (!((w >> (idx & 63)) & 1)) ok = false;
    }
    return __all_sync(0xffffffffu, ok);
}

// ---- bitmap helpers --------------------------------------------------------------------------------------------------
// is the bitmap of block b non-zero (bitmap.isZero, bitmap.go:74-81)?  All 32 lanes call with the same b; the result is uniform.
static __device__ __forceinline__ bool block_alive_warp(const uint64_t* __restrict__ reg, const BatchView& B, uint32_t b) {
    const uint64_t lo = B.blk_word_off[b], hi = B.blk_word_off[b + 1];
    bool any = false;
    for (uint64_t w = lo + lane_id(); w < hi; w += 32) any |= reg[w] != 0;
    return __any_sync(0xffffffffu, any);
}
// number of rows still selected in block b (bitmap.onesCount); uniform result
static __device__ __forceinline__ uint32_t block_ones_warp(const uint64_t* __restrict__ reg, const BatchView& B, uint32_t b) {
    const uint64_t lo = B.blk_word_off[b], hi = B.blk_word_off[b + 1];
    uint32_t n = 0;
    for (uint64_t w = lo + lane_id(); w < hi; w += 32) n += __popcll(reg[w]);
#pragma unroll
    for (int d = 16; d; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
    return n;
}
static __global__ void k_andnot(uint64_t* __restrict__ a, const uint64_t* __restrict__ b, uint64_t n) {   // bitmap.andNot bitmap.go:99-111
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] &= ~b[i];
}

// ---- AND / OR bloom pre-pass (filterAnd.matchBloomFilters filter_and.go:76-111, filterOr.matchBloomFilters filter_or.go:80-115) ----
// one warp per block; a failing block gets its bitmap words zeroed (bm.resetBits()).
static __global__ void k_prepass(DevProgram P, BatchView B, uint32_t pp_begin, uint32_t pp_count, const int* __restrict__ slots /* per prepass entry */,
                          int is_or, uint64_t* __restrict__ reg, unsigned long long* __restrict__ stats) {
    uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B.nblocks || !block_alive_warp(reg, B, b)) return;
    bool pass = is_or ? false : true;
    unsigned long long bloom_bytes = 0;
    for (uint32_t e = 0; e < pp_count; e++) {
        const DevPrepass& pp = P.prepass[pp_begin + e];
        int slot = slots[e];
        const DevColumn* c = slot >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot] : nullptr;
        bool ok;
        bool skip = false;   // OR: "continue" without a verdict
        if (c && c->kind == COL_CONST) {
            // matchStringByAllTokens(v, tokens)
            const uint32_t* to = (const uint32_t*)(P.blob + pp.tok_offs_off);
            const uint8_t* v = B.hdr + c->meta_off;
            ok = true;
            for (uint32_t t = 0; t < pp.ntokens && ok; t++) ok = match_phrase(v, c->meta_len, P.blob + pp.tok_blob_off + to[t], to[t + 1] - to[t]);
        } else if (!c || c->kind == COL_MISSING) {
            ok = false; skip = true;
        } else if (c->vt == VT_DICT) {
            // matchDictValuesByAllTokens: dict values joined with ',' (filter_and.go:198-208); a token never contains ','
            // so a phrase occurrence lies inside one value; value edges behave like the ',' separator (non-token char).
            const uint32_t* dof = (const uint32_t*)(B.hdr + c->meta_off);
            const uint8_t* dv = B.hdr + c->meta_off + 4 * (c->dict_len + 1);
            const uint32_t* to = (const uint32_t*)(P.blob + pp.tok_offs_off);
            ok = true;
            for (uint32_t t = 0; t < pp.ntokens && ok; t++) {
                bool found = false;
                for (uint32_t d = 0; d < c->dict_len && !found; d++) found = match_phrase(dv + dof[d], dof[d + 1] - dof[d], P.blob + pp.tok_blob_off + to[t], to[t + 1] - to[t]);
                ok = found;
            }
        } else {
            bloom_bytes += 8ull * pp.nhashes;
            ok = bloom_contains_all_warp(B.hdr + c->bloom_off, c->bloom_words, P.u64s + pp.hashes_off, pp.nhashes);
        }
        if (is_or) { if (!skip && ok) { pass = true; break; } }
        else if (!ok) { pass = false; break; }
    }
    if (is_or && pp_count == 0) pass = true;
    if (lane_id() == 0 && bloom_bytes) atomicAdd(&stats[ST_BLOOM_BYTES], bloom_bytes);
    if (!pass) for (uint64_t w = B.blk_word_off[b] + lane_id(); w < B.blk_word_off[b + 1]; w += 32) reg[w] = 0;
}

// ---- per (block, leaf) header dispatch: const / missing / dict / typed columns + leaf-level bloom probe ----------------------------
// filterPhrase.applyToBlockSearch filter_phrase.go:61-111, filterPrefix :59-106, filterExact :186-235, filterIn :120-185,
// filterRegexp :78-127 and the match*By* helpers they call.  One warp per block, all lanes run the same scalar logic.
// The same kernel decides bm.isZero() for the block and appends the block to the work lists of the kernels that follow: blocks whose lens
// items must be decoded, the 64 KiB tiles of the row-agnostic scan, blocks of the per-row matcher.  The lists are unordered (appended with
// one atomic per CTA and list): every consumer only needs the set.
#define VL_PLAN_WARPS 8
enum { WC_LENS = 0, WC_TILES = 1, WC_ROW = 2, WC_LENS2 = 3, WC_COUNT = 4 };   // WC_LENS2: the second column of a two-column leaf
#define VL_TILE_BYTES 65536u                  /* row bytes per work item of the substring scan */
// One work item of the substring scan, self-contained so that the streaming side needs one 16-byte load per tile and no column header.
struct __align__(16) ScanTile {
    uint64_t off;      // arena byte offset of the tile's first byte
    uint32_t bytes;    // row bytes in the tile: VL_TILE_BYTES, less for a block's last tile
    uint32_t block;
};
static __global__ void __launch_bounds__(VL_PLAN_WARPS * 32) k_plan_leaf(DevProgram P, BatchView B, uint32_t leaf_idx, int slot, const uint64_t* __restrict__ reg,
                            uint8_t* __restrict__ action, uint64_t* __restrict__ payload, uint32_t* __restrict__ lens_blocks, uint32_t* __restrict__ row_blocks,
                            ScanTile* __restrict__ tiles, uint32_t* __restrict__ work_count,
                            unsigned long long* __restrict__ stats, uint8_t* __restrict__ need = nullptr) {
    // need != NULL: PROBE pass of a bloom-first upload (phase 1: headers, bloom filters and dict tables are on the device, no values yet).
    // `reg` then only carries which blocks are still alive behind the AND / OR bloom pre-passes of the leaf's ancestors; the kernel runs the
    // same header dispatch and bloom probes and sets need[block * nfields + slot] when the leaf would go on to read the column's values.
    // Nothing else is written.  Every block the real scan reads values of is marked: the real scan reaches a leaf with a subset of the rows
    // (hence blocks) the probe reaches it with, and the gates below do not depend on the rows.
    __shared__ uint32_t s_cnt[VL_PLAN_WARPS][3], s_off[VL_PLAN_WARPS][3];
    __shared__ unsigned long long s_stat[VL_PLAN_WARPS][4];
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t b = blockIdx.x * VL_PLAN_WARPS + warp;
    const DevLeaf& L = P.leaves[leaf_idx];
    uint8_t act = ACT_NONE; uint64_t pay = 0;
    unsigned long long bloom_bytes = 0, values_bytes = 0, scan_bytes = 0, scan_off = 0; int err = 0;
    uint32_t need_lens = 0, need_row = 0, ntiles = 0;
    const bool valid = b < B.nblocks;
    const uint32_t ones = valid ? block_ones_warp(reg, B, b) : 0;
    const bool alive = ones != 0;
    if (alive && L.kind == F_NOOP) act = ACT_ALL;
    else if (alive) {
    act = ACT_ALL;
    uint32_t rows = B.blk_rows[b];
    const DevColumn* c = slot >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot] : nullptr;
    const uint8_t* nd = P.blob + L.needle_off; uint32_t nl = L.needle_len;
    if ((L.kind == F_IN && L.in_count == 0) || L.always_none) act = ACT_NONE;   // fi.values.isEmpty(); minLen > maxLen, minValue > maxValue
    else if (L.kind == F_TIME) {   // filterTime.applyToBlockSearch filter_time.go:114-137: header-level decisions first
        const int64_t mn = (int64_t)L.aux0, mx = (int64_t)L.aux1;
        if (!B.ts || B.ts[b].mt == 0) { act = ACT_NONE; err = ERR_NO_TIMESTAMPS; }
        else if (mn > B.ts[b].max || mx < B.ts[b].first) act = ACT_NONE;
        else if (mn <= B.ts[b].first && mx >= B.ts[b].max) act = ACT_ALL;
        else { act = ACT_TIME; need_row = 1; }
    }
    else if (c && c->kind == COL_CONST) {
        if (L.kind == F_VALUE_TYPE) act = L.aux0 == VTYPE_CONST ? ACT_ALL : ACT_NONE;   // filter_value_type.go:46-52
        else act = leaf_match_string(P, L, B.hdr + c->meta_off, c->meta_len) ? ACT_ALL : ACT_NONE;
    } else if (!c || c->kind == COL_MISSING) {
        switch (L.kind) {
        case F_PHRASE: case F_EXACT: case F_EXACT_PREFIX: act = nl == 0 ? ACT_ALL : ACT_NONE; break;
        case F_PREFIX: act = ACT_NONE; break;
        case F_IN: act = L.in_has_empty ? ACT_ALL : ACT_NONE; break;
        case F_REGEXP: act = regex_match(P.regexes[L.regex], P.blob, nullptr, 0) ? ACT_ALL : ACT_NONE; break;
        case F_LEN_RANGE: act = L.aux0 == 0 ? ACT_ALL : ACT_NONE; break;                                // matchLenRange("", min, max)
        case F_STRING_RANGE: act = (nl == 0 && L.needle2_len > 0) ? ACT_ALL : ACT_NONE; break;           // "" >= min && "" < max
        case F_IPV4_RANGE: case F_VALUE_TYPE: case F_RANGE: act = ACT_NONE; break;
        case F_ANY_CASE_PHRASE: act = nl == 0 ? ACT_ALL : ACT_NONE; break;                               // filter_any_case_phrase.go:88-95
        case F_ANY_CASE_PREFIX: act = ACT_NONE; break;                                                   // filter_any_case_prefix.go:92-97
        case F_SEQUENCE: case F_CONTAINS_ALL: case F_CONTAINS_ANY: act = leaf_match_string(P, L, nullptr, 0) ? ACT_ALL : ACT_NONE; break;   // the predicate on ""
        }
    } else if (L.kind == F_VALUE_TYPE) {
        act = L.aux0 == c->vt ? ACT_ALL : ACT_NONE;   // valueType.String() == wanted name (filter_value_type.go:59-66); no payload is read
    } else if (c->vt == VT_DICT) {
        const uint32_t* dof = (const uint32_t*)(B.hdr + c->meta_off);
        const uint8_t* dv = B.hdr + c->meta_off + 4 * (c->dict_len + 1);
        uint32_t mask = 0;
        for (uint32_t d = 0; d < c->dict_len; d++) if (leaf_match_string(P, L, dv + dof[d], dof[d + 1] - dof[d])) mask |= 1u << d;
        if (mask == 0) act = ACT_NONE; else { act = ACT_DICT; pay = mask; }
    } else {
        uint32_t vt = c->vt;
        const uint8_t* bloom = B.hdr + c->bloom_off;
        auto probe = [&](const uint64_t* h, uint32_t nh) -> bool {
            if (nh == 0) return true;
            bloom_bytes += 8ull * nh;
            return bloom_contains_all_warp(bloom, c->bloom_words, h, nh);
        };
        const uint64_t* H = P.u64s + L.hashes_off; uint32_t nH = L.nhashes;
        if (vt == VT_STRING) {
            bool ok = true;
            if (L.kind == F_IN) {
                // matchBloomFilterAnyTokenSet filter_in.go:202-218
                ok = probe(H, L.nhashes);
                if (ok && !(L.in_skip_sets || (uint64_t)L.in_nsets > 10ull * rows)) {
                    bool any = false;
                    const uint32_t* sets = P.u32s + L.in_sets_off;
                    for (uint32_t s = 0; s < L.in_nsets && !any; s++) { bloom_bytes += 8ull * sets[2 * s + 1]; any = bloom_contains_all_warp(bloom, c->bloom_words, P.u64s + sets[2 * s], sets[2 * s + 1]); }
                    ok = any;
                }
            } else if (L.kind == F_CONTAINS_ANY) {
                // matchValuesAnyPhrase filter_contains_any.go:170-189: the common tokens, then EVERY phrase's own tokens (the reference keeps the
                // phrases that pass; a phrase that does not pass cannot match a row, so trying all of them on the rows gives the same bits)
                ok = probe(H, L.nhashes);
                if (ok) {
                    bool any = false;
                    const uint32_t* sets = P.u32s + L.in_sets_off;
                    for (uint32_t s = 0; s < L.in_nsets; s++) { bloom_bytes += 8ull * sets[2 * s + 1]; any |= bloom_contains_all_warp(bloom, c->bloom_words, P.u64s + sets[2 * s], sets[2 * s + 1]); }
                    ok = any;
                }
            } else if (L.kind == F_ANY_CASE_PHRASE || L.kind == F_ANY_CASE_PREFIX || L.kind == F_RANGE) ok = true;   // i(...): tokens are case sensitive, range(): no tokens - no probe
            else ok = probe(H, L.nhashes);
            if (!ok) act = ACT_NONE;
            else if (need) { act = ACT_ROW; values_bytes = 1; }   // probe: the values would be read
            else if (c->data_const) act = leaf_match_string(P, L, B.arena + c->data_off, (uint32_t)c->data_len) ? ACT_ALL : ACT_NONE, values_bytes = 1;
            else {
                act = L.str_strategy == STR_SCAN ? ACT_SCAN : L.str_strategy == STR_ALL ? ACT_ALL : ACT_ROW; values_bytes = 1;
                // short rows (ids, paths, codes ...): candidates of the row-agnostic scan become dense relative to the bytes streamed and
                // each costs a warp-wide verification, so such blocks take the per-row matcher instead (same predicate, same result)
                if (act == ACT_SCAN && c->data_len < (uint64_t)VL_SHORT_ROW_BYTES * rows) act = ACT_ROW;
                // few rows of the block are still selected (an earlier filter of an AND chain was selective): visit just those, like
                // bm.forEachSetBit does, instead of streaming the whole block
                if (act == ACT_SCAN && (uint64_t)ones * 16 < rows) act = ACT_ROW;
            }
        } else {
            // numeric / ipv4 / iso8601 columns
            uint32_t w = width_of_vt(vt);
            bool fixed_ok = c->lens_type >= 4 && c->lens_const == w && c->data_len == (uint64_t)rows * w && !c->data_const;
            const TypedNeedle& tn = L.typed[vt];
            // i(phrase) / i(prefix*) on typed columns: the phrase / prefix filter's path with the lower-cased needle and this filter's tokens; on
            // iso8601 columns the upper-cased needle and tokens (filter_any_case_phrase.go:103-126)
            uint32_t kind = L.kind;
            if (kind == F_ANY_CASE_PHRASE || kind == F_ANY_CASE_PREFIX) {
                kind = kind == F_ANY_CASE_PHRASE ? F_PHRASE : F_PREFIX;
                if (vt == VT_ISO8601) { H = P.u64s + L.hashes2_off; nH = L.nhashes2; nd = P.blob + L.needle2_off; nl = L.needle2_len; }
            }
            auto in_range = [&]() -> bool {
                switch (vt) {
                case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: case VT_IPV4: return tn.val >= c->min_value && tn.val <= c->max_value;
                case VT_INT64: case VT_ISO8601: return tn.sval >= (int64_t)c->min_value && tn.sval <= (int64_t)c->max_value;
                case VT_FLOAT64: { double f = __longlong_as_double((long long)tn.val), mn = __longlong_as_double((long long)c->min_value), mx = __longlong_as_double((long long)c->max_value); return !(f < mn) && !(f > mx); }
                }
                return false;
            };
            auto exact_path = [&]() {   // match*ByExactValue -> matchBinaryValue (filter_exact.go:237-364)
                if (!tn.ok || !in_range()) { act = ACT_NONE; return; }
                if (!probe(H, nH)) { act = ACT_NONE; return; }
                act = fixed_ok ? ACT_FIXED_EQ : ACT_ROW_EQ; pay = tn.val;
            };
            auto tostring_path = [&](bool use_bloom) {
                if (use_bloom && !probe(H, nH)) { act = ACT_NONE; return; }
                act = ACT_ROW;
            };
            const bool is_uintN = vt == VT_UINT8 || vt == VT_UINT16 || vt == VT_UINT32 || vt == VT_UINT64;
            switch (kind) {
            case F_EXACT: exact_path(); break;
            case F_PHRASE:
                if (vt == VT_FLOAT64) { if (!L.f64_phrase_gate) act = ACT_NONE; else if (L.f64_exact_form) exact_path(); else tostring_path(true); }
                else if (vt == VT_IPV4 || vt == VT_ISO8601) { if (tn.ok) exact_path(); else tostring_path(true); }
                else exact_path();
                break;
            case F_PREFIX:
                if (nl == 0) act = ACT_ALL;
                else if (vt == VT_UINT8 || vt == VT_UINT16 || vt == VT_UINT32 || vt == VT_UINT64) { if (!tn.ok || tn.val > c->max_value) act = ACT_NONE; else tostring_path(false); }
                else if (vt == VT_INT64) { bool dash = nl == 1 && nd[0] == '-'; if (!dash && (!tn.ok || !in_range())) act = ACT_NONE; else tostring_path(false); }
                else if (vt == VT_FLOAT64) { if (!L.f64_prefix_gate) act = ACT_NONE; else tostring_path(true); }
                else tostring_path(true);
                break;
            case F_REGEXP: tostring_path(true); break;
            case F_IN:
                if (L.in_typed_cnt[vt] == 0) act = ACT_NONE;
                else {
                    bool ok = probe(H, L.nhashes);
                    if (ok && !(L.in_skip_sets || (uint64_t)L.in_nsets > 10ull * rows)) {
                        bool any = false;
                        const uint32_t* sets = P.u32s + L.in_sets_off;
                        for (uint32_t s = 0; s < L.in_nsets && !any; s++) { bloom_bytes += 8ull * sets[2 * s + 1]; any = bloom_contains_all_warp(bloom, c->bloom_words, P.u64s + sets[2 * s], sets[2 * s + 1]); }
                        ok = any;
                    }
                    act = !ok ? ACT_NONE : fixed_ok ? ACT_FIXED_IN : ACT_ROW_IN;
                }
                break;
            case F_SEQUENCE:         // filter_sequence.go:139-258
                if (is_uintN || vt == VT_INT64) { if (L.in_count > 1) act = ACT_NONE; else exact_path(); }          // one phrase: the exact value
                else if (vt == VT_FLOAT64) tostring_path(true);
                else if (L.in_count == 1 && tn.ok) exact_path();                                                  // ipv4 / iso8601, one phrase that is a whole value
                else tostring_path(true);
                break;
            case F_CONTAINS_ALL:     // filter_contains_all.go:168-189 (matchAllValues), :191-300
                if (is_uintN) {
                    const uint32_t n_values = (uint32_t)L.aux0;   // distinct non-empty values
                    if (n_values == 0) act = ACT_ALL;
                    else if (n_values != 1 || L.in_typed_cnt[vt] != 1) act = ACT_NONE;
                    else if (!probe(H, nH)) act = ACT_NONE;
                    else { act = fixed_ok ? ACT_FIXED_EQ : ACT_ROW_EQ; pay = P.u64s[L.in_typed_off[vt]]; }
                } else tostring_path(true);
                break;
            case F_CONTAINS_ANY:     // filter_contains_any.go:120-168: uintN like in(), the rest like the strings path over the value's text
                if (is_uintN) {
                    if (L.in_typed_cnt[vt] == 0) act = ACT_NONE;
                    else {
                        bool ok = probe(H, nH);
                        if (ok && !(L.in_skip_sets || (uint64_t)L.in_nsets > 10ull * rows)) {
                            bool any = false;
                            const uint32_t* sets = P.u32s + L.in_sets_off;
                            for (uint32_t s = 0; s < L.in_nsets && !any; s++) { bloom_bytes += 8ull * sets[2 * s + 1]; any = bloom_contains_all_warp(bloom, c->bloom_words, P.u64s + sets[2 * s], sets[2 * s + 1]); }
                            ok = any;
                        }
                        act = !ok ? ACT_NONE : fixed_ok ? ACT_FIXED_IN : ACT_ROW_IN;
                    }
                } else {
                    bool ok = probe(H, nH);
                    if (ok) {
                        bool any = false;
                        const uint32_t* sets = P.u32s + L.in_sets_off;
                        for (uint32_t s = 0; s < L.in_nsets; s++) { bloom_bytes += 8ull * sets[2 * s + 1]; any |= bloom_contains_all_warp(bloom, c->bloom_words, P.u64s + sets[2 * s], sets[2 * s + 1]); }
                        ok = any;
                    }
                    act = ok ? ACT_ROW : ACT_NONE;
                }
                break;
            case F_RANGE: {          // match*ByRange filter_range.go:216-347: header min / max first, then the encoded values themselves
                const double fmn = __longlong_as_double((long long)L.rng_fmin), fmx = __longlong_as_double((long long)L.rng_fmax);
                if (is_uintN) act = (fmx < 0 || L.rng_ulo > c->max_value || L.rng_uhi < c->min_value) ? ACT_NONE : ACT_ROW;
                else if (vt == VT_INT64) act = (L.rng_ilo > (int64_t)c->max_value || L.rng_ihi < (int64_t)c->min_value) ? ACT_NONE : ACT_ROW;
                else if (vt == VT_FLOAT64) act = (fmn > __longlong_as_double((long long)c->max_value) || fmx < __longlong_as_double((long long)c->min_value)) ? ACT_NONE : ACT_ROW;
                else if (vt == VT_IPV4) act = (c->min_value > (uint64_t)L.rng_iphi || c->max_value < (uint64_t)L.rng_iplo) ? ACT_NONE : ACT_ROW;
                else act = (fmx < 0 || L.rng_ilo > (int64_t)c->max_value || L.rng_ihi < (int64_t)c->min_value) ? ACT_NONE : ACT_ROW;   // iso8601: nanoseconds
                break;
            }
            case F_EXACT_PREFIX: {   // match*ByExactPrefix filter_exact_prefix.go:105-273
                const bool is_uint = vt == VT_UINT8 || vt == VT_UINT16 || vt == VT_UINT32 || vt == VT_UINT64;
                if (nl == 0) act = ACT_ALL;
                else if (is_uint) act = (L.nhashes > 0 || !tn.ok || tn.val > c->max_value) ? ACT_NONE : ACT_ROW;   // matchMinMaxExactPrefix
                else if (vt == VT_INT64) {
                    bool dash = nl == 1 && nd[0] == '-';
                    if (L.nhashes > 0) act = ACT_NONE;
                    else if (!dash && (!tn.ok || tn.sval > (int64_t)c->max_value || tn.sval < (int64_t)c->min_value)) act = ACT_NONE;
                    else act = ACT_ROW;
                }
                else if (vt == VT_FLOAT64) act = (L.nhashes > 2 * 6 || !probe(H, L.nhashes)) ? ACT_NONE : ACT_ROW;
                else if (vt == VT_IPV4) act = (!(L.gates & GATE_DIGIT_PREFIX) || L.nhashes > 3 * 6 || !probe(H, L.nhashes)) ? ACT_NONE : ACT_ROW;
                else act = (!(L.gates & GATE_DIGIT_PREFIX) || !probe(H, L.nhashes)) ? ACT_NONE : ACT_ROW;   // iso8601
                break;
            }
            case F_LEN_RANGE: {      // match*ByLenRange filter_len_range.go:209-348
                const uint64_t mn = L.aux0, mx = L.aux1;
                uint8_t tmp[24];
                if (vt == VT_UINT8 || vt == VT_UINT16 || vt == VT_UINT32 || vt == VT_UINT64) {
                    const uint64_t maxd = vt == VT_UINT8 ? 3 : vt == VT_UINT16 ? 5 : vt == VT_UINT32 ? 10 : 20;
                    if (mn > maxd || mx == 0) act = ACT_NONE;
                    else if (mx < (uint64_t)fmt_u64(tmp, c->min_value) || mn > (uint64_t)fmt_u64(tmp, c->max_value)) act = ACT_NONE;   // matchMinMaxValueLen
                    else act = ACT_ROW;
                } else if (vt == VT_INT64) {
                    if (mn > 21 || mx == 0) act = ACT_NONE;
                    else { int a = fmt_i64(tmp, (int64_t)c->min_value), b2 = fmt_i64(tmp, (int64_t)c->max_value); act = (uint64_t)(a > b2 ? a : b2) < mn ? ACT_NONE : ACT_ROW; }
                } else if (vt == VT_FLOAT64) act = (mn > 24 || mx == 0) ? ACT_NONE : ACT_ROW;
                else if (vt == VT_IPV4) act = (mn > 15 || mx < 7) ? ACT_NONE : ACT_ROW;
                else act = (mn > 24 || mx < 24) ? ACT_NONE : ACT_ALL;   // iso8601: every value is 24 characters long, nothing is read
                break;
            }
            case F_STRING_RANGE:     // match*ByStringRange filter_string_range.go:88-224
                if (vt == VT_INT64) act = (L.gates & GATE_SR_INT) ? ACT_ROW : ACT_NONE;
                else if (vt == VT_FLOAT64) act = (L.gates & GATE_SR_FLOAT) ? ACT_ROW : ACT_NONE;
                else act = (L.gates & GATE_SR_UINT) ? ACT_ROW : ACT_NONE;
                break;
            case F_IPV4_RANGE:       // filter_ipv4_range.go:113-131, matchIPv4ByRange :176-191
                if (vt != VT_IPV4) act = ACT_NONE;
                else act = (c->min_value > L.aux1 || c->max_value < L.aux0) ? ACT_NONE : ACT_ROW;
                break;
            }
        }
        if (act >= ACT_DICT || values_bytes) values_bytes = lens_stored_bytes(*c, rows) + c->data_len;   // getValuesForColumn was reached
    }
    if (c && c->kind == COL_VALUES && c->vt == VT_DICT && act == ACT_DICT) values_bytes = lens_stored_bytes(*c, rows) + c->data_len;
    if (need) {
        if (c && c->kind == COL_VALUES && (values_bytes || act >= ACT_DICT) && lane_id() == 0) need[(uint64_t)b * B.nfields + slot] = 1;
        act = ACT_NONE; values_bytes = 0; bloom_bytes = 0; err = 0;
    } else if (c && c->kind == COL_VALUES && c->values_state != VALUES_STAGED && (values_bytes || act >= ACT_DICT)) {
        // cannot happen unless the probe pass and this dispatch disagree: fail loudly rather than read values that were never uploaded
        act = ACT_NONE; values_bytes = 0; err = ERR_VALUES_ABSENT;
    }
    if (c && c->kind == COL_VALUES && (act == ACT_SCAN || act >= ACT_ROW)) {
        need_lens = 1;
        if (act == ACT_SCAN) { ntiles = (uint32_t)((c->data_len + VL_TILE_BYTES - 1) / VL_TILE_BYTES); scan_bytes = c->data_len; scan_off = c->data_off; }
        else need_row = 1;
    }
    }
    if (need) return;   // probe pass: uniform for the whole grid
    if (lane_id() == 0) {
        if (valid) { action[b] = act; payload[b] = pay; }
        if (err) atomicMax(&stats[ST_ERROR], (unsigned long long)err);
        s_cnt[warp][0] = need_lens; s_cnt[warp][1] = ntiles; s_cnt[warp][2] = need_row;
        s_stat[warp][0] = bloom_bytes; s_stat[warp][1] = values_bytes; s_stat[warp][2] = values_bytes ? 1 : 0; s_stat[warp][3] = scan_bytes;
    }
    __syncthreads();
    if (threadIdx.x < 3) {            // one atomic per CTA and list
        uint32_t tot = 0;
        for (int w = 0; w < VL_PLAN_WARPS; w++) { s_off[w][threadIdx.x] = tot; tot += s_cnt[w][threadIdx.x]; }
        const uint32_t base = tot ? atomicAdd(&work_count[threadIdx.x], tot) : 0;
        for (int w = 0; w < VL_PLAN_WARPS; w++) s_off[w][threadIdx.x] += base;
    } else if (threadIdx.x >= 32 && threadIdx.x < 36) {
        const int k = threadIdx.x - 32;
        unsigned long long tot = 0;
        for (int w = 0; w < VL_PLAN_WARPS; w++) tot += s_stat[w][k];
        if (tot) atomicAdd(&stats[k == 0 ? ST_BLOOM_BYTES : k == 1 ? ST_VALUES_BYTES : k == 2 ? ST_COLUMNS_READ : ST_SCAN_BYTES], tot);
    }
    __syncthreads();
    if (need_lens && lane_id() == 0) lens_blocks[s_off[warp][0]] = b;
    if (need_row && lane_id() == 0) row_blocks[s_off[warp][2]] = b;
    for (uint32_t k = lane_id(); k < ntiles; k += 32) {
        const uint32_t t0 = k * VL_TILE_BYTES;
        tiles[s_off[warp][1] + k] = ScanTile{scan_off + t0, (uint32_t)min(scan_bytes - t0, (unsigned long long)VL_TILE_BYTES), b};
    }
}

// ---- on-disk columns: header checks of the lens block (unmarshalUint64Items, encoding.go:246-336) once the device has regenerated it ----
// The uint block type byte sits right in front of the lens items (lens_off - 1).  status[0] = max error code.
struct OndiskCol { uint64_t col; uint64_t lens_total; uint64_t rows; };
static __global__ void k_finish_ondisk_cols(const uint8_t* __restrict__ arena, DevColumn* __restrict__ cols, const OndiskCol* __restrict__ oc, uint32_t n,
                                            unsigned long long* __restrict__ status) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    DevColumn& c = cols[oc[i].col];
    const uint64_t total = oc[i].lens_total, rows = oc[i].rows;
    unsigned err = 0;
    if (total < 1) err = 1;
    else {
        const uint8_t* p = arena + c.lens_off - 1;
        uint32_t lt = p[0];
        if (lt > 7) err = 2;
        else {
            uint64_t want = lt < 4 ? (rows << lt) : (1ull << (lt - 4));
            if (total - 1 != want) err = 3;
            else {
                c.lens_type = (uint8_t)lt;
                if (lt >= 4) {
                    uint64_t v = 0; for (uint64_t k = 0; k < want; k++) v = (v << 8) | p[1 + k];
                    if (v > 0xFFFFFFFFull) err = 4;
                    else { c.lens_const = (uint32_t)v; c.data_const = (rows >= 2 && c.data_len == v) ? 1 : 0; }   // encoding.go:113-120
                }
            }
        }
    }
    if (err) atomicMax(&status[0], (unsigned long long)err);
}
// ---- late staging of a kept batch (vlscan_stage_selected) ------------------------------------------------------------------------------
// the column table entries of the cells staged by one call
struct ColPatch { uint64_t col; DevColumn c; };
static __global__ void k_patch_cols(DevColumn* __restrict__ cols, const ColPatch* __restrict__ p, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cols[p[i].col] = p[i].c;
}
// *count += the blocks with marks[b] != 0 whose column `slot` is a values column without its values on the device
static __global__ void k_unstaged_count(BatchView B, const uint32_t* __restrict__ marks, int slot, unsigned long long* __restrict__ count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || marks[b] == 0) return;
    const DevColumn& c = B.cols[(uint64_t)b * B.nfields + slot];
    if (c.kind == COL_VALUES && c.values_state != VALUES_STAGED) atomicAdd(count, 1ull);
}

// ---- lens decode -> byte offset of every 8th row (unmarshalUint64Items + the offsets implied by encoding.go:122-130) --------------------
// row_off8[8 * w + g] = byte offset (within the block's data) of row 64 * (w - first word of the block) + 8 * g, for every bitmap word w of the
// block.  One warp per block of the lens work list, one lane per bitmap word.  Sums are taken in 64 bits: a lens block whose items do not add
// up to the data length (encoding.go:124-126) is reported, never wrapped into agreement.
static __global__ void k_lens_offsets(BatchView B, int slot, const uint32_t* __restrict__ lens_blocks, const uint32_t* __restrict__ work_count,
                               uint32_t* __restrict__ row_off8, uint8_t* __restrict__ ready, unsigned long long* __restrict__ stats, int wc_idx = WC_LENS) {
    // one WARP per block of the lens work list (a block of 2000..6400 rows has 32..100 bitmap words: a whole CTA per block left most of its
    // threads idle between barriers); lane = bitmap word, 32 words per step, the running sum travels in a register
    const uint32_t nwork = work_count[wc_idx];
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5, lane = lane_id();
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nwork; j += warps) {
        const uint32_t b = lens_blocks[j];
        if (ready[b]) continue;   // uniform per warp
        const DevColumn& c = B.cols[(uint64_t)b * B.nfields + slot];
        if (c.values_state != VALUES_STAGED) {   // a kept batch's cell whose values are still on the host: never read, never marked ready
            if (lane == 0) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_VALUES_ABSENT);
            continue;
        }
        const uint32_t rows = B.blk_rows[b];
        const uint64_t w0 = B.blk_word_off[b]; const uint32_t nw = (uint32_t)(B.blk_word_off[b + 1] - w0);
        const uint8_t* lens = B.arena + c.lens_off;
        if (c.lens_type >= 4) {   // one const item: nothing to decode, the consumers divide
            if (lane == 0) {
                if ((unsigned long long)rows * c.lens_const != c.data_len) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_LENS_MISMATCH);
                ready[b] = 1;
            }
            continue;
        }
        unsigned long long carry = 0;
        for (uint32_t base = 0; base < nw; base += 32) {
            const uint32_t w = base + lane;
            uint32_t g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            unsigned long long sum = 0;
            if (w < nw) {
                const uint32_t r0 = w * 64, r1 = min(rows, r0 + 64);
                if (c.lens_type == 0) {
                    if (r1 - r0 == 64) {   // 64 u8 lens = four 16-byte vectors (r0 is a multiple of 64; lens_off is 16-byte aligned)
                        const uint4* v = (const uint4*)(lens + r0);
#pragma unroll
                        for (int q = 0; q < 4; q++) { uint4 x = v[q]; g[2 * q] = __vsadu4(x.x, 0) + __vsadu4(x.y, 0); g[2 * q + 1] = __vsadu4(x.z, 0) + __vsadu4(x.w, 0); }
                    } else for (uint32_t r = r0; r < r1; r++) g[(r - r0) >> 3] += lens[r];
#pragma unroll
                    for (int q = 0; q < 8; q++) sum += g[q];
                } else {
                    unsigned long long g64[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                    for (uint32_t r = r0; r < r1; r++) g64[(r - r0) >> 3] += c.lens_type == 3 ? ld_be64(lens + 8 * (uint64_t)r) : (unsigned long long)row_len(c, lens, r);
#pragma unroll
                    for (int q = 0; q < 8; q++) { sum += g64[q]; g[q] = (uint32_t)min(g64[q], 0xFFFFFFFFull); }
                    if (sum > 0xFFFFFFFFull) sum = 0x100000000ull;   // cannot equal a data length (< 4 GiB); keeps the running sum from wrapping
                }
            }
            unsigned long long incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
            const unsigned long long excl = carry + incl - sum;
            if (w < nw) {
                uint32_t o = (uint32_t)min(excl, 0xFFFFFFFFull);
                uint4 a, bq;
                a.x = o; o += g[0]; a.y = o; o += g[1]; a.z = o; o += g[2]; a.w = o; o += g[3];
                bq.x = o; o += g[4]; bq.y = o; o += g[5]; bq.z = o; o += g[6]; bq.w = o;
                uint4* dst = (uint4*)(row_off8 + ((w0 + w) << 3));
                dst[0] = a; dst[1] = bq;
            }
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) {
            if (carry != c.data_len) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_LENS_MISMATCH);   // encoding.go:124-126
            ready[b] = 1;
        }
    }
}

// ---- the hot kernel: row-agnostic substring scan over the decoded strings payload -------------------------------------------------------
// Replaces bm.forEachSetBit(func(idx){ matchPhrase(values[idx], phrase) }) (filter_phrase.go:201-270, bitmap.go:128-153),
// matchPrefix (filter_prefix.go:318-352) and the strings.Index(literal) loop of regexutil (regex.go:162-212).
//
// Filter.  Every thread streams 16-byte vectors of the block's concatenated row bytes and looks only at ALIGNED 4-byte words.  An occurrence of
// the needle that starts at byte r (0..3) of some word leaves min(4 - r, L) of its bytes in that word and min(4, L - (4 - r)) in the next one;
// the host picks, per r, the word that carries more needle bytes and hands the kernel its (mask, pattern) pair and the distance `delta[r]` from
// that word back to the start of the occurrence.  A word of the stream that equals one of the four patterns under its mask is a candidate:
// <= 4 LOP3 + 4 ISETP per word, no funnel shifts, no bytes from the neighbour lane.  For needles of >= 7 bytes all four masks are full (every
// occurrence covers a whole aligned word) and the instantiation without masks is used.
//
// Verification.  Candidates are verified by the lane that found them, all lanes of a warp in parallel: full compare, byte offset -> row through
// row_off8 (interpolation guess, bracket check, binary search, then at most 8 lens items), rejection of occurrences that straddle a row, the
// boundary rules of the filter kind, atomicOr of the row's bit.  An occurrence in the reference's retry loop ("pos++; continue") is any
// occurrence, so occurrences are independent and order-free -- that is what makes the row-agnostic formulation exact.
struct ScanParams {
    uint32_t mode;            // SCAN_*
    uint32_t needle_off, needle_len;
    uint32_t pat[4], msk[4];  // per start alignment r: (word & msk[r]) == pat[r]
    int32_t delta[4];         // occurrence start = byte address of the matching word + delta[r]
    uint32_t nd16[4];         // the first 16 needle bytes (little-endian words), compared out of registers
    uint8_t starts_tok, ends_tok;
    int32_t regex;
};

static __device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {   // two aligned loads + a funnel shift; reads up to 7 bytes past p
    const uint32_t* a = (const uint32_t*)((uintptr_t)p & ~(uintptr_t)3);
    return __funnelshift_r(a[0], a[1], 8 * (uint32_t)((uintptr_t)p & 3));
}

// Verification of one candidate occurrence at byte `pos` of block b's data by a single lane.
static __device__ __forceinline__ void scan_verify_lane(const DevProgram& P, const BatchView& B, const DevColumn& c, const ScanParams& sp, uint32_t b,
                                                     const uint32_t* __restrict__ row_off8, uint32_t pos, uint64_t* __restrict__ leaf_bm) {
    // everything the chain below depends on is requested up front: column header fields, the block's row count and first bitmap word
    const uint8_t* data = B.arena + c.data_off;
    const uint32_t L = sp.needle_len, n = (uint32_t)c.data_len;
    const uint32_t lens_type = c.lens_type, lens_const = c.lens_const;
    const uint8_t* lens = B.arena + c.lens_off;
    const uint32_t rows = B.blk_rows[b];
    const uint64_t w0 = B.blk_word_off[b];
    if ((uint64_t)pos + L > n) return;
    // the filter only vouches for some of the L bytes.  Payloads keep >= 32 readable bytes past data_len, so whole words may be compared.
    {
        const uint32_t head = L < 16 ? L : 16;
#pragma unroll
        for (uint32_t k = 0; k < 16; k += 4) {
            if (k >= head) break;
            const uint32_t m = head - k >= 4 ? 0xFFFFFFFFu : (1u << (8 * (head - k))) - 1;
            if ((ld_u32_unaligned(data + pos + k) ^ sp.nd16[k >> 2]) & m) return;
        }
        const uint8_t* nd = P.blob + sp.needle_off;
        for (uint32_t k = 16; k < L; k++) if (data[pos + k] != nd[k]) return;
    }
    // byte offset -> row
    uint32_t r, off, len;
    if (lens_type >= 4) {
        len = lens_const;
        if (len == 0) return;
        r = pos / len; off = r * len;
        if (r >= rows) return;
    } else {
        const uint32_t* ro = row_off8 + (w0 << 3);
        const uint32_t n8 = (rows + 7) >> 3;
        // last group of 8 rows that starts at or before pos.  Row lengths of one block are close to uniform, so pos * n8 / n is almost always
        // within one group of the answer: check that bracket first, fall back to the whole range.
        uint32_t lo, hi;
        {
            const uint32_t g = min((uint32_t)(__uint2float_rz(pos) * __fdividef(__uint2float_rz(n8), __uint2float_rz(n))), n8 - 1);
            lo = g ? g - 1 : 0; hi = min(g + 1, n8 - 1);
            if (!(ro[lo] <= pos && (hi + 1 >= n8 || ro[hi + 1] > pos))) { lo = 0; hi = n8 - 1; }
        }
        while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (ro[mid] <= pos) lo = mid; else hi = mid - 1; }
        // the row holding pos is the LAST row whose start is <= pos (zero-length rows share a start with their successor)
        const uint32_t r0 = lo * 8, kmax = min(8u, rows - r0);
        uint32_t o = ro[lo];
        r = r0; off = o; len = 0;
        if (lens_type == 0) {
            const uint2 lw = *(const uint2*)(lens + r0);   // r0 is a multiple of 8 and lens_off is 16-byte aligned
            const uint64_t l8 = ((uint64_t)lw.y << 32) | lw.x;
            for (uint32_t k = 0; k < kmax && o <= pos; k++) { const uint32_t l = (uint32_t)(l8 >> (8 * k)) & 0xFF; r = r0 + k; off = o; len = l; o += l; }
        } else {
            for (uint32_t k = 0; k < kmax && o <= pos; k++) { const uint32_t l = row_len(c, lens, r0 + k); r = r0 + k; off = o; len = l; o += l; }
        }
        if (pos < off || pos - off >= len) return;
    }
    if ((uint64_t)off + len > n) return;   // malformed lens (reported by k_lens_offsets): never read outside the payload
    if (pos + L > off + len) return;       // the occurrence straddles a row boundary
    const uint8_t* s = data + off; const uint32_t p = pos - off;
    bool hit;
    switch (sp.mode) {
    case SCAN_PHRASE: hit = phrase_boundaries_ok(s, len, p, L, sp.starts_tok, sp.ends_tok); break;
    case SCAN_PREFIX: hit = phrase_boundaries_ok(s, len, p, L, sp.starts_tok, false); break;
    case SCAN_CONTAINS: hit = true; break;
    case SCAN_RX_DOTPLUS: hit = p + L < len; break;
    case SCAN_RX_TAIL: {   // the needle is the literal of a `PREFIX.*LITERAL` expression: it matches iff PREFIX occurs entirely before this occurrence
        const DevRegex& R = P.regexes[sp.regex];
        hit = find_bytes(s, p, P.blob + R.prefix_off, R.prefix_len, 0) >= 0;
        break;
    }
    default: {             // SCAN_RX_SUFFIX: the needle is the literal prefix, the remainder of the row goes through the suffix automaton
        const DevRegex& R = P.regexes[sp.regex];
        if (R.tail_len) hit = find_bytes(s + p + L, len - p - L, P.blob + R.tail_off, R.tail_len, 0) >= 0;   // suffix `.*LIT`
        else hit = dfa_run(R, P.blob, s + p + L, len - p - L);
        break;
    }
    }
    if (hit) atomicOr((unsigned long long*)&leaf_bm[w0 + (r >> 6)], 1ull << (r & 63));
}

#define VL_SCAN_THREADS 256
#define VL_SCAN_CTAS 4                         /* resident CTAs per SM the register budget is set for (__launch_bounds__) */
#define VL_SCAN_UNROLL 4                       /* independent 16-byte loads per thread and round */
#define VL_SCAN_ROUNDS 4                       /* rounds per tile */
#define VL_SCAN_STAGES 2                       /* rounds held in registers: STAGES - 1 rounds are in flight while one is evaluated */
#define VL_SCAN_ROUND_BYTES (VL_SCAN_THREADS * 16)
#define VL_SCAN_QSTRIDE (VL_TILE_BYTES / VL_SCAN_UNROLL)                          /* distance between a thread's loads of one round */
static_assert(VL_TILE_BYTES == VL_SCAN_ROUND_BYTES * VL_SCAN_UNROLL * VL_SCAN_ROUNDS, "tile size");
static_assert(VL_SCAN_ROUNDS % VL_SCAN_STAGES == 0 && VL_SCAN_STAGES >= 2, "every round of a tile uses the same register stage in every tile");

template <bool MASKED>
static __device__ __forceinline__ uint32_t scan_word_hits(uint32_t w, const ScanParams& sp) {   // bit r: the word matches pattern r
    if (MASKED) return (uint32_t)((w & sp.msk[0]) == sp.pat[0]) | (uint32_t)((w & sp.msk[1]) == sp.pat[1]) << 1 | (uint32_t)((w & sp.msk[2]) == sp.pat[2]) << 2 | (uint32_t)((w & sp.msk[3]) == sp.pat[3]) << 3;
    return (uint32_t)(w == sp.pat[0]) | (uint32_t)(w == sp.pat[1]) << 1 | (uint32_t)(w == sp.pat[2]) << 2 | (uint32_t)(w == sp.pat[3]) << 3;
}

// does any of the four words of v match one of the four (mask, pattern) pairs?  -> 0 / 1
template <bool MASKED>
static __device__ __forceinline__ uint32_t scan_vector_hit(const uint4& v, const ScanParams& sp) {
    uint32_t h;
    if (MASKED) {
        asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
            "lop3.b32 t, %1, %5, %9, 0x28;\n\tsetp.eq.u32 p, t, 0;\n\t"
            "lop3.b32 t, %1, %6, %10, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %1, %7, %11, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %1, %8, %12, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %2, %5, %9, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %2, %6, %10, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %2, %7, %11, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %2, %8, %12, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %3, %5, %9, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %3, %6, %10, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %3, %7, %11, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %3, %8, %12, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %4, %5, %9, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %4, %6, %10, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %4, %7, %11, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "lop3.b32 t, %4, %8, %12, 0x28;\n\tsetp.eq.or.u32 p, t, 0, p;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(h)
            : "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(sp.pat[0]), "r"(sp.pat[1]), "r"(sp.pat[2]), "r"(sp.pat[3]), "r"(sp.msk[0]), "r"(sp.msk[1]), "r"(sp.msk[2]), "r"(sp.msk[3]));
    } else {
        asm("{\n\t.reg .pred p;\n\t"
            "setp.eq.u32 p, %1, %5;\n\tsetp.eq.or.u32 p, %1, %6, p;\n\tsetp.eq.or.u32 p, %1, %7, p;\n\tsetp.eq.or.u32 p, %1, %8, p;\n\t"
            "setp.eq.or.u32 p, %2, %5, p;\n\tsetp.eq.or.u32 p, %2, %6, p;\n\tsetp.eq.or.u32 p, %2, %7, p;\n\tsetp.eq.or.u32 p, %2, %8, p;\n\t"
            "setp.eq.or.u32 p, %3, %5, p;\n\tsetp.eq.or.u32 p, %3, %6, p;\n\tsetp.eq.or.u32 p, %3, %7, p;\n\tsetp.eq.or.u32 p, %3, %8, p;\n\t"
            "setp.eq.or.u32 p, %4, %5, p;\n\tsetp.eq.or.u32 p, %4, %6, p;\n\tsetp.eq.or.u32 p, %4, %7, p;\n\tsetp.eq.or.u32 p, %4, %8, p;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(h)
            : "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(sp.pat[0]), "r"(sp.pat[1]), "r"(sp.pat[2]), "r"(sp.pat[3]));
    }
    return h;
}

// Candidates are not verified where they are found.  A lane whose 16-byte vector holds a candidate word appends (block, byte position of the
// VECTOR) to a queue in shared memory and goes on streaming; out of the queue, the CTA's 256 threads take one vector each, re-read it (it is
// still in L2), enumerate its candidate words / alignments and verify them.  Verifying in place costs a chain of ~6 dependent memory round trips
// (column header, row offsets, lens items, neighbouring bytes) during which the other 31 lanes of the warp wait; in the drain all lanes are
// busy and the chains overlap.  The streaming side does not enumerate the candidates itself (4 compares on each of a lane's 16 words, by
// every lane of a warp in which ANY lane had a hit): at dense selectivities that enumeration dominates the kernel's instructions.  It only ballots which lanes have a hit in each of their four vectors and reserves queue
// slots with one shared-memory atomic per vector index.  The queue is drained when a tile ends with at least VL_SCAN_QFLUSH entries, and when
// the CTA has run out of tiles.  A vector that finds the queue full is handled by its lane on the spot.
#define VL_SCAN_QCAP 2048
#define VL_SCAN_QFLUSH 192
// pos: the low 32 bits of the arena byte offset of a 16-byte vector.  Offsets inside one column's data are < 4 GiB, so the drain gets the
// vector's offset inside the block's data back exactly as pos - (uint32_t)data_off (mod 2^32) without the streaming side reading the column.
struct ScanCand { uint32_t block, pos; };

// all candidates of one vector: word i matches pattern r => an occurrence may start at pos + 4 i + delta[r]
template <bool MASKED>
static __device__ __forceinline__ void scan_vector(const DevProgram& P, const BatchView& B, const DevColumn& c, const ScanParams& sp, uint32_t b,
                                                    const uint32_t* __restrict__ row_off8, uint32_t pos, uint64_t* __restrict__ leaf_bm) {
    const uint32_t n = (uint32_t)c.data_len;
    // vectors past the end of the data were streamed as zeros; a zero word can only match a pattern of NUL bytes, rejected by the bounds below
    const uint4 v = pos < n ? __ldg((const uint4*)(B.arena + c.data_off + pos)) : make_uint4(0, 0, 0, 0);
    // All candidates of the vector are collected first (bit 4 i + r: word i matches pattern r) and verified in ONE loop: with the verification
    // nested inside the loop over the words, the lanes of a draining warp - each with its candidate in a different word - took turns through four
    // copies of it, a quarter of the lanes at a time (ncu at 50 % candidate rows: 7.6 active lanes per instruction, 60 % of all instructions).
    uint32_t m = scan_word_hits<MASKED>(v.x, sp) | scan_word_hits<MASKED>(v.y, sp) << 4 | scan_word_hits<MASKED>(v.z, sp) << 8 | scan_word_hits<MASKED>(v.w, sp) << 12;
    while (m) {
        const int j = __ffs((int)m) - 1; m &= m - 1;
        const int64_t q = (int64_t)pos + (j & ~3) + sp.delta[j & 3];
        if (q < 0 || q + (int64_t)sp.needle_len > (int64_t)n) continue;
        scan_verify_lane(P, B, c, sp, b, row_off8, (uint32_t)q, leaf_bm);
    }
}

// This thread's VL_SCAN_UNROLL vectors of one round of a tile, 16 KiB apart (a warp's requests spread over more L2 slices / HBM channels than
// adjacent 4 KiB slices would).  A round that lies wholly inside the tile (every round of a full tile) loads at immediate offsets from one
// pointer without predicates; a round that holds the end of a block's last tile checks each vector and streams the ones past the end as zeros
// (a zero word can only match a pattern of NUL bytes, rejected by the bounds in scan_vector).  A record with bytes == 0 loads nothing.
static __device__ __forceinline__ void scan_load_round(uint4 (&v)[VL_SCAN_UNROLL], const BatchView& B, const ScanTile& tl, int round) {
    const uint32_t base = (uint32_t)round * VL_SCAN_ROUND_BYTES + threadIdx.x * 16;
    const uint8_t* __restrict__ ptr = B.arena + tl.off + base;
    if ((uint32_t)(round + 1) * VL_SCAN_ROUND_BYTES + (VL_SCAN_UNROLL - 1) * VL_SCAN_QSTRIDE <= tl.bytes) {   // uniform
#pragma unroll
        for (int u = 0; u < VL_SCAN_UNROLL; u++) v[u] = __ldg((const uint4*)(ptr + u * VL_SCAN_QSTRIDE));
    } else {
        // payloads keep >= 32 readable bytes past data_len: a vector load that starts inside the tile is always in bounds
#pragma unroll
        for (int u = 0; u < VL_SCAN_UNROLL; u++) v[u] = base + u * VL_SCAN_QSTRIDE < tl.bytes ? __ldg((const uint4*)(ptr + u * VL_SCAN_QSTRIDE)) : make_uint4(0, 0, 0, 0);
    }
}

// Filter of one round and queueing of its candidate vectors.  `pos` = low 32 bits of the arena offset of the thread's first vector of the
// round.  Returns true when this lane had a candidate vector that found the queue full.
// The queueing code is inline on purpose: with a call inside the stream ptxas parks the loop state in local memory around every round.
template <bool MASKED>
static __device__ __forceinline__ bool scan_round(const uint4 (&v)[VL_SCAN_UNROLL], const ScanParams& sp, uint32_t b, uint32_t pos, ScanCand* s_q, uint32_t* s_cnt) {
    static_assert(VL_SCAN_UNROLL == 4, "one ballot per vector index below");
    // bit u of `hits`: vector u holds a word equal to one of the four patterns (one predicate chain of 16 x setp.eq.or per vector)
    uint32_t hits = 0;
#pragma unroll
    for (int u = 0; u < VL_SCAN_UNROLL; u++) hits |= scan_vector_hit<MASKED>(v[u], sp) << u;
    if (!__any_sync(0xffffffffu, hits != 0)) return false;
    // some lane has a candidate: the whole warp reserves queue slots with ONE shared-memory atomic per round (lane 0 adds the number of
    // candidate vectors of all four vector indices); a lane's slot = the warp's base + the vectors of lower indices + those of lower lanes
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t b0 = __ballot_sync(0xffffffffu, hits & 1), b1 = __ballot_sync(0xffffffffu, hits & 2), b2 = __ballot_sync(0xffffffffu, hits & 4), b3 = __ballot_sync(0xffffffffu, hits & 8);
    const uint32_t n0 = __popc(b0), n1 = n0 + __popc(b1), n2 = n1 + __popc(b2), n3 = n2 + __popc(b3);
    uint32_t at0 = 0;
    if (lane == 0) at0 = atomicAdd(s_cnt, n3);
    at0 = __shfl_sync(0xffffffffu, at0, 0);
    const uint32_t below = (1u << lane) - 1u;
    const uint32_t bal[4] = {b0, b1, b2, b3}, first[4] = {at0, at0 + n0, at0 + n1, at0 + n2};
    bool overflow = false;
#pragma unroll
    for (int u = 0; u < VL_SCAN_UNROLL; u++) {
        if (!(hits >> u & 1)) continue;
        const uint32_t at = first[u] + __popc(bal[u] & below);
        if (at < VL_SCAN_QCAP) s_q[at] = ScanCand{b, pos + u * VL_SCAN_QSTRIDE}; else overflow = true;
    }
    return overflow;
}

// The re-scan of a tile whose candidate vectors did not all fit the queue: every vector of the tile, candidates verified where they are found.
template <bool MASKED>
static __device__ __noinline__ void scan_tile_inplace(const DevProgram& P, const BatchView& B, int slot, const ScanParams& sp, const ScanTile tl,
                                                      const uint32_t* __restrict__ row_off8, uint64_t* __restrict__ leaf_bm) {
    const DevColumn& c = B.cols[(uint64_t)tl.block * B.nfields + slot];
    const uint32_t tile0 = (uint32_t)(tl.off - c.data_off);
    for (uint32_t p = threadIdx.x * 16; p < tl.bytes; p += VL_SCAN_ROUND_BYTES) scan_vector<MASKED>(P, B, c, sp, tl.block, row_off8, tile0 + p, leaf_bm);
}
template <bool MASKED>
static __device__ __noinline__ void scan_drain(const DevProgram& P, const BatchView& B, int slot, const ScanParams& sp, const uint32_t* __restrict__ row_off8,
                                               uint64_t* __restrict__ leaf_bm, const ScanCand* s_q, uint32_t count) {
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) {
        const ScanCand e = s_q[i];
        const DevColumn& c = B.cols[(uint64_t)e.block * B.nfields + slot];
        scan_vector<MASKED>(P, B, c, sp, e.block, row_off8, e.pos - (uint32_t)c.data_off, leaf_bm);
    }
}

static __device__ __forceinline__ ScanTile scan_tile_at(const ScanTile* __restrict__ tiles, uint32_t t, uint32_t ntiles) {   // bytes == 0: no tile
    if (t >= ntiles) return ScanTile{0, 0, 0};
    const uint4 r = __ldg((const uint4*)(tiles + t));
    return ScanTile{(uint64_t)r.y << 32 | r.x, r.z, r.w};
}

// Persistent grid: SMs (132 on an H100) x VL_SCAN_CTAS resident CTAs x 256 threads, each CTA strides over the tile list built by k_plan_leaf.
// A CTA's tiles form one software pipeline: the loads of the round VL_SCAN_STAGES - 1 ahead (near the end of a tile: of the next tile) go out
// before the current round is evaluated, the next tile's record is fetched a whole tile ahead, and the next tile's first rounds are in flight
// across the end-of-tile barrier and drain.
template <bool MASKED>
static __global__ void __launch_bounds__(VL_SCAN_THREADS, VL_SCAN_CTAS) k_substr_scan(const __grid_constant__ DevProgram P, const __grid_constant__ BatchView B, int slot, const __grid_constant__ ScanParams sp,
                                                                                      const ScanTile* __restrict__ tiles, const uint32_t* __restrict__ work_count,
                                                                                      const uint32_t* __restrict__ row_off8, uint64_t* __restrict__ leaf_bm) {
    __shared__ ScanCand s_q[VL_SCAN_QCAP];
    __shared__ uint32_t s_cnt, s_t, s_ntiles;
    __shared__ ScanTile s_next;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    uint32_t ntiles = work_count[WC_TILES];
    ScanTile cur = scan_tile_at(tiles, blockIdx.x, ntiles), next = scan_tile_at(tiles, blockIdx.x + gridDim.x, ntiles);
    uint4 v[VL_SCAN_STAGES][VL_SCAN_UNROLL];
#pragma unroll
    for (int s = 0; s < VL_SCAN_STAGES - 1; s++) scan_load_round(v[s], B, cur, s);
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        bool overflow = false;
#pragma unroll
        for (int r = 0; r < VL_SCAN_ROUNDS; r++) {
            const int ahead = r + VL_SCAN_STAGES - 1;
            if (ahead < VL_SCAN_ROUNDS) scan_load_round(v[ahead % VL_SCAN_STAGES], B, cur, ahead);
            else scan_load_round(v[ahead % VL_SCAN_STAGES], B, next, ahead - VL_SCAN_ROUNDS);
            overflow |= scan_round<MASKED>(v[r % VL_SCAN_STAGES], sp, cur.block, (uint32_t)cur.off + (uint32_t)r * VL_SCAN_ROUND_BYTES + threadIdx.x * 16, s_q, &s_cnt);
        }
        // end of the tile: drain the queue if it is worth a pass of the whole CTA (thread 0 decides; the barrier makes the decision uniform),
        // or if some candidate vector of this tile did not fit
        if (__syncthreads_or((threadIdx.x == 0 && s_cnt >= VL_SCAN_QFLUSH) || overflow)) {
            // No register of the stream lives across the calls below (the call ABI would park it in local memory): the loop state goes
            // through shared memory and the rounds already issued for the next tile are issued again afterwards.
            if (threadIdx.x == 0) { s_t = t; s_ntiles = ntiles; s_next = next; }
            // candidates that did not fit were dropped: the tile is gone over again with verification in place (bits are OR-ed, so the
            // candidates that did make it into the queue and are verified again below change nothing)
            if (__syncthreads_or(overflow)) scan_tile_inplace<MASKED>(P, B, slot, sp, cur, row_off8, leaf_bm);
            scan_drain<MASKED>(P, B, slot, sp, row_off8, leaf_bm, s_q, min(s_cnt, (uint32_t)VL_SCAN_QCAP));
            __syncthreads();
            if (threadIdx.x == 0) s_cnt = 0;
            t = s_t; ntiles = s_ntiles; next = s_next;
            __syncthreads();
#pragma unroll
            for (int s = 0; s < VL_SCAN_STAGES - 1; s++) scan_load_round(v[s], B, next, s);
        }
        cur = next;
        next = scan_tile_at(tiles, t + 2 * gridDim.x, ntiles);
    }
    __syncthreads();
    scan_drain<MASKED>(P, B, slot, sp, row_off8, leaf_bm, s_q, min(s_cnt, (uint32_t)VL_SCAN_QCAP));
}

// ---- dict LUT / fixed-width equality / typed in(): one thread per bitmap word ---------------------------------------------------------------
// matchEncodedValuesDict filter_phrase.go:272-289, matchBinaryValue filter_exact.go:356-364, matchAnyValue filter_in.go:187-200
static __global__ void k_word_match(DevProgram P, BatchView B, uint32_t leaf_idx, int slot, const uint8_t* __restrict__ action, const uint64_t* __restrict__ payload, const uint64_t* __restrict__ reg,
                             uint64_t* __restrict__ leaf_bm, unsigned long long* __restrict__ stats) {
    uint64_t gw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gw >= B.nwords) return;
    uint32_t b = B.word_block[gw];
    uint8_t act = action[b];
    if (act != ACT_DICT && act != ACT_FIXED_EQ && act != ACT_FIXED_IN) return;
    if (!reg[gw]) { leaf_bm[gw] = 0; return; }   // no selected row left in these 64 (bm.forEachSetBit visits none)
    const DevColumn& c = B.cols[(uint64_t)b * B.nfields + slot];
    const DevLeaf& L = P.leaves[leaf_idx];
    uint32_t rows = B.blk_rows[b];
    uint32_t r0 = (uint32_t)(gw - B.blk_word_off[b]) * 64, r1 = min(rows, r0 + 64);
    const uint8_t* data = B.arena + c.data_off;
    uint64_t bits = 0, pay = payload[b];
    if (act == ACT_DICT) {
        // dict ids: 1 byte per row; lens must be const 1 (or a per-row u8 block of ones for single-row blocks)
        bool bad = false;
        if (r1 - r0 == 64 && ((c.data_off + r0) & 15) == 0) {
            const uint4* v = (const uint4*)(data + r0);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                uint4 x = __ldg(v + q); uint32_t ww[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) { uint32_t id = (ww[i] >> (8 * j)) & 0xFF; bad |= id >= c.dict_len; bits |= (uint64_t)((pay >> (id & 7)) & 1) << (q * 16 + i * 4 + j); }
            }
        } else for (uint32_t r = r0; r < r1; r++) { uint32_t id = data[r]; bad |= id >= c.dict_len; bits |= (uint64_t)((pay >> (id & 7)) & 1) << (r - r0); }
        if (bad) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_DICT_INDEX);   // "too big index for dict value" filter_phrase.go:284-286
    } else {
        uint32_t w = width_of_vt(c.vt);
        for (uint32_t r = r0; r < r1; r++) {
            uint64_t v = load_fixed_be(data + (uint64_t)r * w, w);
            bool hit = act == ACT_FIXED_EQ ? v == pay : in_contains_typed(L, P.u64s, c.vt, v);
            bits |= (uint64_t)hit << (r - r0);
        }
    }
    leaf_bm[gw] = bits;
}

// ---- generic per-row matcher: one warp per bitmap word, lanes take rows l and l+32 ------------------------------------------------------------
// exact / in() / regexp-without-literal-prefix on string columns; numeric columns that must be formatted to text first.
// Persistent grid over the ACT_ROW work list of k_plan_leaf: work item j = block work_blocks[j]; its bitmap words are dealt out to the CTA's warps.
// The kernel is a chain of dependent loads per block and per bitmap word (work list -> column header -> register word -> lens -> row bytes), so it
// lives on resident warps: capped at 64 registers (4 CTAs per SM; the rarely taken predicates spill a little) it runs the `path:api*` leaf of C4
// in a quarter of the time it took with the 153 registers (1 CTA per SM) the compiler picks on its own.
static __global__ void __launch_bounds__(256, 4) k_row_match(DevProgram P, BatchView B, uint32_t leaf_idx, int slot, const uint32_t* __restrict__ work_blocks,
                                   const uint32_t* __restrict__ work_count, const uint8_t* __restrict__ action, const uint64_t* __restrict__ payload, const uint64_t* __restrict__ reg,
                                   const uint32_t* __restrict__ row_off8, uint64_t* __restrict__ leaf_bm) {
  if (work_count[WC_ROW] == 0) return;   // k_plan_leaf sent no block of the batch to the row matcher for this leaf
  const DevLeaf& L = P.leaves[leaf_idx];
  // Behind a selective filter of an AND chain most bitmap words are zero (like bm.forEachSetBit, bitmap.go:128-153, only rows that are still
  // selected are looked at).  A warp therefore reads 32 consecutive register words at once - one word per lane, coalesced - and goes through
  // the live ones among them one after the other; dead words cost 8 bytes of a coalesced load instead of a dependent round trip each.
  // (work_blocks, the block list, is not walked any more: the words of blocks with another action are dropped by the action test below.)
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5), warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (uint64_t base = warp * 32; base < B.nwords; base += nwarps * 32) {
    uint64_t live_l = 0; uint32_t b_l = 0;
    if (base + lane_id() < B.nwords) {
        live_l = reg[base + lane_id()];
        if (live_l) { b_l = B.word_block[base + lane_id()]; const uint8_t a = action[b_l]; if (a < ACT_ROW || a > ACT_ROW_IN) live_l = 0; }
    }
    uint32_t todo = __ballot_sync(0xffffffffu, live_l != 0);
   while (todo) {
    const int src = __ffs((int)todo) - 1; todo &= todo - 1;
    const uint64_t gw = base + (uint32_t)src;
    const uint64_t live = __shfl_sync(0xffffffffu, live_l, src);
    const uint32_t b = __shfl_sync(0xffffffffu, b_l, src);
    const DevColumn& c = B.cols[(uint64_t)b * B.nfields + slot];
    const uint32_t rows = B.blk_rows[b];
    const uint8_t act = action[b]; const uint64_t pay = payload[b];
    const uint64_t w_lo = B.blk_word_off[b];
    uint32_t r0 = (uint32_t)(gw - w_lo) * 64;
    const uint8_t* data = B.arena + c.data_off;
    const uint8_t* lens = B.arena + c.lens_off;
    uint32_t la = 0, lb = 0;
    uint32_t ra = r0 + lane_id(), rb = r0 + 32 + lane_id();
    if (ra < rows) la = row_len(c, lens, ra);
    if (rb < rows) lb = row_len(c, lens, rb);
    // exclusive offsets: rows r0..r0+31 then r0+32..r0+63
    uint32_t ia = la, ib = lb;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, ia, d), u = __shfl_up_sync(0xffffffffu, ib, d); if (lane_id() >= d) { ia += t; ib += u; } }
    uint32_t tot_a = __shfl_sync(0xffffffffu, ia, 31);
    uint64_t base = c.lens_type >= 4 ? (uint64_t)r0 * c.lens_const : row_off8[gw << 3];
    uint64_t oa = base + ia - la, ob = base + tot_a + ib - lb;
    if (c.data_const) { oa = ob = 0; la = lb = (uint32_t)c.data_len; }   // every row = data (encoding.go:113-120)
    bool ha = false, hb = false;
    uint32_t vt = c.vt;
    auto eval = [&](uint64_t off, uint32_t len) -> bool {
        if (off + len > c.data_len) return false;   // malformed; k_lens_offsets reports the error
        const uint8_t* s = data + off;
        if (vt == VT_STRING) return leaf_match_string(P, L, s, len);
        uint32_t w = width_of_vt(vt);
        if (len != w) return false;
        uint64_t raw = load_fixed_be(s, w);
        if (act == ACT_ROW_EQ) return raw == pay;                              // matchBinaryValue filter_exact.go:356-364
        if (act == ACT_ROW_IN) return in_contains_typed(L, P.u64s, vt, raw);   // matchAnyValue filter_in.go:187-200
        if (L.kind == F_IPV4_RANGE) return raw >= L.aux0 && raw <= L.aux1;     // only ipv4 columns get here (k_plan_leaf)
        if (L.kind == F_RANGE) {
            switch (vt) {
            case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: return raw >= L.rng_ulo && raw <= L.rng_uhi;
            case VT_INT64: { const int64_t v = unzigzag64(raw); return v >= L.rng_ilo && v <= L.rng_ihi; }
            case VT_FLOAT64: { const double f = __longlong_as_double((long long)raw); return f >= __longlong_as_double((long long)L.rng_fmin) && f <= __longlong_as_double((long long)L.rng_fmax); }
            case VT_IPV4: return raw >= L.rng_iplo && raw <= L.rng_iphi;
            default: return (int64_t)raw >= L.rng_ilo && (int64_t)raw <= L.rng_ihi;   // iso8601
            }
        }
        if (vt == VT_FLOAT64) return leaf_match_f64(P, L, raw);
        uint8_t buf[32];
        int n = encoded_to_string(vt, raw, buf);
        if (n < 0) return false;
        return leaf_match_typed_text(P, L, vt, buf, (uint32_t)n);
    };
    if (ra < rows && (live >> lane_id() & 1)) ha = eval(oa, la);
    if (rb < rows && (live >> (32 + lane_id()) & 1)) hb = eval(ob, lb);
    uint32_t lo = __ballot_sync(0xffffffffu, ha), hi = __ballot_sync(0xffffffffu, hb);
    if (lane_id() == 0) leaf_bm[gw] = ((uint64_t)hi << 32) | lo;
   }
  }
}

// ---- fold a leaf result into the running bitmap -------------------------------------------------------------------------------------------------
static __global__ void k_apply_leaf(BatchView B, const uint8_t* __restrict__ action, const uint64_t* __restrict__ leaf_bm, uint64_t* __restrict__ reg) {
    uint64_t gw = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gw >= B.nwords) return;
    uint8_t act = action[B.word_block[gw]];
    if (act == ACT_ALL) return;
    reg[gw] = act == ACT_NONE ? 0 : (reg[gw] & leaf_bm[gw]);
}

// ---- finalize: per-block popcount (bitmap.onesCount bitmap.go:185-191 == blockResult.rowsLen) + totals -------------------------------------------
static __global__ void __launch_bounds__(256) k_finalize(BatchView B, const uint64_t* __restrict__ reg, uint32_t* __restrict__ counts, unsigned long long* __restrict__ stats,
                           unsigned long long* __restrict__ totals4) {
    __shared__ unsigned long long s_acc[8][4];   // per warp: rows, rows matched, blocks matched, bitmap bytes
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t b = blockIdx.x * 8 + warp;
    unsigned long long rows = 0, matched = 0, blocks = 0, bm_bytes = 0;
    if (b < B.nblocks) {
        uint64_t lo = B.blk_word_off[b], hi = B.blk_word_off[b + 1];
        uint32_t n = 0;
        for (uint64_t w = lo + lane_id(); w < hi; w += 32) n += __popcll(reg[w]);
#pragma unroll
        for (int d = 16; d; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
        if (lane_id() == 0) counts[b] = n;
        rows = B.blk_rows[b];
        if (n) { matched = n; blocks = 1; bm_bytes = 8ull * (hi - lo); }
    }
    if (lane_id() == 0) { s_acc[warp][0] = rows; s_acc[warp][1] = matched; s_acc[warp][2] = blocks; s_acc[warp][3] = bm_bytes; }
    __syncthreads();
    if (threadIdx.x < 4) {   // one atomic per CTA and counter instead of six per block
        unsigned long long t = 0;
        for (int w = 0; w < 8; w++) t += s_acc[w][threadIdx.x];
        if (t) {
            if (threadIdx.x == 0) atomicAdd(&totals4[0], t);
            else if (threadIdx.x == 1) { atomicAdd(&stats[ST_ROWS_MATCHED], t); atomicAdd(&totals4[1], t); }
            else if (threadIdx.x == 2) { atomicAdd(&stats[ST_BLOCKS_MATCHED], t); atomicAdd(&totals4[2], t); }
            else atomicAdd(&stats[ST_BITMAP_BYTES], t);
        }
    }
}

// ---- hit-row offsets (bitmap.forEachSetBitReadonly bitmap.go:156-183) ----------------------------------------------------------------------------------
// Single CTA exclusive scan of n words into offs[0 .. n), their total into *total.  It also runs in place (in == offs: the tile sums of
// k_scan_tiles), so no pointer is __restrict__.
template <typename T>
static __global__ void k_scan_cta(const T* in, uint32_t n, uint64_t* offs, uint64_t* total) {
    __shared__ uint64_t s[1024];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        const uint64_t v = i < n ? in[i] : 0;
        s[threadIdx.x] = v;
        __syncthreads();
        for (uint32_t d = 1; d < blockDim.x; d <<= 1) { uint64_t a = threadIdx.x >= d ? s[threadIdx.x - d] : 0; __syncthreads(); s[threadIdx.x] += a; __syncthreads(); }
        if (i < n) offs[i] = carry + s[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry += s[threadIdx.x];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

// ---- timestamps column: encoding.UnmarshalTimestamps on the device (vm/lib/encoding/encoding.go:173-250, nearest_delta2.go:57-90, ------------
// nearest_delta.go, int.go:173-280) and filterTime (lib/logstorage/filter_time.go:114-137) ------------------------------------------------------
// One CTA per block.  The sequential decoder becomes three data-parallel steps (tests/test_timestamps_model_cpu.py proves them equal to it,
// malformed input included): (1) a byte ends a varint iff its continuation bit is clear, so the index of a varint is the number of such bytes in
// front of it (ballot + popcount, CTA running sum) and every varint is assembled from its <= 10 bytes independently; (2) NearestDelta: values =
// first + inclusive scan of the deltas; NearestDelta2: one more inclusive scan in front (deltas of deltas -> deltas), all sums mod 2^64 like Go's
// int64; (3) DeltaConst / Const need no scan.  vals[0 .. rows) receives the timestamps.  Returns false (CTA-uniform) on malformed input:
// a varint longer than 10 bytes or overflowing 64 bits, too few / too many varints, bytes left over.
static __device__ unsigned long long cta_incl_scan_u64(unsigned long long v, unsigned long long* s_warp, unsigned long long* s_carry) {   // all threads of the CTA; carries across calls
    unsigned long long incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane_id() >= d) incl += t; }
    const uint32_t wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane_id() == 31) s_warp[wid] = incl;
    __syncthreads();
    unsigned long long pre = *s_carry;
    for (uint32_t k = 0; k < wid; k++) pre += s_warp[k];
    unsigned long long tot = 0;
    for (uint32_t k = 0; k < nw; k++) tot += s_warp[k];
    __syncthreads();
    if (threadIdx.x == 0) *s_carry += tot;
    __syncthreads();
    return pre + incl;
}
static __device__ bool ts_decode_block(const BatchView& B, uint32_t b, unsigned long long* __restrict__ vals) {
    __shared__ unsigned long long s_warp[32];
    __shared__ unsigned long long s_carry;
    __shared__ uint32_t s_cnt[32];
    __shared__ uint32_t s_ccarry;
    __shared__ int s_bad;
    const DevTimestamps t = B.ts[b];
    const uint32_t R = B.blk_rows[b], len = t.len;
    const uint8_t* raw = B.arena + t.off;
    const unsigned long long first = (unsigned long long)t.first;
    if (threadIdx.x == 0) { s_bad = 0; s_ccarry = 0; s_carry = 0; }
    __syncthreads();
    if (t.mt == MT_CONST) {
        for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) vals[r] = first;
        return len == 0;
    }
    if (t.mt == MT_DELTA_CONST) {
        unsigned long long u = 0; bool ok = len >= 1 && len <= 10;
        if (ok) { for (uint32_t k = 0; k < len; k++) { const uint8_t c = raw[k]; if ((k + 1 < len) != (c >= 0x80)) ok = false; u |= (unsigned long long)(c & 0x7F) << (7 * k); } if (len == 10 && raw[9] > 1) ok = false; }
        const unsigned long long d = (u >> 1) ^ (0ull - (u & 1));
        for (uint32_t r = threadIdx.x; r < R; r += blockDim.x) vals[r] = first + (unsigned long long)r * d;
        return ok;
    }
    if (t.mt != MT_NEAREST_DELTA && t.mt != MT_NEAREST_DELTA2) return false;
    const uint32_t min_rows = t.mt == MT_NEAREST_DELTA2 ? 2u : 1u;
    if (R < min_rows) return false;
    const uint32_t need = R - 1;   // NearestDelta: one delta per row after the first; NearestDelta2: the first delta, then R - 2 deltas of deltas
    // (1) varints
    for (uint32_t base = 0; base < len; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        const uint8_t c = i < len ? raw[i] : 0x80;
        const bool is_end = i < len && c < 0x80;
        const uint32_t m = __ballot_sync(0xffffffffu, is_end);
        if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = __popc(m);
        __syncthreads();
        uint32_t k = s_ccarry + __popc(m & ((1u << lane_id()) - 1));
        for (uint32_t w = 0; w < (threadIdx.x >> 5); w++) k += s_cnt[w];
        if (is_end) {
            uint32_t s0 = i, n = 1;
            while (s0 > 0 && raw[s0 - 1] >= 0x80 && n <= 10) { s0--; n++; }
            unsigned long long u = 0;
            for (uint32_t q = 0; q < n && q < 10; q++) u |= (unsigned long long)(raw[s0 + q] & 0x7F) << (7 * q);
            if (n > 10 || (n == 10 && c > 1) || k >= need) s_bad = 1;
            else vals[1 + k] = (u >> 1) ^ (0ull - (u & 1));
        }
        __syncthreads();
        if (threadIdx.x == 0) { uint32_t tot = 0; for (uint32_t w = 0; w < (blockDim.x >> 5); w++) tot += s_cnt[w]; s_ccarry += tot; }
        __syncthreads();
    }
    if (threadIdx.x == 0 && (s_ccarry != need || (len > 0 && raw[len - 1] >= 0x80))) s_bad = 1;
    __syncthreads();
    if (s_bad) return false;
    // (2) prefix sums, in place
    for (int pass = t.mt == MT_NEAREST_DELTA2 ? 0 : 1; pass < 2; pass++) {
        if (threadIdx.x == 0) s_carry = pass == 1 ? first : 0;
        __syncthreads();
        for (uint32_t base = 0; base < need; base += blockDim.x) {
            const uint32_t i = base + threadIdx.x;
            const unsigned long long v = i < need ? vals[1 + i] : 0;
            const unsigned long long sum = cta_incl_scan_u64(v, s_warp, &s_carry);
            if (i < need) vals[1 + i] = sum;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) vals[0] = first;
    __syncthreads();
    return true;
}

// _time filter on the blocks it only partly covers (the ACT_TIME work list of k_plan_leaf): decode, compare, one 32-bit half of a bitmap word per warp
static __global__ void __launch_bounds__(256) k_time_match(BatchView B, long long mn, long long mx, const uint32_t* __restrict__ row_blocks, const uint32_t* __restrict__ work_count,
                                                            unsigned long long* __restrict__ ts_vals, uint64_t* __restrict__ leaf_bm, unsigned long long* __restrict__ stats) {
    const uint32_t nwork = work_count[WC_ROW];
    for (uint32_t j = blockIdx.x; j < nwork; j += gridDim.x) {
        const uint32_t b = row_blocks[j], R = B.blk_rows[b];
        const uint64_t w0 = B.blk_word_off[b];
        unsigned long long* vals = ts_vals + w0 * 64;
        const bool ok = ts_decode_block(B, b, vals);
        if (!ok && threadIdx.x == 0) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_BAD_TIMESTAMPS);
        const uint32_t rows_padded = (R + 63) / 64 * 64;
        for (uint32_t base = 0; base < rows_padded; base += blockDim.x) {
            const uint32_t r = base + threadIdx.x;
            const long long v = r < R ? (long long)vals[r] : 0;
            const uint32_t m = __ballot_sync(0xffffffffu, ok && r < R && v >= mn && v <= mx);
            if (lane_id() == 0 && r < rows_padded) ((uint32_t*)(leaf_bm + w0))[r >> 5] = m;   // little-endian halves of the 64-bit words
        }
        __syncthreads();
    }
}

// ---- hit materialisation: the selected rows' values and timestamps as blockResult would yield them -------------------------------------------
// (lib/logstorage/block_result.go:491-507 initTimestampsInternal, :529-591 the per-type readers behind getValues; values_encoder.go:1367-1422)
// hit h = (hit_block[h], hit_row[h]) in block order, rows ascending (k_hits_compact).
static __global__ void k_hits_compact(BatchView B, const uint64_t* __restrict__ reg, const uint64_t* __restrict__ offs, uint32_t* __restrict__ hits, uint32_t* __restrict__ hit_block, uint64_t cap) {
    uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B.nblocks) return;
    uint64_t lo = B.blk_word_off[b], hi = B.blk_word_off[b + 1];
    uint64_t out = offs[b];
    for (uint64_t w0 = lo; w0 < hi; w0 += 32) {
        uint64_t w = w0 + lane_id();
        uint64_t bits = w < hi ? reg[w] : 0;
        uint32_t n = __popcll(bits), incl = n;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane_id() >= d) incl += t; }
        uint64_t pos = out + incl - n;
        uint32_t rbase = (uint32_t)(w - lo) * 64;
        while (bits) { int k = __ffsll((long long)bits) - 1; bits &= bits - 1; if (pos < cap) { hits[pos] = rbase + k; hit_block[pos] = b; } pos++; }
        out += __shfl_sync(0xffffffffu, incl, 31);
    }
}
// blocks with hits -> work list: mode 0 = into the lens list those whose cell in column `slot` needs row offsets (cell_needs_offsets), mode 1 =
// into the row list every block with hits (timestamps decode)
static __global__ void k_hit_blocks_list(BatchView B, const uint32_t* __restrict__ counts, int slot, int mode, uint32_t* __restrict__ list, uint32_t* __restrict__ work_count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || counts[b] == 0) return;
    if (mode == 0) {
        if (slot < 0 || !cell_needs_offsets(B.cols[(uint64_t)b * B.nfields + slot])) return;
        list[atomicAdd(&work_count[WC_LENS], 1u)] = b;
    } else list[atomicAdd(&work_count[WC_ROW], 1u)] = b;
}
static __global__ void __launch_bounds__(256) k_ts_decode_list(BatchView B, const uint32_t* __restrict__ row_blocks, const uint32_t* __restrict__ work_count,
                                                                unsigned long long* __restrict__ ts_vals, unsigned long long* __restrict__ stats) {
    const uint32_t nwork = work_count[WC_ROW];
    for (uint32_t j = blockIdx.x; j < nwork; j += gridDim.x) {
        const uint32_t b = row_blocks[j];
        const bool ok = B.ts && B.ts[b].mt && ts_decode_block(B, b, ts_vals + B.blk_word_off[b] * 64);
        if (!ok && threadIdx.x == 0) atomicMax(&stats[ST_ERROR], (unsigned long long)(B.ts && B.ts[b].mt ? ERR_BAD_TIMESTAMPS : ERR_NO_TIMESTAMPS));
        __syncthreads();
    }
}
static __global__ void k_gather_ts(BatchView B, const uint32_t* __restrict__ hits, const uint32_t* __restrict__ hit_block, uint64_t nhits, const unsigned long long* __restrict__ ts_vals,
                                   long long* __restrict__ out) {
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h < nhits) out[h] = (long long)ts_vals[B.blk_word_off[hit_block[h]] * 64 + hits[h]];
}
// ---- the reader of one cell: row r of a column in block b as blockResultColumn.getValues yields it -----------------------------------------------
// Three layers: the encoded bytes of a values cell (cell_raw), its text without formatting (cell_text_raw), its text (cell_text).  Each returns
// an ERR_* code and raises nothing: its caller reports the code with one atomicMax.  row_off8: k_lens_offsets of the cell's slot, built for
// every block with hits whose cell has per-row lens items (cell_needs_offsets).
static __device__ __forceinline__ bool cell_typed(const DevColumn* c) { return c && c->kind == COL_VALUES && c->vt != VT_STRING && c->vt != VT_DICT; }
static __device__ __forceinline__ const DevColumn* cell_at(const BatchView& B, int slot, uint32_t b) { return slot >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot] : nullptr; }
static __device__ __forceinline__ void report_error(unsigned long long* stats, uint32_t err) { if (err) atomicMax(&stats[ST_ERROR], (unsigned long long)err); }
// The encoded bytes of row r of a values cell: the whole payload when every row is that one value (rows >= 2, const lens equal to the data
// length, encoding.go:113-120), else the row's slice by its const or per-row lens item.  A payload that is not on the device (a kept batch
// before vlscan_stage_selected) is ERR_VALUES_ABSENT.
static __device__ __forceinline__ uint32_t cell_raw(const BatchView& B, const DevColumn& c, uint32_t b, uint32_t r, const uint32_t* __restrict__ row_off8, const uint8_t** p, uint32_t* n) {
    if (c.values_state != VALUES_STAGED) return ERR_VALUES_ABSENT;
    uint64_t off = 0; uint32_t len;
    if (c.data_const) len = (uint32_t)c.data_len;
    else if (c.lens_type >= 4) { len = c.lens_const; off = (uint64_t)r * len; }
    else {
        const uint8_t* lens = B.arena + c.lens_off;
        uint32_t o = row_off8[(B.blk_word_off[b] << 3) + (r >> 3)];
        for (uint32_t q = r & ~7u; q < r; q++) o += row_len(c, lens, q);
        off = o; len = row_len(c, lens, r);
    }
    if (off + len > c.data_len) return ERR_LENS_MISMATCH;
    *p = B.arena + c.data_off + off; *n = len;
    return ERR_NONE;
}
// The text of row r without formatting: "" for a field the block does not have (c NULL: no block of the batch has it), the const value, the
// row bytes of a strings cell, the dictionary entry; for a typed cell (cell_typed) the encoded value, whose text is left to the caller.  A dict
// or typed value whose length is not its type's width is ERR_BAD_WIDTH.  On an error the text is "".  One exit: with one return per case the
// facets pass outgrew its registers and spilled.
static __device__ __forceinline__ uint32_t cell_text_raw(const BatchView& B, const DevColumn* c, uint32_t b, uint32_t r, const uint32_t* __restrict__ row_off8, const uint8_t** p,
                                                         uint32_t* n) {
    const uint8_t* src = nullptr; uint32_t len = 0, err = ERR_NONE;
    if (c && c->kind == COL_CONST) { src = B.hdr + c->meta_off; len = c->meta_len; }
    else if (c && c->kind == COL_VALUES) {
        err = cell_raw(B, *c, b, r, row_off8, &src, &len);
        if (!err && c->vt != VT_STRING && len != width_of_vt(c->vt)) err = ERR_BAD_WIDTH;
        if (!err && c->vt == VT_DICT) {
            const uint32_t id = src[0];
            if (id >= c->dict_len) err = ERR_DICT_INDEX;
            else { const uint32_t* dof = (const uint32_t*)(B.hdr + c->meta_off); src = B.hdr + c->meta_off + 4 * (c->dict_len + 1) + dof[id]; len = dof[id + 1] - dof[id]; }
        }
        if (err) len = 0;
    }
    *p = src; *n = len;
    return err;
}
// The text of row r: cell_text_raw with a typed value formatted into buf (VL_FMT_F64_MAX bytes).  Not inlined: inlined, it made the hits and
// two-column kernels spill more.
static __device__ __noinline__ uint32_t cell_text(const BatchView& B, const DevColumn* c, uint32_t b, uint32_t r, const uint32_t* __restrict__ row_off8, uint8_t* buf, const uint8_t** p, uint32_t* n) {
    const uint32_t err = cell_text_raw(B, c, b, r, row_off8, p, n);
    if (!err && cell_typed(c)) {
        const uint64_t raw = load_fixed_be(*p, *n);
        const int k = c->vt == VT_FLOAT64 ? fmt_f64(buf, raw) : encoded_to_string(c->vt, raw, buf);
        *p = buf; *n = k > 0 ? (uint32_t)k : 0;
    }
    return err;
}
// The dict ids of a cell in the plain layout, one byte per row (const lens 1, rows bytes of data), which the dict fast paths read directly;
// NULL for any other cell, whose rows go through the reader.
static __device__ __forceinline__ const uint8_t* plain_dict_ids(const BatchView& B, const DevColumn& c, uint32_t rows) {
    const bool plain = c.kind == COL_VALUES && c.vt == VT_DICT && c.values_state == VALUES_STAGED && c.lens_type >= 4 && c.lens_const == 1 && c.data_len == rows && !c.data_const;
    return plain ? B.arena + c.data_off : nullptr;
}
// The value of column `slot` (-1: a field the batch lacks) in one row as a string.  pass 0: lens[h] = its length; pass 1: the bytes go to out + offs[h].
static __global__ void k_gather_values(BatchView B, int slot, const uint32_t* __restrict__ hits, const uint32_t* __restrict__ hit_block, uint64_t nhits, const uint32_t* __restrict__ row_off8,
                                       int pass, uint32_t* __restrict__ lens_out, const uint64_t* __restrict__ offs, uint8_t* __restrict__ out, unsigned long long* __restrict__ stats) {
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= nhits) return;
    uint8_t buf[VL_FMT_F64_MAX];
    const uint8_t* src; uint32_t len;
    const uint32_t b = hit_block[h];
    report_error(stats, cell_text(B, cell_at(B, slot, b), b, hits[h], row_off8, buf, &src, &len));
    if (pass == 0) { lens_out[h] = len; return; }
    uint8_t* d = out + offs[h];
    for (uint32_t k = 0; k < len; k++) d[k] = src[k];
}
// exclusive scan of u32 lengths into u64 offsets (offs[n] = total): tile sums, scan of the tile sums by one CTA, per-tile prefixes
#define VL_SCAN_TILE 2048
static __global__ void __launch_bounds__(256) k_scan_tiles(const uint32_t* __restrict__ v, uint64_t n, unsigned long long* __restrict__ tile_sums, unsigned long long* __restrict__ offs, int pass) {
    __shared__ unsigned long long s_w[8];
    const uint64_t base = (uint64_t)blockIdx.x * VL_SCAN_TILE + (uint64_t)threadIdx.x * 8;
    unsigned long long x[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { x[k] = base + k < n ? v[base + k] : 0; sum += x[k]; }
    unsigned long long incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane_id() >= d) incl += t; }
    if (lane_id() == 31) s_w[threadIdx.x >> 5] = incl;
    __syncthreads();
    unsigned long long pre = 0, tot = 0;
    for (uint32_t k = 0; k < 8; k++) { if (k < (threadIdx.x >> 5)) pre += s_w[k]; tot += s_w[k]; }
    if (pass == 0) { if (threadIdx.x == 0) tile_sums[blockIdx.x] = tot; return; }
    unsigned long long o = tile_sums[blockIdx.x] + pre + incl - sum;
#pragma unroll
    for (int k = 0; k < 8; k++) { if (base + k < n) offs[base + k] = o; o += x[k]; }
}

// ---- two-column leaves: eq_field(), le_field() / lt_field() (filter_eq_field.go:60-237, filter_le_field.go:93-313) -------------------------------
// leValuesString filter_le_field.go:283-297: numbers when both sides are numbers, else strings (bytewise, the shorter first on a tie)
static __device__ bool le_values_string(const uint8_t* a, uint32_t an, const uint8_t* b2, uint32_t bn, bool excl) {
    const double fa = mn::parse_math_number(a, an);
    if (fa == fa) { const double fb = mn::parse_math_number(b2, bn); if (fb == fb) return excl ? fa < fb : fa <= fb; }
    const uint32_t m = an < bn ? an : bn;
    int cmp = 0;
    for (uint32_t i = 0; i < m && !cmp; i++) cmp = (int)a[i] - (int)b2[i];
    if (!cmp) cmp = an < bn ? -1 : an > bn ? 1 : 0;
    return excl ? cmp < 0 : cmp <= 0;
}
// header-level decisions of a two-column leaf; one warp per block (lane 0 decides), work lists like k_plan_leaf
static __global__ void __launch_bounds__(256) k_plan_pair(DevProgram P, BatchView B, uint32_t leaf_idx, int slot_a, int slot_b, const uint64_t* __restrict__ reg, uint8_t* __restrict__ action,
                                                           uint64_t* __restrict__ payload, uint32_t* __restrict__ lens_a, uint32_t* __restrict__ lens_b, uint32_t* __restrict__ row_blocks,
                                                           uint32_t* __restrict__ work_count, unsigned long long* __restrict__ stats, uint8_t* __restrict__ need = nullptr) {
    // need != NULL: probe pass of a bloom-first upload (see k_plan_leaf): marks the values columns the row kernel would read, writes nothing else
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B.nblocks) return;
    const DevLeaf& L = P.leaves[leaf_idx];
    const bool alive = block_alive_warp(reg, B, b);
    if (lane_id() != 0) return;
    uint8_t act = ACT_NONE; uint64_t mode = PAIR_STRINGS;
    if (alive && !L.always_none) {
        const bool le = L.kind == F_LE_FIELD, excl = L.pair_excl != 0;
        const DevColumn* ca = slot_a >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot_a] : nullptr;
        const DevColumn* cb = slot_b >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot_b] : nullptr;
        const int ka = ca ? ca->kind : COL_MISSING, kb = cb ? cb->kind : COL_MISSING;
        // a const column with an empty value is no column at all for getConstColumnValue (block_search.go:232-276 returns "" for both)
        const bool consta = ka == COL_CONST && ca->meta_len > 0, constb = kb == COL_CONST && cb->meta_len > 0;
        const bool vala = ka == COL_VALUES, valb = kb == COL_VALUES;
        if (consta && constb) {
            const uint8_t* x = B.hdr + ca->meta_off; const uint8_t* y = B.hdr + cb->meta_off;
            const bool m = le ? le_values_string(x, ca->meta_len, y, cb->meta_len, excl) : bytes_equal(x, ca->meta_len, y, cb->meta_len);
            act = m ? ACT_ALL : ACT_NONE;
        } else if (consta || constb) act = ACT_PAIR;                                      // one const: row strings
        else if (!vala && !valb) act = (le && excl) ? ACT_NONE : ACT_ALL;                  // both fields missing: "" against ""
        else if (!vala || !valb) act = ACT_PAIR;                                          // one missing: row strings
        else if (ca->vt != cb->vt || ca->vt == VT_STRING) act = ACT_PAIR;
        else { act = ACT_PAIR; mode = ca->vt == VT_DICT ? PAIR_DICT : PAIR_BINARY; }
        if (act == ACT_PAIR && need) {
            if (vala) need[(uint64_t)b * B.nfields + slot_a] = 1;
            if (valb) need[(uint64_t)b * B.nfields + slot_b] = 1;
            return;
        }
        if (act == ACT_PAIR && ((vala && ca->values_state != VALUES_STAGED) || (valb && cb->values_state != VALUES_STAGED))) {
            atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_VALUES_ABSENT); act = ACT_NONE;
        }
        if (act == ACT_PAIR) {
            unsigned long long vb = 0, cols = 0;
            if (vala) { vb += lens_stored_bytes(*ca, B.blk_rows[b]) + ca->data_len; cols++; if (cell_needs_offsets(*ca)) lens_a[atomicAdd(&work_count[WC_LENS], 1u)] = b; }
            if (valb) { vb += lens_stored_bytes(*cb, B.blk_rows[b]) + cb->data_len; cols++; if (cell_needs_offsets(*cb)) lens_b[atomicAdd(&work_count[WC_LENS2], 1u)] = b; }
            row_blocks[atomicAdd(&work_count[WC_ROW], 1u)] = b;
            atomicAdd(&stats[ST_VALUES_BYTES], vb); atomicAdd(&stats[ST_COLUMNS_READ], cols);
        }
    }
    if (need) return;
    action[b] = act; payload[b] = mode;
}
static __device__ __noinline__ bool pair_match_row(const DevProgram& P, const BatchView& B, const DevLeaf& L, const DevColumn* ca, const DevColumn* cb, uint32_t b, uint32_t r, uint32_t mode,
                                                   const uint32_t* __restrict__ ro_a, const uint32_t* __restrict__ ro_b, unsigned long long* __restrict__ stats) {
    const bool le = L.kind == F_LE_FIELD, excl = L.pair_excl != 0;
    const uint8_t *x, *y; uint32_t xn, yn;
    if (mode == PAIR_BINARY) {
        uint32_t err = cell_raw(B, *ca, b, r, ro_a, &x, &xn);
        if (!err) err = cell_raw(B, *cb, b, r, ro_b, &y, &yn);
        if (err) { report_error(stats, err); return false; }
        if (!le) return bytes_equal(x, xn, y, yn);                                        // applyFilterBinValue: same type, same binary form
        if (ca->vt == VT_INT64 && xn == 8 && yn == 8) { const int64_t u = unzigzag64(ld_be64(x)), v = unzigzag64(ld_be64(y)); return excl ? u < v : u <= v; }
        if (ca->vt == VT_FLOAT64 && xn == 8 && yn == 8) { const double u = __longlong_as_double((long long)ld_be64(x)), v = __longlong_as_double((long long)ld_be64(y)); return excl ? u < v : u <= v; }
        return le_values_string(x, xn, y, yn, excl);   // uintN, ipv4, iso8601: their big-endian encodings go through leValuesString as they are (:246-252)
    }
    uint8_t bufa[VL_FMT_F64_MAX], bufb[VL_FMT_F64_MAX];
    uint32_t err = cell_text(B, ca, b, r, ro_a, bufa, &x, &xn);
    if (!err) err = cell_text(B, cb, b, r, ro_b, bufb, &y, &yn);
    if (err) { report_error(stats, err); return false; }
    return le ? le_values_string(x, xn, y, yn, excl) : bytes_equal(x, xn, y, yn);   // PAIR_DICT compares the entries, PAIR_STRINGS the string forms: same code
}
// three CTAs per SM: left to itself ptxas gives the reader's call chain 128 registers and the kernel two, which measured slower
static __global__ void __launch_bounds__(256, 3) k_row_pair(DevProgram P, BatchView B, uint32_t leaf_idx, int slot_a, int slot_b, const uint32_t* __restrict__ row_blocks, const uint32_t* __restrict__ work_count,
                                                          const uint64_t* __restrict__ payload, const uint64_t* __restrict__ reg, const uint32_t* __restrict__ ro_a, const uint32_t* __restrict__ ro_b,
                                                          uint64_t* __restrict__ leaf_bm, unsigned long long* __restrict__ stats) {
    const uint32_t nwork = work_count[WC_ROW];
    const DevLeaf& L = P.leaves[leaf_idx];
    for (uint32_t j = blockIdx.x; j < nwork; j += gridDim.x) {
        const uint32_t b = row_blocks[j], rows = B.blk_rows[b], mode = (uint32_t)payload[b];
        const DevColumn* ca = slot_a >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot_a] : nullptr;
        const DevColumn* cb = slot_b >= 0 ? &B.cols[(uint64_t)b * B.nfields + slot_b] : nullptr;
        const uint64_t w_lo = B.blk_word_off[b], w_hi = B.blk_word_off[b + 1];
        for (uint64_t gw = w_lo + (threadIdx.x >> 5); gw < w_hi; gw += blockDim.x >> 5) {
            const uint64_t live = reg[gw];   // only rows that are still selected (bm.forEachSetBit)
            if (!live) { if (lane_id() == 0) leaf_bm[gw] = 0; continue; }
            const uint32_t r0 = (uint32_t)(gw - w_lo) * 64, ra = r0 + lane_id(), rb = ra + 32;
            bool ha = false, hb = false;
            if (ra < rows && (live >> lane_id() & 1)) ha = pair_match_row(P, B, L, ca, cb, b, ra, mode, ro_a, ro_b, stats);
            if (rb < rows && (live >> (32 + lane_id()) & 1)) hb = pair_match_row(P, B, L, ca, cb, b, rb, mode, ro_a, ro_b, stats);
            const uint32_t lo = __ballot_sync(0xffffffffu, ha), hi = __ballot_sync(0xffffffffu, hb);
            if (lane_id() == 0) leaf_bm[gw] = ((uint64_t)hi << 32) | lo;
        }
    }
}

// ---- digest of the result bitmaps (bench / tests; the oracle computes the same over its own bitmaps, oracle/vlo_api.cpp vlo_scan_generated) -------
// xor over the blocks [block_lo, block_hi) of XXH64(the block's bitmap words as bytes) * (2 * key + 1), key = key_base + block index in the batch.
static __global__ void k_bitmap_digest(BatchView B, const uint64_t* __restrict__ reg, uint32_t block_lo, uint32_t block_hi, uint64_t key_base, unsigned long long* __restrict__ out) {
    const uint32_t b = block_lo + blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long d = 0;
    if (b < block_hi) {
        const uint64_t lo = B.blk_word_off[b], hi = B.blk_word_off[b + 1];
        d = xxh64((const uint8_t*)(reg + lo), (uint32_t)((hi - lo) * 8)) * (2 * (key_base + b) + 1);
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) d ^= __shfl_xor_sync(0xffffffffu, d, s);
    if (lane_id() == 0 && d) atomicXor(out, d);
}

// ---- `stats by (_time:step offset off, f1, ...) count()` over the selected rows: the aggregation of /select/logsql/hits --------------------------
// (app/vlselect/logsql/logsql.go:116-219 builds it, lib/logstorage/block_result.go:760-848 buckets `_time`).  A group is (bucket, the text of every
// by-field as cell_text yields it).  Groups live in an open-addressing table whose slot holds only a 64-bit tag: the high half of the key's hash
// and 1 + the index of a representative hit.  A key is found by comparing the bucket and the texts with the representative's, byte for byte,
// so two keys share a slot only when they are equal: a hash collision costs a probe, never a wrong count.  A hit insert that would claim a slot
// beyond the table's load limit raises the overflow flag; the host then grows the table and runs the pass again.
#define VL_HITS_MAX_BY 4
#define VL_HITS_CODES 4096   // (block, dict entry) pre-aggregation: at most 8 dict entries per by-field, so 8^VL_HITS_MAX_BY codes
struct HitsQuery {
    int64_t step, offset;
    uint32_t calendar, nby;
    int slot[VL_HITS_MAX_BY];                   // batch field slot of every by-field; -1: no block of the batch has it
    const uint32_t* row_off8[VL_HITS_MAX_BY];   // k_lens_offsets of that slot
};
struct HitsView {
    const uint32_t* hits; const uint32_t* hit_block;                 // build_hit_list
    const long long* blk_bucket; const uint8_t* blk_multi;           // k_hits_classify
    const unsigned long long* ts_vals;                               // k_ts_decode_list of the multi-bucket blocks
};
struct HitsTable {
    unsigned long long* tags;    // [mask + 1]: 0 = empty, else (key hash >> 32) << 32 | (representative hit + 1)
    unsigned long long* cnt;     // [mask + 1]
    unsigned long long* state;   // [0] slots claimed, [1] overflow, [2] groups emitted
    uint64_t mask, limit;
    uint32_t* hit_slot;          // k_hits_group<true>: the slot of every hit (vlscan_hits_sums)
    uint32_t* slot_group;        // [mask + 1], k_hits_emit: the group index of every occupied slot, or NULL
};

// Blocks with hits: the buckets of their minimum and maximum timestamps.  Where they are equal every row of the block is in that bucket (the
// fast path of getBucketedTimestampValues :769-783) and the timestamps are never decoded; the others go into the decode list.
static __global__ void k_hits_classify(BatchView B, const uint32_t* __restrict__ counts, HitsQuery q, long long* __restrict__ blk_bucket, uint8_t* __restrict__ blk_multi,
                                       uint32_t* __restrict__ row_blocks, uint32_t* __restrict__ work_count, unsigned long long* __restrict__ stats) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || counts[b] == 0) return;
    if (!B.ts || B.ts[b].mt == 0) { blk_bucket[b] = 0; blk_multi[b] = 0; atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_NO_TIMESTAMPS); return; }
    const int64_t lo = truncate_timestamp(B.ts[b].first, q.step, q.offset, q.calendar), hi = truncate_timestamp(B.ts[b].max, q.step, q.offset, q.calendar);
    blk_bucket[b] = lo; blk_multi[b] = lo != hi;
    if (lo != hi) row_blocks[atomicAdd(&work_count[WC_ROW], 1u)] = b;
}
static __device__ __forceinline__ int64_t hit_bucket(const BatchView& B, const HitsQuery& q, const HitsView& V, uint32_t b, uint32_t r) {
    return V.blk_multi[b] ? truncate_timestamp((int64_t)V.ts_vals[B.blk_word_off[b] * 64 + r], q.step, q.offset, q.calendar) : (int64_t)V.blk_bucket[b];
}
static __device__ __forceinline__ uint64_t mix64(uint64_t z) { z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ULL; z ^= z >> 27; z *= 0x94D049BB133111EBULL; return z ^ (z >> 31); }
// The key tables of the hits and the facets: open addressing, a slot holds a count and a 64-bit tag, the high half of the key's hash and 1 + the
// index of a representative hit (0: empty).  key_table_add adds c to the slot of the key of hit `rep`: a slot whose hash half matches holds the
// key only when same(its representative) says so, so a hash collision costs a probe, never a wrong count; an empty slot is claimed by CAS when
// may_claim() allows it.  The caller's policy acts on the outcome; *at (when given) receives the slot of a found or claimed key.
enum { KEY_FOUND = 0, KEY_CLAIMED = 1, KEY_NOT_PLACED = 2 };   // not placed: the table is full, or may_claim() declined a new key
template <typename Same, typename MayClaim>
static __device__ __forceinline__ int key_table_add(unsigned long long* tags, unsigned long long* cnt, uint64_t mask, uint64_t hash, uint64_t rep, uint64_t c, Same same, MayClaim may_claim,
                                                     uint64_t* at = nullptr) {
    const unsigned long long tag = (hash & 0xFFFFFFFF00000000ull) | (rep + 1);
    uint64_t s = hash & mask;
    for (uint64_t p = 0; p <= mask; p++, s = (s + 1) & mask) {
        unsigned long long cur = *(volatile unsigned long long*)&tags[s];
        if (cur == 0) {
            if (!may_claim()) return KEY_NOT_PLACED;
            cur = atomicCAS(&tags[s], 0ull, tag);
            if (cur == 0) { atomicAdd(&cnt[s], (unsigned long long)c); if (at) *at = s; return KEY_CLAIMED; }
        }
        if ((cur >> 32) != (hash >> 32)) continue;
        if (same((cur & 0xFFFFFFFFull) - 1)) { atomicAdd(&cnt[s], (unsigned long long)c); if (at) *at = s; return KEY_FOUND; }
    }
    return KEY_NOT_PLACED;
}
// Runs of equal keys (key, sub) among the lanes of a warp, in lane order: a lane without `valid` is in no run, and `merge` false puts every lane
// in a run of its own.  Returns the run's length at its last lane (the run's head is lane - length + 1), 0 at every other lane.
static __device__ __forceinline__ uint32_t warp_run_end(bool valid, bool merge, uint64_t key, uint32_t sub) {
    const uint32_t lane = lane_id();
    const uint64_t pk = __shfl_up_sync(0xffffffffu, key, 1);
    const uint32_t ps = __shfl_up_sync(0xffffffffu, sub, 1);
    const int pv = __shfl_up_sync(0xffffffffu, (int)valid, 1);
    const int same_prev = merge && lane > 0 && valid && pv && pk == key && ps == sub;
    const uint32_t heads = __ballot_sync(0xffffffffu, valid && !same_prev);
    const int same_next = __shfl_down_sync(0xffffffffu, same_prev, 1);
    if (!valid || (lane < 31 && same_next)) return 0;
    const uint32_t head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
    return lane - head + 1;
}
static __device__ uint64_t hits_key_hash(const BatchView& B, const HitsQuery& q, int64_t bucket, uint32_t b, uint32_t r, unsigned long long* stats) {
    uint64_t h = mix64((uint64_t)bucket);
    uint8_t buf[VL_FMT_F64_MAX];
    for (uint32_t f = 0; f < q.nby; f++) {
        const uint8_t* src; uint32_t len;
        report_error(stats, cell_text(B, cell_at(B, q.slot[f], b), b, r, q.row_off8[f], buf, &src, &len));
        h = (h ^ len) * 0x100000001B3ull;
        for (uint32_t k = 0; k < len; k++) h = (h ^ src[k]) * 0x100000001B3ull;
        h = mix64(h);
    }
    return h;
}
static __device__ bool hits_same_texts(const BatchView& B, const HitsQuery& q, uint32_t b1, uint32_t r1, uint32_t b2, uint32_t r2, unsigned long long* stats) {
    uint8_t buf1[VL_FMT_F64_MAX], buf2[VL_FMT_F64_MAX];
    for (uint32_t f = 0; f < q.nby; f++) {
        const uint8_t *s1, *s2; uint32_t l1, l2;
        report_error(stats, max(cell_text(B, cell_at(B, q.slot[f], b1), b1, r1, q.row_off8[f], buf1, &s1, &l1), cell_text(B, cell_at(B, q.slot[f], b2), b2, r2, q.row_off8[f], buf2, &s2, &l2)));
        if (l1 != l2) return false;
        for (uint32_t k = 0; k < l1; k++) if (s1[k] != s2[k]) return false;
    }
    return true;
}
// add `c` rows with the key of hit `hit` = row r of block b, whose bucket is `bucket`; returns the key's slot (meaningless once the pass overflowed:
// the host runs it again)
static __device__ uint32_t hits_insert(const BatchView& B, const HitsQuery& q, const HitsView& V, const HitsTable& T, int64_t bucket, uint64_t hit, uint32_t b, uint32_t r, uint64_t c,
                                       unsigned long long* stats) {
    if (*(volatile unsigned long long*)&T.state[1]) return 0;
    const uint64_t hash = hits_key_hash(B, q, bucket, b, r, stats);
    uint64_t at = 0;
    const int got = key_table_add(T.tags, T.cnt, T.mask, hash, hit, c, [&](uint64_t rep) {
        const uint32_t rb = V.hit_block[rep], rr = V.hits[rep];
        return hit_bucket(B, q, V, rb, rr) == bucket && hits_same_texts(B, q, b, r, rb, rr, stats);
    }, [] { return true; }, &at);
    if (got == KEY_NOT_PLACED || (got == KEY_CLAIMED && atomicAdd(&T.state[0], 1ull) >= T.limit)) atomicExch(&T.state[1], 1ull);
    return (uint32_t)at;
}
// One CTA per block with hits.  When every by-field of the block is a const or absent column, or a dict cell in the plain layout
// (plain_dict_ids), its key is a function of (bucket, dict ids): a single-bucket block counts its rows per dict-id code in shared memory and
// inserts one representative per code (with no by-fields: one insert of the block's count); a multi-bucket block merges runs of equal
// (bucket, code) inside each warp first.  Other cells (strings, typed, dict cells in any other layout) insert row by row.  SLOTS: also write the
// slot of every hit to T.hit_slot, for the value sums of vlscan_hits_sums (the hits-only instance compiles to the code it had without it).
template <bool SLOTS>
static __global__ void __launch_bounds__(256) k_hits_group(BatchView B, HitsQuery q, HitsView V, HitsTable T, const uint32_t* __restrict__ counts, const uint64_t* __restrict__ hit_offs,
                                                            unsigned long long* __restrict__ stats) {
    __shared__ uint32_t s_cnt[VL_HITS_CODES], s_rep[VL_HITS_CODES];
    for (uint32_t b = blockIdx.x; b < B.nblocks; b += gridDim.x) {
        const uint32_t n = counts[b];
        if (n == 0) continue;
        const uint64_t h0 = hit_offs[b];
        bool agg = true;
        uint32_t codes = 1, stride[VL_HITS_MAX_BY];
        const uint8_t* ids[VL_HITS_MAX_BY];
        for (uint32_t f = 0; f < q.nby; f++) {
            stride[f] = codes; ids[f] = nullptr;
            if (q.slot[f] < 0) continue;
            const DevColumn& c = B.cols[(uint64_t)b * B.nfields + q.slot[f]];
            if (c.kind != COL_VALUES) continue;
            const uint32_t width = c.dict_len ? c.dict_len : 1;
            ids[f] = plain_dict_ids(B, c, B.blk_rows[b]);   // code_of reads ids only while agg holds
            if (!ids[f] || codes * width > VL_HITS_CODES) { agg = false; continue; }
            codes *= width;
        }
        auto code_of = [&](uint32_t r) { uint32_t k = 0; for (uint32_t f = 0; f < q.nby; f++) if (ids[f]) k += ids[f][r] * stride[f]; return k; };
        if (agg && !V.blk_multi[b]) {
            const int64_t bucket = V.blk_bucket[b];
            if (codes == 1) {
                if (!SLOTS) { if (threadIdx.x == 0) hits_insert(B, q, V, T, bucket, h0, b, V.hits[h0], n, stats); continue; }
                if (threadIdx.x == 0) s_rep[0] = hits_insert(B, q, V, T, bucket, h0, b, V.hits[h0], n, stats);
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) T.hit_slot[h0 + i] = s_rep[0];
                __syncthreads();
                continue;
            }
            for (uint32_t k = threadIdx.x; k < codes; k += blockDim.x) { s_cnt[k] = 0; s_rep[k] = 0xFFFFFFFFu; }
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
                const uint32_t k = code_of(V.hits[h0 + i]);
                if (k >= codes) { atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_DICT_INDEX); continue; }
                atomicAdd(&s_cnt[k], 1u); atomicMin(&s_rep[k], i);
            }
            __syncthreads();
            for (uint32_t k = threadIdx.x; k < codes; k += blockDim.x)
                if (s_cnt[k]) { const uint32_t s = hits_insert(B, q, V, T, bucket, h0 + s_rep[k], b, V.hits[h0 + s_rep[k]], s_cnt[k], stats); if (SLOTS) s_rep[k] = s; }
            __syncthreads();
            if (SLOTS) {
                for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) { const uint32_t k = code_of(V.hits[h0 + i]); if (k < codes) T.hit_slot[h0 + i] = s_rep[k]; }
                __syncthreads();
            }
            continue;
        }
        for (uint32_t base = 0; base < n; base += blockDim.x) {
            const uint32_t i = base + threadIdx.x;
            const bool valid = i < n;
            const uint32_t r = valid ? V.hits[h0 + i] : 0;
            const int64_t bucket = valid ? hit_bucket(B, q, V, b, r) : 0;
            const uint32_t k = valid && agg ? code_of(r) : 0;
            const uint32_t run = warp_run_end(valid, agg, (uint64_t)bucket, k);
            uint32_t s = 0;
            if (run) s = hits_insert(B, q, V, T, bucket, h0 + i, b, r, run, stats);
            if (SLOTS) {   // every lane of a run takes the slot of the run's last lane
                const uint32_t ends = __ballot_sync(0xffffffffu, run != 0);
                const uint32_t mine = ends & (0xffffffffu << lane_id());
                s = __shfl_sync(0xffffffffu, s, mine ? __ffs(mine) - 1 : 0);
                if (valid) T.hit_slot[h0 + i] = s;
            }
        }
    }
}
// occupied slots -> groups: representative (row, block), bucket, count
static __global__ void k_hits_emit(BatchView B, HitsQuery q, HitsView V, HitsTable T, uint32_t* __restrict__ rep_rows, uint32_t* __restrict__ rep_blocks, long long* __restrict__ buckets,
                                   unsigned long long* __restrict__ out_counts) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > T.mask) return;
    const unsigned long long tag = T.tags[s];
    if (!tag) return;
    const uint64_t rep = (tag & 0xFFFFFFFFull) - 1;
    const uint64_t g = atomicAdd(&T.state[2], 1ull);
    if (T.slot_group) T.slot_group[s] = (uint32_t)g;
    const uint32_t b = V.hit_block[rep], r = V.hits[rep];
    rep_rows[g] = r; rep_blocks[g] = b; buckets[g] = hit_bucket(B, q, V, b, r); out_counts[g] = T.cnt[s];
}

// ---- `stats by (_time:step offset off, f1, ...) sum(v...) avg(v...)`: per group and value field the sum and the count of its numbers -------------
// (lib/logstorage/stats_sum.go, stats_avg.go; grouping pipe_stats.go:552-626, 700-730).  The reference updates a group once per block whose
// selected rows all have its key, through blockResultColumn.sumValues (block_result.go:2501-2600), and row by row through getFloatValueAtRow
// (:2402-2448) otherwise.  The two read a cell differently (stats_number); which one applies is decided per block from the slots of its hits
// (k_hits_group<true>).  A sum is exact: the finite numbers of a (group, field) are added as three 31-bit integer digits in units of
// 2^(frame - 92), frame = ilogb of the largest |number| of that (group, field), found by a first pass.  Integer adds commute, so the result does not
// depend on the order of rows, blocks or atomics: it is the exact sum of the numbers (each cut to 2^(frame - 92), which keeps every integer below
// 2^53 exact) rounded once on the host.  +-Inf and NaN numbers set flags instead.
#define VL_STATS_MAX_VALUES 4
#define VL_STATS_FRAME_BIAS 1101   // frame + bias > 0 for every finite nonzero double (ilogb >= -1074); 0 = no such number yet
struct StatsQuery {
    uint32_t nv;
    int slot[VL_STATS_MAX_VALUES];                   // batch field slot of every value field; -1: no block of the batch has it (or `_time`)
    const uint32_t* row_off8[VL_STATS_MAX_VALUES];   // k_lens_offsets of that slot
};
struct StatsAcc {   // per (group, value field), index g * nv + f
    unsigned long long* digits;   // [3 * G * nv]: the digit sums, high digit first (two's complement int64)
    unsigned long long* count;    // the numbers counted (avg's count)
    int* frame;                   // ilogb of the largest finite nonzero |number| + VL_STATS_FRAME_BIAS, 0 = none (pass 0)
    unsigned* flags;              // 1: a +Inf number, 2: a -Inf number, 4: a NaN number, 8: a counted term that is not -0 (pass 0)
};
struct StatsPart { long long d0, d1, d2; unsigned long long cnt; int frame; unsigned flags; };
static __device__ __forceinline__ void stats_combine(StatsPart& a, const StatsPart& b) {
    a.d0 += b.d0; a.d1 += b.d1; a.d2 += b.d2; a.cnt += b.cnt; a.frame = max(a.frame, b.frame); a.flags |= b.flags;
}
static __device__ __forceinline__ StatsPart stats_shfl_up(const StatsPart& a, uint32_t d) {
    StatsPart o;
    o.d0 = __shfl_up_sync(0xffffffffu, a.d0, d); o.d1 = __shfl_up_sync(0xffffffffu, a.d1, d); o.d2 = __shfl_up_sync(0xffffffffu, a.d2, d);
    o.cnt = __shfl_up_sync(0xffffffffu, a.cnt, d); o.frame = __shfl_up_sync(0xffffffffu, a.frame, d); o.flags = __shfl_up_sync(0xffffffffu, a.flags, d);
    return o;
}
static __device__ __forceinline__ StatsPart stats_shfl_xor(const StatsPart& a, uint32_t m) {
    StatsPart o;
    o.d0 = __shfl_xor_sync(0xffffffffu, a.d0, m); o.d1 = __shfl_xor_sync(0xffffffffu, a.d1, m); o.d2 = __shfl_xor_sync(0xffffffffu, a.d2, m);
    o.cnt = __shfl_xor_sync(0xffffffffu, a.cnt, m); o.frame = __shfl_xor_sync(0xffffffffu, a.frame, m); o.flags = __shfl_xor_sync(0xffffffffu, a.flags, m);
    return o;
}
// add `cnt` to the count and the number x (when has): pass 0 its frame or its Inf / NaN flag, pass 1 its digits relative to `frame`.  The
// reference's sum is -0 only when every term it adds is -0, so pass 0 also flags a term that is not (8)
template <int PASS>
static __device__ __forceinline__ void stats_add(StatsPart& a, double x, bool has, uint32_t cnt, int frame) {
    a.cnt += cnt;
    if (PASS == 0 && has && (x != 0.0 || !signbit(x))) a.flags |= 8;
    if (!has || x == 0.0) return;
    if (isnan(x)) { a.flags |= 4; return; }
    if (isinf(x)) { a.flags |= x > 0 ? 1 : 2; return; }
    if (PASS == 0) { a.frame = max(a.frame, ilogb(x) + VL_STATS_FRAME_BIAS); return; }
    // |x| < 2^(frame + 1), so |y| < 2^93; each step below subtracts the leading bits of y, which is exact
    double y = scalbn(x, 92 - (frame - VL_STATS_FRAME_BIAS));
    const long long d0 = (long long)scalbn(y, -62); y -= scalbn((double)d0, 62);
    const long long d1 = (long long)scalbn(y, -31); y -= scalbn((double)d1, 31);
    a.d0 += d0; a.d1 += d1; a.d2 += (long long)y;
}
template <int PASS>
static __device__ __forceinline__ void stats_commit(const StatsAcc& A, uint64_t i, const StatsPart& a) {
    if (PASS == 0) {
        if (a.cnt) atomicAdd(&A.count[i], a.cnt);
        if (a.frame) atomicMax(&A.frame[i], a.frame);
        if (a.flags) atomicOr(&A.flags[i], a.flags);
    } else {
        if (a.d0) atomicAdd(&A.digits[3 * i], (unsigned long long)a.d0);
        if (a.d1) atomicAdd(&A.digits[3 * i + 1], (unsigned long long)a.d1);
        if (a.d2) atomicAdd(&A.digits[3 * i + 2], (unsigned long long)a.d2);
    }
}
// The number of row r of a value cell (*has) and how many numbers it counts (the return value).  whole: every selected row of the block is in one
// group (sumValues), else getFloatValueAtRow.  They differ: sumValues reads strings and dict entries with tryParseNumber (durations, byte sizes,
// ...; a dict entry whose number is NaN is none) and counts every row of a float64 cell, NaN or not; getFloatValueAtRow reads them with
// tryParseFloat64 and counts a float64 row only when it is not NaN.  Both read a const value with tryParseFloat64 (sumValues counts it
// rows times: k_stats_values handles that case), integers as float64(v), and nothing from ipv4 / iso8601 cells or a field the block lacks.
static __device__ __forceinline__ uint32_t stats_number(const BatchView& B, const DevColumn* c, uint32_t b, uint32_t r, const uint32_t* __restrict__ ro, bool whole, double* x,
                                                        bool* has, unsigned long long* stats) {
    *has = false;
    if (!c || (c->kind != COL_CONST && c->kind != COL_VALUES)) return 0;
    const uint8_t* p; uint32_t n;
    const uint32_t err = cell_text_raw(B, c, b, r, ro, &p, &n);
    if (err) { report_error(stats, err); return 0; }
    const vl::mn::Span sp{p, n};
    if (c->kind == COL_CONST || c->vt == VT_STRING || c->vt == VT_DICT) {
        if (c->kind == COL_VALUES && whole) *has = vl::mn::parse_number(sp, x) && !(c->vt == VT_DICT && isnan(*x));
        else *has = vl::mn::parse_f64_internal(sp, false, x);
        return *has;
    }
    const uint64_t raw = load_fixed_be(p, n);
    switch (c->vt) {
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: *x = (double)raw; *has = true; return 1;
    case VT_INT64: *x = (double)unzigzag64(raw); *has = true; return 1;
    case VT_FLOAT64: *x = __longlong_as_double((long long)raw); *has = !isnan(*x); return whole || *has;
    }
    return 0;
}
// One CTA per block with hits (grid-stride), each value field in turn.  A block whose hits all have one slot is one group: its numbers are
// reduced over the CTA and committed once (a const cell: tryParseFloat64(v) * rows, counted rows times, as sumValues does).  Other blocks reduce
// runs of equal groups inside each warp and commit once per run.  PASS 0 finds the counts, frames and flags; PASS 1 adds the digits.
// Two launches per call, so the reference's order of float adds is not reproduced; the bound that leaves is in DESIGN §3.13.
template <int PASS>
static __global__ void __launch_bounds__(256) k_stats_values(BatchView B, StatsQuery sq, HitsView V, const uint32_t* __restrict__ hit_slot, const uint32_t* __restrict__ slot_group,
                                                             StatsAcc A, const uint32_t* __restrict__ counts, const uint64_t* __restrict__ hit_offs, unsigned long long* __restrict__ stats) {
    __shared__ StatsPart s_warp[8];
    for (uint32_t b = blockIdx.x; b < B.nblocks; b += gridDim.x) {
        const uint32_t n = counts[b];
        if (n == 0) continue;
        const uint64_t h0 = hit_offs[b];
        const uint32_t s0 = hit_slot[h0];
        bool same = true;
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) same = same && hit_slot[h0 + i] == s0;
        const bool whole = __syncthreads_and(same);
        const uint32_t g0 = slot_group[s0];
        for (uint32_t f = 0; f < sq.nv; f++) {
            const DevColumn* c = cell_at(B, sq.slot[f], b);
            if (whole) {
                const int frame = PASS ? A.frame[(uint64_t)g0 * sq.nv + f] : 0;
                StatsPart a{0, 0, 0, 0, 0, 0};
                double x; bool has;
                if (c && c->kind == COL_CONST) {
                    if (threadIdx.x == 0 && stats_number(B, c, b, V.hits[h0], sq.row_off8[f], false, &x, &has, stats)) stats_add<PASS>(a, x * (double)n, true, n, frame);
                } else {
                    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
                        const uint32_t k = stats_number(B, c, b, V.hits[h0 + i], sq.row_off8[f], true, &x, &has, stats);
                        stats_add<PASS>(a, x, has, k, frame);
                    }
                    if (PASS == 0 && a.cnt) a.flags |= 8;   // sumValues starts its sum at +0, so a counted block adds no -0
                }
#pragma unroll
                for (uint32_t m = 16; m; m >>= 1) stats_combine(a, stats_shfl_xor(a, m));
                if (lane_id() == 0) s_warp[threadIdx.x >> 5] = a;
                __syncthreads();
                if (threadIdx.x == 0) {
                    for (uint32_t w = 1; w < (blockDim.x >> 5); w++) stats_combine(a, s_warp[w]);
                    stats_commit<PASS>(A, (uint64_t)g0 * sq.nv + f, a);
                }
                __syncthreads();
                continue;
            }
            for (uint32_t base = 0; base < n; base += blockDim.x) {
                const uint32_t i = base + threadIdx.x;
                const bool valid = i < n;
                const uint32_t g = valid ? slot_group[hit_slot[h0 + i]] : 0xFFFFFFFFu;
                StatsPart a{0, 0, 0, 0, 0, 0};
                if (valid) {
                    double x; bool has;
                    const uint32_t k = stats_number(B, c, b, V.hits[h0 + i], sq.row_off8[f], false, &x, &has, stats);
                    stats_add<PASS>(a, x, has, k, PASS ? A.frame[(uint64_t)g * sq.nv + f] : 0);
                }
                // segmented inclusive scan over runs of equal g in lane order; the last lane of a run holds its total
                const uint32_t lane = lane_id();
                const uint32_t gp = __shfl_up_sync(0xffffffffu, g, 1);
                bool head = lane == 0 || gp != g;
#pragma unroll
                for (uint32_t d = 1; d < 32; d <<= 1) {
                    const StatsPart o = stats_shfl_up(a, d);
                    const bool oh = __shfl_up_sync(0xffffffffu, head, d);
                    if (lane >= d && !head) { stats_combine(a, o); head = oh; }
                }
                const uint32_t gn = __shfl_down_sync(0xffffffffu, g, 1);
                if (valid && (lane == 31 || gn != g)) stats_commit<PASS>(A, (uint64_t)g * sq.nv + f, a);
            }
        }
    }
}

// ---- the N newest selected rows: `/select/logsql/query?limit=N` (app/vlselect/logsql/logsql.go:1005-1080 getLastNQueryResults) ----------------
// Timestamps inside a block never decrease (the writer refuses anything else, lib/logstorage/block.go:182,346), so every selected row of block b
// lies in [min_b, max_b] of its header.  A weighted radix select over the minimums of the blocks with hits at or above the floor (weight: their
// selected rows) gives T_lo, the limit-th largest: at least `limit` selected rows are >= T_lo, so only blocks with max_b >= T_lo can hold a
// returned row, and every other block gets no per-row work.  The selected rows >= T_lo of those blocks are compacted in (block, row) order; the
// same radix select over their timestamps (weight 1) gives T_N, the limit-th largest.  Rows above T_N are in; of the rows equal to T_N the last
// ones in (block, row) order (a prefix count over the ties), which is getLastNRows after a stable sort by _time.
// Radix select: int64 keys with the sign bit flipped (unsigned order = signed order), VL_RADIX_PASSES passes of 8 bits from the top.  The state
// (RS_*) stays on the device, so the passes need no host round trip: after the last pass RS_PREFIX is the flipped limit-th largest key and RS_K
// how many keys equal to it are needed; RS_SHORT = the weights add up to less than the limit.
enum { RS_PREFIX = 0, RS_MASK = 1, RS_K = 2, RS_SHORT = 3, RS_COUNT = 4 };
#define VL_RADIX_PASSES 8
#define VL_SIGN64 0x8000000000000000ull
static __device__ __forceinline__ long long radix_key(const unsigned long long* st) { return (long long)(st[RS_PREFIX] ^ VL_SIGN64); }
// weighted histogram of the next digit of the keys that match the prefix chosen so far (weights == NULL: every key weighs 1)
static __global__ void __launch_bounds__(256) k_radix_hist(const long long* __restrict__ keys, const uint32_t* __restrict__ weights, uint64_t n, const unsigned long long* __restrict__ st,
                                                            int shift, unsigned long long* __restrict__ hist) {
    __shared__ unsigned long long s_h[256];
    s_h[threadIdx.x] = 0;
    __syncthreads();
    if (!st[RS_SHORT]) {
        const unsigned long long prefix = st[RS_PREFIX], mask = st[RS_MASK];
        const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
        for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += stride) {   // warp-uniform trip count: the match below takes every lane
            const uint64_t i = base + threadIdx.x;
            uint32_t w = 0, d = 0;
            if (i < n) {
                const unsigned long long u = (unsigned long long)keys[i] ^ VL_SIGN64;
                w = (u & mask) != prefix ? 0u : weights ? weights[i] : 1u;
                d = (uint32_t)(u >> shift) & 255u;
            }
            if (weights) {   // block minimums: few keys, spread out
                if (w) atomicAdd(&s_h[d], (unsigned long long)w);
            } else {         // row timestamps share their high digits: one shared atomic per group of equal digits in the warp
                const uint32_t peers = __match_any_sync(0xffffffffu, w ? d : 256u);
                if (w && lane_id() == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&s_h[d], (unsigned long long)__popc(peers));
            }
        }
    }
    __syncthreads();
    if (s_h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], s_h[threadIdx.x]);
}
// the digit of this pass: the largest d whose keys, with those of the digits above it, reach the limit
static __global__ void k_radix_pick(const unsigned long long* __restrict__ hist, int shift, unsigned long long limit, unsigned long long* __restrict__ st) {
    if (threadIdx.x != 0 || st[RS_SHORT]) return;
    unsigned long long k = st[RS_K];
    if (shift == 64 - 8) {
        unsigned long long total = 0;
        for (int d = 0; d < 256; d++) total += hist[d];
        if (total < limit) { st[RS_SHORT] = 1; return; }
        k = limit;
    }
    unsigned long long above = 0;
    int d = 255;
    for (; d > 0; d--) {
        if (above + hist[d] >= k) break;
        above += hist[d];
    }
    st[RS_PREFIX] |= (unsigned long long)d << shift; st[RS_MASK] |= 0xFFull << shift; st[RS_K] = k - above;
}
// the key of the block threshold: the header minimum of a block with hits, weighted by its selected rows when it is at or above the floor
static __global__ void k_last_block_keys(BatchView B, const uint32_t* __restrict__ counts, long long floor_ts, long long* __restrict__ keys, uint32_t* __restrict__ weights,
                                         unsigned long long* __restrict__ stats) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks) return;
    uint32_t w = counts[b];
    long long key = 0;
    if (w) {
        if (!B.ts || B.ts[b].mt == 0) { atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_NO_TIMESTAMPS); w = 0; }
        else { key = B.ts[b].first; if (key < floor_ts) w = 0; }
    }
    keys[b] = key; weights[b] = w;
}
// T_lo = the block threshold, or the floor when the weights add up to less than the limit.  Candidate blocks (blocks with hits and max_b >= T_lo)
// go into cand; those whose minimum and maximum differ also into the decode list (WC_ROW; a flat block's rows all carry its minimum).
static __device__ __forceinline__ long long last_threshold(const unsigned long long* st, long long floor_ts) { return st[RS_SHORT] ? floor_ts : radix_key(st); }
static __global__ void k_last_candidates(BatchView B, const uint32_t* __restrict__ counts, long long floor_ts, const unsigned long long* __restrict__ st, uint32_t* __restrict__ cand,
                                         uint32_t* __restrict__ decode, uint32_t* __restrict__ work_count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || counts[b] == 0 || !B.ts || B.ts[b].mt == 0) return;
    const DevTimestamps& t = B.ts[b];
    if (t.max < last_threshold(st, floor_ts)) return;
    cand[atomicAdd(&work_count[WC_LENS2], 1u)] = b;
    if (t.first != t.max) decode[atomicAdd(&work_count[WC_ROW], 1u)] = b;
}
// One CTA per candidate block: its selected rows with ts >= T_lo.  pass 0: their number -> cand_rows[b]; pass 1: (ts, block, row) at offs[b] + rank,
// rows ascending.  A decoded timestamp outside the block's header range is reported (ERR_TS_HEADER).
static __global__ void __launch_bounds__(256) k_last_rows(BatchView B, const uint64_t* __restrict__ reg, const uint32_t* __restrict__ cand, const uint32_t* __restrict__ work_count,
                                                           const unsigned long long* __restrict__ ts_vals, long long floor_ts, const unsigned long long* __restrict__ st, int pass,
                                                           uint32_t* __restrict__ cand_rows, const uint64_t* __restrict__ offs, long long* __restrict__ out_ts, uint32_t* __restrict__ out_blk,
                                                           uint32_t* __restrict__ out_row, unsigned long long* __restrict__ stats) {
    __shared__ uint32_t s_warp[8];
    const uint32_t nwork = work_count[WC_LENS2];
    const long long lo = last_threshold(st, floor_ts);
    const uint32_t lane = lane_id(), wid = threadIdx.x >> 5;
    for (uint32_t j = blockIdx.x; j < nwork; j += gridDim.x) {
        const uint32_t b = cand[j], R = B.blk_rows[b];
        const uint64_t w0 = B.blk_word_off[b];
        const long long mn = B.ts[b].first, mx = B.ts[b].max;
        const unsigned long long* vals = ts_vals + w0 * 64;
        uint64_t o = pass ? offs[b] : 0;
        bool bad = false;
        for (uint32_t base = 0; base < R; base += blockDim.x) {
            const uint32_t r = base + threadIdx.x;
            long long t = mn;
            bool f = false;
            if (r < R) {
                if (mn != mx) { t = (long long)vals[r]; bad |= t < mn || t > mx; }
                f = (reg[w0 + (r >> 6)] >> (r & 63) & 1) && t >= lo;
            }
            const uint32_t m = __ballot_sync(0xffffffffu, f);
            if (lane == 0) s_warp[wid] = __popc(m);
            __syncthreads();
            uint32_t pre = 0, tot = 0;
            for (uint32_t k = 0; k < (blockDim.x >> 5); k++) { const uint32_t c = s_warp[k]; pre += k < wid ? c : 0; tot += c; }
            if (pass && f) {
                const uint64_t p = o + pre + __popc(m & ((1u << lane) - 1));
                out_ts[p] = t; out_blk[p] = b; out_row[p] = r;
            }
            o += tot;
            __syncthreads();
        }
        if (bad) atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_TS_HEADER);
        if (pass == 0 && threadIdx.x == 0) cand_rows[b] = (uint32_t)o;
    }
}
// eq[i] = candidate i carries T_N (the ties whose prefix count decides which of them stay)
static __global__ void k_last_ties(const long long* __restrict__ cts, uint64_t n, const unsigned long long* __restrict__ st, uint32_t* __restrict__ eq) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) eq[i] = !st[RS_SHORT] && cts[i] == radix_key(st);
}
// the chosen candidates: ts > T_N, or ts == T_N among the last RS_K ties (eq_offs: exclusive prefix count of the ties, eq_offs[n] = all of them);
// every candidate when there are no more than the limit.  Output order is arbitrary (the host sorts the <= limit rows); blk_mark[b] = 1 for their blocks.
static __global__ void k_last_choose(const long long* __restrict__ cts, const uint32_t* __restrict__ cblk, const uint32_t* __restrict__ crow, uint64_t n, const unsigned long long* __restrict__ st,
                                     const uint64_t* __restrict__ eq_offs, long long* __restrict__ out_ts, uint32_t* __restrict__ out_blk, uint32_t* __restrict__ out_row,
                                     unsigned long long* __restrict__ out_n, uint32_t* __restrict__ blk_mark) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long t = cts[i];
    if (!st[RS_SHORT]) {
        const long long tn = radix_key(st);
        if (t < tn || (t == tn && eq_offs[i] < eq_offs[n] - st[RS_K])) return;
    }
    const unsigned long long p = atomicAdd(out_n, 1ull);
    out_ts[p] = t; out_blk[p] = cblk[i]; out_row[p] = crow[i];
    blk_mark[cblk[i]] = 1;
}

// ---- `| facets` over the selected rows: the state of one pipeFacetsProcessorShard that saw them (lib/logstorage/pipe_facets.go:162-282) -----------
// A key is (class, 64-bit number) for FK_U64 / FK_NEG (the u64 and negative64 maps of hitsMapAdaptive, hits_map.go:85-115) and FK_TIME (`_time`:
// its RFC3339Nano text is a function of the timestamp), or its text for FK_STR.  Every field has an open-addressing table of `cap` slots whose slot
// holds only a 64-bit tag: the high half of the key's hash and 1 + the hit index of a representative row.  A probe whose hash half matches derives
// the representative's key again and compares it (texts byte for byte), so a hash collision costs a probe, never a wrong count.  Claiming key
// number max_values + 1 drops the field; cap >= 2 * min(max_values + 1, selected rows), so a table never fills.
enum { FK_U64 = 0, FK_NEG = 1, FK_STR = 2, FK_TIME = 3 };
enum { FR_SKIP = 0, FR_OK = 1, FR_DROP = 2 };
#define VL_FACET_SLOTS 1024   // per-CTA pre-aggregation table of a (field, block) work item; it takes new keys up to half full
struct FacetField {
    int slot, is_time;                       // slot -1: no block of the batch has the field
    const uint32_t* row_off8;                // k_lens_offsets of the slot
    const uint64_t* toffs; const uint8_t* tbytes;   // texts of every hit (k_gather_values) when a block with hits stores the field as float64 / ipv4 / iso8601
};
struct FacetsArgs {
    const FacetField* fields; uint32_t nf;
    const uint32_t* blocks; uint32_t nblocks;   // the blocks with hits
    uint64_t max_values, max_len;
    const uint32_t* hits; const uint32_t* hit_block; const uint64_t* hit_offs; const uint32_t* counts;   // build_hit_list
    const unsigned long long* ts_vals;       // k_ts_decode_list of the blocks with hits whose timestamps are not all equal
    unsigned long long* tags; unsigned long long* cnt;   // [nf * cap]
    unsigned long long* nkeys; unsigned int* dropped;    // [nf]
    uint64_t cap;
};
struct FKey { uint32_t cls, len; uint64_t num, hash; const uint8_t* src; };

// uint64StringLen / int64StringLen (pipe_facets.go:240-282): 20 for every n >= 10^10
static __device__ __forceinline__ uint32_t facet_u64_len(uint64_t n) {
    if (n >= 10000000000ull) return 20;
    uint32_t k = 1;
    for (uint64_t p = 10; n >= p; p *= 10) k++;
    return k;
}
static __device__ __forceinline__ uint32_t facet_i64_len(int64_t v) {
    if (v >= 0) return facet_u64_len((uint64_t)v);
    return v == INT64_MIN ? 21 : 1 + facet_u64_len((uint64_t)(-v));
}
// length of marshalTimestampRFC3339NanoString in UTC: "2006-01-02T15:04:05Z", plus "." and the fraction without its trailing zeros
static __device__ __forceinline__ uint32_t facet_rfc3339_len(int64_t ts) {
    int64_t frac = ts % 1000000000LL;
    if (frac < 0) frac += 1000000000LL;
    if (!frac) return 20;
    uint32_t len = 30;
    while (frac % 10 == 0) { frac /= 10; len--; }
    return len;
}
static __device__ __forceinline__ void facet_num_key(FKey& k, uint32_t cls, uint64_t num) {
    k.cls = cls; k.num = num; k.src = nullptr; k.len = 0; k.hash = mix64(num ^ (0x9E3779B97F4A7C15ull * (cls + 1)));
}
// hitsMapAdaptive.updateStateGeneric (hits_map.go:85-97): tryParseUint64, then a '-' text through tryParseInt64, else the bytes
static __device__ __forceinline__ void facet_text_key(FKey& k, const uint8_t* s, uint32_t n) {
    uint64_t v;
    if (mn::parse_u64(mn::Span{s, n}, &v)) { facet_num_key(k, FK_U64, v); return; }
    if (n > 1 && s[0] == '-' && mn::parse_u64(mn::Span{s + 1, n - 1}, &v) && v <= (1ull << 63)) { facet_num_key(k, FK_NEG, 0ull - v); return; }
    uint64_t h = 0xCBF29CE484222325ull;
    for (uint32_t i = 0; i < n; i++) h = (h ^ s[i]) * 0x100000001B3ull;
    k.cls = FK_STR; k.num = 0; k.src = s; k.len = n; k.hash = mix64(h ^ n);
}
// the key of field F in hit h = row r of block b.  FR_SKIP: no key (an empty value, a field the block does not have); FR_DROP: the value is
// too long for max_value_len, which drops the field (updateStateGeneric / updateStateUint64 / updateStateInt64, pipe_facets.go:222-307).
// float64 / ipv4 / iso8601 texts come from F.tbytes, formatted before the pass: no formatter runs here.
static __device__ __forceinline__ int facet_row_key(const BatchView& B, const FacetsArgs& A, const FacetField& F, uint32_t b, uint32_t r, uint64_t h, FKey& k,
                                                    unsigned long long* __restrict__ stats) {
    if (F.is_time) {
        const DevTimestamps& t = B.ts[b];
        const int64_t ts = t.first == t.max ? t.first : (int64_t)A.ts_vals[B.blk_word_off[b] * 64 + r];
        facet_num_key(k, FK_TIME, (uint64_t)ts);
        return facet_rfc3339_len(ts) > A.max_len ? FR_DROP : FR_OK;
    }
    if (F.slot < 0) return FR_SKIP;
    const DevColumn& c = B.cols[(uint64_t)b * B.nfields + F.slot];
    const uint8_t* src; uint32_t len;
    const uint32_t err = cell_text_raw(B, &c, b, r, F.row_off8, &src, &len);
    report_error(stats, err);
    if (!err && cell_typed(&c)) {
        if (c.vt == VT_UINT8 || c.vt == VT_UINT16 || c.vt == VT_UINT32 || c.vt == VT_UINT64 || c.vt == VT_INT64) {
            const uint64_t raw = load_fixed_be(src, len);
            if (c.vt != VT_INT64) {
                facet_num_key(k, FK_U64, raw);
                return A.max_len <= 20 && facet_u64_len(raw) > A.max_len ? FR_DROP : FR_OK;
            }
            const int64_t v = unzigzag64(raw);
            facet_num_key(k, v >= 0 ? FK_U64 : FK_NEG, (uint64_t)v);
            return A.max_len <= 21 && facet_i64_len(v) > A.max_len ? FR_DROP : FR_OK;
        }
        if (!F.toffs) return FR_SKIP;
        src = F.tbytes + F.toffs[h]; len = (uint32_t)(F.toffs[h + 1] - F.toffs[h]);
    }
    if (len == 0) return FR_SKIP;
    if (len > A.max_len) return FR_DROP;
    facet_text_key(k, src, len);
    return FR_OK;
}
static __device__ __forceinline__ bool facet_same_key(const BatchView& B, const FacetsArgs& A, const FacetField& F, const FKey& k, uint64_t h,
                                                      unsigned long long* __restrict__ stats) {
    FKey o;
    if (facet_row_key(B, A, F, A.hit_block[h], A.hits[h], h, o, stats) != FR_OK || o.cls != k.cls) return false;
    if (k.cls != FK_STR) return o.num == k.num;
    if (o.len != k.len) return false;
    for (uint32_t i = 0; i < k.len; i++) if (o.src[i] != k.src[i]) return false;
    return true;
}
// count c rows of key k (representative: hit `rep`) in the table of field f, which drops the field when it claims key number max_values + 1 or
// finds no slot
static __device__ __forceinline__ void facet_add_global(const BatchView& B, const FacetsArgs& A, const FacetField& F, uint32_t f, const FKey& k, uint64_t rep, uint64_t c,
                                                        unsigned long long* __restrict__ stats) {
    if (*(volatile unsigned int*)&A.dropped[f]) return;
    const int got = key_table_add(A.tags + (uint64_t)f * A.cap, A.cnt + (uint64_t)f * A.cap, A.cap - 1, k.hash, rep, c,
                                  [&](uint64_t rh) { return facet_same_key(B, A, F, k, rh, stats); }, [] { return true; });
    if (got == KEY_NOT_PLACED || (got == KEY_CLAIMED && atomicAdd(&A.nkeys[f], 1ull) >= A.max_values)) atomicExch(&A.dropped[f], 1u);
}

// Blocks with hits whose timestamps are not all equal (minimum != maximum): the decode list of the `_time` facet.  Flat blocks are one key each.
static __global__ void k_facets_ts_list(BatchView B, const uint32_t* __restrict__ counts, uint32_t* __restrict__ row_blocks, uint32_t* __restrict__ work_count,
                                        unsigned long long* __restrict__ stats) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || counts[b] == 0) return;
    if (!B.ts || B.ts[b].mt == 0) { atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_NO_TIMESTAMPS); return; }
    if (B.ts[b].first != B.ts[b].max) row_blocks[atomicAdd(&work_count[WC_ROW], 1u)] = b;
}

// 1 in *flag when a block with hits stores column `slot` as float64 / ipv4 / iso8601: the field's texts are then formatted before the pass
static __global__ void k_facets_formatted(BatchView B, const uint32_t* __restrict__ blocks, uint32_t nblocks, int slot, unsigned int* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblocks) return;
    const DevColumn& c = B.cols[(uint64_t)blocks[i] * B.nfields + slot];
    if (c.kind == COL_VALUES && (c.vt == VT_FLOAT64 || c.vt == VT_IPV4 || c.vt == VT_ISO8601)) *flag = 1;
}

// One CTA per (block with hits, field) work item, after a look at the field's dropped flag.  A const cell and a flat `_time` cell are one insert of
// the block's count; a dict cell counts its ids in shared memory and inserts each entry with hits once (forEachDictValueWithHits,
// block_result.go:2381-2400); `_time` rows merge runs of equal timestamps inside each warp; other cells count their rows in a CTA table first and
// insert each of its keys once.  Row loops look at the dropped flag again every blockDim.x rows.
static __global__ void __launch_bounds__(256) k_facets(BatchView B, FacetsArgs A, unsigned long long* __restrict__ stats) {
    __shared__ unsigned long long s_tag[VL_FACET_SLOTS], s_cnt[VL_FACET_SLOTS];
    __shared__ unsigned long long s_used;
    __shared__ uint32_t s_dcnt[8], s_drep[8];
    __shared__ uint32_t s_stop;
    const uint64_t nitems = (uint64_t)A.nblocks * A.nf;
    for (uint64_t j = blockIdx.x; j < nitems; j += gridDim.x) {
        const uint32_t b = A.blocks[j / A.nf], f = (uint32_t)(j % A.nf);
        const uint32_t n = A.counts[b];
        const FacetField F = A.fields[f];
        if (F.is_time ? (!B.ts || B.ts[b].mt == 0) : F.slot < 0) continue;
        __syncthreads();   // the previous item is done with the shared state
        if (threadIdx.x == 0) { s_stop = *(volatile unsigned int*)&A.dropped[f]; s_used = 0; }
        __syncthreads();
        if (s_stop) continue;
        const uint64_t h0 = A.hit_offs[b];
        const DevColumn* c = F.is_time ? nullptr : &B.cols[(uint64_t)b * B.nfields + F.slot];
        if (c && c->kind != COL_CONST && c->kind != COL_VALUES) continue;
        FKey k;
        if (F.is_time ? B.ts[b].first == B.ts[b].max : c->kind == COL_CONST) {   // one key for the whole block
            if (threadIdx.x == 0) {
                const int fr = facet_row_key(B, A, F, b, A.hits[h0], h0, k, stats);
                if (fr == FR_DROP) atomicExch(&A.dropped[f], 1u);
                else if (fr == FR_OK) facet_add_global(B, A, F, f, k, h0, n, stats);
            }
            continue;
        }
        const uint8_t* ids = F.is_time ? nullptr : plain_dict_ids(B, *c, B.blk_rows[b]);
        if (ids) {
            if (threadIdx.x < 8) { s_dcnt[threadIdx.x] = 0; s_drep[threadIdx.x] = 0xFFFFFFFFu; }
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
                const uint32_t id = ids[A.hits[h0 + i]];
                if (id >= c->dict_len || id >= 8) { atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_DICT_INDEX); continue; }
                atomicAdd(&s_dcnt[id], 1u); atomicMin(&s_drep[id], i);
            }
            __syncthreads();
            if (threadIdx.x < c->dict_len && s_dcnt[threadIdx.x]) {
                const uint64_t rep = h0 + s_drep[threadIdx.x];
                const int fr = facet_row_key(B, A, F, b, A.hits[rep], rep, k, stats);
                if (fr == FR_DROP) atomicExch(&A.dropped[f], 1u);
                else if (fr == FR_OK) facet_add_global(B, A, F, f, k, rep, s_dcnt[threadIdx.x], stats);
            }
            continue;
        }
        if (F.is_time) {   // non-decreasing in practice: runs of equal timestamps become one insert
            for (uint32_t base = 0; base < n; base += blockDim.x) {
                if (base) {
                    __syncthreads();
                    if (threadIdx.x == 0 && *(volatile unsigned int*)&A.dropped[f]) s_stop = 1;
                    __syncthreads();
                    if (s_stop) break;
                }
                const uint32_t i = base + threadIdx.x;
                const bool valid = i < n;
                int fr = FR_SKIP;
                if (valid) fr = facet_row_key(B, A, F, b, A.hits[h0 + i], h0 + i, k, stats);
                if (fr == FR_DROP) atomicExch(&A.dropped[f], 1u);
                const bool ok = fr == FR_OK;
                const uint32_t run = warp_run_end(ok, true, ok ? k.num : 0, 0);
                if (run) facet_add_global(B, A, F, f, k, h0 + i - (run - 1), run, stats);
            }
            continue;
        }
        for (uint32_t s = threadIdx.x; s < VL_FACET_SLOTS; s += blockDim.x) { s_tag[s] = 0; s_cnt[s] = 0; }
        __syncthreads();
        for (uint32_t base = 0; base < n; base += blockDim.x) {
            if (base) {
                __syncthreads();
                if (threadIdx.x == 0 && *(volatile unsigned int*)&A.dropped[f]) s_stop = 1;
                __syncthreads();
                if (s_stop) break;
            }
            const uint32_t i = base + threadIdx.x;
            if (i >= n) continue;
            const int fr = facet_row_key(B, A, F, b, A.hits[h0 + i], h0 + i, k, stats);
            if (fr == FR_DROP) { atomicExch(&A.dropped[f], 1u); s_stop = 1; }
            else if (fr == FR_OK) {   // the CTA table declines a new key once it is half full; such keys go to the field's table at once
                const int got = key_table_add(s_tag, s_cnt, VL_FACET_SLOTS - 1, k.hash, h0 + i, 1, [&](uint64_t rh) { return facet_same_key(B, A, F, k, rh, stats); },
                                              [&] { return *(volatile unsigned long long*)&s_used < VL_FACET_SLOTS / 2; });
                if (got == KEY_CLAIMED) atomicAdd(&s_used, 1ull);
                else if (got == KEY_NOT_PLACED) facet_add_global(B, A, F, f, k, h0 + i, 1, stats);
            }
        }
        __syncthreads();
        if (s_stop) continue;
        for (uint32_t s = threadIdx.x; s < VL_FACET_SLOTS; s += blockDim.x) {
            const unsigned long long tag = s_tag[s];
            if (!tag) continue;
            const uint64_t rep = (tag & 0xFFFFFFFFull) - 1;
            if (facet_row_key(B, A, F, b, A.hits[rep], rep, k, stats) == FR_OK) facet_add_global(B, A, F, f, k, rep, s_cnt[s], stats);
        }
    }
}
// occupied slots of the fields that were not dropped -> entries, field after field from base[f]: representative (row, block), class, number, hits
static __global__ void __launch_bounds__(256) k_facets_emit(BatchView B, FacetsArgs A, const uint64_t* __restrict__ base, unsigned long long* __restrict__ cursor,
                                                            uint32_t* __restrict__ rep_rows, uint32_t* __restrict__ rep_blocks, uint32_t* __restrict__ cls,
                                                            unsigned long long* __restrict__ nums, unsigned long long* __restrict__ hits_out, unsigned long long* __restrict__ stats) {
    const uint64_t total = (uint64_t)A.nf * A.cap;
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < total; s += (uint64_t)gridDim.x * blockDim.x) {
        const unsigned long long tag = A.tags[s];
        const uint32_t f = (uint32_t)(s / A.cap);
        if (!tag || A.dropped[f]) continue;
        const uint64_t rep = (tag & 0xFFFFFFFFull) - 1;
        const uint32_t b = A.hit_block[rep], r = A.hits[rep];
        FKey k;
        facet_row_key(B, A, A.fields[f], b, r, rep, k, stats);
        const uint64_t e = base[f] + atomicAdd(&cursor[f], 1ull);
        rep_rows[e] = r; rep_blocks[e] = b; cls[e] = k.cls; nums[e] = k.num; hits_out[e] = A.cnt[s];
    }
}

}  // namespace vl
