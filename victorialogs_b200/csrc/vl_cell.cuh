// Device helpers shared by the scan kernels (vl_kernels.cuh) and the aggregation kernels (vl_agg.cuh): the lens items of a values cell, the
// reader of one cell, the text of a typed value and the timestamps decoder.  No kernels: a plain __device__ function is emitted only in the
// translation unit whose kernels call it, so including this header from both adds no copies.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vl_hd.cuh"
#include "vl_mathnum.cuh"
#include "vl_types.h"

namespace vl {

static __device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
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
// ---- bucketed texts of a by-field (newValuesBucketedForColumn, lib/logstorage/block_result.go:703-739, 935-1764) -----------------------------
// A typed value v (uint8..uint64 / ipv4 as stored, int64 and iso8601 as int64 bits, float64 as bits) -> its bucket in the same form
static __device__ __forceinline__ uint64_t typed_bucket(uint32_t vt, const BucketSpec& bk, uint64_t v) {
    switch (vt) {
    case VT_INT64: return (uint64_t)trunc_i64((int64_t)v, bk.i64_col_size, bk.i64_off);
    case VT_FLOAT64: return f64_bits(trunc_f64(f64_of_bits(v), bk));
    case VT_IPV4: return trunc_u32((uint32_t)v, bk.u32_size, bk.u32_off);
    case VT_ISO8601: return (uint64_t)truncate_timestamp((int64_t)v, bk.i64_size, bk.i64_off, bk.calendar);
    }
    return trunc_u64(v, bk.u64_size, bk.u64_off);
}
// The header fast path of the typed kinds: the buckets of the column's minimum and maximum (the header keeps int64 as plain bits, ipv4 in the
// low 32 bits); when they are equal every row of the block has that bucket.  float64 buckets compare as numbers: a NaN minimum and maximum
// fall into one finite bucket.
static __device__ __forceinline__ bool typed_header_bucket(const DevColumn& c, const BucketSpec& bk, uint64_t* lo) {
    const uint64_t a = typed_bucket(c.vt, bk, c.min_value), z = typed_bucket(c.vt, bk, c.max_value);
    *lo = a;
    return c.vt == VT_FLOAT64 ? f64_of_bits(a) == f64_of_bits(z) : a == z;
}
// The bucketed text of row r: a typed value truncated (`fast`: the block's bucket `lo` from typed_header_bucket) and formatted into buf
// (VL_FMT_F64_MAX bytes); any other text through bucket_text.
static __device__ __noinline__ uint32_t cell_text_bucketed(const BatchView& B, const DevColumn* c, uint32_t b, uint32_t r, const uint32_t* __restrict__ row_off8, const BucketSpec* bk,
                                                           bool fast, uint64_t lo, uint8_t* buf, const uint8_t** p, uint32_t* n) {
    const uint8_t* s; uint32_t len;
    uint32_t err = ERR_NONE;
    if (!cell_typed(c)) {
        err = cell_text_raw(B, c, b, r, row_off8, &s, &len);
        *n = bucket_text(*bk, s, len, buf, p);
        return err;
    }
    uint64_t v = lo;
    if (!fast) {
        err = cell_text_raw(B, c, b, r, row_off8, &s, &len);
        const uint64_t raw = err ? 0 : load_fixed_be(s, len);
        v = typed_bucket(c->vt, *bk, c->vt == VT_INT64 ? (uint64_t)unzigzag64(raw) : raw);
    }
    int k = 0;
    switch (c->vt) {
    case VT_INT64: k = fmt_i64(buf, (int64_t)v); break;
    case VT_FLOAT64: k = fmt_f64(buf, v); break;
    case VT_IPV4: k = fmt_ipv4(buf, (uint32_t)v); break;
    case VT_ISO8601: k = fmt_iso8601(buf, (int64_t)v); break;
    default: k = fmt_u64(buf, v);
    }
    *p = buf; *n = err ? 0 : (uint32_t)k;
    return err;
}

// The dict ids of a cell in the plain layout, one byte per row (const lens 1, rows bytes of data), which the dict fast paths read directly;
// NULL for any other cell, whose rows go through the reader.
static __device__ __forceinline__ const uint8_t* plain_dict_ids(const BatchView& B, const DevColumn& c, uint32_t rows) {
    const bool plain = c.kind == COL_VALUES && c.vt == VT_DICT && c.values_state == VALUES_STAGED && c.lens_type >= 4 && c.lens_const == 1 && c.data_len == rows && !c.data_const;
    return plain ? B.arena + c.data_off : nullptr;
}

}  // namespace vl
