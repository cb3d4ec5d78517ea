// CUDA kernels of the aggregations over the last scan's result (sm_90a): the hit list, the gathers of values and timestamps, the hits
// histogram and its value sums, the N newest rows and the facets.  Only vl_agg.cu includes this file.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "vl_mathnum.cuh"
#include "vl_cell.cuh"

namespace vl {

// ---- values of a kept batch left on the host (hit_row_offsets names the field before any kernel reads them) ---------------------------
// *count += the blocks with marks[b] != 0 whose column `slot` is a values column without its values on the device
static __global__ void k_unstaged_count(BatchView B, const uint32_t* __restrict__ marks, int slot, unsigned long long* __restrict__ count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || marks[b] == 0) return;
    const DevColumn& c = B.cols[(uint64_t)b * B.nfields + slot];
    if (c.kind == COL_VALUES && c.values_state != VALUES_STAGED) atomicAdd(count, 1ull);
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
    uint32_t bucketed;                          // bit f: by-field f has a bucket, buckets[f] (device memory: a kernel parameter passed on by
    const BucketSpec* buckets;                  // reference to the noinline reader would be copied to the stack first)
};
struct HitsView {
    const uint32_t* hits; const uint32_t* hit_block;                 // build_hit_list
    const long long* blk_bucket; const uint8_t* blk_multi;           // k_hits_classify
    const unsigned long long* ts_vals;                               // k_ts_decode_list of the multi-bucket blocks
    const uint8_t* by_fast; const unsigned long long* by_lo;         // k_hits_classify, [block * nby + by-field]: typed_header_bucket
    const struct KeyTexts* keys;                                     // [nby], device memory: the texts of every hit of the bucketed by-fields
};
struct KeyTexts { const uint64_t* offs; const uint8_t* bytes; };     // the text of hit h: bytes[offs[h] .. offs[h + 1]) (k_hits_key_texts)
struct HitsTable {
    unsigned long long* tags;    // [mask + 1]: 0 = empty, else (key hash >> 32) << 32 | (representative hit + 1)
    unsigned long long* cnt;     // [mask + 1]
    unsigned long long* state;   // [0] slots claimed, [1] overflow, [2] groups emitted
    uint64_t mask, limit;
    uint32_t* hit_slot;          // k_hits_group<true>: the slot of every hit (vlscan_hits_sums)
    uint32_t* slot_group;        // [mask + 1], k_hits_emit: the group index of every occupied slot, or NULL
};

// Blocks with hits: the buckets of their minimum and maximum timestamps.  Where they are equal every row of the block is in that bucket (the
// fast path of getBucketedTimestampValues :769-783) and the timestamps are never decoded; the others go into the decode list.  Likewise for every
// bucketed by-field stored as a typed column: by_fast = the header fast path of its kind holds, by_lo = the block's bucket then.
static __global__ void k_hits_classify(BatchView B, const uint32_t* __restrict__ counts, HitsQuery q, long long* __restrict__ blk_bucket, uint8_t* __restrict__ blk_multi,
                                       uint8_t* __restrict__ by_fast, unsigned long long* __restrict__ by_lo, uint32_t* __restrict__ row_blocks,
                                       uint32_t* __restrict__ work_count, unsigned long long* __restrict__ stats) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B.nblocks || counts[b] == 0) return;
    for (uint32_t f = 0; f < q.nby; f++) {
        if (!(q.bucketed >> f & 1)) continue;
        const DevColumn* c = cell_at(B, q.slot[f], b);
        uint64_t lo = 0;
        by_fast[(uint64_t)b * q.nby + f] = cell_typed(c) && typed_header_bucket(*c, q.buckets[f], &lo);
        by_lo[(uint64_t)b * q.nby + f] = lo;
    }
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
// the key text of by-field f in hit h = row r of block b: cell_text, or the bucketed text gathered before the pass (no bucketing code runs in
// the grouping kernels: called from them, it made them spill four times as much)
static __device__ __forceinline__ uint32_t by_text(const BatchView& B, const HitsQuery& q, const HitsView& V, uint32_t f, uint64_t h, uint32_t b, uint32_t r, uint8_t* buf,
                                                   const uint8_t** p, uint32_t* n) {
    if (q.bucketed >> f & 1) {
        const KeyTexts& t = V.keys[f];
        *p = t.bytes + t.offs[h]; *n = (uint32_t)(t.offs[h + 1] - t.offs[h]);
        return ERR_NONE;
    }
    return cell_text(B, cell_at(B, q.slot[f], b), b, r, q.row_off8[f], buf, p, n);
}
static __device__ uint64_t hits_key_hash(const BatchView& B, const HitsQuery& q, const HitsView& V, int64_t bucket, uint64_t hit, uint32_t b, uint32_t r, unsigned long long* stats) {
    uint64_t h = mix64((uint64_t)bucket);
    uint8_t buf[VL_FMT_F64_MAX];
    for (uint32_t f = 0; f < q.nby; f++) {
        const uint8_t* src; uint32_t len;
        report_error(stats, by_text(B, q, V, f, hit, b, r, buf, &src, &len));
        h = (h ^ len) * 0x100000001B3ull;
        for (uint32_t k = 0; k < len; k++) h = (h ^ src[k]) * 0x100000001B3ull;
        h = mix64(h);
    }
    return h;
}
static __device__ bool hits_same_texts(const BatchView& B, const HitsQuery& q, const HitsView& V, uint64_t h1, uint32_t b1, uint32_t r1, uint64_t h2, uint32_t b2, uint32_t r2,
                                       unsigned long long* stats) {
    uint8_t buf1[VL_FMT_F64_MAX], buf2[VL_FMT_F64_MAX];
    for (uint32_t f = 0; f < q.nby; f++) {
        const uint8_t *s1, *s2; uint32_t l1, l2;
        report_error(stats, max(by_text(B, q, V, f, h1, b1, r1, buf1, &s1, &l1), by_text(B, q, V, f, h2, b2, r2, buf2, &s2, &l2)));
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
    const uint64_t hash = hits_key_hash(B, q, V, bucket, hit, b, r, stats);
    uint64_t at = 0;
    const int got = key_table_add(T.tags, T.cnt, T.mask, hash, hit, c, [&](uint64_t rep) {
        const uint32_t rb = V.hit_block[rep], rr = V.hits[rep];
        return hit_bucket(B, q, V, rb, rr) == bucket && hits_same_texts(B, q, V, hit, b, r, rep, rb, rr, stats);
    }, [] { return true; }, &at);
    if (got == KEY_NOT_PLACED || (got == KEY_CLAIMED && atomicAdd(&T.state[0], 1ull) >= T.limit)) atomicExch(&T.state[1], 1ull);
    return (uint32_t)at;
}
// One CTA per block with hits.  When every by-field of the block is a const or absent column, or a dict cell in the plain layout
// (plain_dict_ids), its key is a function of (bucket, dict ids): a single-bucket block counts its rows per dict-id code in shared memory and
// inserts one representative per code (with no by-fields: one insert of the block's count); a multi-bucket block merges runs of equal
// (bucket, code) inside each warp first.  Other cells (strings, typed, dict cells in any other layout) insert row by row.  SLOTS: also write the
// slot of every hit to T.hit_slot, for the value sums of vlscan_hits_sums (the hits-only instance compiles to the code it had without it).
// Resident CTAs per SM: four for the hits-only instance (64 registers; left free, ptxas gives it 80, three CTAs, and the pass over 1e8 rows
// ran 5% slower on an H100), three for the one with slots (80 registers, as it gets on its own).
template <bool SLOTS>
static __global__ void __launch_bounds__(256, SLOTS ? 3 : 4) k_hits_group(BatchView B, HitsQuery q, HitsView V, HitsTable T, const uint32_t* __restrict__ counts, const uint64_t* __restrict__ hit_offs,
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
            if (c.kind != COL_VALUES || ((q.bucketed >> f & 1) && V.by_fast[(uint64_t)b * q.nby + f])) continue;   // one text in the whole block
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

// The bucketed text of by-field f in the n rows (rows[i], blocks[i]): k_gather_values with cell_text_bucketed.  Run over every hit before the
// grouping pass (HitsView.key_offs / key_bytes) and over the groups' representatives after it.
static __global__ void k_hits_key_texts(BatchView B, HitsQuery q, HitsView V, uint32_t f, const uint32_t* __restrict__ rows, const uint32_t* __restrict__ blocks, uint64_t n, int pass,
                                        uint32_t* __restrict__ lens_out, const uint64_t* __restrict__ offs, uint8_t* __restrict__ out, unsigned long long* __restrict__ stats) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t buf[VL_FMT_F64_MAX];
    const uint8_t* src; uint32_t len;
    const uint32_t b = blocks[i];
    const uint64_t k = (uint64_t)b * q.nby + f;
    report_error(stats, cell_text_bucketed(B, cell_at(B, q.slot[f], b), b, rows[i], q.row_off8[f], q.buckets + f, V.by_fast[k], V.by_lo[k], buf, &src, &len));
    if (pass == 0) { lens_out[i] = len; return; }
    uint8_t* d = out + offs[i];
    for (uint32_t k = 0; k < len; k++) d[k] = src[k];
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

// ---- `stats by (_time:step offset off, f1, ...) histogram(v...)`: per group and value field the numbers counted per vmrange ---------------------
// (lib/logstorage/stats_histogram.go; metrics.Histogram.Update).  Both reference paths read a cell the same way, so, unlike the sums, nothing
// depends on whether a block's hits fall in one group.  The index of a number is a binary search over the VL_VMR_BOUNDS boundaries the host
// computed from its restatement of Go's Log10 (vl_agg.cu, vmr_bounds): no transcendental runs on the device, and the host's
// vlscan_vmrange_index, the same search, gives the same index by construction.  Counts are exact integers in a table keyed by
// (g * nv + f) * VL_VMRANGES + index, which grows like the hits table.
#define VL_VMRANGES 488
#define VL_VMR_BOUNDS 487   // bound k: the least double whose index is k + 1
struct VmrTable {
    unsigned long long* keys;    // [mask + 1]: 0 = empty, else key + 1
    unsigned long long* cnt;     // [mask + 1]
    unsigned long long* state;   // [0] slots claimed, [1] overflow, [2] entries compacted, [3] (block, value field) cells on the header fast path
    uint64_t mask, limit;
};
// Histogram.Update's index of x: -1 for NaN and x < 0 (-0 is not below 0 and lands in index 0)
static __device__ __forceinline__ int vmr_index(const double* bounds, double x) {
    if (isnan(x) || x < 0) return -1;
    uint32_t lo = 0, hi = VL_VMR_BOUNDS;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (bounds[m] <= x) lo = m + 1; else hi = m; }
    return (int)lo;
}
// add c to `key`; a claim beyond the load limit, or a full table, raises the overflow flag and the host runs the pass again on a larger table
static __device__ void vmr_add(const VmrTable& M, uint64_t key, uint64_t c) {
    if (*(volatile unsigned long long*)&M.state[1]) return;
    uint64_t s = mix64(key) & M.mask;
    for (uint64_t p = 0; p <= M.mask; p++, s = (s + 1) & M.mask) {
        unsigned long long cur = *(volatile unsigned long long*)&M.keys[s];
        if (cur == 0) {
            cur = atomicCAS(&M.keys[s], 0ull, (unsigned long long)key + 1);
            if (cur == 0) {
                if (atomicAdd(&M.state[0], 1ull) >= M.limit) atomicExch(&M.state[1], 1ull);
                atomicAdd(&M.cnt[s], (unsigned long long)c);
                return;
            }
        }
        if (cur == key + 1) { atomicAdd(&M.cnt[s], (unsigned long long)c); return; }
    }
    atomicExch(&M.state[1], 1ull);
}
// One CTA per block with hits (grid-stride), each value field in turn.  Where every row of the cell has one index it is found once: a const
// cell (one tryParseNumber), or a uint8..uint64 cell / an int64 cell with minimum >= 0 whose header minimum and maximum have one index (the
// header fast path; float64 stays off it, its NaN rows count nothing).  A dict cell in the plain layout maps its entries once.  Other cells read
// every hit's number (stats_number's sumValues reading is the histogram's: tryParseNumber, float64(n), the stored double).  A block whose hits
// are one group then counts its indexes in shared memory and adds one entry per index, else runs of equal (group, index) in each warp add once.
static __global__ void __launch_bounds__(256) k_stats_vmranges(BatchView B, StatsQuery sq, HitsView V, const uint32_t* __restrict__ hit_slot,
                                                               const uint32_t* __restrict__ slot_group, const double* __restrict__ bounds, VmrTable M,
                                                               const uint32_t* __restrict__ counts, const uint64_t* __restrict__ hit_offs, unsigned long long* __restrict__ stats) {
    __shared__ double s_bounds[VL_VMR_BOUNDS];
    __shared__ uint32_t s_hist[VL_VMRANGES];
    __shared__ int s_dict[256], s_one;
    const int PER_ROW = 0x7FFFFFFF;
    for (uint32_t i = threadIdx.x; i < VL_VMR_BOUNDS; i += blockDim.x) s_bounds[i] = bounds[i];
    __syncthreads();
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
            if (!c || (c->kind != COL_CONST && c->kind != COL_VALUES)) continue;
            const uint8_t vt = c->kind == COL_VALUES ? c->vt : VT_STRING;
            if (vt == VT_IPV4 || vt == VT_ISO8601) continue;
            const uint8_t* ids = vt == VT_DICT ? plain_dict_ids(B, *c, B.blk_rows[b]) : nullptr;
            if (threadIdx.x == 0) {
                int one = PER_ROW;
                if (c->kind == COL_CONST) {
                    double x;
                    one = vl::mn::parse_number(vl::mn::Span{B.hdr + c->meta_off, c->meta_len}, &x) ? vmr_index(s_bounds, x) : -1;
                } else if (vt == VT_UINT8 || vt == VT_UINT16 || vt == VT_UINT32 || vt == VT_UINT64 || (vt == VT_INT64 && (long long)c->min_value >= 0)) {
                    const int lo = vmr_index(s_bounds, (double)c->min_value), hi = vmr_index(s_bounds, (double)c->max_value);
                    if (lo == hi) { one = lo; atomicAdd(&M.state[3], 1ull); }
                }
                s_one = one;
            }
            if (ids)
                for (uint32_t k = threadIdx.x; k < c->dict_len; k += blockDim.x) {
                    const uint32_t* dof = (const uint32_t*)(B.hdr + c->meta_off);
                    double x;
                    s_dict[k] = vl::mn::parse_number(vl::mn::Span{B.hdr + c->meta_off + 4 * (c->dict_len + 1) + dof[k], dof[k + 1] - dof[k]}, &x) ? vmr_index(s_bounds, x) : -1;
                }
            __syncthreads();
            const int one = s_one;
            auto index_at = [&](uint32_t r) -> int {
                if (one != PER_ROW) return one;
                if (ids) {
                    if (ids[r] < c->dict_len) return s_dict[ids[r]];
                    atomicMax(&stats[ST_ERROR], (unsigned long long)ERR_DICT_INDEX);
                    return -1;
                }
                double x; bool has;
                stats_number(B, c, b, r, sq.row_off8[f], true, &x, &has, stats);
                return has ? vmr_index(s_bounds, x) : -1;
            };
            auto key = [&](uint32_t g, int x) { return ((uint64_t)g * sq.nv + f) * VL_VMRANGES + (uint32_t)x; };
            if (whole && one != PER_ROW) {
                if (threadIdx.x == 0 && one >= 0) vmr_add(M, key(g0, one), n);
            } else if (whole) {
                for (uint32_t k = threadIdx.x; k < VL_VMRANGES; k += blockDim.x) s_hist[k] = 0;
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) { const int x = index_at(V.hits[h0 + i]); if (x >= 0) atomicAdd(&s_hist[x], 1u); }
                __syncthreads();
                for (uint32_t k = threadIdx.x; k < VL_VMRANGES; k += blockDim.x) if (s_hist[k]) vmr_add(M, key(g0, (int)k), s_hist[k]);
            } else {
                for (uint32_t base = 0; base < n; base += blockDim.x) {
                    const uint32_t i = base + threadIdx.x;
                    const bool valid = i < n;
                    const uint32_t g = valid ? slot_group[hit_slot[h0 + i]] : 0;
                    const int x = valid ? index_at(V.hits[h0 + i]) : -1;
                    const uint32_t run = warp_run_end(x >= 0, true, g, (uint32_t)x);
                    if (run) vmr_add(M, key(g, x), run);
                }
            }
            __syncthreads();   // s_one, s_dict and s_hist are rewritten for the next field
        }
    }
}
// the occupied slots of the vmrange table -> (key, count) entries, in no particular order (the host sorts them)
static __global__ void k_vmr_compact(VmrTable M, unsigned long long* __restrict__ out_keys, unsigned long long* __restrict__ out_cnt) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > M.mask) return;
    const unsigned long long k = M.keys[s];
    if (!k) return;
    const uint64_t e = atomicAdd(&M.state[2], 1ull);
    out_keys[e] = k - 1; out_cnt[e] = M.cnt[s];
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
