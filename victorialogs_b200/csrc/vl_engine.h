// Internal host-side structures of libvlscan.so shared by vl_engine.cu (staging, scan interpreter, C ABI), vl_agg.cu (the aggregations
// over a scan's result), vl_gen.cu (synthetic batch generator) and vl_zstd.cu (device ZSTD decoder driver).
//
// This header holds no device code.  A __global__ is defined in exactly one file, and exactly one .cu includes that file: nvcc emits every
// non-template static kernel in each translation unit that includes its definition, launched there or not, so a kernel header included
// twice compiles and ships its kernels twice.  vl_kernels.cuh belongs to vl_engine.cu, vl_agg.cuh to vl_agg.cu; device helpers both use
// are plain __device__ functions in vl_cell.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../include/vlscan.h"
#include "vl_types.h"
#include "vl_zstd.h"
#include "vl_zstd_walk.h"   // BadInput
#include "vl_hostpool.h"

namespace vl {

void set_thread_error(const std::string& s);
#define VL_CUDA(call)                                                                                                   \
    do {                                                                                                                \
        cudaError_t e__ = (call);                                                                                       \
        if (e__ != cudaSuccess) throw CudaFail(std::string(#call) + ": " + cudaGetErrorString(e__), (int)e__);        \
    } while (0)
struct CudaFail { std::string msg; int code; CudaFail(std::string m, int c) : msg(std::move(m)), code(c) {} };

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    void ensure(size_t n) {
        if (n <= cap) return;
        if (p) VL_CUDA(cudaFree(p));
        p = nullptr; cap = 0;
        size_t want = n + std::min<size_t>(n / 8, (size_t)256 << 20) + 256;   // growth slack, capped: a 150 GB arena must not ask for 170 GB
        VL_CUDA(cudaMalloc(&p, want)); cap = want;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};



static const size_t kArenaAlign = 16;
static const size_t kArenaPad = 32;   // readable slack after every payload (vector loads past the end, see k_substr_scan)
inline uint64_t arena_reserve(uint64_t& cursor, uint64_t len) {
    uint64_t off = (cursor + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
    cursor = off + len + kArenaPad;
    return off;
}

}  // namespace vl

// opaque C ABI types
struct vlscan_batch {
    int device = 0;
    uint32_t nfields = 0;
    std::vector<std::string> field_names;
    uint64_t nblocks = 0, nwords = 0, rows = 0;
    uint64_t arena_bytes = 0, harena_bytes = 0;
    vl::DevBuf arena, cols, blk_rows, blk_word_off, word_block, init_bitmap, ts;
    vl::DevBuf harena;                    // bloom-first staging only: header payloads (bloom filters, const values, dict tables) of phase 1
    bool split_hdr = false;               // the columns' bloom_off / meta_off refer to `harena`, not to `arena`
    std::vector<vl::DevColumn> h_cols;    // bloom-first staging: the column table between the two phases
    bool has_ts = false;                  // some block came with its timestamps column
    std::vector<uint32_t> h_rows;
    std::vector<uint64_t> h_word_off;
    std::vector<uint32_t> slot_vt_mask;   // per field slot: bit vt set when some block stores the field with that valueType
    // kept batches (vlscan_scan_batch_keep) only:
    std::vector<vl::DevBuf> late;         // one region per vlscan_stage_selected call; late cells address it by an offset from `arena` (DESIGN §3.12)
    size_t late_used = 0;                 // regions holding payloads of the current batch (the others are reused by later calls; there are as many
                                          // regions as stage calls one kept batch ever received, each at its largest size, until the batch is freed)
    struct CellSig { uint64_t len0 = 0, len1 = 0; uint32_t stage = 0; };   // a values column: ONDISK (values_len, 0), DECODED (lens_items_len, data_len)
    std::vector<CellSig> h_sig;           // per (block, field) cell, as the keep call was given it
    std::vector<uint32_t> h_ncols;        // per block: the number of columns it was described with
    void note_columns(const std::vector<vl::DevColumn>& cols) {
        slot_vt_mask.assign(nfields, 0);
        for (size_t i = 0; i < cols.size(); i++) if (cols[i].kind == vl::COL_VALUES) slot_vt_mask[i % nfields] |= 1u << cols[i].vt;
    }
    // batch field slot of a canonical field name, -1 when no block of the batch has it
    int field_slot(const std::string& name) const {
        for (uint32_t s = 0; s < nfields; s++) if (field_names[s] == name) return (int)s;
        return -1;
    }
    vl::BatchView view() const {
        vl::BatchView v;
        v.arena = arena.as<uint8_t>(); v.hdr = split_hdr ? harena.as<uint8_t>() : arena.as<uint8_t>(); v.cols = cols.as<vl::DevColumn>(); v.blk_rows = blk_rows.as<uint32_t>();
        v.blk_word_off = blk_word_off.as<uint64_t>(); v.word_block = word_block.as<uint32_t>();
        v.ts = has_ts ? ts.as<vl::DevTimestamps>() : nullptr;
        v.nblocks = (uint32_t)nblocks; v.nfields = nfields; v.nwords = nwords;
        return v;
    }
    uint64_t device_bytes() const {
        uint64_t n = arena.cap + harena.cap + cols.cap + blk_rows.cap + blk_word_off.cap + word_block.cap + init_bitmap.cap + ts.cap;
        for (const vl::DevBuf& r : late) n += r.cap;
        return n;
    }
    ~vlscan_batch() {
        cudaSetDevice(device); arena.release(); harena.release(); cols.release(); blk_rows.release(); blk_word_off.release(); word_block.release(); init_bitmap.release(); ts.release();
        for (vl::DevBuf& r : late) r.release();
    }
};

struct vlscan_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;        // compute stream: kernels, small copies, results
    cudaStream_t copy_stream = nullptr;   // host -> device payload copies of vlscan_batch_upload / vlscan_scan_batch
    std::string err;
    uint64_t launches = 0;
    // scratch (grow-only)
    vl::DevBuf action, payload, leaf_bm, lens_blocks, work_count, stats, totals, counts, slots, tiles;   // tiles: ScanTile work list of k_substr_scan
    vl::DevBuf lens_blocks2;               // second lens work list of a two-column leaf
    vl::DevBuf row_blocks;                 // block work list: row-level blocks of the scan; the timestamps decode list of vlscan_gather_timestamps,
                                           // vlscan_hits_stats and vlscan_facets
    vl::DevBuf hit_offs, hits;             // build_hit_list: first hit of every block, row of each hit (hit_offs also: vlscan_last_rows' selected
                                           // row count, vlscan_result_digest's digest)
    std::vector<vl::DevBuf> regs;          // bitmap registers of the tree interpreter
    std::vector<vl::DevBuf> row_off8;      // per batch field slot: byte offset of every 8th row (k_lens_offsets)
    std::vector<vl::DevBuf> ready;         // per batch field slot: row_off8 computed for block b in this scan
    std::vector<char> ready_cleared;
    vl::DevBuf hit_block, glens, goffs, gtiles, gout, gstat;   // build_hit_list: block of each hit; text_offsets / text_bytes (vlscan_gather_values,
                                           // hits, last rows, facets): value lengths / offsets, exclusive_scan's tile sums, output staging; the error slot
    vl::DevBuf ts_vals;                    // decoded timestamps / running sums, 8 bytes per row of the batch (k_time_match, decode_listed_timestamps)
    vl::DevBuf hslot;                      // vlscan_hits_sums / _vmranges: the group-table slot of every hit (k_hits_group<true>)
    vl::DevBuf vagg;                       // vlscan_hits_vmranges: the boundaries, the vmrange table and its compacted entries, laid out by Carve
    vl::DevBuf hblk, htab, hgrp;           // laid out by Carve.  vlscan_hits_stats: per-block bucket + multi-bucket flag, the group table (tags,
                                           // counts, state), the emitted groups.  vlscan_last_rows: per-block keys / candidate offsets / weights /
                                           // counts / marks and the candidate and decode lists, the radix select states, the chosen rows.
                                           // vlscan_facets: hblk the field table, entry bases / cursors, work counter, flag and blocks with hits;
                                           // hgrp the emitted entries and the string representatives (htab unused)
    vl::DevBuf lcand;                      // vlscan_last_rows: the candidate rows (timestamp, block, row), laid out by Carve
    vl::DevBuf ftab;                       // vlscan_facets: the per-field tables (tags, counts) and states
    std::vector<vl::DevBuf> ftxt;          // vlscan_facets: per requested field, the texts of every hit when the field is stored as float64 / ipv4 / iso8601
    vl::DevBuf need;                       // bloom-first probe pass: one byte per (block, field), set when the column's values must be staged
    const void* bf_prog = nullptr; int bf_skip = 0;   // adaptive bloom-first: after a probe that pruned next to nothing, the next calls with the same program stage everything at once
    vl::DevBuf zsrc, zcols, ztest;         // compressed staging of on-disk values blocks; their column list; test output
    vl::ZstdDev* zdev = nullptr;           // device ZSTD decoder scratch (vl_zstd.cu)
    void* pinned = nullptr; size_t pinned_cap = 0;
    vl::HostPool* pool = nullptr;          // packing threads, started by the first upload from pageable memory
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> scan_events; size_t scan_events_used = 0;
    // last scan
    const vlscan_batch* last_batch = nullptr;   // the batch of the last scan: must stay alive until its results have been fetched
    uint64_t last_nblocks = 0, last_nwords = 0, last_rows = 0;   // host-side facts about it, kept here so that counters never touch a freed batch
    vlscan_batch* recycle = nullptr;       // staging batch reused by vlscan_scan_batch and vlscan_scan_batch_keep
    bool kept = false;                     // the last result is a kept batch (`recycle`, alive until the next scan on this ctx)
    vl::DevBuf patch, unstaged;            // vlscan_stage_selected: the column table entries it rewrites; a counter of unstaged cells with selected rows
    bool has_result = false;
    uint64_t last_launches = 0;
    int sm_count = 132;                    // H100 SXM; vlscan_ctx_create reads the device's own count
    int scan_occ[2] = {1, 1};              // resident CTAs per SM of k_substr_scan<false> / <true> on this device
    int row_occ = 1;                       // ... and of k_row_match (its persistent grid is exactly the resident set)
    void* ensure_pinned(size_t n);
};

namespace vl {
// fills word_block / init_bitmap / blk_* device arrays of a batch from host row counts (shared by upload + generate)
void finish_batch_layout(vlscan_ctx* ctx, vlscan_batch* b, const std::vector<uint32_t>& rows);

// row_off8 of column `slot` (k_lens_offsets) for the blocks in `list` (wc[wc_slot] of them) that this scan has not computed yet; ready[slot]
// is cleared by the first call of a scan.  Returns ctx->row_off8[slot].  Errors go to stats.
const uint32_t* row_offsets(vlscan_ctx* ctx, const BatchView& B, int slot, const uint32_t* list, const uint32_t* wc, unsigned long long* stats, int wc_slot);

// ---- error plumbing --------------------------------------------------------------------------------------------------
template <class F> int guarded(vlscan_ctx* ctx, F&& f) {
    try { f(); return 0; }
    catch (const CudaFail& e) { set_thread_error(e.msg); if (ctx) ctx->err = e.msg; return e.code > 0 ? e.code : 1; }
    catch (const BadInput& e) { set_thread_error(e.msg); if (ctx) ctx->err = e.msg; return -1; }
    catch (const ProgError& e) { set_thread_error(e.what()); if (ctx) ctx->err = e.what(); return -2; }
    catch (const std::exception& e) { set_thread_error(e.what()); if (ctx) ctx->err = e.what(); return -3; }
}

inline void launch_check(vlscan_ctx* ctx) { ctx->launches++; VL_CUDA(cudaGetLastError()); }
inline unsigned cdiv(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }

// the canonical names of a caller's n field names ("" is `_msg`: getCanonicalColumnName)
inline std::vector<std::string> canonical_names(const char* const* names, const size_t* lens, uint32_t n, const char* what) {
    if (n && (!names || !lens)) throw BadInput(std::string(what) + ": field names missing");
    std::vector<std::string> out;
    for (uint32_t f = 0; f < n; f++) out.push_back(lens[f] ? std::string(names[f], lens[f]) : "_msg");
    return out;
}
}  // namespace vl
