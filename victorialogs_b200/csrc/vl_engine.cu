// libvlscan.so: staging of column blocks into HBM, the filter-tree interpreter that drives the scan kernels (vl_kernels.cuh), the result
// digest and the rest of the C ABI declared in include/vlscan.h; the aggregations over a scan's result are in vl_agg.cu.  There is no CPU
// code path for the scan itself: without a CUDA device every computing entry point fails with an error.
#include <dlfcn.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <limits>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include "vl_copier.h"
#include "vl_engine.h"
#include "vl_kernels.cuh"
#include "vl_program.h"
#include "vl_part.h"
#include "vl_mathnum.cuh"

using namespace vl;

namespace vl {
static thread_local std::string g_thread_err;
void set_thread_error(const std::string& s) { g_thread_err = s; }
}  // namespace vl

struct vlscan_program {
    Program p;
    struct Image { DevBuf leaves, prepass, regexes, blob, u64s, u32s; DevProgram view; };
    std::map<int, std::unique_ptr<Image>> images;
    std::mutex mu;
    const DevProgram& image(int device, cudaStream_t st) {
        std::lock_guard<std::mutex> g(mu);
        auto it = images.find(device);
        if (it != images.end()) return it->second->view;
        auto im = std::make_unique<Image>();
        auto up = [&](DevBuf& b, const void* src, size_t n) { b.ensure(std::max<size_t>(n, 16)); if (n) VL_CUDA(cudaMemcpyAsync(b.p, src, n, cudaMemcpyHostToDevice, st)); };
        up(im->leaves, p.leaves.data(), p.leaves.size() * sizeof(DevLeaf));
        up(im->prepass, p.prepass.data(), p.prepass.size() * sizeof(DevPrepass));
        up(im->regexes, p.regexes.data(), p.regexes.size() * sizeof(DevRegex));
        up(im->blob, p.blob.data(), p.blob.size());
        up(im->u64s, p.u64s.data(), p.u64s.size() * 8);
        up(im->u32s, p.u32s.data(), p.u32s.size() * 4);
        VL_CUDA(cudaStreamSynchronize(st));
        im->view = DevProgram{im->leaves.as<DevLeaf>(), im->prepass.as<DevPrepass>(), im->regexes.as<DevRegex>(), im->blob.as<uint8_t>(), im->u64s.as<uint64_t>(), im->u32s.as<uint32_t>()};
        auto& ref = *im;
        images[device] = std::move(im);
        return ref.view;
    }
    ~vlscan_program() { for (auto& kv : images) { cudaSetDevice(kv.first); kv.second->leaves.release(); kv.second->prepass.release(); kv.second->regexes.release(); kv.second->blob.release(); kv.second->u64s.release(); kv.second->u32s.release(); } }
};

struct vlscan_host_blocks {
    void* pinned = nullptr; size_t bytes = 0;
    std::vector<vlscan_block> blocks;
    std::vector<vlscan_column> cols;
    std::vector<std::string> fields;
    std::vector<std::vector<uint32_t>> dict_offsets;
    std::vector<std::unique_ptr<std::vector<uint8_t>>> owned;   // dict tables rebuilt from a part's column headers
    std::vector<uint64_t> source;                               // vlscan_part_blocks: index of each block inside the part
};
struct vlscan_part { vl::part::PartReader r; };

void* vlscan_ctx::ensure_pinned(size_t n) {
    if (n <= pinned_cap) return pinned;
    if (pinned) cudaFreeHost(pinned);
    pinned = nullptr; pinned_cap = 0;
    VL_CUDA(cudaMallocHost(&pinned, n));
    pinned_cap = n;
    return pinned;
}

namespace {

// ---- libzstd, COMPRESSION only: vlscan_host_blocks_compress plays the reference's writer (marshalBytesBlock, encoding.go:343-360) so that
// benches and tests can feed on-disk-stage blocks.  Nothing on the scan path calls into it: frames are decoded on the device (vl_zstd.cuh).
struct ZstdWriter {
    size_t (*compress)(void*, size_t, const void*, size_t, int) = nullptr;
    size_t (*bound)(size_t) = nullptr;
    unsigned (*is_error)(size_t) = nullptr;
    bool ok = false;
    ZstdWriter() {
        void* h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        compress = (decltype(compress))dlsym(h, "ZSTD_compress");
        bound = (decltype(bound))dlsym(h, "ZSTD_compressBound");
        is_error = (decltype(is_error))dlsym(h, "ZSTD_isError");
        ok = compress && bound && is_error;
    }
};
ZstdWriter& zstd_writer() { static ZstdWriter z; return z; }

}  // namespace

// ---- batch layout shared with the generator ------------------------------------------------------------------------------
namespace vl {
void finish_batch_layout(vlscan_ctx* ctx, vlscan_batch* b, const std::vector<uint32_t>& rows) {
    b->nblocks = rows.size();
    b->h_rows = rows;
    b->h_word_off.assign(rows.size() + 1, 0);
    b->rows = 0;
    for (size_t i = 0; i < rows.size(); i++) { b->h_word_off[i + 1] = b->h_word_off[i] + (rows[i] + 63) / 64; b->rows += rows[i]; }
    b->nwords = b->h_word_off.back();
    std::vector<uint32_t> wb(b->nwords);
    std::vector<uint64_t> init(b->nwords);
    for (size_t i = 0; i < rows.size(); i++) {
        for (uint64_t w = b->h_word_off[i]; w < b->h_word_off[i + 1]; w++) { wb[w] = (uint32_t)i; init[w] = ~0ull; }
        uint32_t tail = rows[i] & 63;   // bitmap.setBits: tail bits beyond bitsLen stay zero (bitmap.go:62-72)
        if (tail) init[b->h_word_off[i + 1] - 1] = (~0ull) >> (64 - tail);
    }
    b->blk_rows.ensure(std::max<size_t>(rows.size() * 4, 16));
    b->blk_word_off.ensure((rows.size() + 1) * 8);
    b->word_block.ensure(std::max<size_t>(b->nwords * 4, 16));
    b->init_bitmap.ensure(std::max<size_t>(b->nwords * 8, 16));
    if (!rows.empty()) VL_CUDA(cudaMemcpyAsync(b->blk_rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    VL_CUDA(cudaMemcpyAsync(b->blk_word_off.p, b->h_word_off.data(), (rows.size() + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (b->nwords) {
        VL_CUDA(cudaMemcpyAsync(b->word_block.p, wb.data(), b->nwords * 4, cudaMemcpyHostToDevice, ctx->stream));
        VL_CUDA(cudaMemcpyAsync(b->init_bitmap.p, init.data(), b->nwords * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    VL_CUDA(cudaStreamSynchronize(ctx->stream));   // wb / init are stack-owned
}
}  // namespace vl

// ---- upload --------------------------------------------------------------------------------------------------------------
// The on-disk values blocks of a batch in (block, column) order; each one's place in the compressed staging buffer is a running sum that
// starts behind 512 bytes of headroom (the device bit readers load whole aligned words around a stream).  Returns the end of the last one.
// need (may be NULL = all): need[block * nfields + field] != 0 for the columns whose values are staged (phase 2 of a bloom-first upload).
// at (may be NULL): at[block * nfields + field] = the index in zv of that cell's block (the first, should a block list the field twice).
static uint64_t collect_values_blocks(const vlscan_block* blocks, uint64_t nblocks, std::vector<ZValuesBlock>& zv, const uint8_t* need = nullptr, uint32_t nfields = 0, std::vector<size_t>* at = nullptr) {
    uint64_t zc = 512;
    if (at) at->assign((size_t)nblocks * nfields, SIZE_MAX);
    for (uint64_t b = 0; b < nblocks; b++)
        for (uint32_t k = 0; k < blocks[b].ncols; k++) {
            const vlscan_column& c = blocks[b].cols[k];
            if (c.kind != VLSCAN_COL_VALUES || c.stage != VLSCAN_STAGE_ONDISK) continue;
            if (need && (c.field >= nfields || !need[b * nfields + c.field])) continue;
            if (at && c.field < nfields && (*at)[b * nfields + c.field] == SIZE_MAX) (*at)[b * nfields + c.field] = zv.size();
            zv.push_back({c.values, (size_t)c.values_len, zc});
            zc += c.values_len;
        }
    return zc;
}
static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

namespace {
// One staging step of a batch into one device region (see do_upload).  The helpers below describe cells into the host column table and
// collect what the region receives; which of them run for which cells is the step's business.  commit() then fills the region.
struct Upload {
    vlscan_ctx* ctx; vlscan_batch* out; const vlscan_block* blocks; uint64_t nblocks; uint32_t nfields; vlscan_stats* stats;
    const std::vector<char>* need_bloom;
    std::vector<DevColumn>& cols = out->h_cols;   // the steps after the header step continue with the table it left
    const bool dbg = getenv("VLSCAN_DEBUG_TIMING") != nullptr; const double t_start = now_s();
    Copier io{ctx};
    std::vector<uint32_t> rows = std::vector<uint32_t>(nblocks);
    std::vector<Piece> pieces;   // host -> region
    std::vector<std::unique_ptr<std::vector<uint8_t>>> owned;   // dict metadata built here
    uint64_t cursor = 16;   // the first 16 bytes stay unused so that every payload has a readable byte in front of it
    // On-disk values blocks are not copied into the region: their bytes go to the compressed staging buffer as they are and the device
    // regenerates them (vl_zstd.cuh) into regions placed behind everything that is copied, so that host memory laid out like
    // the copied part still goes out as one DMA.  Region offsets are relative to `regen_base` until commit() has sized that part.
    ZstdJob zjob;
    uint64_t regen_cursor = 0;
    struct Ondisk { uint64_t col; uint32_t lens_frame, data_frame; uint64_t lens_rel, data_rel; };
    std::vector<Ondisk> ondisk;
    std::vector<OndiskCol> ocols;
    struct TsFrame { uint64_t block; uint32_t frame; uint64_t rel; };
    std::vector<TsFrame> ts_frames;
    std::vector<DevTimestamps> tsv;   // empty until some block comes with its timestamps column
    // the on-disk values blocks (zv_of: cell -> index in zv / zinfo) and the places of the ZSTD timestamps blocks (by block)
    std::vector<ZValuesBlock> zv; std::vector<ZValuesInfo> zinfo; std::vector<size_t> zv_of; std::vector<uint64_t> ts_zoff; size_t zbad = SIZE_MAX; std::string zmsg;
    uint64_t add_piece(const uint8_t* src, uint64_t len) { uint64_t off = arena_reserve(cursor, len); if (len) pieces.push_back({src, len, off}); return off; }
    // f(block, column, cell) for every column of every block, in order, behind the block's checks and (with `ts`) its timestamps column
    template <class F> void walk(bool ts, F&& f) {
        for (uint64_t b = 0; b < nblocks; b++) {
            const vlscan_block& blk = blocks[b];
            if (blk.rows > (8u << 20)) throw BadInput("block rows exceed maxRowsPerBlock (8Mi)");   // consts.go:24
            rows[b] = (uint32_t)blk.rows;
            if (ts) timestamps(blk, b);
            for (uint32_t k = 0; k < blk.ncols; k++) {
                if (blk.cols[k].field >= nfields) throw BadInput("column refers to a field outside the batch field table");
                f(blk, blk.cols[k], (size_t)b * nfields + blk.cols[k].field);
            }
        }
    }
    // The compressed bytes of the on-disk values blocks (those marked in `need`, or all) and, with `ts`, of the ZSTD timestamps blocks are
    // shipped first, so that the DMA engine is busy while the host walks frame and block headers.
    void sources(const uint8_t* need, bool ts) {
        uint64_t zc = collect_values_blocks(blocks, nblocks, zv, need, nfields, &zv_of);
        for (const ZValuesBlock& v : zv) if (v.n) io.src.push_back({v.p, v.n, v.zoff});
        ts_zoff.resize(ts ? nblocks : 0);
        for (uint64_t b = 0; b < nblocks && ts; b++) {
            const vlscan_block& blk = blocks[b];
            if (blk.ts_marshal_type != MT_ZSTD_NEAREST_DELTA2 && blk.ts_marshal_type != MT_ZSTD_NEAREST_DELTA) continue;
            if (blk.timestamps_len > vl::part::kMaxTimestampsBlockSize) throw BadInput("timestamps block size cannot exceed 8 MiB");   // getTimestamps block_search.go:490-493
            ts_zoff[b] = zc;
            if (blk.timestamps_len) io.src.push_back({blk.timestamps, blk.timestamps_len, zc});
            zc += blk.timestamps_len;
        }
        if (!io.src.empty()) { ctx->zsrc.ensure(zc + 512); io.send_sources(ctx->zsrc.as<uint8_t>()); }
        // frame, block and section headers of all of them, on several host threads; a malformed block is reported when values() gets to it
        zinfo.resize(zv.size());
        const double t_w = now_s();
        if (!zv.empty()) zjob.add_values_blocks(zv.data(), zv.size(), host_threads(), zinfo.data(), &zbad, &zmsg);
        if (dbg) fprintf(stderr, "[vlscan upload] header walk of %zu values blocks on %d host threads: %.1f ms (after %.1f ms of collecting and enqueueing the copies)\n",
                         zv.size(), host_threads(), 1e3 * (now_s() - t_w), 1e3 * (t_w - t_start));
    }
    // kind, const value, bloom filter and dict table of a column; `payload` stages or defers the values, whose pieces come before the bloom filter
    template <class F> void header(const vlscan_column& c, size_t i, F&& payload) {
        DevColumn& d = cols[i];
        if (d.kind != COL_MISSING) throw BadInput("duplicate column for one field in a block");
        if (c.kind == VLSCAN_COL_CONST) {
            d.kind = COL_CONST; d.meta_len = (uint32_t)c.const_len; d.meta_off = add_piece(c.const_value, c.const_len);
            return;
        }
        if (c.kind != VLSCAN_COL_VALUES) throw BadInput("unknown column kind");
        if (c.value_type < VT_STRING || c.value_type >= VT_MAX) throw BadInput("unknown valueType");
        d.kind = COL_VALUES; d.vt = c.value_type; d.min_value = c.min_value; d.max_value = c.max_value;
        payload();
        if (c.bloom_len % 8) throw BadInput("cannot unmarshal bloomFilter from src with size not multiple by 8");   // bloomfilter.go:59-61
        if (need_bloom && !(*need_bloom)[c.field]) { d.bloom_words = 0; d.bloom_off = add_piece(c.bloom, 0); }
        else { d.bloom_words = (uint32_t)(c.bloom_len / 8); d.bloom_off = add_piece(c.bloom, c.bloom_len); }
        if (c.value_type == VT_DICT) {
            if (c.dict_len > 8) throw BadInput("valuesDict may contain max 8 items");
            d.dict_len = c.dict_len;
            uint32_t total = c.dict_len ? c.dict_offsets[c.dict_len] : 0;
            d.meta_len = total;
            if (c.dict_len && c.dict_blob == (const uint8_t*)c.dict_offsets + 4 * (c.dict_len + 1)) {
                d.meta_off = add_piece((const uint8_t*)c.dict_offsets, 4 * (c.dict_len + 1) + total);   // caller memory already has the device layout
            } else {
                auto meta = std::make_unique<std::vector<uint8_t>>();
                meta->resize(4 * (c.dict_len + 1) + total);
                if (c.dict_len) memcpy(meta->data(), c.dict_offsets, 4 * (c.dict_len + 1)); else memset(meta->data(), 0, 4);
                if (total) memcpy(meta->data() + 4 * (c.dict_len + 1), c.dict_blob, total);
                d.meta_off = add_piece(meta->data(), meta->size());
                owned.push_back(std::move(meta));
            }
        }
    }
    // the values payload of a column: on-disk stage -> regenerated by the device decoder, decoded stage -> copied
    void values(const vlscan_block& blk, const vlscan_column& c, size_t ci) {
        DevColumn& d = cols[ci];
        if (c.stage == VLSCAN_STAGE_ONDISK) {
            // stringsBlockUnmarshaler.unmarshal: bytesBlock(lens) ++ bytesBlock(data) (encoding.go:83-108).  The host reads the
            // containers, the frame header and the block headers; the payload is regenerated on the device.
            const size_t z = zv_of[ci];
            if (z >= zbad) throw BadInput(zmsg);
            const uint64_t lens_len = zinfo[z].lens_len, data_len = zinfo[z].data_len;
            if (data_len > 0xFFFFFFFFull) throw BadInput("values block too large");
            // the uint block type byte lands on offset 15 of its region, so the lens items behind it are 16-byte aligned
            const uint64_t lr = arena_reserve(regen_cursor, lens_len + 15), dr = arena_reserve(regen_cursor, data_len);
            d.lens_off = lr + 16; d.data_off = dr; d.data_len = data_len;
            ondisk.push_back({ci, (uint32_t)(2 * z), (uint32_t)(2 * z + 1), lr + 15, dr});   // frames 2z, 2z + 1: lens and data
            ocols.push_back({ci, lens_len, blk.rows});   // lens header checks + lens_type / lens_const / data_const: k_finish_ondisk_cols
        } else if (c.stage == VLSCAN_STAGE_DECODED) {
            const uint8_t* lens_items = c.lens_items; const uint64_t lens_len = c.lens_items_len, data_len = c.data_len;
            // unmarshalUint64Items header checks (encoding.go:246-336)
            if (lens_len < 1) throw BadInput("cannot unmarshal uint64 block type from empty src");
            uint8_t lt = lens_items[0];
            if (lt > 7) throw BadInput("unexpected uint64 block type");
            uint64_t want = lt < 4 ? (blk.rows << lt) : (1ull << (lt - 4));
            if (lens_len - 1 != want) throw BadInput("unexpected block length for uint items");
            d.lens_type = lt;
            if (lt >= 4) { uint64_t v = 0; for (uint64_t i = 0; i < want; i++) v = (v << 8) | lens_items[1 + i]; if (v > 0xFFFFFFFFull) throw BadInput("row length does not fit 32 bits"); d.lens_const = (uint32_t)v; }
            if (data_len > 0xFFFFFFFFull) throw BadInput("values block too large");
            d.lens_off = add_piece(lens_items + 1, lens_len - 1);
            d.data_off = add_piece(c.data, data_len); d.data_len = data_len;
            // decode rule of encoding.go:113-120: rows >= 2, all lens equal, len(data) == lens[0] => every row = data
            d.data_const = (blk.rows >= 2 && lt >= 4 && data_len == d.lens_const) ? 1 : 0;
        } else throw BadInput("unknown values stage");
    }
    // the timestamps column of a block that has one: encoded deltas as stored + timestampsHeader (block_header.go:990-997)
    void timestamps(const vlscan_block& blk, uint64_t b) {
        if (!blk.ts_marshal_type) return;
        if (blk.ts_marshal_type > MT_NEAREST_DELTA) throw BadInput("unknown MarshalType of a timestamps block");
        if (blk.timestamps_len > vl::part::kMaxTimestampsBlockSize) throw BadInput("timestamps block size cannot exceed 8 MiB");
        if (tsv.empty()) { tsv.resize(nblocks); memset(tsv.data(), 0, nblocks * sizeof(DevTimestamps)); }
        DevTimestamps& t = tsv[b];
        t.first = blk.min_timestamp; t.max = blk.max_timestamp;
        if (blk.ts_marshal_type == MT_ZSTD_NEAREST_DELTA2 || blk.ts_marshal_type == MT_ZSTD_NEAREST_DELTA) {
            uint64_t regen = 0; uint32_t id = 0;
            zjob.add_frame(blk.timestamps, blk.timestamps_len, ts_zoff[b], &regen, &id);   // throws on a malformed frame header
            if (regen > 10ull * blk.rows + 16) throw BadInput("cannot unmarshal timestamps: the decompressed block is larger than its varints can be");
            t.mt = blk.ts_marshal_type == MT_ZSTD_NEAREST_DELTA2 ? MT_NEAREST_DELTA2 : MT_NEAREST_DELTA;
            t.len = (uint32_t)regen;
            ts_frames.push_back({b, id, arena_reserve(regen_cursor, regen)});
        } else {
            t.mt = (uint8_t)blk.ts_marshal_type; t.len = (uint32_t)blk.timestamps_len;
            t.off = add_piece(blk.timestamps, blk.timestamps_len);
        }
    }

    // Places the regenerated regions behind the copied part, sizes `region` and fills it; returns its size.  patch (may be NULL = the whole
    // column table): the cells of a late region, whose table entries alone are sent.  layout: a new batch, whose layout tables are built too.
    uint64_t commit(DevBuf& region, const std::vector<uint64_t>* patch, bool layout) {
        const uint64_t regen_base = (cursor + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
        for (const Ondisk& o : ondisk) {
            DevColumn& d = cols[o.col];
            d.lens_off += regen_base; d.data_off += regen_base;
            zjob.set_dst(o.lens_frame, regen_base + o.lens_rel); zjob.set_dst(o.data_frame, regen_base + o.data_rel);
        }
        for (const TsFrame& tf : ts_frames) { tsv[tf.block].off = regen_base + tf.rel; zjob.set_dst(tf.frame, regen_base + tf.rel); }
        const bool have_z = !ondisk.empty() || !ts_frames.empty();
        if (have_z) cursor = regen_base + regen_cursor;
        const uint64_t bytes = cursor + kArenaPad;
        const double t_desc = now_s();
        region.ensure(bytes);
        const double t_alloc = now_s();
        // Late cells keep the arena-relative addressing of every kernel: their offsets are taken from the batch arena's base to the late region
        // (modulo 2^64, so a region below the arena works too), and k_finish_ondisk_cols reads them against that base as well.
        uint8_t* cols_base = region.as<uint8_t>();
        std::vector<ColPatch> patches;
        if (patch) {
            const uint64_t delta = (uint64_t)(uintptr_t)region.p - (uint64_t)(uintptr_t)out->arena.p;
            cols_base = out->arena.as<uint8_t>();
            patches.resize(patch->size());
            for (size_t i = 0; i < patch->size(); i++) {
                DevColumn& d = cols[(*patch)[i]];
                d.lens_off += delta; d.data_off += delta;
                patches[i].col = (*patch)[i]; patches[i].c = d;
            }
        }
        // the region is cleared on the compute stream; the copy stream takes over from there
        cudaStream_t cs = ctx->copy_stream;
        cudaEvent_t ev_cleared = io.events.make(), ev_copied = io.events.make();
        VL_CUDA(cudaMemsetAsync(region.p, 0, bytes, ctx->stream));
        VL_CUDA(cudaEventRecord(ev_cleared, ctx->stream));
        VL_CUDA(cudaStreamWaitEvent(cs, ev_cleared, 0));
        // The decoder is enqueued BEFORE anything below that can block this thread (packing pageable pieces through the staging ring, copies
        // from pageable vectors): each launch group then runs as soon as its compressed bytes have landed, beside the DMA of the later ones.
        const double t_h2d = dbg ? now_s() : 0;
        double t_zrun = 0;
        if (have_z) {
            zjob.set_group_hook([&](uint64_t src_end) { io.wait_sources(ctx->stream, src_end); });
            zjob.run(ctx, ctx->zsrc.as<uint8_t>(), region.as<uint8_t>());
            io.ship_sources(UINT64_MAX);
            if (dbg) t_zrun = now_s();
        }
        io.copy(pieces, region.as<uint8_t>());
        // the column table, or only the entries of a late region's cells: the table on the device has what k_finish_ondisk_cols derived since
        DevBuf& table = patch ? ctx->patch : out->cols;
        const void* entries = patch ? (const void*)patches.data() : (const void*)cols.data();
        const size_t table_bytes = patch ? patches.size() * sizeof(ColPatch) : cols.size() * sizeof(DevColumn);
        table.ensure(std::max<size_t>(table_bytes, 16));
        if (table_bytes) VL_CUDA(cudaMemcpyAsync(table.p, entries, table_bytes, cudaMemcpyHostToDevice, cs));
        io.h2d += table_bytes;
        if (!patch) out->has_ts = !tsv.empty();   // a late region leaves the timestamps alone
        if (!tsv.empty()) {
            out->ts.ensure(nblocks * sizeof(DevTimestamps));
            VL_CUDA(cudaMemcpyAsync(out->ts.p, tsv.data(), nblocks * sizeof(DevTimestamps), cudaMemcpyHostToDevice, cs));
            io.h2d += nblocks * sizeof(DevTimestamps);
        }
        VL_CUDA(cudaEventRecord(ev_copied, cs));
        if (!patches.empty()) {
            VL_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied, 0));
            k_patch_cols<<<cdiv(patches.size(), 128), 128, 0, ctx->stream>>>(out->cols.as<DevColumn>(), ctx->patch.as<ColPatch>(), (uint32_t)patches.size());
            launch_check(ctx);
        }
        const double t_enq = dbg ? now_s() : 0;
        if (have_z) {
            // the on-disk payloads are being regenerated in HBM; derive lens_type / lens_const / data_const from the regenerated lens blocks
            VL_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied, 0));
            ctx->zcols.ensure(16 + ocols.size() * sizeof(OndiskCol));
            VL_CUDA(cudaMemsetAsync(ctx->zcols.p, 0, 16, ctx->stream));
            VL_CUDA(cudaMemcpyAsync(ctx->zcols.as<uint8_t>() + 16, ocols.data(), ocols.size() * sizeof(OndiskCol), cudaMemcpyHostToDevice, ctx->stream));
            if (!ocols.empty()) {
                k_finish_ondisk_cols<<<cdiv(ocols.size(), 128), 128, 0, ctx->stream>>>(cols_base, out->cols.as<DevColumn>(), (const OndiskCol*)(ctx->zcols.as<uint8_t>() + 16),
                                                                                         (uint32_t)ocols.size(), ctx->zcols.as<unsigned long long>());
                launch_check(ctx);
            }
            io.h2d += ocols.size() * sizeof(OndiskCol);
            zjob.check(ctx);   // synchronises the stream
            unsigned long long cst[2] = {0, 0};
            VL_CUDA(cudaMemcpy(cst, ctx->zcols.p, 16, cudaMemcpyDeviceToHost));
            static const char* what[] = {"", "cannot unmarshal uint64 block type from empty src", "unexpected uint64 block type", "unexpected block length for uint items", "row length does not fit 32 bits"};
            if (cst[0]) throw BadInput(what[std::min<unsigned long long>(cst[0], 4)]);
        }
        VL_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied, 0));
        double t_copy = 0;
        if (dbg) { VL_CUDA(cudaStreamSynchronize(ctx->stream)); t_copy = now_s(); }
        if (nfields) out->note_columns(cols);
        if (layout) finish_batch_layout(ctx, out, rows);   // synchronises the stream => `owned`, `cols`, staging are safe to drop
        else VL_CUDA(cudaStreamSynchronize(ctx->stream));  // the layout tables are there since the header step
        if (dbg) fprintf(stderr, "[vlscan upload] blocks=%llu arena=%.1f MB h2d=%.1f MB pieces=%zu+%zu pinned=%d: describe %.1f ms, alloc %.1f ms, copy %.1f ms (%.1f GB/s), "
                                 "zstd %llu frames / %llu blocks / %llu sequences: enqueue %.1f ms, decode %.1f ms; layout %.1f ms\n", (unsigned long long)nblocks,
                         bytes / 1e6, io.h2d / 1e6, pieces.size(), io.src.size(), (int)io.all_pinned, 1e3 * (t_desc - t_start), 1e3 * (t_alloc - t_desc), 1e3 * (t_enq - (t_zrun > 0 ? t_zrun : t_h2d)), io.h2d / 1e9 / std::max(t_copy - t_start, 1e-9),
                         (unsigned long long)zjob.frames(), (unsigned long long)zjob.compressed_blocks(), (unsigned long long)zjob.sequences(), 1e3 * (t_zrun > 0 ? t_zrun - t_h2d : 0), 1e3 * (t_copy - t_enq), 1e3 * (now_s() - t_copy));
        if (layout) io.h2d += out->nwords * 12 + nblocks * 12;
        if (stats) stats->h2d_bytes += io.h2d;
        return bytes;
    }
};
}  // namespace

// need_bloom (may be NULL = all): per batch field, whether the program that will scan this batch ever probes that field's bloom filters.  A filter
// nobody probes stays on the host (the reference reads a column's bloom filter lazily, only when a filter asks for it: getBloomFilterForColumn,
// block_search.go:411-439); the column is staged with an empty filter, which no kernel touches.
//
// mode: UP_FULL stages everything in one go.  A bloom-first upload (vlscan_scan_batch, the reference's lazy order: a column's values are read only
// after its bloom filter let the block through, block_search.go:411-439 then :444-474) runs the function twice around the probe pass:
// UP_HEADERS stages what the header dispatch and the bloom probes look at (const values, bloom filters, dict tables -> batch->harena) and
// leaves every values payload on the host (VALUES_DEFERRED); UP_VALUES then stages the timestamps and the values of the columns the probe marked in
// `need` (-> batch->arena) and flags the others VALUES_ABSENT.
// UP_LATE (vlscan_stage_selected on a kept batch) stages the values of the columns marked in `need` into a new region of the batch
// (batch->late), leaves every other cell as it is and rewrites only the staged cells' entries of the device column table.
// A failed upload drains both streams before the error leaves it: nothing may still read the caller's buffers.
enum UploadMode { UP_FULL = 0, UP_HEADERS = 1, UP_VALUES = 2, UP_LATE = 3 };
static void do_upload(vlscan_ctx* ctx, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields, const vlscan_block* blocks,
                      uint64_t nblocks, vlscan_batch* out, vlscan_stats* stats, const std::vector<char>* need_bloom = nullptr, UploadMode mode = UP_FULL,
                      const uint8_t* need = nullptr, uint64_t* zframes = nullptr) {
    VL_CUDA(cudaSetDevice(ctx->device));
    if (nblocks > 0xFFFFFFF0ull) throw BadInput("too many blocks in one batch");
    out->device = ctx->device; out->nfields = nfields;
    Upload u{ctx, out, blocks, nblocks, nfields, stats, need_bloom};
    if (mode == UP_FULL || mode == UP_HEADERS) {   // a new batch: the late regions of the previous one are free
        for (uint32_t f = 0; f < nfields; f++) out->field_names.emplace_back(field_names[f], field_name_lens[f]);
        u.cols.assign((size_t)nblocks * std::max<uint32_t>(nfields, 1), DevColumn{});
        memset(u.cols.data(), 0, u.cols.size() * sizeof(DevColumn));
        out->late_used = 0; out->split_hdr = mode == UP_HEADERS;
    } else if (u.cols.size() != (size_t)nblocks * std::max<uint32_t>(nfields, 1) || !need) throw BadInput("internal: values phase of a bloom-first upload without its header phase");
    try {
        switch (mode) {
        case UP_FULL:
            u.sources(nullptr, true);
            u.walk(true, [&](const vlscan_block& blk, const vlscan_column& c, size_t i) { u.header(c, i, [&] { u.values(blk, c, i); }); });
            out->arena_bytes = u.commit(out->arena, nullptr, true);
            out->harena_bytes = 0;
            std::vector<DevColumn>().swap(out->h_cols);   // only a bloom-first upload needs the table again
            break;
        case UP_HEADERS:
            u.walk(false, [&](const vlscan_block&, const vlscan_column& c, size_t i) {
                u.header(c, i, [&] {
                    if (c.stage != VLSCAN_STAGE_ONDISK && c.stage != VLSCAN_STAGE_DECODED) throw BadInput("unknown values stage");
                    u.cols[i].values_state = VALUES_DEFERRED;
                });
            });
            out->harena_bytes = u.commit(out->harena, nullptr, true);
            break;
        case UP_VALUES:
            u.sources(need, true);
            u.walk(true, [&](const vlscan_block& blk, const vlscan_column& c, size_t i) {
                if (c.kind != VLSCAN_COL_VALUES) return;
                u.cols[i].values_state = need[i] ? VALUES_STAGED : VALUES_ABSENT;
                if (need[i]) u.values(blk, c, i);
            });
            out->arena_bytes = u.commit(out->arena, nullptr, false);
            break;
        case UP_LATE: {
            std::vector<uint64_t> staged;
            u.sources(need, false);
            u.walk(false, [&](const vlscan_block& blk, const vlscan_column& c, size_t i) {
                if (c.kind != VLSCAN_COL_VALUES || !need[i]) return;
                // `need` marks unstaged cells only: one staged already is a field this block lists twice
                if (u.cols[i].values_state == VALUES_STAGED) throw BadInput("duplicate column for one field in a block");
                u.cols[i].values_state = VALUES_STAGED;
                u.values(blk, c, i);
                staged.push_back(i);
            });
            if (out->late_used == out->late.size()) out->late.emplace_back();
            u.commit(out->late[out->late_used], &staged, false);
            out->late_used++;
            *zframes += u.zjob.frames();
            break;
        }
        }
    } catch (...) {
        cudaStreamSynchronize(ctx->copy_stream); cudaStreamSynchronize(ctx->stream);
        throw;
    }
}

// ---- the filter-tree interpreter --------------------------------------------------------------------------------------------
const uint32_t* vl::row_offsets(vlscan_ctx* ctx, const BatchView& B, int slot, const uint32_t* list, const uint32_t* wc, unsigned long long* stats, int wc_slot) {
    uint8_t* ready = ctx->ready[slot].as<uint8_t>();
    if (!ctx->ready_cleared[slot]) { VL_CUDA(cudaMemsetAsync(ready, 0, B.nblocks, ctx->stream)); ctx->ready_cleared[slot] = 1; }
    k_lens_offsets<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(B, slot, list, wc, ctx->row_off8[slot].as<uint32_t>(), ready, stats, wc_slot); launch_check(ctx);
    return ctx->row_off8[slot].as<uint32_t>();
}

namespace {
struct ScanRun {
    vlscan_ctx* ctx; const vlscan_program* prog; const vlscan_batch* batch;
    DevProgram P; BatchView B; std::vector<int> field_slot;   // program field -> batch field slot or -1
    unsigned long long* stats;
    size_t regs_used = 0;

    uint64_t* new_reg() {
        if (regs_used == ctx->regs.size()) ctx->regs.emplace_back();
        DevBuf& r = ctx->regs[regs_used++];
        r.ensure(std::max<size_t>(B.nwords * 8, 16));
        return r.as<uint64_t>();
    }
    void free_reg() { regs_used--; }
    void copy_reg(uint64_t* dst, const uint64_t* src) { if (B.nwords) VL_CUDA(cudaMemcpyAsync(dst, src, B.nwords * 8, cudaMemcpyDeviceToDevice, ctx->stream)); }
    void andnot(uint64_t* a, const uint64_t* b) { if (!B.nwords) return; k_andnot<<<cdiv(B.nwords, 256), 256, 0, ctx->stream>>>(a, b, B.nwords); launch_check(ctx); }
    void prepass(const PNode& nd, uint64_t* reg) {
        if (nd.prepass_count == 0) return;
        std::vector<int> slots(nd.prepass_count);
        for (int e = 0; e < nd.prepass_count; e++) slots[e] = field_slot[prog->p.prepass[nd.prepass_begin + e].field];
        // slots live in a small device array; successive pre-passes use disjoint regions of it
        size_t off = slots_cursor; slots_cursor += slots.size();
        ctx->slots.ensure(std::max<size_t>(slots_total * 4, 16));
        VL_CUDA(cudaMemcpyAsync(ctx->slots.as<int>() + off, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        k_prepass<<<cdiv((uint64_t)B.nblocks * 32, 128), 128, 0, ctx->stream>>>(P, B, (uint32_t)nd.prepass_begin, (uint32_t)nd.prepass_count, ctx->slots.as<int>() + off,
                                                                             nd.kind == F_OR, reg, stats);
        launch_check(ctx);
    }
    size_t slots_cursor = 0, slots_total = 0;

    void leaf(int leaf_idx, uint64_t* reg) {
        const DevLeaf& L = prog->p.leaves[leaf_idx];
        if (L.kind == F_NOOP) return;
        int slot = L.field >= 0 ? field_slot[L.field] : -1;
        uint8_t* action = ctx->action.as<uint8_t>(); uint64_t* payload = ctx->payload.as<uint64_t>(); uint64_t* leaf_bm = ctx->leaf_bm.as<uint64_t>();
        uint32_t* lens_blocks = ctx->lens_blocks.as<uint32_t>(); uint32_t* row_blocks = ctx->row_blocks.as<uint32_t>(); uint32_t* wc = ctx->work_count.as<uint32_t>();
        ScanTile* tiles = ctx->tiles.as<ScanTile>();
        VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
        if (L.kind == F_EQ_FIELD || L.kind == F_LE_FIELD) {   // two columns, row by row (filter_eq_field.go, filter_le_field.go)
            const int slot_b = field_slot[L.field2];
            uint32_t* lens_b = ctx->lens_blocks2.as<uint32_t>();
            k_plan_pair<<<cdiv((uint64_t)B.nblocks * 32, 256), 256, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, slot_b, reg, action, payload, lens_blocks, lens_b, row_blocks, wc, stats);
            launch_check(ctx);
            if (B.nwords) {
                const int persistent = ctx->sm_count * 8;
                const uint32_t *ro_a = nullptr, *ro_b = nullptr;
                for (int side = 0; side < 2; side++) {
                    const int sl = side ? slot_b : slot;
                    if (sl >= 0) (side ? ro_b : ro_a) = row_offsets(ctx, B, sl, side ? lens_b : lens_blocks, wc, stats, side ? WC_LENS2 : WC_LENS);
                }
                k_row_pair<<<persistent, 256, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, slot_b, row_blocks, wc, payload, reg, ro_a, ro_b, leaf_bm, stats); launch_check(ctx);
                k_apply_leaf<<<cdiv(B.nwords, 256), 256, 0, ctx->stream>>>(B, action, leaf_bm, reg); launch_check(ctx);
            }
            return;
        }
        // bm.isZero() per block, header dispatch + leaf bloom probe -> per-block action, and the work lists of the kernels below
        k_plan_leaf<<<cdiv(B.nblocks, VL_PLAN_WARPS), VL_PLAN_WARPS * 32, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, reg, action, payload, lens_blocks, row_blocks, tiles, wc, stats);
        launch_check(ctx);
        if (slot >= 0 && B.nwords) {
            // which kernels can have work is known from the value types this field takes in the batch (header dispatch is per block,
            // on the device, but a field that is never a plain string column cannot produce ACT_SCAN, etc.)
            const uint32_t vts = batch->slot_vt_mask.empty() ? ~0u : batch->slot_vt_mask[slot];
            const bool has_string = vts >> VT_STRING & 1, has_dict = vts >> VT_DICT & 1;
            const bool has_numeric = (vts & ~((1u << VT_STRING) | (1u << VT_DICT))) != 0;
            const bool may_scan = L.str_strategy == STR_SCAN && has_string;
            const bool may_row = (has_string && L.str_strategy != STR_ALL) || has_numeric;   // also the fallback of scan leaves for blocks with short rows (k_plan_leaf)
            const uint32_t* ro = may_scan || may_row ? row_offsets(ctx, B, slot, lens_blocks, wc, stats, WC_LENS) : nullptr;
            // row-agnostic substring scan
            if (may_scan) {
                VL_CUDA(cudaMemsetAsync(leaf_bm, 0, B.nwords * 8, ctx->stream));
                ScanParams sp; memset(&sp, 0, sizeof sp);
                sp.mode = L.scan_mode; sp.needle_off = L.scan_needle_off; sp.needle_len = L.scan_needle_len; sp.starts_tok = L.starts_tok; sp.ends_tok = L.ends_tok; sp.regex = L.regex;
                const bool masked = fill_scan_patterns(prog->p.blob.data() + L.scan_needle_off, L.scan_needle_len, sp.pat, sp.msk, sp.delta, sp.nd16);
                if (L.scan_mode == SCAN_CONTAINS || L.scan_mode >= SCAN_RX_DOTPLUS) { sp.starts_tok = sp.ends_tok = 0; }
                auto& evp = next_scan_events();
                VL_CUDA(cudaEventRecord(evp.first, ctx->stream));
                // persistent CTAs: exactly the resident set (SMs x resident CTAs per SM), each striding over the tile table
                if (masked) k_substr_scan<true><<<ctx->sm_count * ctx->scan_occ[1], VL_SCAN_THREADS, 0, ctx->stream>>>(P, B, slot, sp, tiles, wc, ro, leaf_bm);
                else k_substr_scan<false><<<ctx->sm_count * ctx->scan_occ[0], VL_SCAN_THREADS, 0, ctx->stream>>>(P, B, slot, sp, tiles, wc, ro, leaf_bm);
                launch_check(ctx);
                VL_CUDA(cudaEventRecord(evp.second, ctx->stream));
            }
            // per-row matcher (string exact / in / general regexp; numeric columns through text); persistent grid over the ACT_ROW work list
            if (may_row) { k_row_match<<<ctx->sm_count * ctx->row_occ, 256, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, row_blocks, wc, action, payload, reg, ro, leaf_bm); launch_check(ctx); }
            if (has_dict || has_numeric) { k_word_match<<<cdiv(B.nwords, 128), 128, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, action, payload, reg, leaf_bm, stats); launch_check(ctx); }
        }
        if (L.kind == F_TIME && B.nwords) {   // blocks the range only partly covers: decode their timestamps, compare per row
            ctx->ts_vals.ensure(B.nwords * 64 * 8);
            k_time_match<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(B, (long long)L.aux0, (long long)L.aux1, row_blocks, wc, ctx->ts_vals.as<unsigned long long>(), leaf_bm, stats);
            launch_check(ctx);
        }
        if (B.nwords) { k_apply_leaf<<<cdiv(B.nwords, 256), 256, 0, ctx->stream>>>(B, action, leaf_bm, reg); launch_check(ctx); }
    }
    std::pair<cudaEvent_t, cudaEvent_t>& next_scan_events() {
        if (ctx->scan_events_used == ctx->scan_events.size()) { cudaEvent_t a, b; VL_CUDA(cudaEventCreate(&a)); VL_CUDA(cudaEventCreate(&b)); ctx->scan_events.emplace_back(a, b); }
        return ctx->scan_events[ctx->scan_events_used++];
    }
    // ---- probe pass of a bloom-first upload: which (block, column) values can the program reach? ------------------------------------------
    // `reg` only says which blocks are still alive: the AND / OR bloom pre-passes of a leaf's ancestors zero the blocks they rule out
    // (exactly what they do to the bitmaps of the real scan); leaves do not touch it.  The real scan hands a leaf a subset of these rows, so
    // the blocks whose values it reads are a subset of the blocks marked here.
    void probe_leaf(int leaf_idx, const uint64_t* reg, uint8_t* need) {
        const DevLeaf& L = prog->p.leaves[leaf_idx];
        if (L.kind == F_NOOP || L.kind == F_TIME) return;   // timestamps always travel with the block
        const int slot = L.field >= 0 ? field_slot[L.field] : -1;
        if (L.kind == F_EQ_FIELD || L.kind == F_LE_FIELD) {
            k_plan_pair<<<cdiv((uint64_t)B.nblocks * 32, 256), 256, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, field_slot[L.field2], reg, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stats, need);
        } else {
            if (slot < 0) return;   // a field the batch does not have: nothing to stage
            k_plan_leaf<<<cdiv(B.nblocks, VL_PLAN_WARPS), VL_PLAN_WARPS * 32, 0, ctx->stream>>>(P, B, (uint32_t)leaf_idx, slot, reg, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stats, need);
        }
        launch_check(ctx);
    }
    void probe_node(int id, uint64_t* reg, uint8_t* need) {
        const PNode& nd = prog->p.nodes[id];
        switch (nd.kind) {
        case F_NOOP: break;
        case F_AND: case F_OR: {
            uint64_t* r = reg;
            if (nd.prepass_count) { r = new_reg(); copy_reg(r, reg); prepass(nd, r); }
            for (int k : nd.kids) probe_node(k, r, need);
            if (nd.prepass_count) free_reg();
            break;
        }
        case F_NOT: probe_node(nd.kids[0], reg, need); break;
        default: probe_leaf(nd.leaf, reg, need);
        }
    }
    // applyToBlockSearch of the combinators: filter_and.go:58-74, filter_or.go:55-78, filter_not.go:38-46
    void node(int id, uint64_t* reg) {
        const PNode& nd = prog->p.nodes[id];
        switch (nd.kind) {
        case F_NOOP: break;
        case F_AND: prepass(nd, reg); for (int k : nd.kids) node(k, reg); break;
        case F_OR: {
            prepass(nd, reg);
            uint64_t* res = new_reg(); uint64_t* tmp = new_reg();
            copy_reg(res, reg);
            for (int k : nd.kids) { copy_reg(tmp, res); node(k, tmp); andnot(res, tmp); }
            andnot(reg, res);
            free_reg(); free_reg();
            break;
        }
        case F_NOT: { uint64_t* tmp = new_reg(); copy_reg(tmp, reg); node(nd.kids[0], tmp); andnot(reg, tmp); free_reg(); break; }
        default: leaf(nd.leaf, reg);
        }
    }
};
}  // namespace

static void read_stats(vlscan_ctx* ctx, vlscan_stats* st, bool check_error) {
    unsigned long long h[ST_COUNT];
    VL_CUDA(cudaMemcpyAsync(h, ctx->stats.p, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    VL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (check_error && h[ST_ERROR]) {
        static const char* const msg[] = {"", "cannot unmarshal strings: row lengths do not add up to the data length", "too big index for dict value",
                                          "unexpected length for binary representation of a number", "", "", "the filter needs the timestamps of a block that was handed over without them", "cannot unmarshal timestamps",
                                          "internal: a filter reached the values of a column that the bloom-first probe pass had left on the host"};
        throw BadInput(msg[std::min<unsigned long long>(h[ST_ERROR], 8)]);
    }
    if (!st) return;
    st->values_bytes += h[ST_VALUES_BYTES]; st->bloom_probe_bytes += h[ST_BLOOM_BYTES]; st->columns_read += h[ST_COLUMNS_READ];
    st->bitmap_bytes += h[ST_BITMAP_BYTES]; st->rows_matched += h[ST_ROWS_MATCHED]; st->blocks_matched += h[ST_BLOCKS_MATCHED];
    st->scan_kernel_bytes += h[ST_SCAN_BYTES];
    float ms = 0;
    VL_CUDA(cudaEventElapsedTime(&ms, ctx->ev_begin, ctx->ev_end)); st->gpu_ms += ms;
    for (size_t i = 0; i < ctx->scan_events_used; i++) { VL_CUDA(cudaEventElapsedTime(&ms, ctx->scan_events[i].first, ctx->scan_events[i].second)); st->scan_kernel_ms += ms; }
}

static void do_scan(vlscan_ctx* ctx, const vlscan_program* prog, const vlscan_batch* batch, vlscan_stats* stats) {
    VL_CUDA(cudaSetDevice(ctx->device));
    if (batch->device != ctx->device) throw BadInput("batch lives on another device than the ctx");
    ScanRun run{ctx, prog, batch};
    run.P = const_cast<vlscan_program*>(prog)->image(ctx->device, ctx->stream);
    run.B = batch->view();
    const Program& pr = prog->p;
    run.field_slot.assign(pr.fields.size(), -1);
    for (size_t f = 0; f < pr.fields.size(); f++) for (uint32_t s = 0; s < batch->nfields; s++) if (batch->field_names[s] == pr.fields[f]) run.field_slot[f] = (int)s;
    for (auto& nd : pr.nodes) run.slots_total += nd.prepass_count;
    uint64_t nb = std::max<uint64_t>(batch->nblocks, 1), nw = std::max<uint64_t>(batch->nwords, 1);
    ctx->action.ensure(nb); ctx->payload.ensure(nb * 8); ctx->leaf_bm.ensure(nw * 8);
    ctx->lens_blocks.ensure(nb * 4); ctx->lens_blocks2.ensure(nb * 4); ctx->row_blocks.ensure(nb * 4); ctx->work_count.ensure(WC_COUNT * 4);
    {   // upper bound of 64 KiB tiles of any single column: every payload byte belongs to one column, plus one partial tile per block
        uint64_t max_tiles = batch->arena_bytes / VL_TILE_BYTES + nb + 16;
        ctx->tiles.ensure(max_tiles * sizeof(ScanTile));
    }
    ctx->stats.ensure(ST_COUNT * 8); ctx->totals.ensure(32); ctx->counts.ensure(nb * 4);
    if (ctx->row_off8.size() < batch->nfields) { ctx->row_off8.resize(batch->nfields); ctx->ready.resize(batch->nfields); }
    ctx->ready_cleared.assign(batch->nfields, 0);
    for (uint32_t s = 0; s < batch->nfields; s++) { ctx->row_off8[s].ensure(nw * 32); ctx->ready[s].ensure(nb); }
    uint64_t launches0 = ctx->launches;
    ctx->scan_events_used = 0;
    run.stats = ctx->stats.as<unsigned long long>();
    VL_CUDA(cudaEventRecord(ctx->ev_begin, ctx->stream));
    VL_CUDA(cudaMemsetAsync(ctx->stats.p, 0, ST_COUNT * 8, ctx->stream));
    VL_CUDA(cudaMemsetAsync(ctx->totals.p, 0, 32, ctx->stream));
    // bm.init(rows); bm.setBits()   (block_search.go:213-214)
    uint64_t* reg = run.new_reg();
    run.copy_reg(reg, batch->init_bitmap.as<uint64_t>());
    if (batch->nblocks) {
        run.node(pr.root, reg);
        k_finalize<<<cdiv(batch->nblocks, 8), 256, 0, ctx->stream>>>(run.B, reg, ctx->counts.as<uint32_t>(), run.stats, ctx->totals.as<unsigned long long>());
        launch_check(ctx);
    }
    VL_CUDA(cudaEventRecord(ctx->ev_end, ctx->stream));
    ctx->last_batch = batch; ctx->has_result = true; ctx->kept = false; ctx->last_launches = ctx->launches - launches0;
    ctx->last_nblocks = batch->nblocks; ctx->last_nwords = batch->nwords; ctx->last_rows = batch->rows;
    if (stats) {
        read_stats(ctx, stats, true);
        stats->blocks += batch->nblocks; stats->rows += batch->rows; stats->gpu_launches += ctx->launches - launches0;
    }
}

// The probe pass between the two phases of a bloom-first upload: runs the program's bloom pre-passes, header dispatch and leaf bloom probes on a
// batch whose values are still on the host and returns need[block * nfields + field] = 1 for every values column some filter can reach.
static void do_probe(vlscan_ctx* ctx, const vlscan_program* prog, const vlscan_batch* batch, std::vector<uint8_t>& need) {
    VL_CUDA(cudaSetDevice(ctx->device));
    ScanRun run{ctx, prog, batch};
    run.P = const_cast<vlscan_program*>(prog)->image(ctx->device, ctx->stream);
    run.B = batch->view();
    const Program& pr = prog->p;
    run.field_slot.assign(pr.fields.size(), -1);
    for (size_t f = 0; f < pr.fields.size(); f++) for (uint32_t s = 0; s < batch->nfields; s++) if (batch->field_names[s] == pr.fields[f]) run.field_slot[f] = (int)s;
    for (auto& nd : pr.nodes) run.slots_total += nd.prepass_count;
    const size_t cells = (size_t)batch->nblocks * batch->nfields;
    need.assign(cells, 0);
    if (!cells || !batch->nwords) return;
    ctx->need.ensure(std::max<size_t>(cells, 16)); ctx->stats.ensure(ST_COUNT * 8);
    VL_CUDA(cudaMemsetAsync(ctx->need.p, 0, cells, ctx->stream));
    VL_CUDA(cudaMemsetAsync(ctx->stats.p, 0, ST_COUNT * 8, ctx->stream));
    run.stats = ctx->stats.as<unsigned long long>();
    uint64_t* reg = run.new_reg();
    run.copy_reg(reg, batch->init_bitmap.as<uint64_t>());
    run.probe_node(pr.root, reg, ctx->need.as<uint8_t>());
    VL_CUDA(cudaMemcpyAsync(need.data(), ctx->need.p, cells, cudaMemcpyDeviceToHost, ctx->stream));
    VL_CUDA(cudaStreamSynchronize(ctx->stream));
}

// ---- C ABI -------------------------------------------------------------------------------------------------------------------
extern "C" {

int vlscan_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

vlscan_ctx* vlscan_ctx_create(int device) {
    vlscan_ctx* ctx = new vlscan_ctx();
    int rc = guarded(nullptr, [&] {
        int n = vlscan_device_count();
        if (n <= 0) throw CudaFail("no CUDA device is available: libvlscan has no CPU fallback", 100);
        ctx->device = ((device % n) + n) % n;
        VL_CUDA(cudaSetDevice(ctx->device));
        VL_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        VL_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        VL_CUDA(cudaEventCreate(&ctx->ev_begin)); VL_CUDA(cudaEventCreate(&ctx->ev_end));
        cudaDeviceProp prop; VL_CUDA(cudaGetDeviceProperties(&prop, ctx->device)); ctx->sm_count = prop.multiProcessorCount;
        // resident CTAs per SM of the two scan instantiations on THIS device (the persistent grids are sized by it)
        VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->scan_occ[0], k_substr_scan<false>, VL_SCAN_THREADS, 0));
        VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->scan_occ[1], k_substr_scan<true>, VL_SCAN_THREADS, 0));
        for (int& o : ctx->scan_occ) o = std::max(o, 1);
        VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->row_occ, k_row_match, 256, 0));
        ctx->row_occ = std::max(ctx->row_occ, 1);
    });
    if (rc) { delete ctx; return nullptr; }
    return ctx;
}
void vlscan_ctx_free(vlscan_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (DevBuf* b : {&ctx->action, &ctx->payload, &ctx->leaf_bm, &ctx->lens_blocks, &ctx->row_blocks, &ctx->work_count, &ctx->stats, &ctx->totals, &ctx->counts, &ctx->slots, &ctx->hit_offs, &ctx->hits, &ctx->tiles, &ctx->lens_blocks2}) b->release();
    for (auto& r : ctx->regs) r.release();
    for (auto& r : ctx->row_off8) r.release();
    for (auto& r : ctx->ready) r.release();
    ctx->zsrc.release(); ctx->zcols.release(); ctx->ztest.release(); ctx->ts_vals.release();
    for (DevBuf* b : {&ctx->hit_block, &ctx->glens, &ctx->goffs, &ctx->gtiles, &ctx->gout, &ctx->gstat, &ctx->hslot, &ctx->vagg, &ctx->hblk, &ctx->htab, &ctx->hgrp, &ctx->lcand, &ctx->ftab, &ctx->patch, &ctx->unstaged}) b->release();
    for (DevBuf& b : ctx->ftxt) b.release();
    zstd_dev_free(ctx->zdev);
    delete ctx->pool;
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    delete ctx->recycle;
    for (auto& e : ctx->scan_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    if (ctx->ev_begin) cudaEventDestroy(ctx->ev_begin);
    if (ctx->ev_end) cudaEventDestroy(ctx->ev_end);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}
const char* vlscan_last_error(const vlscan_ctx* ctx) { return ctx ? ctx->err.c_str() : g_thread_err.c_str(); }
void* vlscan_ctx_stream(const vlscan_ctx* ctx) { return (void*)ctx->stream; }
int vlscan_ctx_sync(vlscan_ctx* ctx) { return guarded(ctx, [&] { VL_CUDA(cudaSetDevice(ctx->device)); VL_CUDA(cudaStreamSynchronize(ctx->stream)); }); }

int vlscan_program_create(const void* tree, size_t tree_len, vlscan_program** out) {
    *out = nullptr;
    auto* pg = new vlscan_program();
    int rc = guarded(nullptr, [&] { ProgramBuilder(tree, tree_len, pg->p).build(); });
    if (rc) { delete pg; return rc; }
    *out = pg;
    return 0;
}
void vlscan_program_free(vlscan_program* prog) { delete prog; }
uint32_t vlscan_program_nfields(const vlscan_program* prog) { return (uint32_t)prog->p.fields.size(); }
const char* vlscan_program_field(const vlscan_program* prog, uint32_t i, size_t* len) { if (i >= prog->p.fields.size()) { *len = 0; return nullptr; } *len = prog->p.fields[i].size(); return prog->p.fields[i].data(); }
int64_t vlscan_program_leaf_tokens(const vlscan_program* prog, uint32_t leaf, char* buf, size_t cap) {
    if (leaf >= prog->p.leaf_tokens.size()) return -1;
    std::string s; for (size_t i = 0; i < prog->p.leaf_tokens[leaf].size(); i++) { if (i) s.push_back('\n'); s += prog->p.leaf_tokens[leaf][i]; }
    if (s.size() > cap) return -1;
    memcpy(buf, s.data(), s.size());
    return (int64_t)s.size();
}

int vlscan_eval_predicate(int kind, const void* value, size_t value_len, const void* arg1, size_t arg1_len, const void* arg2, size_t arg2_len, uint64_t aux0, uint64_t aux1) {
    if (value_len > 0xFFFFFFFFull || arg1_len > 0xFFFFFFFFull || arg2_len > 0xFFFFFFFFull) return -1;
    const uint8_t* v = (const uint8_t*)value; const uint32_t vn = (uint32_t)value_len;
    const uint8_t* a = (const uint8_t*)arg1; const uint32_t an = (uint32_t)arg1_len;
    switch (kind) {   // predicates of the kinds that are not wired into the row kernels yet (vl_anycase.cuh)
    case F_REGEXP: {   // arg1 = the expression: compiled like a regexp leaf, matched by the host mirror of the device automaton (const / dict values take this path)
        try { return vl::compile_regex(std::string((const char*)a, an)).match(v, vn) ? 1 : 0; } catch (const vl::RxError& e) { vl::set_thread_error(e.what()); return -2; }
    }
    case 14: return vl::any_case_match(v, vn, a, an, false) ? 1 : 0;
    case 15: return vl::any_case_match(v, vn, a, an, true) ? 1 : 0;
    case 16: return vl::match_sequence(v, vn, vl::PhraseList{a, an}) ? 1 : 0;
    case 17: return vl::match_all_phrases(v, vn, vl::PhraseList{a, an}) ? 1 : 0;
    case 18: return vl::match_any_phrase(v, vn, vl::PhraseList{a, an}) ? 1 : 0;
    }
    if (kind < F_EXACT_PREFIX || kind > F_IPV4_RANGE) return -1;
    return vl::range_predicate(kind, (const uint8_t*)value, (uint32_t)value_len, (const uint8_t*)arg1, (uint32_t)arg1_len, (const uint8_t*)arg2, (uint32_t)arg2_len, aux0, aux1) ? 1 : 0;
}

int64_t vlscan_program_prepass_tokens(const vlscan_program* prog, char* buf, size_t cap) {
    const Program& P = prog->p;
    std::string s;
    for (const PNode& nd : P.nodes) {   // nodes are numbered in pre-order
        if (nd.kind != F_AND && nd.kind != F_OR) continue;
        s += nd.kind == F_AND ? "A" : "O";
        for (int k = 0; k < nd.prepass_count; k++) {
            const DevPrepass& pp = P.prepass[(size_t)nd.prepass_begin + k];
            s += "\t" + P.fields[pp.field];
            const uint32_t* offs = (const uint32_t*)(P.blob.data() + pp.tok_offs_off);
            for (uint32_t t = 0; t < pp.ntokens; t++) { s += "\x1f"; s.append((const char*)P.blob.data() + pp.tok_blob_off + offs[t], offs[t + 1] - offs[t]); }
        }
        s += "\n";
    }
    if (s.size() > cap) return -1;
    memcpy(buf, s.data(), s.size());
    return (int64_t)s.size();
}

int64_t vlscan_program_in_hashes(const vlscan_program* prog, uint32_t leaf, uint64_t* out, size_t cap) {
    const Program& P = prog->p;
    if (leaf >= P.leaves.size() || P.leaves[leaf].kind != F_IN) return -1;
    const DevLeaf& L = P.leaves[leaf];
    std::vector<uint64_t> v;
    v.push_back(L.nhashes); v.insert(v.end(), P.u64s.begin() + L.hashes_off, P.u64s.begin() + L.hashes_off + L.nhashes);
    if (L.in_skip_sets) v.push_back(UINT64_MAX);   // more than maxTokenSetsToInit value sets: none is kept
    else {
        v.push_back(L.in_nsets);
        for (uint32_t k = 0; k < L.in_nsets; k++) {
            const uint32_t off = P.u32s[L.in_sets_off + 2 * k], n = P.u32s[L.in_sets_off + 2 * k + 1];
            v.push_back(n); v.insert(v.end(), P.u64s.begin() + off, P.u64s.begin() + off + n);
        }
    }
    if (v.size() > cap) return -1;
    memcpy(out, v.data(), v.size() * 8);
    return (int64_t)v.size();
}

int64_t vlscan_program_in_typed(const vlscan_program* prog, uint32_t leaf, int value_type, uint64_t* out, size_t cap) {
    const Program& P = prog->p;
    if (leaf >= P.leaves.size() || P.leaves[leaf].kind != F_IN || value_type < VT_UINT8 || value_type >= VT_MAX) return -1;
    const DevLeaf& L = P.leaves[leaf];
    const uint32_t n = L.in_typed_cnt[value_type];
    if (n > cap) return -1;
    if (n) memcpy(out, P.u64s.data() + L.in_typed_off[value_type], (size_t)n * 8);
    return (int64_t)n;
}

int vlscan_parse_typed(int value_type, const void* s, size_t len, uint64_t* out) {
    const std::string v((const char*)s, len);
    uint64_t u = 0; int64_t i = 0; double f = 0; uint32_t ip = 0;
    switch (value_type) {
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: if (!vl::parse_u64(v, &u)) return 0; *out = u; return 1;
    case VT_INT64: if (!vl::parse_i64(v, &i)) return 0; *out = (uint64_t)i; return 1;
    case VT_FLOAT64: if (!vl::parse_f64_exact(v, &f)) return 0; memcpy(out, &f, 8); return 1;
    case VT_IPV4: if (!vl::parse_ipv4(v, &ip)) return 0; *out = ip; return 1;
    case VT_ISO8601: if (!vl::parse_iso8601(v, &i)) return 0; *out = (uint64_t)i; return 1;
    }
    return -1;
}

double vlscan_parse_math_number(const void* s, size_t len) {
    if (len > 0xFFFFFFFFull) return NAN;
    return vl::mn::parse_math_number((const uint8_t*)s, (uint32_t)len);
}

int vlscan_format_float64(uint64_t ieee_bits, char* buf, size_t cap) {
    uint8_t tmp[VL_FMT_F64_MAX];
    int n = vl::fmt_f64(tmp, ieee_bits);
    if ((size_t)n > cap) return -1;
    memcpy(buf, tmp, (size_t)n);
    return n;
}

int vlscan_batch_upload(vlscan_ctx* ctx, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields, const vlscan_block* blocks,
                        uint64_t nblocks, vlscan_batch** out, vlscan_stats* stats) {
    *out = nullptr;
    auto* b = new vlscan_batch();
    int rc = guarded(ctx, [&] { do_upload(ctx, field_names, field_name_lens, nfields, blocks, nblocks, b, stats); });
    if (rc) { delete b; return rc; }
    *out = b;
    return 0;
}
void vlscan_batch_free(vlscan_batch* batch) { delete batch; }
uint64_t vlscan_batch_nblocks(const vlscan_batch* b) { return b->nblocks; }
uint64_t vlscan_batch_rows(const vlscan_batch* b) { return b->rows; }
uint64_t vlscan_batch_words(const vlscan_batch* b) { return b->nwords; }
uint64_t vlscan_batch_device_bytes(const vlscan_batch* b) { return b->device_bytes(); }

int vlscan_batch_download(vlscan_ctx* ctx, const vlscan_batch* batch, vlscan_host_blocks** out) {
    *out = nullptr;
    auto* hb = new vlscan_host_blocks();
    int rc = guarded(ctx, [&] {
        VL_CUDA(cudaSetDevice(ctx->device));
        if (batch->split_hdr) throw BadInput("a batch staged bloom-first cannot be downloaded");
        hb->bytes = batch->arena_bytes;
        VL_CUDA(cudaMallocHost(&hb->pinned, std::max<size_t>(hb->bytes, 16)));
        std::vector<DevColumn> cols((size_t)batch->nblocks * batch->nfields);
        VL_CUDA(cudaMemcpyAsync(hb->pinned, batch->arena.p, hb->bytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (!cols.empty()) VL_CUDA(cudaMemcpyAsync(cols.data(), batch->cols.p, cols.size() * sizeof(DevColumn), cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
        hb->fields = batch->field_names;
        const uint8_t* base = (const uint8_t*)hb->pinned;
        hb->blocks.resize(batch->nblocks);
        hb->cols.reserve(cols.size());
        // the lens type byte is not stored in the arena: rebuild "type + items" views in a side buffer kept alive by dict_offsets storage
        std::vector<size_t> first(batch->nblocks + 1, 0);
        for (uint64_t b = 0; b < batch->nblocks; b++) {
            first[b] = hb->cols.size();
            for (uint32_t f = 0; f < batch->nfields; f++) {
                const DevColumn& d = cols[(size_t)b * batch->nfields + f];
                if (d.kind == COL_MISSING) continue;
                vlscan_column c; memset(&c, 0, sizeof c);
                c.field = f;
                if (d.kind == COL_CONST) { c.kind = VLSCAN_COL_CONST; c.const_value = base + d.meta_off; c.const_len = d.meta_len; hb->cols.push_back(c); continue; }
                c.kind = VLSCAN_COL_VALUES; c.value_type = d.vt; c.stage = VLSCAN_STAGE_DECODED; c.dict_len = d.dict_len; c.min_value = d.min_value; c.max_value = d.max_value;
                uint64_t items = d.lens_type < 4 ? ((uint64_t)batch->h_rows[b] << d.lens_type) : (1ull << (d.lens_type - 4));
                // lens items are preceded in the arena by alignment slack; the type byte is materialised in the byte right before them
                uint8_t* tb = (uint8_t*)hb->pinned + d.lens_off - 1;
                *tb = d.lens_type;
                c.lens_items = tb; c.lens_items_len = items + 1;
                c.data = base + d.data_off; c.data_len = d.data_len;
                c.bloom = base + d.bloom_off; c.bloom_len = (uint64_t)d.bloom_words * 8;
                if (d.vt == VT_DICT) { c.dict_offsets = (const uint32_t*)(base + d.meta_off); c.dict_blob = base + d.meta_off + 4 * (d.dict_len + 1); }
                hb->cols.push_back(c);
            }
        }
        first[batch->nblocks] = hb->cols.size();
        for (uint64_t b = 0; b < batch->nblocks; b++) { hb->blocks[b].rows = batch->h_rows[b]; hb->blocks[b].ncols = (uint32_t)(first[b + 1] - first[b]); hb->blocks[b].cols = hb->cols.data() + first[b]; }
        if (batch->has_ts && batch->nblocks) {   // the timestamps columns, in their plain marshal types (ZSTD ones were inflated at upload)
            std::vector<DevTimestamps> ts(batch->nblocks);
            VL_CUDA(cudaMemcpy(ts.data(), batch->ts.p, ts.size() * sizeof(DevTimestamps), cudaMemcpyDeviceToHost));
            for (uint64_t b = 0; b < batch->nblocks; b++) {
                if (!ts[b].mt) continue;
                vlscan_block& blk = hb->blocks[b];
                blk.ts_marshal_type = ts[b].mt; blk.timestamps = base + ts[b].off; blk.timestamps_len = ts[b].len;
                blk.min_timestamp = ts[b].first; blk.max_timestamp = ts[b].max;
            }
        }
    });
    if (rc) { if (hb->pinned) cudaFreeHost(hb->pinned); delete hb; return rc; }
    *out = hb;
    return 0;
}
// The reference's writer for one values block: marshalBytesBlock(lens items) ++ marshalBytesBlock(data) (encoding.go:16-50, 343-370)
static void marshal_bytes_block(std::vector<uint8_t>& dst, const uint8_t* src, size_t n) {
    if (n < 128) { dst.push_back(0); dst.push_back((uint8_t)n); dst.insert(dst.end(), src, src + n); return; }
    ZstdWriter& z = zstd_writer();
    if (!z.ok) throw BadInput("libzstd.so.1 is not available for compressing values blocks");
    int level = n <= 512 ? 1 : n <= 4096 ? 2 : 3;   // getCompressLevel, encoding.go:362-370
    size_t cap = z.bound(n), old = dst.size();
    dst.push_back(1);
    dst.resize(old + 1 + 10 + cap);
    size_t got = z.compress(dst.data() + old + 11, cap, src, n, level);
    if (z.is_error(got)) throw BadInput("ZSTD_compress failed");
    uint8_t vu[10]; int k = 0; uint64_t v = got; while (v >= 0x80) { vu[k++] = (uint8_t)(v | 0x80); v >>= 7; } vu[k++] = (uint8_t)v;   // MarshalVarUint64
    memcpy(dst.data() + old + 1, vu, k);
    memmove(dst.data() + old + 1 + k, dst.data() + old + 11, got);
    dst.resize(old + 1 + k + got);
}

int vlscan_host_blocks_compress(const vlscan_host_blocks* in, int threads, vlscan_host_blocks** out) {
    *out = nullptr;
    auto* hb = new vlscan_host_blocks();
    int rc = guarded(nullptr, [&] {
        const size_t ncols = in->cols.size();
        std::vector<std::vector<uint8_t>> packed(ncols);
        std::atomic<size_t> next{0}; std::atomic<bool> failed{false}; std::string fail_msg; std::mutex mu;
        auto work = [&] {
            for (;;) {
                size_t i0 = next.fetch_add(64); if (i0 >= ncols || failed) return;
                for (size_t i = i0; i < std::min(ncols, i0 + 64); i++) {
                    const vlscan_column& c = in->cols[i];
                    if (c.kind != VLSCAN_COL_VALUES) continue;
                    try {
                        if (c.stage == VLSCAN_STAGE_ONDISK) packed[i].assign(c.values, c.values + c.values_len);
                        else { marshal_bytes_block(packed[i], c.lens_items, c.lens_items_len); marshal_bytes_block(packed[i], c.data, c.data_len); }
                    } catch (const BadInput& e) { std::lock_guard<std::mutex> g(mu); fail_msg = e.msg; failed = true; return; }
                }
            }
        };
        int nt = threads > 0 ? threads : (int)std::max(1u, std::thread::hardware_concurrency());
        std::vector<std::thread> pool; for (int t = 1; t < nt; t++) pool.emplace_back(work);
        work(); for (auto& t : pool) t.join();
        if (failed) throw BadInput(fail_msg);
        // layout: [copied part: consts, blooms, dict tables, strided exactly like the upload arena][values blocks, back to back]
        uint64_t cursor = 16, vbytes = 0;
        std::vector<uint64_t> off_a(ncols, 0), off_b(ncols, 0), off_v(ncols, 0);
        for (size_t i = 0; i < ncols; i++) {
            const vlscan_column& c = in->cols[i];
            if (c.kind == VLSCAN_COL_CONST) { off_a[i] = arena_reserve(cursor, c.const_len); continue; }
            off_a[i] = arena_reserve(cursor, c.bloom_len);
            if (c.value_type == VT_DICT) off_b[i] = arena_reserve(cursor, 4 * (c.dict_len + 1) + (c.dict_len ? c.dict_offsets[c.dict_len] : 0));
            off_v[i] = vbytes; vbytes += packed[i].size();
        }
        const uint64_t vbase = (cursor + kArenaPad + 63) / 64 * 64;
        hb->bytes = vbase + vbytes + 64;
        VL_CUDA(cudaMallocHost(&hb->pinned, hb->bytes));
        uint8_t* base = (uint8_t*)hb->pinned;
        memset(base, 0, vbase);
        hb->fields = in->fields; hb->cols = in->cols; hb->blocks = in->blocks;
        for (size_t i = 0; i < ncols; i++) {
            vlscan_column& c = hb->cols[i];
            if (c.kind == VLSCAN_COL_CONST) { if (c.const_len) memcpy(base + off_a[i], c.const_value, c.const_len); c.const_value = base + off_a[i]; continue; }
            if (c.bloom_len) memcpy(base + off_a[i], c.bloom, c.bloom_len);
            c.bloom = base + off_a[i];
            if (c.value_type == VT_DICT) {
                uint32_t total = c.dict_len ? c.dict_offsets[c.dict_len] : 0;
                uint8_t* m = base + off_b[i];
                if (c.dict_len) memcpy(m, c.dict_offsets, 4 * (c.dict_len + 1)); else memset(m, 0, 4);
                if (total) memcpy(m + 4 * (c.dict_len + 1), c.dict_blob, total);
                c.dict_offsets = (const uint32_t*)m; c.dict_blob = m + 4 * (c.dict_len + 1);
            }
            memcpy(base + vbase + off_v[i], packed[i].data(), packed[i].size());
            c.stage = VLSCAN_STAGE_ONDISK; c.values = base + vbase + off_v[i]; c.values_len = packed[i].size();
            c.lens_items = nullptr; c.lens_items_len = 0; c.data = nullptr; c.data_len = 0;
            std::vector<uint8_t>().swap(packed[i]);
        }
        size_t k = 0;
        for (size_t b = 0; b < hb->blocks.size(); b++) { hb->blocks[b].cols = hb->cols.data() + k; k += hb->blocks[b].ncols; }
    });
    if (rc) { if (hb->pinned) cudaFreeHost(hb->pinned); delete hb; return rc; }
    *out = hb;
    return 0;
}

int vlscan_zstd_inspect(const void* bytes_block, size_t len, uint64_t out[5]) {
    return guarded(nullptr, [&] {
        ZstdJob job;
        uint64_t regen = 0; uint32_t id = 0;
        size_t used = job.add_bytes_block((const uint8_t*)bytes_block, len, 512, &regen, &id);
        out[0] = used; out[1] = regen; out[2] = job.blocks(); out[3] = job.compressed_blocks(); out[4] = job.sequences();
    });
}

int vlscan_zstd_walk_digest(const vlscan_block* blocks, uint64_t nblocks, int threads, uint64_t out[12]) {
    return guarded(nullptr, [&] {
        std::vector<ZValuesBlock> zv;
        collect_values_blocks(blocks, nblocks, zv);
        std::vector<ZValuesInfo> info(zv.size());
        ZstdJob job; size_t bad = SIZE_MAX; std::string msg;
        const double t0 = now_s();
        if (!zv.empty()) job.add_values_blocks(zv.data(), zv.size(), threads, info.data(), &bad, &msg);
        const double t1 = now_s();
        if (bad != SIZE_MAX) throw BadInput("values block " + std::to_string(bad) + ": " + msg);
        job.prepare();
        const double t2 = now_s();
        job.digest(out);
        uint64_t h = 5; for (const ZValuesInfo& x : info) { h = (h ^ x.lens_len) * 0x9E3779B97F4A7C15ull; h = (h ^ x.data_len) * 0x9E3779B97F4A7C15ull; h ^= h >> 29; }
        out[0] ^= h;
        out[4] = job.frames(); out[5] = job.blocks(); out[6] = job.groups(); out[7] = job.compressed_blocks(); out[8] = job.sequences();
        out[9] = (uint64_t)((t1 - t0) * 1e9); out[10] = (uint64_t)((t2 - t1) * 1e9); out[11] = 0;
    });
}

// the device decoder on independent frames given as host pointers (metadata of a part, parity tests)
static void zstd_decompress_frames(vlscan_ctx* ctx, uint32_t nframes, const void* const* frames, const size_t* frame_lens, void* dst, const uint64_t* dst_offsets) {
    {
        VL_CUDA(cudaSetDevice(ctx->device));
        ZstdJob job;
        std::vector<uint8_t> packed(512, 0);
        for (uint32_t i = 0; i < nframes; i++) {
            uint64_t regen = 0; uint32_t id = 0;
            job.add_frame((const uint8_t*)frames[i], frame_lens[i], packed.size(), &regen, &id);
            if (regen != dst_offsets[i + 1] - dst_offsets[i]) throw BadInput("cannot decompress block: frame content size differs from the destination size");
            job.set_dst(id, 16 + dst_offsets[i]);
            packed.insert(packed.end(), (const uint8_t*)frames[i], (const uint8_t*)frames[i] + frame_lens[i]);
        }
        const uint64_t total = nframes ? dst_offsets[nframes] : 0;
        ctx->zsrc.ensure(packed.size() + 512); ctx->ztest.ensure(16 + total + 64);
        VL_CUDA(cudaMemcpyAsync(ctx->zsrc.p, packed.data(), packed.size(), cudaMemcpyHostToDevice, ctx->stream));
        VL_CUDA(cudaMemsetAsync(ctx->ztest.p, 0xA5, 16 + total + 64, ctx->stream));
        job.run(ctx, ctx->zsrc.as<uint8_t>(), ctx->ztest.as<uint8_t>());
        job.check(ctx);
        if (total) VL_CUDA(cudaMemcpy(dst, ctx->ztest.as<uint8_t>() + 16, total, cudaMemcpyDeviceToHost));
    }
}

int vlscan_zstd_decompress(vlscan_ctx* ctx, uint32_t nframes, const void* const* frames, const size_t* frame_lens, void* dst, const uint64_t* dst_offsets) {
    return guarded(ctx, [&] { zstd_decompress_frames(ctx, nframes, frames, frame_lens, dst, dst_offsets); });
}

// ---- part directory reader (vl_part.h) ------------------------------------------------------------------------------------
int vlscan_part_open(vlscan_ctx* ctx, const char* path, vlscan_inflate_fn inflate, void* user, vlscan_part** out) {
    *out = nullptr;
    auto* p = new vlscan_part();
    int rc = guarded(ctx, [&] {
        if (!inflate && !ctx) throw BadInput("vlscan_part_open needs a ctx (device ZSTD decoder) or an inflate callback");
        vl::part::Inflate inf;
        if (inflate) inf = [&](const uint8_t* f, size_t n, uint8_t* dst, size_t dn) { if (inflate(user, f, n, dst, dn) != 0) throw BadInput("the inflate callback failed on a metadata frame of the part"); };
        else inf = [&](const uint8_t* f, size_t n, uint8_t* dst, size_t dn) { const void* fr[1] = {f}; const size_t ln[1] = {n}; const uint64_t offs[2] = {0, dn}; zstd_decompress_frames(ctx, 1, fr, ln, dst, offs); };
        p->r.open(path, inf);
    });
    if (rc) { delete p; return rc; }
    *out = p;
    return 0;
}
void vlscan_part_free(vlscan_part* part) { delete part; }
void vlscan_part_header(const vlscan_part* part, uint64_t out[8]) {
    const vl::part::PartHeader& h = part->r.ph;
    out[0] = h.FormatVersion; out[1] = h.CompressedSizeBytes; out[2] = h.UncompressedSizeBytes; out[3] = h.RowsCount; out[4] = h.BlocksCount;
    out[5] = (uint64_t)h.MinTimestamp; out[6] = (uint64_t)h.MaxTimestamp; out[7] = h.BloomValuesShardsCount;
}
uint64_t vlscan_part_nblocks(const vlscan_part* part) { return part->r.blockHeaders.size(); }
int vlscan_part_block_header(const vlscan_part* part, uint64_t i, uint64_t out[15]) {
    return guarded(nullptr, [&] {
        if (i >= part->r.blockHeaders.size()) throw BadInput("block index outside the part");
        const vl::part::BlockHeader& b = part->r.blockHeaders[i];
        out[0] = b.sid.accountID; out[1] = b.sid.projectID; out[2] = b.sid.hi; out[3] = b.sid.lo; out[4] = b.uncompressedSizeBytes; out[5] = b.rowsCount;
        out[6] = b.tsOffset; out[7] = b.tsSize; out[8] = (uint64_t)b.minTimestamp; out[9] = (uint64_t)b.maxTimestamp; out[10] = b.tsMarshalType;
        out[11] = b.chIndexOffset; out[12] = b.chIndexSize; out[13] = b.chOffset; out[14] = b.chSize;
    });
}
int vlscan_part_timestamps(const vlscan_part* part, uint64_t i, const uint8_t** data, uint64_t* len) {
    return guarded(nullptr, [&] {
        if (i >= part->r.blockHeaders.size()) throw BadInput("block index outside the part");
        const vl::part::BlockHeader& b = part->r.blockHeaders[i];
        if (b.tsSize > vl::part::kMaxTimestampsBlockSize) throw BadInput("timestamps block size is too big");   // getTimestamps block_search.go:490-493
        *data = part->r.timestamps_file().at(b.tsOffset, b.tsSize, "a timestamps block"); *len = b.tsSize;
    });
}
uint32_t vlscan_part_ncolumn_names(const vlscan_part* part) { return (uint32_t)part->r.columnNames.size(); }
const char* vlscan_part_column_name(const vlscan_part* part, uint32_t i, size_t* len) { if (i >= part->r.columnNames.size()) { *len = 0; return nullptr; } const std::string& s = part->r.columnNames[i]; *len = s.size(); return s.data(); }
int vlscan_part_blocks(const vlscan_part* part, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields, uint64_t block_lo, uint64_t block_hi,
                       int64_t min_timestamp, int64_t max_timestamp, vlscan_host_blocks** out) {
    *out = nullptr;
    auto* hb = new vlscan_host_blocks();
    int rc = guarded(nullptr, [&] {
        std::vector<std::string> fields;
        for (uint32_t f = 0; f < nfields; f++) { std::string n(field_names[f], field_name_lens[f]); fields.push_back(n.empty() ? "_msg" : n); }
        for (size_t a = 0; a < fields.size(); a++) for (size_t b = a + 1; b < fields.size(); b++) if (fields[a] == fields[b]) throw BadInput("duplicate field name");
        vl::part::Described d;
        part->r.describe(fields, block_lo, block_hi, min_timestamp, max_timestamp, d);
        hb->fields = std::move(d.fields); hb->cols = std::move(d.cols); hb->blocks = std::move(d.blocks); hb->owned = std::move(d.owned); hb->source = std::move(d.source);
        for (const vlscan_column& c : hb->cols) hb->bytes += c.const_len + c.values_len + c.bloom_len;
    });
    if (rc) { delete hb; return rc; }
    *out = hb;
    return 0;
}
const uint64_t* vlscan_host_blocks_source(const vlscan_host_blocks* hb, uint64_t* n) { *n = hb->source.size(); return hb->source.data(); }

const vlscan_block* vlscan_host_blocks_get(const vlscan_host_blocks* hb, uint64_t* nblocks, uint32_t* nfields) { *nblocks = hb->blocks.size(); *nfields = (uint32_t)hb->fields.size(); return hb->blocks.data(); }
const char* vlscan_host_blocks_field(const vlscan_host_blocks* hb, uint32_t i, size_t* len) { if (i >= hb->fields.size()) { *len = 0; return nullptr; } *len = hb->fields[i].size(); return hb->fields[i].data(); }
uint64_t vlscan_host_blocks_bytes(const vlscan_host_blocks* hb) { return hb->bytes; }
void vlscan_host_blocks_free(vlscan_host_blocks* hb) { if (!hb) return; if (hb->pinned) cudaFreeHost(hb->pinned); delete hb; }

int vlscan_scan_resident(vlscan_ctx* ctx, const vlscan_program* prog, const vlscan_batch* batch, vlscan_stats* stats) {
    return guarded(ctx, [&] { do_scan(ctx, prog, batch, stats); });
}

int vlscan_last_scan_stats(vlscan_ctx* ctx, vlscan_stats* stats) {
    return guarded(ctx, [&] {
        if (!ctx->has_result) throw BadInput("no scan on this ctx yet");
        VL_CUDA(cudaSetDevice(ctx->device));
        read_stats(ctx, stats, true);
        stats->blocks += ctx->last_nblocks; stats->rows += ctx->last_rows; stats->gpu_launches += ctx->last_launches;
    });
}

int vlscan_fetch_results(vlscan_ctx* ctx, uint64_t* out_bitmap_words, uint32_t* out_match_counts, vlscan_stats* stats) {
    return guarded(ctx, [&] {
        if (!ctx->has_result) throw BadInput("no scan result to fetch on this ctx");
        VL_CUDA(cudaSetDevice(ctx->device));
        uint64_t d2h = 0;   // bitmaps and counts live in ctx scratch: no access to the batch here
        if (out_bitmap_words && ctx->last_nwords) { VL_CUDA(cudaMemcpyAsync(out_bitmap_words, ctx->regs[0].p, ctx->last_nwords * 8, cudaMemcpyDeviceToHost, ctx->stream)); d2h += ctx->last_nwords * 8; }
        if (out_match_counts && ctx->last_nblocks) { VL_CUDA(cudaMemcpyAsync(out_match_counts, ctx->counts.p, ctx->last_nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream)); d2h += ctx->last_nblocks * 4; }
        read_stats(ctx, nullptr, true);
        if (stats) stats->d2h_bytes += d2h;
    });
}

int vlscan_result_digest(vlscan_ctx* ctx, uint64_t block_lo, uint64_t block_hi, uint64_t key_base, uint64_t* out_digest) {
    return guarded(ctx, [&] {
        if (!ctx->has_result) throw BadInput("no scan result on this ctx");
        if (block_lo > block_hi || block_hi > ctx->last_nblocks) throw BadInput("block range outside the batch of the last scan");
        VL_CUDA(cudaSetDevice(ctx->device));
        ctx->hit_offs.ensure(16);
        VL_CUDA(cudaMemsetAsync(ctx->hit_offs.p, 0, 8, ctx->stream));
        if (block_hi > block_lo) {
            k_bitmap_digest<<<cdiv(block_hi - block_lo, 128), 128, 0, ctx->stream>>>(ctx->last_batch->view(), ctx->regs[0].as<uint64_t>(), (uint32_t)block_lo, (uint32_t)block_hi, key_base, ctx->hit_offs.as<unsigned long long>());
            launch_check(ctx);
        }
        VL_CUDA(cudaMemcpyAsync(out_digest, ctx->hit_offs.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
    });
}

int vlscan_totals_sum(vlscan_ctx* const* ctxs, int nctx, uint64_t out4[4]) {
    out4[0] = out4[1] = out4[2] = out4[3] = 0;
    for (int i = 0; i < nctx; i++) {
        vlscan_ctx* ctx = ctxs[i];
        int rc = guarded(ctx, [&] {
            if (!ctx->has_result) throw BadInput("no scan result on this ctx");
            VL_CUDA(cudaSetDevice(ctx->device));
            unsigned long long t[4];
            VL_CUDA(cudaMemcpyAsync(t, ctx->totals.p, 32, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaStreamSynchronize(ctx->stream));
            for (int k = 0; k < 4; k++) out4[k] += t[k];
        });
        if (rc) return rc;
    }
    return 0;
}

int vlscan_result_device_ptrs(vlscan_ctx* ctx, void** bitmap_words, void** match_counts, void** totals4) {
    if (!ctx->has_result) { ctx->err = "no scan result on this ctx"; return -1; }
    if (bitmap_words) *bitmap_words = ctx->regs[0].p;
    if (match_counts) *match_counts = ctx->counts.p;
    if (totals4) *totals4 = ctx->totals.p;
    return 0;
}

// what vlscan_stage_selected checks a values column's descriptor against: its stage and payload lengths
static vlscan_batch::CellSig cell_sig(const vlscan_column& c) {
    vlscan_batch::CellSig g;
    g.stage = c.stage;
    if (c.stage == VLSCAN_STAGE_ONDISK) g.len0 = c.values_len; else { g.len0 = c.lens_items_len; g.len1 = c.data_len; }
    return g;
}

// The body of vlscan_scan_batch and vlscan_scan_batch_keep.  keep = false is vlscan_scan_batch as it always was.  keep = true always stages in two
// phases (UP_HEADERS, then UP_VALUES with a `need` mask): the probe pass decides the values of the program's fields when it runs, else all of
// them are marked; cells of the other fields (output fields) keep their values on the host.  The batch then stays the ctx's last result.
static int scan_batch_impl(vlscan_ctx* ctx, const vlscan_program* prog, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields,
                           const vlscan_block* blocks, uint64_t nblocks, uint64_t* out_bitmap_words, uint32_t* out_match_counts, vlscan_stats* stats, bool keep) {
    // the staging batch (HBM arena + descriptor tables) is recycled across calls of this ctx: a search worker submits batch after
    // batch, so cudaMalloc / cudaFree of a multi-GB arena per call would sit on the critical path
    vlscan_batch* b = ctx->recycle ? ctx->recycle : new vlscan_batch();
    ctx->recycle = nullptr;
    b->field_names.clear(); b->slot_vt_mask.clear();
    uint64_t launches0 = ctx->launches;
    // which fields' bloom filters the program can ever probe: leaves with token hashes (or in() / contains_any() token sets) and the per-field
    // tokens of the AND / OR pre-passes; and (keep) which batch fields the program references at all
    std::vector<char> need_bloom(nfields, 0), in_prog(nfields, 0);
    {
        const Program& P = prog->p;
        auto mark = [&](std::vector<char>& m, int field) { for (uint32_t s = 0; s < nfields; s++) if (std::string(field_names[s], field_name_lens[s]) == P.fields[field]) m[s] = 1; };
        for (const DevLeaf& L : P.leaves) if (L.nhashes || L.nhashes2 || L.in_nsets) mark(need_bloom, L.field);
        for (const DevPrepass& pp : P.prepass) if (pp.nhashes) mark(need_bloom, pp.field);
        if (keep) for (size_t f = 0; f < P.fields.size(); f++) mark(in_prog, (int)f);
    }
    // Bloom-first staging (the reference reads a column's values only after the block got past the bloom filters, block_search.go:411-474): when
    // the program probes bloom filters at all, the headers and bloom filters go first, a probe pass marks the columns some filter can reach,
    // and only their values cross PCIe and get decoded.  VLSCAN_BLOOM_FIRST = 0 never, 2 always, 1 (default) adaptive: after a probe that
    // pruned less than 1/8 of the values bytes the next 7 calls with the same program stage everything at once (the probe serialises the
    // bloom copy with the decode, which costs more than it saves when nearly every block is read anyway).
    int bf = 1;
    if (const char* e = getenv("VLSCAN_BLOOM_FIRST")) bf = atoi(e);
    bool probes = false;
    for (char c : need_bloom) probes |= c != 0;
    if (ctx->bf_prog != (const void*)prog) { ctx->bf_prog = prog; ctx->bf_skip = 0; }
    const bool probe = bf != 0 && probes && nblocks > 0 && (bf == 2 || ctx->bf_skip == 0);
    if (!probe && ctx->bf_skip > 0) ctx->bf_skip--;
    int rc;
    if (probe || keep) {
        rc = guarded(ctx, [&] {
            do_upload(ctx, field_names, field_name_lens, nfields, blocks, nblocks, b, stats, &need_bloom, UP_HEADERS);
            std::vector<uint8_t> need;
            if (probe) do_probe(ctx, prog, b, need);
            else {   // keep without a probe: every values cell of the program's own fields
                need.assign(std::max<size_t>((size_t)nblocks * nfields, 1), 0);   // never empty: the values phase needs a mask, also for no block or no field
                for (uint64_t i = 0; i < nblocks; i++)
                    for (uint32_t k = 0; k < blocks[i].ncols; k++) if (blocks[i].cols[k].field < nfields && in_prog[blocks[i].cols[k].field]) need[i * nfields + blocks[i].cols[k].field] = 1;
            }
            // the adaptive rule weighs what the probe saved on the fields it can prune: with keep, the program's fields only
            uint64_t vals_all = 0, vals_need = 0, cols_all = 0, cols_need = 0;
            for (uint64_t i = 0; i < nblocks; i++)
                for (uint32_t k = 0; k < blocks[i].ncols; k++) {
                    const vlscan_column& c = blocks[i].cols[k];
                    if (c.kind != VLSCAN_COL_VALUES || c.field >= nfields) continue;
                    const bool needed = need[i * nfields + c.field] != 0;
                    cols_all++; cols_need += needed;
                    if (keep && !in_prog[c.field]) continue;
                    const uint64_t n = c.stage == VLSCAN_STAGE_ONDISK ? c.values_len : c.lens_items_len + c.data_len;
                    vals_all += n;
                    if (needed) vals_need += n;
                }
            if (stats && probe) { stats->staged_columns += cols_need; stats->pruned_columns += cols_all - cols_need; }   // as vlscan_scan_batch: 0 / 0 without a probe
            if (probe && vals_need * 8 > vals_all * 7) ctx->bf_skip = 7;
            do_upload(ctx, field_names, field_name_lens, nfields, blocks, nblocks, b, stats, &need_bloom, UP_VALUES, need.data());
            if (keep) {   // what vlscan_stage_selected checks its descriptors against
                b->h_sig.assign((size_t)nblocks * nfields, vlscan_batch::CellSig{});
                b->h_ncols.resize(nblocks);
                for (uint64_t i = 0; i < nblocks; i++) {
                    b->h_ncols[i] = blocks[i].ncols;
                    for (uint32_t k = 0; k < blocks[i].ncols; k++) {
                        const vlscan_column& c = blocks[i].cols[k];
                        if (c.kind == VLSCAN_COL_VALUES) b->h_sig[i * nfields + c.field] = cell_sig(c);
                    }
                }
            }
        });
    } else rc = guarded(ctx, [&] { do_upload(ctx, field_names, field_name_lens, nfields, blocks, nblocks, b, stats, &need_bloom); });
    if (!rc) rc = vlscan_scan_resident(ctx, prog, b, nullptr);
    if (!rc) rc = vlscan_fetch_results(ctx, out_bitmap_words, out_match_counts, stats);
    if (!rc && stats) {
        rc = guarded(ctx, [&] { read_stats(ctx, stats, true); stats->blocks += b->nblocks; stats->rows += b->rows; stats->gpu_launches += ctx->launches - launches0; });
    }
    if (keep && !rc) ctx->kept = true;   // the result of vlscan_scan_resident above stays, on the batch it staged
    else { ctx->has_result = false; ctx->last_batch = nullptr; ctx->kept = false; }
    ctx->recycle = b;
    return rc;
}

int vlscan_scan_batch(vlscan_ctx* ctx, const vlscan_program* prog, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields,
                      const vlscan_block* blocks, uint64_t nblocks, uint64_t* out_bitmap_words, uint32_t* out_match_counts, vlscan_stats* stats) {
    return scan_batch_impl(ctx, prog, field_names, field_name_lens, nfields, blocks, nblocks, out_bitmap_words, out_match_counts, stats, false);
}

int vlscan_scan_batch_keep(vlscan_ctx* ctx, const vlscan_program* prog, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields,
                           const vlscan_block* blocks, uint64_t nblocks, uint64_t* out_bitmap_words, uint32_t* out_match_counts, vlscan_stats* stats) {
    if (!ctx || !prog) return guarded(nullptr, [&] { throw BadInput(!ctx ? "vlscan_scan_batch_keep needs a vlscan_ctx on a CUDA device (there is no CPU fallback)" : "vlscan_scan_batch_keep: no program"); });
    return scan_batch_impl(ctx, prog, field_names, field_name_lens, nfields, blocks, nblocks, out_bitmap_words, out_match_counts, stats, true);
}

int vlscan_stage_selected(vlscan_ctx* ctx, const vlscan_block* blocks, uint64_t nblocks, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields,
                          const uint32_t* block_list, uint64_t nlist, uint64_t out_info[4]) {
    uint64_t info[4] = {0, 0, 0, 0};   // cells staged, cells already staged, H2D bytes, frames through the device decoder
    bool staging = false;
    const int rc = guarded(ctx, [&] {
        if (nfields == 0) throw BadInput("vlscan_stage_selected needs at least one field");
        const std::vector<std::string> names = canonical_names(field_names, field_name_lens, nfields, "vlscan_stage_selected");
        if (nlist && !block_list) throw BadInput("vlscan_stage_selected: block list missing");
        if (!ctx) throw BadInput("vlscan_stage_selected needs a vlscan_ctx on a CUDA device (there is no CPU fallback)");
        if (!ctx->has_result || !ctx->kept || !ctx->recycle || ctx->last_batch != ctx->recycle) throw BadInput("no kept scan on this ctx (vlscan_scan_batch_keep keeps one until the next scan)");
        vlscan_batch* b = ctx->recycle;
        VL_CUDA(cudaSetDevice(ctx->device));
        const uint32_t nf = b->nfields;
        std::vector<char> want(nf, 0);
        for (const std::string& n : names) {
            const int slot = b->field_slot(n);
            if (slot < 0) throw BadInput("field `" + n + "` is not a field of the kept batch");
            want[slot] = 1;
        }
        if (!blocks || nblocks != b->nblocks) throw BadInput("the block descriptors differ from those of the kept scan: " + std::to_string(nblocks) + " blocks instead of " + std::to_string(b->nblocks));
        std::vector<uint8_t> sel(nblocks, 0);
        if (block_list) {
            for (uint64_t i = 0; i < nlist; i++) {
                if (block_list[i] >= nblocks) throw BadInput("block_list[" + std::to_string(i) + "] = " + std::to_string(block_list[i]) + " is outside the kept batch of " + std::to_string(nblocks) + " blocks");
                sel[block_list[i]] = 1;
            }
        } else if (nblocks) {   // every block with selected rows
            std::vector<uint32_t> cnt(nblocks);
            VL_CUDA(cudaMemcpyAsync(cnt.data(), ctx->counts.p, nblocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaStreamSynchronize(ctx->stream));
            for (uint64_t i = 0; i < nblocks; i++) sel[i] = cnt[i] != 0;
        }
        // the descriptors of the blocks this call reads must be the ones the keep call staged from
        auto mismatch = [&](uint64_t i, const char* what) { return BadInput("the block descriptors differ from those of the kept scan: block " + std::to_string(i) + ", " + what); };
        for (uint64_t i = 0; i < nblocks; i++) {
            if (!sel[i]) continue;
            const vlscan_block& blk = blocks[i];
            if (blk.rows != b->h_rows[i]) throw mismatch(i, "row count");
            if (blk.ncols != b->h_ncols[i] || (blk.ncols && !blk.cols)) throw mismatch(i, "column count");
            for (uint32_t k = 0; k < blk.ncols; k++) {
                const vlscan_column& c = blk.cols[k];
                if (c.field >= nf) throw mismatch(i, "field of a column");
                const DevColumn& d = b->h_cols[i * nf + c.field];
                if (c.kind == VLSCAN_COL_CONST) { if (d.kind != COL_CONST || d.meta_len != c.const_len) throw mismatch(i, "const column"); }
                else if (c.kind == VLSCAN_COL_VALUES) {
                    if (d.kind != COL_VALUES || d.vt != c.value_type) throw mismatch(i, "column kind or value type");
                    const vlscan_batch::CellSig want = cell_sig(c), &had = b->h_sig[i * nf + c.field];
                    if (had.stage != want.stage || had.len0 != want.len0 || had.len1 != want.len1) throw mismatch(i, "values stage or payload lengths");
                } else throw mismatch(i, "column kind");
            }
        }
        // const, dict tables and absent cells are on the device (or nothing) already; values cells whose payload the keep call left on the host are staged
        std::vector<uint8_t> need((size_t)nblocks * nf, 0);
        for (uint64_t i = 0; i < nblocks; i++) {
            if (!sel[i]) continue;
            for (uint32_t s = 0; s < nf; s++) {
                const DevColumn& d = b->h_cols[i * nf + s];
                if (!want[s] || d.kind != COL_VALUES) continue;
                if (d.values_state == VALUES_STAGED) info[1]++;
                else { need[i * nf + s] = 1; info[0]++; }
            }
        }
        if (!info[0]) return;
        vlscan_stats st;
        memset(&st, 0, sizeof st);
        staging = true;
        do_upload(ctx, nullptr, nullptr, nf, blocks, nblocks, b, &st, nullptr, UP_LATE, need.data(), &info[3]);
        info[2] = st.h2d_bytes;
    });
    if (rc && staging) {   // a half-staged batch is not a result any more
        ctx->has_result = false; ctx->last_batch = nullptr; ctx->kept = false;
        info[0] = info[1] = info[2] = info[3] = 0;
    }
    if (out_info && !rc) memcpy(out_info, info, sizeof info);
    return rc;
}

}  // extern "C"
