// Host side of the device ZSTD decoder, the part that never touches CUDA: the tables a decode job hands to the device (frames, ZSTD blocks
// with scratch offsets and table slots, launch groups, work lists) and how they are built - block by block, or for a whole batch of
// values blocks on several threads.  vl_zstd.cu adds the device buffers and the launches; tests build this header alone with
// ThreadSanitizer (tests/host_asan/harness.cpp, mode "walk").
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <array>
#include <atomic>
#include <exception>
#include <functional>
#include <string>
#include <thread>
#include <vector>
#include "vl_zstd.h"
#include "vl_zstd_types.h"
#include "vl_zstd_walk.h"

namespace vl {

using namespace zs;

// scratch limits of one launch group (groups are cut at frame boundaries)
// A group must hold enough blocks to fill the device for the lane-per-block phases (132 SMs x 56 sequence lanes = 7.4 k blocks per
// wave on an H100) and enough frames for the warp-per-frame executor (~8 k in flight): small groups decode less efficiently.  On the other hand
// group g is decoded while the bytes of group g+1 are still being copied, so the FIRST group decides when the decoder starts and the LAST
// one is the tail that nothing hides.  With uniform groups a decode-bound batch (C3) wants the large limits, a DMA-bound one (C2) half
// of them.  So the limits are tapered: a small first group, large ones in the middle,
// small ones over the last twelfth of the sequences (walk_values_blocks knows every frame's needs before it cuts).
// VLSCAN_ZSTD_GROUP_SCALE (tuning only): a fixed multiplier for all groups instead; 4 = the round-1 limits.
inline uint64_t group_scale_env() { static const uint64_t v = [] { const char* e = getenv("VLSCAN_ZSTD_GROUP_SCALE"); long x = e ? atol(e) : 0; return (uint64_t)(x < 0 ? 0 : x > 64 ? 64 : x); }(); return v; }
static const uint64_t kGroupLitsUnit = 512ull << 20, kGroupSeqsUnit = 64ull << 20;
static const uint32_t kGroupSlotsUnit = 32u << 10;

struct Group { uint32_t frame_lo, frame_hi; uint32_t huf_lo, huf_hi, lit_lo, lit_hi, seq_lo, seq_hi, ord_lo, ord_hi; };

// scratch a frame needs (or, as a running total, the scratch of its launch group used up in front of it)
struct FrameUse { uint64_t lits, seqs; uint32_t huf, fse; };

struct ZstdJobImpl {
    std::vector<ZFrame> frames;
    std::vector<ZBlock> blocks;
    std::vector<Group> groups;
    std::vector<uint32_t> lists;   // work lists of all groups (prepare)
    // running scratch use of the open group
    uint64_t g_lits = 0, g_seqs = 0; uint32_t g_huf = 0, g_fse = 0; uint32_t g_frame_lo = 0;
    uint64_t limit_scale = group_scale_env() ? group_scale_env() : 4;   // multiplier of the group limits for the frame being admitted
    uint64_t max_lits = 0, max_seqs = 0; uint32_t max_huf = 0, max_fse = 0;
    uint64_t n_compressed = 0, n_seqs = 0;
    int threads = 0;               // host threads for the table-sized passes (add_values_blocks sets it)
    bool prepared = false, ran = false;
    std::function<void(uint64_t)> group_hook;

    void close_group_at(uint32_t f) {   // f = number of frames committed so far
        if (g_frame_lo == f) return;
        Group g{}; g.frame_lo = g_frame_lo; g.frame_hi = f;
        groups.push_back(g);
        max_lits = std::max(max_lits, g_lits); max_seqs = std::max(max_seqs, g_seqs); max_huf = std::max(max_huf, g_huf); max_fse = std::max(max_fse, g_fse);
        g_lits = g_seqs = 0; g_huf = g_fse = 0; g_frame_lo = f;
    }
    void close_group() { close_group_at((uint32_t)frames.size()); }

    static FrameUse frame_use(const ZBlock* b, uint32_t cnt) {
        FrameUse u{0, 0, 0, 0};
        for (uint32_t i = 0; i < cnt; i++) {
            if (b[i].type != ZB_COMPRESSED) continue;
            if (b[i].lit_type >= ZL_COMPRESSED) u.lits += b[i].lit_regen;
            u.seqs += b[i].nseq; u.huf += b[i].huf_own != Z_PREDEF; u.fse += b[i].fse_own != Z_PREDEF;
        }
        return u;
    }
    // Frame number f (the next one) needs `u`: cuts the launch group in front of it when the group's scratch would overflow, and returns the
    // scratch of the group used up in front of the frame.
    FrameUse admit_frame(uint32_t f, const FrameUse& u) {
        const uint64_t m = limit_scale;
        if (g_frame_lo != f && (g_lits + u.lits > kGroupLitsUnit * m || g_seqs + u.seqs > kGroupSeqsUnit * m || g_huf + u.huf > kGroupSlotsUnit * m || g_fse + u.fse > kGroupSlotsUnit * m)) close_group_at(f);
        FrameUse base{g_lits, g_seqs, g_huf, g_fse};
        g_lits += u.lits; g_seqs += u.seqs; g_huf += u.huf; g_fse += u.fse;
        return base;
    }
    // Slots and scratch offsets inside a frame were numbered from 0 by the parser; rebase them into the launch group.
    static void place_blocks(ZBlock* b, uint32_t cnt, FrameUse base, uint64_t& n_compressed, uint64_t& n_seqs) {
        for (uint32_t i = 0; i < cnt; i++) {
            ZBlock& B = b[i];
            if (B.type != ZB_COMPRESSED) continue;
            if (B.lit_type >= ZL_COMPRESSED) { B.lit_off = base.lits; base.lits += B.lit_regen; }
            B.seq_base = base.seqs; base.seqs += B.nseq;
            if (B.huf_own != Z_PREDEF) B.huf_own += base.huf;
            if (B.huf_slot != Z_PREDEF) B.huf_slot += base.huf;
            if (B.fse_own != Z_PREDEF) B.fse_own += base.fse;
            if (B.ll_slot != Z_PREDEF) B.ll_slot += base.fse;
            if (B.of_slot != Z_PREDEF) B.of_slot += base.fse;
            if (B.ml_slot != Z_PREDEF) B.ml_slot += base.fse;
            n_compressed++; n_seqs += B.nseq;
        }
    }

    // Assigns scratch to the blocks [blk_lo, end) of the frame that was just parsed and appends the frame.
    void commit_frame(ZFrame fr) {
        const uint32_t cnt = (uint32_t)blocks.size() - fr.blk_lo;
        const FrameUse base = admit_frame((uint32_t)frames.size(), frame_use(blocks.data() + fr.blk_lo, cnt));
        place_blocks(blocks.data() + fr.blk_lo, cnt, base, n_compressed, n_seqs);
        fr.blk_hi = (uint32_t)blocks.size();
        frames.push_back(fr);
    }

    // ---- the walk of a whole batch on several threads ---------------------------------------------------------------------------------
    // Thread t walks the values blocks [lo_t, hi_t) into a block vector of its own (frames go straight to their final place: values
    // block i is frames 2i and 2i+1).  A sequential pass over the per-frame scratch needs then cuts the launch groups exactly like
    // commit_frame would have, and the threads move their blocks to the final place, rebased into their group.  The result does not
    // depend on the number of threads.
    struct Shard { std::vector<ZBlock> blocks; size_t lo = 0, hi = 0, bad = SIZE_MAX; std::string msg; uint64_t n_compressed = 0, n_seqs = 0; };

    // f(0) .. f(T-1), f(0) on the calling thread; whatever a worker throws is rethrown here once all of them are done
    template <class F> static void on_threads(int T, F&& f) {
        std::vector<std::exception_ptr> err((size_t)T);
        auto guarded_f = [&f, &err](int t) { try { f(t); } catch (...) { err[(size_t)t] = std::current_exception(); } };
        std::vector<std::thread> pool;
        for (int t = 1; t < T; t++) pool.emplace_back(guarded_f, t);
        guarded_f(0);
        for (auto& th : pool) th.join();
        for (auto& e : err) if (e) std::rethrow_exception(e);
    }

    void walk_values_blocks(const ZValuesBlock* v, size_t n, int nthreads, ZValuesInfo* info, size_t* bad, std::string* msg) {
        if (2 * (uint64_t)n > 0xFFFFFFF0ull) throw BadInput("too many values blocks in one batch");
        const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)nthreads, n / 256 + 1));
        threads = T;
        frames.assign(2 * n, ZFrame{});
        std::vector<FrameUse> use(2 * n);
        std::vector<Shard> sh((size_t)T);
        for (int t = 0; t < T; t++) { sh[t].lo = n * (size_t)t / (size_t)T; sh[t].hi = n * (size_t)(t + 1) / (size_t)T; }
        on_threads(T, [&](int t) {
            Shard& S = sh[t];
            S.blocks.reserve((S.hi - S.lo) * 2 + (S.hi - S.lo) / 2 + 16);
            for (size_t i = S.lo; i < S.hi; i++) {
                try {
                    ZFrame &f1 = frames[2 * i], &f2 = frames[2 * i + 1];
                    const size_t c1 = zwalk::parse_bytes_block_into(S.blocks, (uint32_t)(2 * i), v[i].p, v[i].n, v[i].zoff, f1);
                    const size_t c2 = zwalk::parse_bytes_block_into(S.blocks, (uint32_t)(2 * i + 1), v[i].p + c1, v[i].n - c1, v[i].zoff + c1, f2);
                    if (c1 + c2 != v[i].n) throw BadInput("unexpected non-empty tail after reading bytes block with strings");
                    info[i].lens_len = f1.fcs; info[i].data_len = f2.fcs;
                    use[2 * i] = frame_use(S.blocks.data() + f1.blk_lo, f1.blk_hi - f1.blk_lo);
                    use[2 * i + 1] = frame_use(S.blocks.data() + f2.blk_lo, f2.blk_hi - f2.blk_lo);
                } catch (const BadInput& e) { S.bad = i; S.msg = e.msg; return; }
            }
        });
        for (int t = 0; t < T; t++) if (sh[t].bad != SIZE_MAX) { *bad = sh[t].bad; *msg = sh[t].msg; frames.clear(); return; }
        // scratch need -> scratch base; the group limits follow the position in the batch (see the top of this file)
        uint64_t total_seqs = 0, seen = 0;
        for (size_t f = 0; f < 2 * n; f++) total_seqs += use[f].seqs;
        for (size_t f = 0; f < 2 * n; f++) {
            if (!group_scale_env()) limit_scale = (groups.empty() || seen > total_seqs - total_seqs / 12) ? 1 : 4;
            seen += use[f].seqs;
            use[f] = admit_frame((uint32_t)f, use[f]);
        }
        if (!group_scale_env()) limit_scale = 1;   // frames added one by one after the walk (timestamps) join the last, small group
        std::vector<size_t> base((size_t)T + 1, 0);
        for (int t = 0; t < T; t++) base[t + 1] = base[t] + sh[t].blocks.size();
        if (base[T] > 0xFFFFFFF0ull) throw BadInput("too many ZSTD blocks in one batch");
        blocks.resize(base[T]);
        on_threads(T, [&](int t) {
            Shard& S = sh[t];
            if (!S.blocks.empty()) memcpy(blocks.data() + base[t], S.blocks.data(), S.blocks.size() * sizeof(ZBlock));
            std::vector<ZBlock>().swap(S.blocks);
            for (size_t f = 2 * S.lo; f < 2 * S.hi; f++) {
                ZFrame& fr = frames[f];
                fr.blk_lo += (uint32_t)base[t]; fr.blk_hi += (uint32_t)base[t];
                place_blocks(blocks.data() + fr.blk_lo, fr.blk_hi - fr.blk_lo, use[f], S.n_compressed, S.n_seqs);
            }
        });
        for (int t = 0; t < T; t++) { n_compressed += sh[t].n_compressed; n_seqs += sh[t].n_seqs; }
    }

    // Work lists of every launch group, in one array: blocks with a Huffman description | blocks with Huffman streams | blocks with sequences |
    // frames ordered by size (largest first: the tail of a launch is then made of short frames)
    void prepare() {
        if (prepared) return;
        prepared = true;
        close_group();
        const size_t G = groups.size();
        std::vector<std::vector<uint32_t>> gl(G);
        std::vector<std::array<uint32_t, 4>> cnt(G);
        std::atomic<size_t> next{0};
        const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(threads, 1), G));
        on_threads(T, [&](int) {
            std::vector<std::pair<uint32_t, uint32_t>> v; std::vector<uint32_t> count;
            for (;;) {
                const size_t gi = next.fetch_add(1);
                if (gi >= G) return;
                const Group& g = groups[gi];
                std::vector<uint32_t>& L = gl[gi];
                const uint32_t blo = frames[g.frame_lo].blk_lo, bhi = frames[g.frame_hi - 1].blk_hi;
                // appends the second members of v ordered by descending first member, ties in input order
                auto by_desc = [&] {
                    uint32_t kmax = 0; for (auto& e : v) kmax = std::max(kmax, e.first);
                    if (v.size() >= 64 && kmax < (1u << 16)) {   // counting sort: the keys are sizes in coarse units
                        count.assign((size_t)kmax + 2, 0);
                        for (auto& e : v) count[kmax - e.first + 1]++;
                        for (uint32_t k = 0; k <= kmax; k++) count[k + 1] += count[k];
                        const size_t at = L.size(); L.resize(at + v.size());
                        for (auto& e : v) L[at + count[kmax - e.first]++] = e.second;
                    } else {
                        std::stable_sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return a.first > b.first; });
                        for (auto& e : v) L.push_back(e.second);
                    }
                    v.clear();
                };
                for (uint32_t i = blo; i < bhi; i++) if (blocks[i].type == ZB_COMPRESSED && blocks[i].lit_type == ZL_COMPRESSED) L.push_back(i);
                cnt[gi][0] = (uint32_t)L.size();
                for (uint32_t i = blo; i < bhi; i++) if (blocks[i].type == ZB_COMPRESSED && blocks[i].lit_type >= ZL_COMPRESSED) v.push_back({blocks[i].lit_regen >> 9, i});
                by_desc(); cnt[gi][1] = (uint32_t)L.size();
                for (uint32_t i = blo; i < bhi; i++) if (blocks[i].type == ZB_COMPRESSED && blocks[i].nseq) v.push_back({blocks[i].nseq >> 6, i});
                by_desc(); cnt[gi][2] = (uint32_t)L.size();
                for (uint32_t i = g.frame_lo; i < g.frame_hi; i++) v.push_back({(uint32_t)(frames[i].fcs >> 10), i});
                by_desc(); cnt[gi][3] = (uint32_t)L.size();
            }
        });
        size_t total = 0; for (auto& L : gl) total += L.size();
        if (total > 0xFFFFFFF0ull) throw BadInput("too many ZSTD blocks in one batch");
        lists.resize(total);
        size_t off = 0;
        for (size_t gi = 0; gi < G; gi++) {
            Group& g = groups[gi];
            g.huf_lo = (uint32_t)off; g.huf_hi = g.lit_lo = (uint32_t)(off + cnt[gi][0]); g.lit_hi = g.seq_lo = (uint32_t)(off + cnt[gi][1]);
            g.seq_hi = g.ord_lo = (uint32_t)(off + cnt[gi][2]); g.ord_hi = (uint32_t)(off + cnt[gi][3]);
            if (!gl[gi].empty()) memcpy(lists.data() + off, gl[gi].data(), gl[gi].size() * 4);
            off += gl[gi].size();
        }
    }

    // copies n bytes on the job's host threads (the descriptor tables are ~100 bytes per ZSTD block)
    void spread_copy(void* dst, const void* src, size_t n) const {
        const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(threads, 1), n / (4u << 20) + 1));
        on_threads(T, [&](int t) { const size_t lo = n * (size_t)t / (size_t)T, hi = n * (size_t)(t + 1) / (size_t)T; if (hi > lo) memcpy((uint8_t*)dst + lo, (const uint8_t*)src + lo, hi - lo); });
    }

    // Everything run() hands to the device, field by field (padding bytes stay out of it).
    void digest(uint64_t out[4]) const {
        const ZstdJobImpl& J = *this;
        auto mix = [](uint64_t& h, uint64_t v) { h = (h ^ v) * 0x9E3779B97F4A7C15ull; h ^= h >> 29; };
        uint64_t h0 = 1, h1 = 2, h2 = 3, h3 = 4;
        for (const ZFrame& f : J.frames) { mix(h0, f.dst); mix(h0, f.fcs); mix(h0, ((uint64_t)f.blk_lo << 32) | f.blk_hi); }
        for (const ZBlock& b : J.blocks) {
            mix(h1, b.src); mix(h1, b.lit_off); mix(h1, b.seq_base); mix(h1, ((uint64_t)b.size << 32) | b.frame); mix(h1, ((uint64_t)b.lit_hdr << 32) | b.lit_regen);
            mix(h1, ((uint64_t)b.lit_comp << 32) | b.nseq); mix(h1, ((uint64_t)b.seq_hdr << 32) | b.huf_slot); mix(h1, ((uint64_t)b.huf_own << 32) | b.fse_own);
            mix(h1, ((uint64_t)b.ll_slot << 32) | b.of_slot); mix(h1, ((uint64_t)b.ml_slot << 32) | ((uint64_t)b.type << 24) | ((uint64_t)b.lit_type << 16) | ((uint64_t)b.lit_streams << 8) | b.modes); mix(h1, b.rep_known);
        }
        for (const Group& g : J.groups) for (uint32_t x : {g.frame_lo, g.frame_hi, g.huf_lo, g.huf_hi, g.lit_lo, g.lit_hi, g.seq_lo, g.seq_hi, g.ord_lo, g.ord_hi}) mix(h2, x);
        for (uint64_t x : {J.max_lits, J.max_seqs, (uint64_t)J.max_huf, (uint64_t)J.max_fse, J.n_compressed, J.n_seqs, (uint64_t)J.groups.size()}) mix(h2, x);
        for (uint32_t x : J.lists) mix(h3, x);
        out[0] = h0; out[1] = h1; out[2] = h2; out[3] = h3;
    }
};

}  // namespace vl
