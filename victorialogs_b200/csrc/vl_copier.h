// The host -> device transport of the batch uploads in vl_engine.cu.
#pragma once
#include <dlfcn.h>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <utility>
#include <vector>
#include "vl_engine.h"

namespace vl {

// Host threads for the header walk and the descriptor tables of an upload: VLSCAN_HOST_THREADS, else up to 16 (one process per GPU shares the
// box with its peers).  0 selects the single-threaded block-by-block walk.
inline int host_threads() {
    if (const char* e = getenv("VLSCAN_HOST_THREADS")) return std::max(0, std::min(256, atoi(e)));
    return (int)std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
}

// every event of an upload lives here: destroyed when the upload is left, by return or by exception (a worker that keeps hitting malformed
// parts must not leak one event per batch)
struct EventBag {
    std::vector<cudaEvent_t> all;
    cudaEvent_t make() { cudaEvent_t e; VL_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); all.push_back(e); return e; }
    ~EventBag() { for (cudaEvent_t e : all) cudaEventDestroy(e); }
};
struct Piece { const uint8_t* src; uint64_t len; uint64_t dst; };

// The host -> device transport of an upload.  All payload copies run on the ctx's copy stream; the compute stream picks them up through events.
// Runs of pieces that are contiguous on both sides (src stride == dst stride) and live in pinned host memory go out as one cudaMemcpyAsync;
// everything else is packed through a pinned staging ring.
class Copier {
public:
    EventBag events;
    uint64_t h2d = 0;
    bool all_pinned = true;   // no piece took the staging ring
    std::vector<Piece> src;   // the compressed sources of the device decoder: src[0, src_sent) are on their way
    explicit Copier(vlscan_ctx* ctx) : ctx(ctx), cs(ctx->copy_stream) {}

    // pieces [i0, i1) of the list (all of it by default) to `base`; the staging ring is flushed at the end of every call
    void copy(const std::vector<Piece>& pieces, uint8_t* base, size_t i0 = 0, size_t i1 = SIZE_MAX) {
        dev_base = base;
        size_t i = i0;
        const size_t end = std::min(i1, pieces.size());
        while (i < end) {
            // maximal run of pieces laid out identically on both sides (same stride between source and destination)
            size_t j = i;
            while (j + 1 < end && pieces[j + 1].src > pieces[j].src && pieces[j + 1].src - pieces[i].src == (ptrdiff_t)(pieces[j + 1].dst - pieces[i].dst)) j++;
            // one DMA for the whole run (gaps, i.e. alignment slack, included) only when the run lies inside a single page-locked allocation: two
            // pinned buffers that merely line up could have pageable memory between them
            if (pinned(pieces[i].src, (pieces[j].dst - pieces[i].dst) + pieces[j].len)) {
                flush();
                // (split at piece boundaries every ~128 MB so that consumers can be released chunk by chunk)
                for (size_t a = i; a <= j;) {
                    size_t b2 = a;
                    while (b2 < j && (pieces[b2].dst + pieces[b2].len) - pieces[a].dst < (128ull << 20)) b2++;
                    const uint64_t len = (pieces[b2].dst - pieces[a].dst) + pieces[b2].len;
                    VL_CUDA(cudaMemcpyAsync(dev_base + pieces[a].dst, pieces[a].src, len, cudaMemcpyHostToDevice, cs));
                    if (marking) mark(pieces[b2].dst + pieces[b2].len);
                    h2d += len; a = b2 + 1;
                }
                i = j + 1;
                continue;
            }
            all_pinned = false;
            need_stage();
            for (; i <= j; i++) {
                const Piece& pc = pieces[i];
                uint64_t done = 0;
                while (done < pc.len) {
                    if (chunk_open && (chunk_dst + fill != pc.dst + done || fill == CH)) flush();
                    if (!chunk_open) { chunk_open = true; chunk_dst = pc.dst + done; fill = 0; }
                    size_t take = (size_t)std::min<uint64_t>(pc.len - done, CH - fill);
                    segs.push_back({pc.src + done, fill, take});
                    fill += take; done += take;
                }
                // pack the space up to the next piece as zeros when it follows closely, so chunks stay large: between two pieces of the copied part
                // there is nothing but alignment slack and empty reservations (a bloom filter left on the host is 48 bytes of them), zero in the
                // arena already.  With a 64-byte limit every timestamps block of a part was a chunk, a DMA and an event of its own: 16 k per batch.
                if (i + 1 < end) {
                    uint64_t gap = pieces[i + 1].dst - (pc.dst + pc.len);
                    if (gap <= 1024 && fill + gap < CH) { if (gap) segs.push_back({nullptr, fill, (size_t)gap}); fill += gap; } else flush();
                }
            }
        }
        flush();
    }
    // The compressed sources go to `zbase`, and while they do, `marks` records (end offset, event) pairs.  Page-locked sources are enqueued
    // right away (asynchronous DMA).  Pageable sources (a part's mmap()ed files) have to be packed through the staging ring by this thread:
    // that is done lazily, launch group by launch group, from wait_sources, so that the device decodes group g while the host packs group
    // g + 1 (packing it all here would finish before the first kernel starts).
    void send_sources(uint8_t* zbase) { src_base = zbase; if (pinned(src[0].src, src[0].len)) ship_sources(UINT64_MAX); }
    void ship_sources(uint64_t limit) {   // enqueue every source piece that starts below `limit`
        size_t hi = src_sent;
        while (hi < src.size() && src[hi].dst < limit) hi++;
        if (hi == src_sent) return;
        marking = true; copy(src, src_base, src_sent, hi); marking = false;
        src_sent = hi;
    }
    // the decoder's group hook: stream `s` waits for the sources up to `src_end` only, so the group starts while later bytes are in flight
    void wait_sources(cudaStream_t s, uint64_t src_end) {
        ship_sources(src_end);
        for (auto& m : marks) if (m.first >= src_end) { VL_CUDA(cudaStreamWaitEvent(s, m.second, 0)); return; }
        if (!marks.empty()) VL_CUDA(cudaStreamWaitEvent(s, marks.back().second, 0));
    }

private:
    static constexpr size_t CH = 64u << 20;
    vlscan_ctx* ctx; cudaStream_t cs;
    uint8_t* stage = nullptr; cudaEvent_t evs[2] = {nullptr, nullptr}; int cur = 0; size_t fill = 0; uint64_t chunk_dst = 0; bool chunk_open = false;
    uint8_t* dev_base = nullptr;   // destination buffer of the pieces being copied
    uint8_t* src_base = nullptr; size_t src_sent = 0;
    bool marking = false;
    std::vector<std::pair<uint64_t, cudaEvent_t>> marks;
    // Packing pageable memory (a part's mmap()ed files) into the ring is a memcpy, ~10 GB/s on one core and page faults on cold files: the
    // segments of a chunk are only recorded while the pieces are walked, and copied by all host threads when the chunk is flushed
    // (each thread takes an equal byte range of the chunk).
    struct Seg { const uint8_t* src; size_t at, len; };   // src == nullptr: zeros
    std::vector<Seg> segs;
    uintptr_t pageable_lo = 1, pageable_hi = 0, locked_lo = 1, locked_hi = 0;

    void mark(uint64_t end_off) { cudaEvent_t e = events.make(); VL_CUDA(cudaEventRecord(e, cs)); marks.push_back({end_off, e}); }
    void pack_chunk(uint8_t* buf, size_t bytes) {
        const int nt = (int)std::min<size_t>(std::max(1, host_threads()), bytes / (1u << 20) + 1);
        auto work = [&](int t) {
            const size_t lo = bytes * (size_t)t / nt, hi = bytes * (size_t)(t + 1) / nt;
            size_t i = std::upper_bound(segs.begin(), segs.end(), lo, [](size_t v, const Seg& g) { return v < g.at; }) - segs.begin();
            if (i) i--;
            for (; i < segs.size() && segs[i].at < hi; i++) {
                const Seg& g = segs[i];
                const size_t a = std::max(g.at, lo), b = std::min(g.at + g.len, hi);
                if (a >= b) continue;
                if (g.src) memcpy(buf + a, g.src + (a - g.at), b - a); else memset(buf + a, 0, b - a);
            }
        };
        if (nt <= 1) { work(0); return; }
        if (!ctx->pool) ctx->pool = new HostPool;
        ctx->pool->run(nt, work);
    }
    void flush() {
        if (!chunk_open || !fill) { chunk_open = false; fill = 0; segs.clear(); return; }
        pack_chunk(stage + (size_t)cur * CH, fill);
        segs.clear();
        VL_CUDA(cudaMemcpyAsync(dev_base + chunk_dst, stage + (size_t)cur * CH, fill, cudaMemcpyHostToDevice, cs));
        VL_CUDA(cudaEventRecord(evs[cur], cs));
        if (marking) mark(chunk_dst + fill);
        h2d += fill; cur ^= 1; fill = 0; chunk_open = false;
        VL_CUDA(cudaEventSynchronize(evs[cur]));
    }
    static bool is_pinned(const void* p) { cudaPointerAttributes a; if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; } return a.type == cudaMemoryTypeHost; }
    // Is [p, p + len) inside ONE page-locked allocation?  The runtime API only classifies single addresses; the driver knows the range of the
    // allocation an address belongs to (cuPointerGetAttribute RANGE_START_ADDR / RANGE_SIZE).  libcuda is always there when a device is.
    // Pointer queries cost microseconds each and a part's descriptors come as tens of thousands of small pieces (timestamps, const values) out of
    // the same mmap()ed files: the last answers are remembered.  A 2 MiB-aligned region around a pageable address is taken as pageable as a whole
    // (if a page-locked allocation begins inside it, its pieces merely take the staging ring), a page-locked allocation by its exact range.
    bool pinned(const uint8_t* p, uint64_t len) {
        typedef int (*attr_fn)(void*, int, unsigned long long);
        static const attr_fn fn = [] { void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL); return h ? (attr_fn)dlsym(h, "cuPointerGetAttribute") : (attr_fn) nullptr; }();
        const uintptr_t a = (uintptr_t)p;
        if (a >= pageable_lo && a < pageable_hi) return false;
        if (a >= locked_lo && a + len <= locked_hi) return true;
        if (!is_pinned(p)) { pageable_lo = a & ~(uintptr_t)((2u << 20) - 1); pageable_hi = pageable_lo + (2u << 20); return false; }
        if (!fn) return len <= 1 || (len <= 4096 && is_pinned(p + len - 1));   // no driver entry point: only what single-address checks can vouch for
        unsigned long long base = 0; size_t size = 0;
        if (fn(&base, 11 /* CU_POINTER_ATTRIBUTE_RANGE_START_ADDR */, (unsigned long long)(uintptr_t)p) != 0 || fn(&size, 12 /* CU_POINTER_ATTRIBUTE_RANGE_SIZE */, (unsigned long long)(uintptr_t)p) != 0) return false;
        if (size) { locked_lo = (uintptr_t)base; locked_hi = (uintptr_t)(base + size); }
        return (unsigned long long)(uintptr_t)p >= base && (unsigned long long)(uintptr_t)p + len <= base + size;
    }
    void need_stage() {
        if (stage) return;
        stage = (uint8_t*)ctx->ensure_pinned(2 * CH);
        for (int k = 0; k < 2; k++) { evs[k] = events.make(); VL_CUDA(cudaEventRecord(evs[k], cs)); }
    }
};

}  // namespace vl
