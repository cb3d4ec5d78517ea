// libvlscan.so: the aggregations over the last scan's result, driven from the host: the hit list and the gathers of values and timestamps
// (vlscan_fetch_hits, vlscan_gather_*), the hits histogram, its value sums and vmranges (vlscan_hits_stats, _sums, _vmranges), the N newest rows
// (vlscan_last_rows) and the facets (vlscan_facets).  Their kernels are in vl_agg.cuh; row offsets come from the scan's row_offsets.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <limits>
#include <mutex>
#include <string>
#include <string_view>
#include <vector>
#include "vl_engine.h"
#include "vl_agg.cuh"

using namespace vl;

namespace {

// Typed arrays laid out in one scratch buffer at 16-byte alignment: take() every array, then place() grows the buffer once, sets the pointers
// and returns the bytes laid out.
struct Carve {
    size_t off = 0;
    std::vector<std::function<void(uint8_t*)>> set;
    template <class T> Carve& take(T*& p, uint64_t n) { const size_t o = off; off += (n * sizeof(T) + 15) & ~(size_t)15; set.push_back([&p, o](uint8_t* base) { p = (T*)(base + o); }); return *this; }
    size_t place(DevBuf& buf) { buf.ensure(std::max<size_t>(off, 16)); for (auto& f : set) f(buf.as<uint8_t>()); return off; }
};

// ---- the by-field buckets: the query's size and offset converted as the reference converts them (include/vlscan.h, vlscan_hits_stats) --------
// Go's float -> integer conversions on amd64: int64 and int32 by CVTTSD2SQ / CVTTSD2SL (NaN and out of range -> the minimum), uint32 through
// int64, uint64 by the compiler's split at 2^63.
int32_t go_int32_of_float(double f) { return f > -2147483649.0 && f < 2147483648.0 ? (int32_t)f : INT32_MIN; }
uint64_t go_uint64_of_float(double f) {
    const double c = 9223372036854775808.0;
    return f < c ? (uint64_t)mn::int64_of_float(f) : (uint64_t)mn::int64_of_float(f - c) | (1ull << 63);
}
// math.Pow10
double go_pow10(int n) {
    static const double tab[32] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20,
                                   1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31};
    static const double pos32[10] = {1e0, 1e32, 1e64, 1e96, 1e128, 1e160, 1e192, 1e224, 1e256, 1e288};
    static const double neg32[11] = {1e-0, 1e-32, 1e-64, 1e-96, 1e-128, 1e-160, 1e-192, 1e-224, 1e-256, 1e-288, 1e-320};
    if (n >= 0 && n <= 308) return pos32[n / 32] * tab[n % 32];
    if (n < 0 && n >= -323) return neg32[-n / 32] / tab[-n % 32];
    return n > 0 ? std::numeric_limits<double>::infinity() : 0.0;
}
// the exponent e of decimal.FromFloat(f) = (v, e) for a finite f > 0 (VictoriaMetrics lib/decimal positiveFloatToDecimal, getDecimalAndScale,
// positiveFloatToDecimalSlow)
int decimal_exponent(double f) {
    uint64_t u = go_uint64_of_float(f);
    int scale = 0;
    if ((double)u == f) {
        if (u < (1ull << 55) && u % 10 != 0) return 0;
        for (; u >= (1ull << 55); u /= 10) scale++;
        if (u % 10 != 0) return scale;
        for (u /= 10, scale++; u != 0 && u % 10 == 0; u /= 10) scale++;
        return scale;
    }
    double prec = 1e12;
    if (f > 1e6 || f < 1e-6) {
        if (f > 1e6) prec = 1e15;
        int e2;
        std::frexp(f, &e2);
        e2 = std::min(std::max(e2, -1022), 1023);
        scale = (int16_t)((double)e2 * 0.30102999566398119521);   // math.Ln2 / math.Ln10
        f *= go_pow10(-scale);
    }
    while (f < prec) {
        double x;
        const double frac = std::modf(f, &x);
        if (frac * prec < x) { f = x; break; }
        if ((1 - frac) * prec < x) { f = x + 1; break; }
        f *= 100;
        scale -= 2;
    }
    return go_uint64_of_float(f) % 10 != 0 ? scale : scale + 1;
}
// BucketSpec of one by-field bucket; an empty string, or why the bucket is rejected
std::string bucket_spec(const vlscan_by_bucket& b, BucketSpec* o) {
    if (!std::isfinite(b.size) || !std::isfinite(b.offset)) return "its size and offset must be finite numbers";
    if (b.calendar > VLSCAN_BUCKET_YEAR) return "unknown calendar bucket kind";
    memset(o, 0, sizeof *o);
    o->enabled = 1; o->calendar = b.calendar; o->offset = b.offset;
    o->u64_size = go_uint64_of_float(b.size); if (o->u64_size == 0) o->u64_size = 1;
    o->u64_off = (uint64_t)mn::int64_of_float(b.offset);
    const int64_t i = mn::int64_of_float(b.size);
    o->i64_size = i <= 0 ? 1 : i;
    o->i64_col_size = i == 0 ? 1 : i;
    o->i64_off = mn::int64_of_float(b.offset);
    o->u32_size = (uint32_t)i; if (o->u32_size == 0) o->u32_size = 1;
    o->u32_off = (uint32_t)go_int32_of_float(b.offset);
    const double size = b.size <= 0 ? 1 : b.size;
    o->p10 = go_pow10(-decimal_exponent(size));
    o->size_p10 = mn::int64_of_float(size * o->p10);
    if (o->size_p10 == 0) return "int64(size * 10^-e) is 0 for its float buckets";
    return "";
}

// ---- the vmrange index of metrics.Histogram.Update (include/vlscan.h, vlscan_hits_vmranges) -----------------------------------------------------
// Go's portable math.Log (math/log.go: the fdlibm reduction by Frexp, s = f / (2 + f), L1..L7, Ln2Hi / Ln2Lo), every step one rounded double
// operation.  The amd64 build of Go runs an assembly archLog that mirrors this algorithm; DESIGN §3.15 states that assumption.
double go_log(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10, L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01,
                 L3 = 2.857142874366239149e-01, L4 = 2.222219843214978396e-01, L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01,
                 L7 = 1.479819860511658591e-01;
    if (std::isnan(x) || x == std::numeric_limits<double>::infinity()) return x;
    if (x < 0) return std::numeric_limits<double>::quiet_NaN();
    if (x == 0) return -std::numeric_limits<double>::infinity();
    int ki;
    double f1 = std::frexp(x, &ki);
    if (f1 < 0.70710678118654752440) { f1 *= 2; ki--; }   // Sqrt2 / 2
    const double f = f1 - 1, k = (double)ki;
    const double s = f / (2 + f), s2 = s * s, s4 = s2 * s2;
    const double t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)));
    const double t2 = s4 * (L2 + s4 * (L4 + s4 * L6));
    const double R = t1 + t2, hfsq = 0.5 * f * f;
    return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f);
}
// Histogram.Update's index from its formula: b = (Log10(v) - e10Min) * bucketsPerDecimal with Log10(x) = Log(x) * (1 / Ln10), 1 / Ln10 the
// correctly rounded constant; lower below 0, upper from 486, else uint(b), one less when b is an integer above 0 (10^n goes to the bucket below)
int vmr_index_formula(double v) {
    if (std::isnan(v) || v < 0) return -1;
    const double b = (go_log(v) * 0x1.bcb7b1526e50ep-2 - (-9.0)) * 18.0;
    if (b < 0) return 0;
    if (b >= 486) return VL_VMRANGES - 1;
    uint64_t idx = (uint64_t)b;
    if (b == (double)idx && idx > 0) idx--;
    return (int)idx + 1;
}
double f64_bits(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }
// bound k - 1 = the least double whose formula index reaches k, found by bisection on the bit patterns of +0 .. +Inf.  The kernels and
// vmr_index_host search this table, so the device gives the host's index by construction.  Built once; the build checks that the formula does
// not decrease for 2000 ulps on either side of every bound, where a search over the bounds would disagree with it.
const std::vector<double>& vmr_bounds() {
    static std::vector<double> bounds;
    static std::string error;
    static std::once_flag once;
    std::call_once(once, [] {
        const uint64_t inf = 0x7FF0000000000000ull;
        for (int k = 1; k < VL_VMRANGES; k++) {
            uint64_t lo = 0, hi = inf;   // index(lo) < k <= index(hi)
            while (hi - lo > 1) { const uint64_t m = lo + (hi - lo) / 2; (vmr_index_formula(f64_bits(m)) >= k ? hi : lo) = m; }
            bounds.push_back(f64_bits(hi));
            int prev = -1;
            for (uint64_t u = hi > 2000 ? hi - 2000 : 0; u <= hi + 2000; u++) {
                const int x = vmr_index_formula(f64_bits(u));
                if (x < prev) error = "the vmrange index decreases near bound " + std::to_string(k);
                prev = x;
            }
        }
    });
    if (!error.empty()) throw BadInput(error);
    return bounds;
}
int vmr_index_host(double v) {
    if (std::isnan(v) || v < 0) return -1;
    const std::vector<double>& b = vmr_bounds();
    return (int)(std::upper_bound(b.begin(), b.end(), v) - b.begin());
}
// the vmrange texts by index: lowerBucketRange, bucketRanges (initBucketRanges: v = Pow10(-9), then v *= Pow(10, 1/18) 486 times, each end
// printed with %.3e), upperBucketRange.  The texts are the same for every multiplier within 16 ulps of 10^(1/18) (a test pins that), so
// they do not depend on how Go's Pow rounds.
const std::vector<std::string>& vmr_texts() {
    static std::vector<std::string> t;
    static std::once_flag once;
    std::call_once(once, [] {
        auto e3 = [](double v) { char b[32]; snprintf(b, sizeof b, "%.3e", v); return std::string(b); };
        const double mult = std::pow(10.0, 1.0 / 18);
        double v = go_pow10(-9);
        t.push_back("0..." + e3(v));
        for (int i = 0; i < VL_VMRANGES - 2; i++) {
            const std::string start = e3(v);
            v *= mult;
            t.push_back(start + "..." + e3(v));
        }
        t.push_back(e3(go_pow10(18)) + "...+Inf");
    });
    return t;
}

}  // namespace

extern "C" {

// ---- hit materialisation ----------------------------------------------------------------------------------------------------------------------
// hits of the last scan on the device: ctx->hits (row inside its block), ctx->hit_block, ctx->hit_offs (first hit of every block); returns their number
static uint64_t build_hit_list(vlscan_ctx* ctx, uint64_t* out_hit_offsets) {
    if (!ctx->has_result) throw BadInput("no scan result on this ctx");
    VL_CUDA(cudaSetDevice(ctx->device));
    const vlscan_batch* b = ctx->last_batch;
    BatchView B = b->view();
    ctx->hit_offs.ensure((b->nblocks + 1) * 8);
    uint64_t* offs = ctx->hit_offs.as<uint64_t>();
    k_scan_cta<uint32_t><<<1, 1024, 0, ctx->stream>>>(ctx->counts.as<uint32_t>(), (uint32_t)b->nblocks, offs, offs + b->nblocks); launch_check(ctx);
    uint64_t total = 0;
    VL_CUDA(cudaMemcpyAsync(&total, offs + b->nblocks, 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_hit_offsets) VL_CUDA(cudaMemcpyAsync(out_hit_offsets, offs, (b->nblocks + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VL_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->hits.ensure(std::max<uint64_t>(total, 4) * 4); ctx->hit_block.ensure(std::max<uint64_t>(total, 4) * 4);
    if (b->nblocks && total) {
        k_hits_compact<<<cdiv((uint64_t)b->nblocks * 32, 256), 256, 0, ctx->stream>>>(B, ctx->regs[0].as<uint64_t>(), offs, ctx->hits.as<uint32_t>(), ctx->hit_block.as<uint32_t>(), total);
        launch_check(ctx);
    }
    ctx->gstat.ensure(ST_COUNT * 8);
    VL_CUDA(cudaMemsetAsync(ctx->gstat.p, 0, ST_COUNT * 8, ctx->stream));
    return total;
}

int vlscan_fetch_hits(vlscan_ctx* ctx, uint32_t* out_hit_rows, uint64_t cap, uint64_t* out_hit_offsets) {
    return guarded(ctx, [&] {
        if (!ctx->has_result) throw BadInput("no scan result to fetch on this ctx");
        const uint64_t total = build_hit_list(ctx, out_hit_offsets);
        if (total > cap) throw BadInput("hit buffer too small");
        if (total) VL_CUDA(cudaMemcpyAsync(out_hit_rows, ctx->hits.p, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
    });
}

static void check_gather_errors(vlscan_ctx* ctx) {
    unsigned long long h[ST_COUNT];
    VL_CUDA(cudaMemcpyAsync(h, ctx->gstat.p, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    VL_CUDA(cudaStreamSynchronize(ctx->stream));
    static const char* const msg[] = {"", "cannot unmarshal strings: row lengths do not add up to the data length", "too big index for dict value", "unexpected length for binary representation of a number", "", "",
                                      "the timestamps of a block with selected rows were not handed over", "cannot unmarshal timestamps",
                                      "the values of a cell with selected rows are not on the device (vlscan_stage_selected stages them)",
                                      "the decoded timestamps of a block contradict the minimum / maximum of its header"};
    if (h[ST_ERROR]) throw BadInput(msg[std::min<unsigned long long>(h[ST_ERROR], 9)]);
}
// the timestamps of the blocks in `list` (wc[WC_ROW] of them) decoded into ctx->ts_vals, at each block's first word * 64; errors go to gstat
static const unsigned long long* decode_listed_timestamps(vlscan_ctx* ctx, const BatchView& B, const uint32_t* list, const uint32_t* wc) {
    ctx->ts_vals.ensure(B.nwords * 64 * 8);
    k_ts_decode_list<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(B, list, wc, ctx->ts_vals.as<unsigned long long>(), ctx->gstat.as<unsigned long long>()); launch_check(ctx);
    return ctx->ts_vals.as<unsigned long long>();
}

int vlscan_gather_timestamps(vlscan_ctx* ctx, int64_t* out_timestamps, uint64_t cap, uint64_t* out_hit_offsets) {
    return guarded(ctx, [&] {
        const uint64_t n = build_hit_list(ctx, out_hit_offsets);
        if (n > cap) throw BadInput("timestamps buffer too small");
        if (!n) return;
        const vlscan_batch* b = ctx->last_batch;
        BatchView B = b->view();
        uint32_t* wc = ctx->work_count.as<uint32_t>(); uint32_t* row_blocks = ctx->row_blocks.as<uint32_t>();
        VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
        k_hit_blocks_list<<<cdiv(b->nblocks, 256), 256, 0, ctx->stream>>>(B, ctx->counts.as<uint32_t>(), -1, 1, row_blocks, wc); launch_check(ctx);
        const unsigned long long* ts_vals = decode_listed_timestamps(ctx, B, row_blocks, wc);
        ctx->gout.ensure(n * 8);
        k_gather_ts<<<cdiv(n, 256), 256, 0, ctx->stream>>>(B, ctx->hits.as<uint32_t>(), ctx->hit_block.as<uint32_t>(), n, ts_vals, ctx->gout.as<long long>()); launch_check(ctx);
        check_gather_errors(ctx);
        VL_CUDA(cudaMemcpy(out_timestamps, ctx->gout.p, n * 8, cudaMemcpyDeviceToHost));
    });
}

// row offsets of the blocks with hits whose cell in column `slot` has per-row lens items (cell_needs_offsets; kept from the scan where it already
// computed them); `with_rows` (default: the scan's counts) != 0 marks the blocks whose offsets are needed.  On a kept batch every such block
// must have the field's values on the device: the call fails naming the field otherwise (the kernels would report ERR_VALUES_ABSENT, which
// cannot say which field it was).
static const uint32_t* hit_row_offsets(vlscan_ctx* ctx, int slot, const std::string& name, const uint32_t* with_rows = nullptr) {
    if (slot < 0) return nullptr;
    BatchView B = ctx->last_batch->view();
    if (ctx->last_batch->split_hdr && B.nblocks) {   // only a bloom-first / kept staging leaves values on the host
        ctx->unstaged.ensure(16);
        VL_CUDA(cudaMemsetAsync(ctx->unstaged.p, 0, 8, ctx->stream));
        k_unstaged_count<<<cdiv(B.nblocks, 256), 256, 0, ctx->stream>>>(B, with_rows ? with_rows : ctx->counts.as<uint32_t>(), slot, ctx->unstaged.as<unsigned long long>());
        launch_check(ctx);
        unsigned long long n = 0;
        VL_CUDA(cudaMemcpyAsync(&n, ctx->unstaged.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
        if (n) throw BadInput("field `" + name + "`: its values are not on the device in " + std::to_string(n) + " block(s) with selected rows (stage them with vlscan_stage_selected)");
    }
    uint32_t* wc = ctx->work_count.as<uint32_t>();
    VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
    k_hit_blocks_list<<<cdiv(B.nblocks, 256), 256, 0, ctx->stream>>>(B, with_rows ? with_rows : ctx->counts.as<uint32_t>(), slot, 0, ctx->lens_blocks.as<uint32_t>(), wc); launch_check(ctx);
    return row_offsets(ctx, B, slot, ctx->lens_blocks.as<uint32_t>(), wc, ctx->gstat.as<unsigned long long>(), WC_LENS);
}
// exclusive scan of the n lengths into offs[0 .. n], offs[n] = the total: tile sums, their scan by one CTA, per-tile prefixes
static void exclusive_scan(vlscan_ctx* ctx, const uint32_t* lens, uint64_t n, uint64_t* offs) {
    const uint64_t ntiles = cdiv(n, VL_SCAN_TILE);
    ctx->gtiles.ensure((ntiles + 1) * 8);
    k_scan_tiles<<<(unsigned)ntiles, 256, 0, ctx->stream>>>(lens, n, ctx->gtiles.as<unsigned long long>(), nullptr, 0); launch_check(ctx);
    k_scan_cta<uint64_t><<<1, 1024, 0, ctx->stream>>>(ctx->gtiles.as<uint64_t>(), (uint32_t)ntiles, ctx->gtiles.as<uint64_t>(), offs + n); launch_check(ctx);
    k_scan_tiles<<<(unsigned)ntiles, 256, 0, ctx->stream>>>(lens, n, ctx->gtiles.as<unsigned long long>(), (unsigned long long*)offs, 1); launch_check(ctx);
}
// texts of column `slot` in the n rows (rows[i], blocks[i]): their lengths and exclusive offsets go to ctx->glens / ctx->goffs (goffs[n] = the
// total, also returned; synchronises), then text_bytes writes the bytes to ctx->gout
// `key` (vlscan_hits_stats, a bucketed by-field): the texts come from k_hits_key_texts instead of k_gather_values
struct HitsKey { HitsQuery q; HitsView V; uint32_t f; };
static uint64_t text_offsets(vlscan_ctx* ctx, int slot, const uint32_t* ro, const uint32_t* rows, const uint32_t* blocks, uint64_t n, const HitsKey* key = nullptr) {
    BatchView B = ctx->last_batch->view();
    ctx->glens.ensure(n * 4); ctx->goffs.ensure((n + 1) * 8);
    if (key) k_hits_key_texts<<<cdiv(n, 128), 128, 0, ctx->stream>>>(B, key->q, key->V, key->f, rows, blocks, n, 0, ctx->glens.as<uint32_t>(), nullptr, nullptr, ctx->gstat.as<unsigned long long>());
    else k_gather_values<<<cdiv(n, 128), 128, 0, ctx->stream>>>(B, slot, rows, blocks, n, ro, 0, ctx->glens.as<uint32_t>(), nullptr, nullptr, ctx->gstat.as<unsigned long long>());
    launch_check(ctx);
    exclusive_scan(ctx, ctx->glens.as<uint32_t>(), n, ctx->goffs.as<uint64_t>());
    uint64_t total = 0;
    VL_CUDA(cudaMemcpyAsync(&total, ctx->goffs.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
    check_gather_errors(ctx);
    return total;
}
static void text_bytes(vlscan_ctx* ctx, int slot, const uint32_t* ro, const uint32_t* rows, const uint32_t* blocks, uint64_t n, uint64_t total, const HitsKey* key = nullptr) {
    ctx->gout.ensure(std::max<uint64_t>(total, 16));
    if (key) k_hits_key_texts<<<cdiv(n, 128), 128, 0, ctx->stream>>>(ctx->last_batch->view(), key->q, key->V, key->f, rows, blocks, n, 1, nullptr, ctx->goffs.as<uint64_t>(), ctx->gout.as<uint8_t>(),
                                                                     ctx->gstat.as<unsigned long long>());
    else k_gather_values<<<cdiv(n, 128), 128, 0, ctx->stream>>>(ctx->last_batch->view(), slot, rows, blocks, n, ro, 1, nullptr, ctx->goffs.as<uint64_t>(), ctx->gout.as<uint8_t>(),
                                                                ctx->gstat.as<unsigned long long>());
    launch_check(ctx);
}
// the texts of column `slot` in the n rows (rows[i], blocks[i]) on the host: text i is bytes[offs[i] .. offs[i + 1])
static void host_texts(vlscan_ctx* ctx, int slot, const uint32_t* ro, const uint32_t* rows, const uint32_t* blocks, uint64_t n, std::vector<uint64_t>& offs,
                       std::vector<uint8_t>& bytes, const HitsKey* key = nullptr) {
    const uint64_t total = text_offsets(ctx, slot, ro, rows, blocks, n, key);
    offs.resize(n + 1); bytes.resize(total);
    text_bytes(ctx, slot, ro, rows, blocks, n, total, key);
    VL_CUDA(cudaMemcpyAsync(offs.data(), ctx->goffs.p, (n + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (total) VL_CUDA(cudaMemcpyAsync(bytes.data(), ctx->gout.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    check_gather_errors(ctx);   // synchronises
}
// rows x fields output: row i is row order[i] of the per-field texts (host_texts); the text of field f in row i ends at out_offsets[i * nf + f + 1]
static void pack_texts(const std::vector<uint64_t>& order, const std::vector<std::vector<uint64_t>>& toffs, const std::vector<std::vector<uint8_t>>& tbytes,
                       uint8_t* out_bytes, uint64_t* out_offsets) {
    const size_t nf = toffs.size();
    uint64_t o = 0;
    for (uint64_t i = 0; i < order.size(); i++)
        for (size_t f = 0; f < nf; f++) {
            const uint64_t a = toffs[f][order[i]], len = toffs[f][order[i] + 1] - a;
            if (len) memcpy(out_bytes + o, tbytes[f].data() + a, len);
            o += len;
            out_offsets[i * nf + f + 1] = o;
        }
}

int vlscan_gather_values(vlscan_ctx* ctx, const char* field, size_t field_len, uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_value_offsets, uint64_t cap_values,
                         uint64_t* out_total_bytes, uint64_t* out_hit_offsets) {
    if (out_total_bytes) *out_total_bytes = 0;
    return guarded(ctx, [&] {
        const uint64_t n = build_hit_list(ctx, out_hit_offsets);
        if (n > cap_values) throw BadInput("value offsets buffer too small");
        if (out_value_offsets) out_value_offsets[0] = 0;
        if (!n) return;
        std::string name(field, field_len); if (name.empty()) name = "_msg";   // getCanonicalColumnName
        const int slot = ctx->last_batch->field_slot(name);
        const uint32_t* ro = hit_row_offsets(ctx, slot, name);
        const uint32_t* rows = ctx->hits.as<uint32_t>(); const uint32_t* blocks = ctx->hit_block.as<uint32_t>();
        const uint64_t total = text_offsets(ctx, slot, ro, rows, blocks, n);
        if (out_total_bytes) *out_total_bytes = total;
        if (total > cap_bytes) throw BadInput("values buffer too small (the needed size is reported)");
        text_bytes(ctx, slot, ro, rows, blocks, n, total);
        if (out_value_offsets) VL_CUDA(cudaMemcpyAsync(out_value_offsets, ctx->goffs.p, (n + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (total) VL_CUDA(cudaMemcpyAsync(out_bytes, ctx->gout.p, total, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
    });
}

static_assert(VLSCAN_HITS_MAX_BY == VL_HITS_MAX_BY, "the ABI's and the kernels' by-field limits differ");
int64_t vlscan_truncate_timestamp(int64_t ts, int64_t step, int64_t offset, uint32_t calendar) { return vl::truncate_timestamp(ts, step, offset, calendar); }
int vlscan_bucket_text(const vlscan_by_bucket* b, const void* s, size_t len, char* out, size_t cap) {
    BucketSpec bk;
    if (!b || len > 0xFFFFFFFFu || !bucket_spec(*b, &bk).empty()) return -2;
    uint8_t buf[VL_FMT_F64_MAX];
    const uint8_t* p;
    const uint32_t n = bucket_text(bk, (const uint8_t*)s, (uint32_t)len, buf, &p);
    if (n > cap) return -1;
    if (n) memcpy(out, p, n);
    return (int)n;
}

static_assert(VLSCAN_STATS_MAX_VALUES == VL_STATS_MAX_VALUES, "the ABI's and the kernels' value-field limits differ");
// the finished sum of one (group, value field) from its digit sums, frame and flags (k_stats_values): NaN without numbers, as newStatsProcessor
// starts it; the exact digit total rounded once otherwise; -0 when every term was -0 (no flag 8), as the reference's float adds give it
static double stats_sum(const int64_t d[3], int frame, unsigned flags, uint64_t count) {
    if (!count) return std::numeric_limits<double>::quiet_NaN();
    if ((flags & 4) || (flags & 3) == 3) return std::numeric_limits<double>::quiet_NaN();
    if (flags & 1) return std::numeric_limits<double>::infinity();
    if (flags & 2) return -std::numeric_limits<double>::infinity();
    if (!frame) return (flags & 8) ? 0.0 : -0.0;
    const __int128 t = ((__int128)d[0] << 62) + ((__int128)d[1] << 31) + (__int128)d[2];
    return std::ldexp((double)t, frame - VL_STATS_FRAME_BIAS - 92);
}

// The value aggregation over the groups of hits_groups (vlscan_hits_sums, vlscan_hits_vmranges).  run: after the groups are emitted, on the
// device state they leave (copies its results to the host; may set info[4..]).  write: the results in the caller's buffers in group order,
// after the groups' capacities passed and before the groups are written (a capacity of its own that is too small fails the call).
struct GroupPass {
    vlscan_ctx* ctx; const BatchView& B; const StatsQuery& sq; const HitsView& V; const HitsTable& T; uint64_t n, G; unsigned grid; uint64_t* info;
};
struct ValueAgg {
    const char* prefix_example;   // the pipe a prefix value field would be, for the error
    std::function<void(Carve&, uint64_t G)> take;   // optional: device arrays laid out after the groups' (ctx->hgrp)
    std::function<void(const GroupPass&)> run;
    std::function<void(const std::vector<uint64_t>& order)> write;
};

// vlscan_hits_stats (agg NULL), vlscan_hits_sums and vlscan_hits_vmranges: one grouping, then the value aggregation over the same groups
static int hits_groups(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, const char* const* value_names, const size_t* value_name_lens, uint32_t nv, const char* what,
                       int64_t* out_buckets, uint64_t* out_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets,
                       uint64_t* out_info, size_t ninfo, const ValueAgg* agg) {
    uint64_t info[6] = {0, 0, 0, 0, 0, 0};   // groups, key bytes, selected rows, blocks whose timestamps were decoded, then the aggregation's
    const int rc = guarded(ctx, [&] {
        if (!q) throw BadInput("no hits query");
        if (q->calendar > VLSCAN_BUCKET_YEAR) throw BadInput("unknown calendar bucket kind");
        if (q->nby > VLSCAN_HITS_MAX_BY) throw BadInput("too many by-fields for the hits aggregation (at most VLSCAN_HITS_MAX_BY = 4)");
        const std::vector<std::string> names = canonical_names(q->by_names, q->by_name_lens, q->nby, what);
        for (const std::string& n : names)
            if (n == "_time") throw BadInput("`_time` cannot be a by-field of the hits aggregation: it is the bucket");
        if (nv > VLSCAN_STATS_MAX_VALUES) throw BadInput(std::string("too many value fields for ") + what + " (at most VLSCAN_STATS_MAX_VALUES = 4)");
        const std::vector<std::string> vnames = canonical_names(value_names, value_name_lens, nv, what);
        for (const std::string& v : vnames)
            if (v.back() == '*') throw BadInput("value field `" + v + "`: a prefix filter such as " + agg->prefix_example + " is not supported by " + what);
        if (!ctx) throw BadInput(std::string(what) + " needs a vlscan_ctx on a CUDA device (there is no CPU fallback)");
        const uint64_t n = build_hit_list(ctx, nullptr);
        if (n >= 0xFFFFFFFFull) throw BadInput("more than 2^32 - 2 selected rows in one batch");
        info[2] = n;
        if (out_key_offsets) out_key_offsets[0] = 0;
        if (!n) return;
        const vlscan_batch* b = ctx->last_batch;
        BatchView B = b->view();
        HitsQuery hq;
        memset(&hq, 0, sizeof hq);
        hq.step = q->step; hq.offset = q->offset; hq.calendar = q->calendar; hq.nby = q->nby;
        for (uint32_t f = 0; f < q->nby; f++) { hq.slot[f] = b->field_slot(names[f]); hq.row_off8[f] = hit_row_offsets(ctx, hq.slot[f], names[f]); }
        BucketSpec specs[VL_HITS_MAX_BY];
        for (uint32_t f = 0; f < q->nby && by_buckets; f++)
            if (by_buckets[f].enabled) {
                const std::string why = bucket_spec(by_buckets[f], &specs[f]);
                if (!why.empty()) throw BadInput("by-field `" + names[f] + "`: bucket rejected: " + why);
                hq.bucketed |= 1u << f;
            }
        StatsQuery sq;
        memset(&sq, 0, sizeof sq);
        sq.nv = nv;
        for (uint32_t f = 0; f < nv; f++) {   // `_time` is the bucket; its value adds nothing (isTime in sumValues / getFloatValueAtRow)
            sq.slot[f] = vnames[f] == "_time" ? -1 : b->field_slot(vnames[f]);
            sq.row_off8[f] = hit_row_offsets(ctx, sq.slot[f], vnames[f]);
        }
        // buckets of the blocks; timestamps decoded only where a block spans several buckets
        unsigned long long* gstat = ctx->gstat.as<unsigned long long>();
        uint32_t* wc = ctx->work_count.as<uint32_t>(); uint32_t* row_blocks = ctx->row_blocks.as<uint32_t>();
        long long* blk_bucket; uint8_t* blk_multi; uint8_t* by_fast; unsigned long long* by_lo; BucketSpec* d_specs; KeyTexts* d_keys;
        Carve().take(blk_bucket, b->nblocks).take(blk_multi, b->nblocks).take(by_fast, b->nblocks * q->nby).take(by_lo, b->nblocks * q->nby).take(d_specs, VL_HITS_MAX_BY)
            .take(d_keys, VL_HITS_MAX_BY).place(ctx->hblk);
        if (hq.bucketed) VL_CUDA(cudaMemcpyAsync(d_specs, specs, sizeof specs, cudaMemcpyHostToDevice, ctx->stream));
        hq.buckets = d_specs;
        VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
        k_hits_classify<<<cdiv(b->nblocks, 256), 256, 0, ctx->stream>>>(B, ctx->counts.as<uint32_t>(), hq, blk_bucket, blk_multi, by_fast, by_lo, row_blocks, wc, gstat);
        launch_check(ctx);
        const unsigned long long* ts_vals = decode_listed_timestamps(ctx, B, row_blocks, wc);
        uint32_t decoded = 0;
        VL_CUDA(cudaMemcpyAsync(&decoded, wc + WC_ROW, 4, cudaMemcpyDeviceToHost, ctx->stream));
        HitsView V{ctx->hits.as<uint32_t>(), ctx->hit_block.as<uint32_t>(), blk_bucket, blk_multi, ts_vals, by_fast, by_lo, d_keys};
        KeyTexts keys[VL_HITS_MAX_BY] = {};
        // the bucketed texts of every hit, kept in ctx->ftxt for the grouping pass
        if (ctx->ftxt.size() < q->nby) ctx->ftxt.resize(q->nby);
        for (uint32_t f = 0; f < q->nby; f++) {
            if (!(hq.bucketed >> f & 1)) continue;
            const HitsKey key{hq, V, f};
            const uint64_t total = text_offsets(ctx, hq.slot[f], hq.row_off8[f], V.hits, V.hit_block, n, &key);
            text_bytes(ctx, hq.slot[f], hq.row_off8[f], V.hits, V.hit_block, n, total, &key);
            DevBuf& T = ctx->ftxt[f];
            T.ensure((n + 1) * 8 + total + 16);
            VL_CUDA(cudaMemcpyAsync(T.p, ctx->goffs.p, (n + 1) * 8, cudaMemcpyDeviceToDevice, ctx->stream));
            if (total) VL_CUDA(cudaMemcpyAsync(T.as<uint8_t>() + (n + 1) * 8, ctx->gout.p, total, cudaMemcpyDeviceToDevice, ctx->stream));
            keys[f] = KeyTexts{T.as<uint64_t>(), T.as<uint8_t>() + (n + 1) * 8};
        }
        if (hq.bucketed) VL_CUDA(cudaMemcpyAsync(d_keys, keys, sizeof keys, cudaMemcpyHostToDevice, ctx->stream));
        // the group table: starts small, grows by 8x while a pass overflows; at 2 x the hit count it cannot overflow
        uint64_t max_cap = 1024; while (max_cap < 2 * n) max_cap <<= 1;
        uint64_t cap = std::min<uint64_t>(max_cap, 1 << 14);
        HitsTable T;
        T.hit_slot = nullptr; T.slot_group = nullptr;
        if (nv) { ctx->hslot.ensure(n * 4); T.hit_slot = ctx->hslot.as<uint32_t>(); }
        unsigned long long state[3];
        const unsigned grid = (unsigned)std::min<uint64_t>(b->nblocks, (uint64_t)ctx->sm_count * 8);
        for (;;) {
            const size_t bytes = Carve().take(T.tags, cap).take(T.cnt, cap).take(T.state, 4).place(ctx->htab);
            T.mask = cap - 1; T.limit = cap == max_cap ? cap : cap / 2;
            VL_CUDA(cudaMemsetAsync(T.tags, 0, bytes, ctx->stream));
            if (nv) k_hits_group<true><<<grid, 256, 0, ctx->stream>>>(B, hq, V, T, ctx->counts.as<uint32_t>(), ctx->hit_offs.as<uint64_t>(), gstat);
            else k_hits_group<false><<<grid, 256, 0, ctx->stream>>>(B, hq, V, T, ctx->counts.as<uint32_t>(), ctx->hit_offs.as<uint64_t>(), gstat);
            launch_check(ctx);
            VL_CUDA(cudaMemcpyAsync(state, T.state, sizeof state, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaStreamSynchronize(ctx->stream));
            if (!state[1]) break;
            if (cap == max_cap) throw BadInput("hits aggregation: group table overflow");
            cap = std::min(cap * 8, max_cap);
        }
        check_gather_errors(ctx);
        const uint64_t G = state[0];
        info[0] = G; info[3] = decoded;
        // the groups, then the texts of their representatives only
        long long* buckets; unsigned long long* counts; uint32_t* rep_rows; uint32_t* rep_blocks;
        Carve cv;
        cv.take(buckets, G).take(counts, G).take(rep_rows, G).take(rep_blocks, G);
        if (nv) cv.take(T.slot_group, cap);
        if (agg && agg->take) agg->take(cv, G);
        cv.place(ctx->hgrp);
        k_hits_emit<<<cdiv(cap, 256), 256, 0, ctx->stream>>>(B, hq, V, T, rep_rows, rep_blocks, buckets, counts); launch_check(ctx);
        if (agg) agg->run(GroupPass{ctx, B, sq, V, T, n, G, grid, info});
        std::vector<int64_t> hb(G); std::vector<uint64_t> hc(G);
        VL_CUDA(cudaMemcpyAsync(hb.data(), buckets, G * 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaMemcpyAsync(hc.data(), counts, G * 8, cudaMemcpyDeviceToHost, ctx->stream));
        std::vector<std::vector<uint64_t>> toffs(q->nby); std::vector<std::vector<uint8_t>> tbytes(q->nby);
        uint64_t key_bytes = 0;
        for (uint32_t f = 0; f < q->nby; f++) {
            const HitsKey key{hq, V, f};
            host_texts(ctx, hq.slot[f], hq.row_off8[f], rep_rows, rep_blocks, G, toffs[f], tbytes[f], (hq.bucketed >> f & 1) ? &key : nullptr);
            key_bytes += tbytes[f].size();
        }
        VL_CUDA(cudaStreamSynchronize(ctx->stream));
        info[1] = key_bytes;
        if (G > cap_groups) throw BadInput("hits groups buffer too small (the needed size is reported)");
        if (key_bytes > cap_key_bytes) throw BadInput("hits key bytes buffer too small (the needed size is reported)");
        if (!out_buckets || !out_counts || (q->nby && (!out_key_offsets || (key_bytes && !out_key_bytes)))) throw BadInput("hits output buffer missing");
        // sorted by bucket, then by the key texts bytewise
        std::vector<uint64_t> order(G);
        for (uint64_t g = 0; g < G; g++) order[g] = g;
        auto text = [&](uint32_t f, uint64_t g) { return std::string_view((const char*)tbytes[f].data() + toffs[f][g], toffs[f][g + 1] - toffs[f][g]); };
        std::sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) {
            if (hb[x] != hb[y]) return hb[x] < hb[y];
            for (uint32_t f = 0; f < q->nby; f++) { const int c = text(f, x).compare(text(f, y)); if (c) return c < 0; }
            return false;
        });
        if (agg) agg->write(order);
        for (uint64_t i = 0; i < G; i++) { out_buckets[i] = hb[order[i]]; out_counts[i] = hc[order[i]]; }
        pack_texts(order, toffs, tbytes, out_key_bytes, out_key_offsets);
    });
    if (out_info) memcpy(out_info, info, ninfo * sizeof(uint64_t));
    return rc;
}

int vlscan_hits_stats(vlscan_ctx* ctx, const vlscan_hits_query* q, int64_t* out_buckets, uint64_t* out_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes,
                      uint64_t* out_key_offsets, uint64_t out_info[4]) {
    return vlscan_hits_stats_bucketed(ctx, q, nullptr, out_buckets, out_counts, cap_groups, out_key_bytes, cap_key_bytes, out_key_offsets, out_info);
}
int vlscan_hits_stats_bucketed(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, int64_t* out_buckets, uint64_t* out_counts,
                               uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets, uint64_t out_info[4]) {
    return hits_groups(ctx, q, by_buckets, nullptr, nullptr, 0, "vlscan_hits_stats", out_buckets, out_counts, cap_groups, out_key_bytes, cap_key_bytes, out_key_offsets,
                       out_info, 4, nullptr);
}

int vlscan_hits_sums(vlscan_ctx* ctx, const vlscan_hits_query* q, const char* const* value_names, const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets,
                     uint64_t* out_counts, double* out_sums, uint64_t* out_value_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes,
                     uint64_t* out_key_offsets, uint64_t out_info[4]) {
    return vlscan_hits_sums_bucketed(ctx, q, nullptr, value_names, value_name_lens, nvalues, out_buckets, out_counts, out_sums, out_value_counts, cap_groups, out_key_bytes,
                                     cap_key_bytes, out_key_offsets, out_info);
}
int vlscan_hits_sums_bucketed(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, const char* const* value_names,
                              const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets, uint64_t* out_counts, double* out_sums,
                              uint64_t* out_value_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets,
                              uint64_t out_info[4]) {
    if (nvalues == 0) {   // a query without value fields is vlscan_hits_stats
        if (out_info) memset(out_info, 0, 4 * sizeof(uint64_t));
        return guarded(ctx, [] { throw BadInput("vlscan_hits_sums: no value fields (vlscan_hits_stats counts without them)"); });
    }
    const uint32_t nv = nvalues;
    std::vector<int64_t> hd; std::vector<uint64_t> hn; std::vector<int> hf; std::vector<unsigned> hfl;
    ValueAgg agg;
    agg.prefix_example = "sum(foo*)";
    StatsAcc A;
    agg.take = [&](Carve& cv, uint64_t G) { cv.take(A.digits, 3 * G * nv).take(A.count, G * nv).take(A.frame, G * nv).take(A.flags, G * nv); };
    agg.run = [&](const GroupPass& P) {   // the value sums: pass 0 counts and frames, pass 1 digits (k_stats_values)
        vlscan_ctx* c = P.ctx;
        const uint64_t G = P.G;
        VL_CUDA(cudaMemsetAsync(A.digits, 0, (uint8_t*)(A.flags + G * nv) - (uint8_t*)A.digits, c->stream));
        unsigned long long* gstat = c->gstat.as<unsigned long long>();
        k_stats_values<0><<<P.grid, 256, 0, c->stream>>>(P.B, P.sq, P.V, P.T.hit_slot, P.T.slot_group, A, c->counts.as<uint32_t>(), c->hit_offs.as<uint64_t>(), gstat); launch_check(c);
        k_stats_values<1><<<P.grid, 256, 0, c->stream>>>(P.B, P.sq, P.V, P.T.hit_slot, P.T.slot_group, A, c->counts.as<uint32_t>(), c->hit_offs.as<uint64_t>(), gstat); launch_check(c);
        hd.resize(3 * G * nv); hn.resize(G * nv); hf.resize(G * nv); hfl.resize(G * nv);
        VL_CUDA(cudaMemcpyAsync(hd.data(), A.digits, hd.size() * 8, cudaMemcpyDeviceToHost, c->stream));
        VL_CUDA(cudaMemcpyAsync(hn.data(), A.count, hn.size() * 8, cudaMemcpyDeviceToHost, c->stream));
        VL_CUDA(cudaMemcpyAsync(hf.data(), A.frame, hf.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        VL_CUDA(cudaMemcpyAsync(hfl.data(), A.flags, hfl.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        check_gather_errors(c);
    };
    agg.write = [&](const std::vector<uint64_t>& order) {
        if (!out_sums || !out_value_counts) throw BadInput("hits output buffer missing");
        for (uint64_t i = 0; i < order.size(); i++)
            for (uint32_t f = 0; f < nv; f++) {
                const uint64_t k = order[i] * nv + f;
                out_sums[i * nv + f] = stats_sum(&hd[3 * k], hf[k], hfl[k], hn[k]);
                out_value_counts[i * nv + f] = hn[k];
            }
    };
    return hits_groups(ctx, q, by_buckets, value_names, value_name_lens, nvalues, "vlscan_hits_sums", out_buckets, out_counts, cap_groups, out_key_bytes, cap_key_bytes,
                       out_key_offsets, out_info, 4, &agg);
}

int vlscan_hits_vmranges(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, const char* const* value_names,
                         const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets, uint64_t* out_counts, uint64_t cap_groups,
                         uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets, uint64_t* out_entry_offsets,
                         uint16_t* out_entry_ranges, uint64_t* out_entry_hits, uint64_t cap_entries, uint64_t out_info[6]) {
    if (nvalues == 0) {
        if (out_info) memset(out_info, 0, 6 * sizeof(uint64_t));
        return guarded(ctx, [] { throw BadInput("vlscan_hits_vmranges: no value fields (histogram takes one field)"); });
    }
    const uint32_t nv = nvalues;
    std::vector<unsigned long long> ek, ec;                   // the table's entries: key (g * nv + f) * VL_VMRANGES + index, hits
    std::vector<std::pair<uint16_t, uint64_t>> entries;       // (index, hits) by (device group, value field), then index
    std::vector<uint64_t> first;                              // the first entry of every (device group, value field)
    ValueAgg agg;
    agg.prefix_example = "histogram(foo*)";
    agg.run = [&](const GroupPass& P) {
        vlscan_ctx* c = P.ctx;
        const std::vector<double>& bounds = vmr_bounds();
        // the vmrange table: starts small, grows by 8x while a pass overflows; at 2 x (hits x value fields) it cannot overflow
        uint64_t max_cap = 1024; while (max_cap < 2 * P.n * nv) max_cap <<= 1;
        uint64_t cap = std::min<uint64_t>(max_cap, 1 << 14);
        VmrTable M;
        double* d_bounds; unsigned long long* out_keys; unsigned long long* out_cnt;
        unsigned long long state[4];
        for (;;) {
            Carve cv;
            cv.take(d_bounds, VL_VMR_BOUNDS).take(M.keys, cap).take(M.cnt, cap).take(M.state, 4).take(out_keys, cap).take(out_cnt, cap).place(c->vagg);
            M.mask = cap - 1; M.limit = cap == max_cap ? cap : cap / 2;
            VL_CUDA(cudaMemcpyAsync(d_bounds, bounds.data(), VL_VMR_BOUNDS * 8, cudaMemcpyHostToDevice, c->stream));
            VL_CUDA(cudaMemsetAsync(M.keys, 0, (uint8_t*)(M.state + 4) - (uint8_t*)M.keys, c->stream));
            k_stats_vmranges<<<P.grid, 256, 0, c->stream>>>(P.B, P.sq, P.V, P.T.hit_slot, P.T.slot_group, d_bounds, M, c->counts.as<uint32_t>(), c->hit_offs.as<uint64_t>(),
                                                             c->gstat.as<unsigned long long>());
            launch_check(c);
            VL_CUDA(cudaMemcpyAsync(state, M.state, sizeof state, cudaMemcpyDeviceToHost, c->stream));
            VL_CUDA(cudaStreamSynchronize(c->stream));
            if (!state[1]) break;
            if (cap == max_cap) throw BadInput("vlscan_hits_vmranges: vmrange table overflow");
            cap = std::min(cap * 8, max_cap);
        }
        const uint64_t E = state[0];
        k_vmr_compact<<<cdiv(cap, 256), 256, 0, c->stream>>>(M, out_keys, out_cnt); launch_check(c);
        ek.resize(E); ec.resize(E);
        if (E) {
            VL_CUDA(cudaMemcpyAsync(ek.data(), out_keys, E * 8, cudaMemcpyDeviceToHost, c->stream));
            VL_CUDA(cudaMemcpyAsync(ec.data(), out_cnt, E * 8, cudaMemcpyDeviceToHost, c->stream));
        }
        check_gather_errors(c);   // synchronises
        P.info[4] = E; P.info[5] = state[3];
        // by (device group, value field) with a counting pass, then by index inside each of them (at most VL_VMRANGES entries)
        first.assign(P.G * nv + 1, 0);
        for (uint64_t e = 0; e < E; e++) first[ek[e] / VL_VMRANGES + 1]++;
        for (size_t k = 1; k < first.size(); k++) first[k] += first[k - 1];
        std::vector<uint64_t> at(first.begin(), first.end() - 1);
        entries.resize(E);
        for (uint64_t e = 0; e < E; e++) entries[at[ek[e] / VL_VMRANGES]++] = {(uint16_t)(ek[e] % VL_VMRANGES), ec[e]};
        for (size_t k = 0; k + 1 < first.size(); k++) std::sort(entries.begin() + first[k], entries.begin() + first[k + 1]);
    };
    agg.write = [&](const std::vector<uint64_t>& order) {
        const uint64_t E = entries.size();
        if (E > cap_entries) throw BadInput("vmrange entries buffer too small (the needed size is reported)");
        if (!out_entry_offsets || (E && (!out_entry_ranges || !out_entry_hits))) throw BadInput("hits output buffer missing");
        uint64_t o = 0;
        out_entry_offsets[0] = 0;
        for (uint64_t i = 0; i < order.size(); i++)
            for (uint32_t f = 0; f < nv; f++) {
                const uint64_t k = order[i] * nv + f;
                for (uint64_t e = first[k]; e < first[k + 1]; e++, o++) { out_entry_ranges[o] = entries[e].first; out_entry_hits[o] = entries[e].second; }
                out_entry_offsets[i * nv + f + 1] = o;
            }
    };
    if (out_entry_offsets) out_entry_offsets[0] = 0;
    return hits_groups(ctx, q, by_buckets, value_names, value_name_lens, nvalues, "vlscan_hits_vmranges", out_buckets, out_counts, cap_groups, out_key_bytes,
                       cap_key_bytes, out_key_offsets, out_info, 6, &agg);
}
int vlscan_vmrange_index(double v) { return vmr_index_host(v); }
int vlscan_vmrange_text(uint32_t index, char* buf, size_t cap) {
    if (index >= VL_VMRANGES) return -2;
    const std::string& t = vmr_texts()[index];
    if (t.size() > cap) return -1;
    memcpy(buf, t.data(), t.size());
    return (int)t.size();
}

// the limit-th largest of the n int64 keys (weights: NULL = 1 each) into the radix state st (RS_COUNT words + VL_RADIX_PASSES histograms), on
// the stream, with no host round trip
static void radix_select(vlscan_ctx* ctx, const long long* keys, const uint32_t* weights, uint64_t n, uint64_t limit, unsigned long long* st) {
    VL_CUDA(cudaMemsetAsync(st, 0, (RS_COUNT + VL_RADIX_PASSES * 256) * 8, ctx->stream));
    const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(cdiv(n, 256), (uint64_t)ctx->sm_count * 8));
    for (int p = 0; p < VL_RADIX_PASSES; p++) {
        const int shift = 64 - 8 * (p + 1);
        unsigned long long* hist = st + RS_COUNT + p * 256;
        k_radix_hist<<<grid, 256, 0, ctx->stream>>>(keys, weights, n, st, shift, hist); launch_check(ctx);
        k_radix_pick<<<1, 32, 0, ctx->stream>>>(hist, shift, limit, st); launch_check(ctx);
    }
}

int vlscan_last_rows(vlscan_ctx* ctx, const vlscan_last_query* q, int64_t* out_timestamps, uint32_t* out_blocks, uint32_t* out_rows, uint64_t cap_rows,
                     uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_offsets, uint64_t out_info[4]) {
    uint64_t info[4] = {0, 0, 0, 0};   // rows returned, value bytes, selected rows, blocks whose timestamps were decoded
    const int rc = guarded(ctx, [&] {
        if (!q) throw BadInput("no last-rows query");
        if (q->limit == 0) throw BadInput("the limit of vlscan_last_rows must be at least 1");
        const std::vector<std::string> names = canonical_names(q->field_names, q->field_name_lens, q->nfields, "vlscan_last_rows");
        for (const std::string& n : names)
            if (n == "_time") throw BadInput("`_time` cannot be a field of vlscan_last_rows: it is returned in out_timestamps");
        if (!ctx) throw BadInput("vlscan_last_rows needs a vlscan_ctx on a CUDA device (there is no CPU fallback)");
        if (!ctx->has_result) throw BadInput("no scan result on this ctx");
        VL_CUDA(cudaSetDevice(ctx->device));
        const vlscan_batch* b = ctx->last_batch;
        BatchView B = b->view();
        const uint64_t nb = b->nblocks, limit = q->limit;
        const long long floor_ts = q->min_timestamp;
        const uint32_t* counts = ctx->counts.as<uint32_t>();
        ctx->gstat.ensure(ST_COUNT * 8);
        VL_CUDA(cudaMemsetAsync(ctx->gstat.p, 0, ST_COUNT * 8, ctx->stream));
        unsigned long long* gstat = ctx->gstat.as<unsigned long long>();
        long long* blk_key; uint64_t* cand_offs; uint32_t* blk_w; uint32_t* cand_rows; uint32_t* blk_mark; uint32_t* cand; uint32_t* decode;
        Carve().take(blk_key, nb).take(cand_offs, nb + 1).take(blk_w, nb).take(cand_rows, nb).take(blk_mark, nb).take(cand, nb).take(decode, nb).place(ctx->hblk);
        const size_t st_words = RS_COUNT + VL_RADIX_PASSES * 256;
        unsigned long long* st_blk; unsigned long long* st_row;
        Carve().take(st_blk, st_words).take(st_row, st_words).place(ctx->htab);
        ctx->hit_offs.ensure((nb + 1) * 8);
        uint64_t* hit_offs = ctx->hit_offs.as<uint64_t>();
        k_scan_cta<uint32_t><<<1, 1024, 0, ctx->stream>>>(counts, (uint32_t)nb, hit_offs, hit_offs + nb); launch_check(ctx);
        // (1) the block threshold T_lo, from the headers alone
        if (nb) { k_last_block_keys<<<cdiv(nb, 256), 256, 0, ctx->stream>>>(B, counts, floor_ts, blk_key, blk_w, gstat); launch_check(ctx); }
        radix_select(ctx, blk_key, blk_w, nb, limit, st_blk);
        // (2) the candidate blocks, the timestamps of those that are not flat, and the count of their selected rows >= T_lo
        uint32_t* wc = ctx->work_count.as<uint32_t>();
        VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
        VL_CUDA(cudaMemsetAsync(cand_rows, 0, nb * 4, ctx->stream));
        VL_CUDA(cudaMemsetAsync(blk_mark, 0, nb * 4, ctx->stream));
        if (nb) { k_last_candidates<<<cdiv(nb, 256), 256, 0, ctx->stream>>>(B, counts, floor_ts, st_blk, cand, decode, wc); launch_check(ctx); }
        const unsigned long long* ts_vals = decode_listed_timestamps(ctx, B, decode, wc);
        const unsigned row_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(nb, (uint64_t)ctx->sm_count * 8));
        k_last_rows<<<row_grid, 256, 0, ctx->stream>>>(B, ctx->regs[0].as<uint64_t>(), cand, wc, ts_vals, floor_ts, st_blk, 0, cand_rows, nullptr, nullptr, nullptr, nullptr, gstat);
        launch_check(ctx);
        k_scan_cta<uint32_t><<<1, 1024, 0, ctx->stream>>>(cand_rows, (uint32_t)nb, cand_offs, cand_offs + nb); launch_check(ctx);
        uint64_t selected = 0, M = 0; unsigned long long blk_short = 0; uint32_t decoded = 0;
        VL_CUDA(cudaMemcpyAsync(&selected, hit_offs + nb, 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaMemcpyAsync(&M, cand_offs + nb, 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaMemcpyAsync(&blk_short, st_blk + RS_SHORT, 8, cudaMemcpyDeviceToHost, ctx->stream));
        VL_CUDA(cudaMemcpyAsync(&decoded, wc + WC_ROW, 4, cudaMemcpyDeviceToHost, ctx->stream));
        check_gather_errors(ctx);   // synchronises
        info[2] = selected; info[3] = decoded;
        if (selected >= 0xFFFFFFFFull) throw BadInput("more than 2^32 - 2 selected rows in one batch");
        // the block weights promise `limit` rows >= T_lo; fewer means a block's timestamps disagree with its header
        if (!blk_short && M < limit) throw BadInput("the decoded timestamps of a block contradict the minimum / maximum of its header");
        const uint64_t n = std::min<uint64_t>(limit, M);
        std::vector<int64_t> hts(n); std::vector<uint32_t> hb(n), hr(n);
        uint32_t* sel_blk = nullptr; uint32_t* sel_row = nullptr;
        if (n) {
            // the candidates in (block, row) order, then (3) the exact top N: T_N, every row above it and the last ties
            long long* cts; uint32_t* cblk; uint32_t* crow;
            Carve().take(cts, M).take(cblk, M).take(crow, M).place(ctx->lcand);
            k_last_rows<<<row_grid, 256, 0, ctx->stream>>>(B, ctx->regs[0].as<uint64_t>(), cand, wc, ts_vals, floor_ts, st_blk, 1, nullptr, cand_offs, cts, cblk, crow, gstat);
            launch_check(ctx);
            radix_select(ctx, cts, nullptr, M, limit, st_row);
            ctx->glens.ensure(M * 4); ctx->goffs.ensure((M + 1) * 8);
            k_last_ties<<<cdiv(M, 256), 256, 0, ctx->stream>>>(cts, M, st_row, ctx->glens.as<uint32_t>()); launch_check(ctx);
            exclusive_scan(ctx, ctx->glens.as<uint32_t>(), M, ctx->goffs.as<uint64_t>());
            long long* sel_ts; unsigned long long* sel_n;
            Carve().take(sel_ts, n).take(sel_n, 1).take(sel_blk, n).take(sel_row, n).place(ctx->hgrp);
            VL_CUDA(cudaMemsetAsync(sel_n, 0, 8, ctx->stream));
            k_last_choose<<<cdiv(M, 256), 256, 0, ctx->stream>>>(cts, cblk, crow, M, st_row, ctx->goffs.as<uint64_t>(), sel_ts, sel_blk, sel_row, sel_n, blk_mark); launch_check(ctx);
            uint64_t chosen = 0;
            VL_CUDA(cudaMemcpyAsync(&chosen, sel_n, 8, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaMemcpyAsync(hts.data(), sel_ts, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaMemcpyAsync(hb.data(), sel_blk, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaMemcpyAsync(hr.data(), sel_row, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaStreamSynchronize(ctx->stream));
            if (chosen != n) throw BadInput("internal: the top-N selection chose " + std::to_string(chosen) + " rows instead of " + std::to_string(n));
        }
        // (4) the texts of the chosen rows only
        std::vector<std::vector<uint64_t>> toffs(q->nfields); std::vector<std::vector<uint8_t>> tbytes(q->nfields);
        uint64_t value_bytes = 0;
        for (uint32_t f = 0; f < q->nfields && n; f++) {
            const int slot = b->field_slot(names[f]);
            host_texts(ctx, slot, hit_row_offsets(ctx, slot, names[f], blk_mark), sel_row, sel_blk, n, toffs[f], tbytes[f]);
            value_bytes += tbytes[f].size();
        }
        if (!q->nfields) check_gather_errors(ctx);   // else host_texts checked them after the last kernel
        info[0] = n; info[1] = value_bytes;
        if (n > cap_rows) throw BadInput("rows buffer too small (the needed size is reported)");
        if (value_bytes > cap_bytes) throw BadInput("value bytes buffer too small (the needed size is reported)");
        if ((n && (!out_timestamps || !out_blocks || !out_rows)) || (q->nfields && !out_offsets) || (value_bytes && !out_bytes)) throw BadInput("last-rows output buffer missing");
        // ascending (timestamp, block, row): getLastNRows' order
        std::vector<uint64_t> order(n);
        for (uint64_t i = 0; i < n; i++) order[i] = i;
        std::sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) {
            if (hts[x] != hts[y]) return hts[x] < hts[y];
            if (hb[x] != hb[y]) return hb[x] < hb[y];
            return hr[x] < hr[y];
        });
        if (out_offsets) out_offsets[0] = 0;
        for (uint64_t i = 0; i < n; i++) { out_timestamps[i] = hts[order[i]]; out_blocks[i] = hb[order[i]]; out_rows[i] = hr[order[i]]; }
        pack_texts(order, toffs, tbytes, out_bytes, out_offsets);
    });
    if (out_info) memcpy(out_info, info, sizeof info);
    return rc;
}

static std::string rfc3339_nano(int64_t ts) {
    uint8_t buf[32];
    return std::string((const char*)buf, fmt_rfc3339nano(buf, ts));
}

int vlscan_facets(vlscan_ctx* ctx, const vlscan_facets_query* q, uint8_t* out_dropped, uint64_t* out_field_offsets, uint64_t* out_hits, uint8_t* out_classes,
                  uint64_t cap_entries, uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_value_offsets, uint64_t out_info[4]) {
    uint64_t info[4] = {0, 0, 0, 0};   // entries, value bytes, selected rows, blocks whose timestamps were decoded
    const int rc = guarded(ctx, [&] {
        if (!q) throw BadInput("no facets query");
        if (q->nfields == 0) throw BadInput("vlscan_facets needs at least one field");
        const std::vector<std::string> names = canonical_names(q->field_names, q->field_name_lens, q->nfields, "vlscan_facets");
        for (auto n = names.begin(); n != names.end(); ++n) {
            if (*n == "_stream" || *n == "_stream_id") throw BadInput("`" + *n + "` facets are not computed by the engine: it does not know the streams of the blocks");
            if (std::find(names.begin(), n, *n) != n) throw BadInput("duplicate facets field `" + *n + "`");
        }
        const uint64_t max_values = q->max_values_per_field ? q->max_values_per_field : VLSCAN_FACETS_DEFAULT_MAX_VALUES;
        const uint64_t max_len = q->max_value_len ? q->max_value_len : VLSCAN_FACETS_DEFAULT_MAX_VALUE_LEN;
        if (!ctx) throw BadInput("vlscan_facets needs a vlscan_ctx on a CUDA device (there is no CPU fallback)");
        const uint64_t n = build_hit_list(ctx, nullptr);
        if (n >= 0xFFFFFFFFull) throw BadInput("more than 2^32 - 2 selected rows in one batch");
        info[2] = n;
        const uint32_t nf = q->nfields;
        std::vector<uint8_t> dropped(nf, 0);
        std::vector<uint64_t> field_off(nf + 1, 0);
        std::vector<uint64_t> ehits, evoff(1, 0);
        std::vector<uint8_t> ecls;
        std::string ebytes;
        if (n) {
            const vlscan_batch* b = ctx->last_batch;
            BatchView B = b->view();
            // small device state: the field table, the entry bases and cursors, a work counter, a flag, the blocks with hits
            FacetField* d_fields; uint64_t* d_base; unsigned long long* d_cursor; uint32_t* d_wc; unsigned int* d_flag; uint32_t* d_blocks;
            Carve().take(d_fields, nf).take(d_base, nf + 1).take(d_cursor, nf).take(d_wc, WC_COUNT).take(d_flag, 1).take(d_blocks, b->nblocks + 1).place(ctx->hblk);
            VL_CUDA(cudaMemsetAsync(d_wc, 0, WC_COUNT * 4, ctx->stream));
            k_hit_blocks_list<<<cdiv(b->nblocks, 256), 256, 0, ctx->stream>>>(B, ctx->counts.as<uint32_t>(), -1, 1, d_blocks, d_wc); launch_check(ctx);
            uint32_t nblk = 0;
            VL_CUDA(cudaMemcpyAsync(&nblk, d_wc + WC_ROW, 4, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaStreamSynchronize(ctx->stream));
            std::vector<FacetField> hf(nf);
            bool has_time = false;
            if (ctx->ftxt.size() < nf) ctx->ftxt.resize(nf);
            for (uint32_t f = 0; f < nf; f++) {
                FacetField& F = hf[f];
                F.is_time = names[f] == "_time";
                F.slot = F.is_time ? -1 : b->field_slot(names[f]);
                F.row_off8 = hit_row_offsets(ctx, F.slot, names[f]);
                F.toffs = nullptr; F.tbytes = nullptr;
                has_time |= F.is_time;
                if (F.slot < 0 || !nblk) continue;
                // a field stored as float64 / ipv4 / iso8601 in a block with hits: the texts of every hit, formatted by the gather kernels first, so
                // that no formatter runs inside the facets pass
                unsigned int formatted = 0;
                VL_CUDA(cudaMemsetAsync(d_flag, 0, 4, ctx->stream));
                k_facets_formatted<<<cdiv(nblk, 256), 256, 0, ctx->stream>>>(B, d_blocks, nblk, F.slot, d_flag); launch_check(ctx);
                VL_CUDA(cudaMemcpyAsync(&formatted, d_flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
                VL_CUDA(cudaStreamSynchronize(ctx->stream));
                if (!formatted) continue;
                const uint64_t total = text_offsets(ctx, F.slot, F.row_off8, ctx->hits.as<uint32_t>(), ctx->hit_block.as<uint32_t>(), n);
                text_bytes(ctx, F.slot, F.row_off8, ctx->hits.as<uint32_t>(), ctx->hit_block.as<uint32_t>(), n, total);
                DevBuf& T = ctx->ftxt[f];
                T.ensure((n + 1) * 8 + total + 16);
                VL_CUDA(cudaMemcpyAsync(T.p, ctx->goffs.p, (n + 1) * 8, cudaMemcpyDeviceToDevice, ctx->stream));
                if (total) VL_CUDA(cudaMemcpyAsync(T.as<uint8_t>() + (n + 1) * 8, ctx->gout.p, total, cudaMemcpyDeviceToDevice, ctx->stream));
                F.toffs = T.as<uint64_t>(); F.tbytes = T.as<uint8_t>() + (n + 1) * 8;
            }
            // one table per field, bounded by the keys it can hold before it is dropped (saturating: max_values may be UINT64_MAX)
            const uint64_t bound = std::min(max_values, n - 1) + 1;
            uint64_t cap = 16;
            while (cap < 2 * bound) cap <<= 1;
            const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)nblk * nf, (uint64_t)ctx->sm_count * 4));
            const uint64_t table_bytes = (uint64_t)nf * cap * 16 + nf * 16 + 64;
            size_t free_b = 0, total_b = 0;
            VL_CUDA(cudaMemGetInfo(&free_b, &total_b));
            if (cap > (1ull << 40) / 16 || table_bytes > ctx->ftab.cap + free_b / 2)
                throw BadInput("vlscan_facets: max_values_per_field = " + std::to_string(max_values) + " needs " + std::to_string(table_bytes >> 20) + " MiB of facet tables for " +
                               std::to_string(nf) + " fields, more than the device has free");
            ctx->ftab.ensure(table_bytes);
            VL_CUDA(cudaMemcpyAsync(d_fields, hf.data(), nf * sizeof(FacetField), cudaMemcpyHostToDevice, ctx->stream));
            FacetsArgs A;
            A.fields = d_fields; A.nf = nf; A.blocks = d_blocks; A.nblocks = nblk; A.max_values = max_values; A.max_len = max_len;
            A.hits = ctx->hits.as<uint32_t>(); A.hit_block = ctx->hit_block.as<uint32_t>(); A.hit_offs = ctx->hit_offs.as<uint64_t>(); A.counts = ctx->counts.as<uint32_t>();
            A.tags = ctx->ftab.as<unsigned long long>(); A.cnt = A.tags + (uint64_t)nf * cap; A.nkeys = A.cnt + (uint64_t)nf * cap; A.dropped = (unsigned int*)(A.nkeys + nf);
            A.cap = cap; A.ts_vals = nullptr;
            VL_CUDA(cudaMemsetAsync(A.tags, 0, table_bytes, ctx->stream));
            unsigned long long* gstat = ctx->gstat.as<unsigned long long>();
            uint32_t decoded = 0;
            if (has_time) {   // timestamps of the blocks with hits that are not flat
                uint32_t* wc = ctx->work_count.as<uint32_t>(); uint32_t* row_blocks = ctx->row_blocks.as<uint32_t>();
                VL_CUDA(cudaMemsetAsync(wc, 0, WC_COUNT * 4, ctx->stream));
                k_facets_ts_list<<<cdiv(b->nblocks, 256), 256, 0, ctx->stream>>>(B, A.counts, row_blocks, wc, gstat); launch_check(ctx);
                A.ts_vals = decode_listed_timestamps(ctx, B, row_blocks, wc);
                VL_CUDA(cudaMemcpyAsync(&decoded, wc + WC_ROW, 4, cudaMemcpyDeviceToHost, ctx->stream));
                check_gather_errors(ctx);
            }
            info[3] = decoded;
            k_facets<<<grid, 256, 0, ctx->stream>>>(B, A, gstat); launch_check(ctx);
            std::vector<unsigned long long> nkeys(nf); std::vector<uint32_t> drop(nf);
            VL_CUDA(cudaMemcpyAsync(nkeys.data(), A.nkeys, nf * 8, cudaMemcpyDeviceToHost, ctx->stream));
            VL_CUDA(cudaMemcpyAsync(drop.data(), A.dropped, nf * 4, cudaMemcpyDeviceToHost, ctx->stream));
            check_gather_errors(ctx);   // synchronises
            for (uint32_t f = 0; f < nf; f++) {
                dropped[f] = drop[f] ? 1 : 0;
                field_off[f + 1] = field_off[f] + (dropped[f] ? 0 : nkeys[f]);
            }
            const uint64_t E = field_off[nf];
            std::vector<uint32_t> cls(E), rrows(E), rblocks(E); std::vector<unsigned long long> nums(E), cnts(E);
            uint32_t* rep_rows; uint32_t* rep_blocks; uint32_t* d_cls; unsigned long long* d_nums; unsigned long long* d_cnts; uint32_t* str_rows; uint32_t* str_blocks;
            Carve().take(rep_rows, E).take(rep_blocks, E).take(d_cls, E).take(d_nums, E).take(d_cnts, E).take(str_rows, E).take(str_blocks, E).place(ctx->hgrp);
            if (E) {   // the entries field after field
                VL_CUDA(cudaMemcpyAsync(d_base, field_off.data(), nf * 8, cudaMemcpyHostToDevice, ctx->stream));
                VL_CUDA(cudaMemsetAsync(d_cursor, 0, nf * 8, ctx->stream));
                k_facets_emit<<<grid, 256, 0, ctx->stream>>>(B, A, d_base, d_cursor, rep_rows, rep_blocks, d_cls, d_nums, d_cnts, gstat); launch_check(ctx);
                VL_CUDA(cudaMemcpyAsync(cls.data(), d_cls, E * 4, cudaMemcpyDeviceToHost, ctx->stream));
                VL_CUDA(cudaMemcpyAsync(nums.data(), d_nums, E * 8, cudaMemcpyDeviceToHost, ctx->stream));
                VL_CUDA(cudaMemcpyAsync(cnts.data(), d_cnts, E * 8, cudaMemcpyDeviceToHost, ctx->stream));
                VL_CUDA(cudaMemcpyAsync(rrows.data(), rep_rows, E * 4, cudaMemcpyDeviceToHost, ctx->stream));
                VL_CUDA(cudaMemcpyAsync(rblocks.data(), rep_blocks, E * 4, cudaMemcpyDeviceToHost, ctx->stream));
                check_gather_errors(ctx);
            }
            for (uint32_t f = 0; f < nf; f++) {
                const uint64_t e0 = field_off[f], ne = field_off[f + 1] - e0;
                if (!ne) continue;
                std::vector<std::string> text(ne);
                // the texts of the string-class representatives only
                std::vector<uint64_t> str_of; std::vector<uint32_t> sr, sb;
                for (uint64_t i = 0; i < ne; i++)
                    if (cls[e0 + i] == FK_STR) { str_of.push_back(i); sr.push_back(rrows[e0 + i]); sb.push_back(rblocks[e0 + i]); }
                if (!str_of.empty()) {
                    const uint64_t ns = str_of.size();
                    VL_CUDA(cudaMemcpyAsync(str_rows, sr.data(), ns * 4, cudaMemcpyHostToDevice, ctx->stream));
                    VL_CUDA(cudaMemcpyAsync(str_blocks, sb.data(), ns * 4, cudaMemcpyHostToDevice, ctx->stream));
                    std::vector<uint64_t> toffs; std::vector<uint8_t> tbytes;
                    host_texts(ctx, hf[f].slot, hf[f].row_off8, str_rows, str_blocks, ns, toffs, tbytes);
                    for (uint64_t k = 0; k < ns; k++) text[str_of[k]].assign((const char*)tbytes.data() + toffs[k], toffs[k + 1] - toffs[k]);
                }
                std::vector<uint8_t> ecl(ne);
                for (uint64_t i = 0; i < ne; i++) {
                    const uint64_t e = e0 + i;
                    char nb[24];
                    switch (cls[e]) {
                    case FK_U64: snprintf(nb, sizeof nb, "%llu", (unsigned long long)nums[e]); text[i] = nb; ecl[i] = VLSCAN_FACET_UINT64; break;
                    case FK_NEG: snprintf(nb, sizeof nb, "%lld", (long long)nums[e]); text[i] = nb; ecl[i] = VLSCAN_FACET_NEGATIVE; break;
                    case FK_TIME: text[i] = rfc3339_nano((int64_t)nums[e]); ecl[i] = VLSCAN_FACET_STRING; break;
                    default: ecl[i] = VLSCAN_FACET_STRING;   // its text was gathered above
                    }
                }
                // hits descending, then text bytewise, then class: a total order, where the reference's sort.Slice leaves ties unordered
                std::vector<uint64_t> order(ne);
                for (uint64_t i = 0; i < ne; i++) order[i] = i;
                std::sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) {
                    if (cnts[e0 + x] != cnts[e0 + y]) return cnts[e0 + x] > cnts[e0 + y];
                    const int c = text[x].compare(text[y]);
                    return c ? c < 0 : ecl[x] < ecl[y];
                });
                for (uint64_t i : order) {
                    ehits.push_back(cnts[e0 + i]); ecls.push_back(ecl[i]);
                    ebytes += text[i]; evoff.push_back(ebytes.size());
                }
            }
        }
        info[0] = ehits.size(); info[1] = ebytes.size();
        if (info[0] > cap_entries) throw BadInput("facets entries buffer too small (the needed size is reported)");
        if (info[1] > cap_bytes) throw BadInput("facets value bytes buffer too small (the needed size is reported)");
        if (!out_dropped || !out_field_offsets || !out_value_offsets || (info[0] && (!out_hits || !out_classes)) || (info[1] && !out_bytes)) throw BadInput("facets output buffer missing");
        memcpy(out_dropped, dropped.data(), nf);
        memcpy(out_field_offsets, field_off.data(), (nf + 1) * 8);
        memcpy(out_value_offsets, evoff.data(), evoff.size() * 8);
        if (info[0]) { memcpy(out_hits, ehits.data(), info[0] * 8); memcpy(out_classes, ecls.data(), info[0]); }
        if (info[1]) memcpy(out_bytes, ebytes.data(), info[1]);
    });
    if (out_info) memcpy(out_info, info, sizeof info);
    return rc;
}

}  // extern "C"
