// TEST INFRASTRUCTURE ONLY: a C++ restatement of `stats by (_time:step offset off, f1, ...) histogram(v...)` (lib/logstorage/stats_histogram.go)
// over oracle blocks, on the bucketed by-fields restatement (vlo_bucket.h) for the keys and the oracle's tryParseNumber.  Both reference paths,
// updateStatsForAllRows and updateStatsForRow, read a number the same way, so every selected row is fed to Histogram.Update on its own.  The
// index is computed from Update's formula with Go's portable math.Log restated here, never from the engine's boundary table.
#pragma once
#include <cmath>
#include <map>
#include "vlo_bucket.h"

namespace vlo {

// math/log.go
inline double go_log(double x) {
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10;
    const double L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01, L3 = 2.857142874366239149e-01, L4 = 2.222219843214978396e-01,
                 L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01, L7 = 1.479819860511658591e-01;
    if (std::isnan(x) || (std::isinf(x) && x > 0)) return x;
    if (x < 0) return NAN;
    if (x == 0) return -INFINITY;
    int ki;
    double f1 = std::frexp(x, &ki);
    if (f1 < 0.70710678118654752440) { f1 *= 2; ki--; }
    const double f = f1 - 1, k = ki;
    const double s = f / (2 + f), s2 = s * s, s4 = s2 * s2;
    const double t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7))), t2 = s4 * (L2 + s4 * (L4 + s4 * L6));
    const double R = t1 + t2, hfsq = 0.5 * f * f;
    return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f);
}
// Histogram.Update: -1 skipped, 0 lower, 1 + bucket index, 487 upper
inline int vmrange_index(double v) {
    if (std::isnan(v) || v < 0) return -1;
    // Go evaluates the untyped constant 1/Ln10 exactly and rounds it once; 1 / (double)Ln10 would round twice and land one ulp off
    static const double inv_ln10 = (double)(1.0L / 2.30258509299404568401799145468436420760110148862877297603332790L);
    const double b = (go_log(v) * inv_ln10 - (-9)) * 18;
    if (b < 0) return 0;
    if (b >= 486) return 487;
    unsigned long idx = (unsigned long)b;
    if (b == (double)idx && idx > 0) idx--;
    return (int)idx + 1;
}

struct VmrGroup {
    uint64_t rows = 0;
    std::vector<std::map<int, uint64_t>> hits;   // per value field: index -> hits
    explicit VmrGroup(size_t nv = 0) : hits(nv) {}
};
using VmrResult = std::map<std::pair<int64_t, std::vector<std::string>>, VmrGroup>;

// the number of row r of a value field (stats_histogram.go:42-168) -> ok, *x
inline bool histogram_number(const HitsField& f, const std::vector<std::string>& items, uint64_t r, double* x) {
    if (f.kind == HITS_FIELD_ABSENT) return false;
    if (f.kind == HITS_FIELD_CONST) return try_parse_number(f.payload, x);
    switch (f.valueType) {
    case VT_STRING: return try_parse_number(items[r], x);
    case VT_DICT: return try_parse_number(f.dict.at((uint8_t)items[r].at(0)), x);
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: case VT_INT64: case VT_FLOAT64: *x = typed_number(f.valueType, items[r]); return true;
    }
    return false;   // ipv4, iso8601
}

inline void vmrange_block(uint64_t rows, const uint64_t* words, sv ts_data, int ts_mt, int64_t min_ts, int64_t max_ts, const std::vector<ByColumn>& by,
                          const std::vector<ByBucket>& buckets, const std::vector<HitsField>& vals, int64_t step, int64_t offset, int calendar, VmrResult& res) {
    std::vector<uint64_t> sel;
    for (uint64_t i = 0; i < rows; i++) if (words[i / 64] >> (i % 64) & 1) sel.push_back(i);
    if (sel.empty()) return;
    if (!ts_mt) throw std::runtime_error("the block has no timestamps");
    std::vector<std::vector<std::string>> texts;
    for (size_t f = 0; f < by.size(); f++) texts.push_back(bucketed_texts(by[f], rows, buckets[f]));
    std::vector<int64_t> ts;
    const int64_t lo = truncate_timestamp(min_ts, step, offset, calendar), hi = truncate_timestamp(max_ts, step, offset, calendar);
    if (lo != hi) ts = unmarshal_int64_array(ts_data, (uint8_t)ts_mt, min_ts, rows);
    std::vector<std::vector<std::string>> items;
    for (const HitsField& f : vals) items.push_back(f.kind == HITS_FIELD_VALUES ? stored_items(f, rows) : std::vector<std::string>());
    for (uint64_t r : sel) {
        std::vector<std::string> key;
        for (auto& t : texts) key.push_back(t[r]);
        auto it = res.try_emplace({lo == hi ? lo : truncate_timestamp(ts[r], step, offset, calendar), std::move(key)}, vals.size()).first;
        it->second.rows++;
        for (size_t f = 0; f < vals.size(); f++) {
            double x;
            if (!histogram_number(vals[f], items[f], r, &x)) continue;
            const int i = vmrange_index(x);
            if (i >= 0) it->second.hits[f][i]++;
        }
    }
}

}  // namespace vlo
