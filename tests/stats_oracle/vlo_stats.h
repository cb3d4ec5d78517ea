// TEST INFRASTRUCTURE ONLY: a C++ restatement of `stats by (_time:step offset off, f1, ...) count(), sum(v...), avg(v...)` over oracle blocks,
// built on the hits restatement (oracle/vlo_hits.h) for the buckets and key texts, the oracle's timestamps and values decode, and the oracle's
// tryParseFloat64 / tryParseNumber (oracle/vlo_mathnum.h).  Per block as pipeStatsProcessorShard.writeBlock feeds it
// (lib/logstorage/pipe_stats.go:552-626, 700-730): a block whose selected rows all have one key goes through blockResultColumn.sumValues
// (block_result.go:2501-2600), any other block row by row through getFloatValueAtRow (:2402-2448); float adds in the reference's order.
#pragma once
#include <cmath>
#include "vlo_hits.h"
#include "vlo_mathnum.h"

namespace vlo {

struct StatsGroup {
    uint64_t rows = 0;
    std::vector<double> sum, abs;     // statsSumProcessor.sum (NaN: none), the sum of |number| (the bound of a reordered sum)
    std::vector<uint64_t> count;      // statsAvgProcessor.count
    std::vector<uint8_t> ints;        // every number an integer
    explicit StatsGroup(size_t nv = 0) : sum(nv, NAN), abs(nv, 0.0), count(nv, 0), ints(nv, 1) {}
    void add(size_t f, double x, uint64_t c) {   // statsSumProcessor.updateState when c > 0; statsAvgProcessor adds c
        count[f] += c;
        if (!c) return;
        sum[f] = std::isnan(sum[f]) ? x : sum[f] + x;
        if (!std::isnan(x)) { abs[f] += std::fabs(x); ints[f] = ints[f] && std::isfinite(x) && x == std::trunc(x); }
    }
};
using StatsResult = std::map<std::pair<int64_t, std::vector<std::string>>, StatsGroup>;

// the stored values of a values column, one item per row (dict ids, typed bytes, strings)
inline std::vector<std::string> stored_items(const HitsField& f, uint64_t rows) {
    const DecodedStringsBlock d = decode_values_block_stage(f.payload);
    std::vector<std::string> out;
    for (sv v : unmarshal_strings(d, rows)) out.emplace_back(v);
    return out;
}
inline uint64_t typed_u64(const std::string& v) {
    uint64_t x = 0;
    for (unsigned char c : v) x = x << 8 | c;   // big-endian, 1 / 2 / 4 / 8 bytes
    return x;
}
inline double typed_number(uint8_t vt, const std::string& v) {
    const uint64_t u = typed_u64(v);
    if (vt == VT_INT64) return (double)unzigzag(u);
    if (vt == VT_FLOAT64) { double f; memcpy(&f, &u, 8); return f; }
    return (double)u;
}

// blockResultColumn.sumValues over the selected rows -> (sum, count)
inline std::pair<double, uint64_t> sum_values(const HitsField& f, uint64_t rows, const std::vector<uint64_t>& sel) {
    const uint64_t n = sel.size();
    if (f.kind == HITS_FIELD_ABSENT) return {0.0, 0};
    if (f.kind == HITS_FIELD_CONST) { double x; return try_parse_float64(f.payload, &x) ? std::make_pair(x * (double)n, n) : std::make_pair(0.0, (uint64_t)0); }
    const std::vector<std::string> items = stored_items(f, rows);
    double s = 0; uint64_t c = 0;
    switch (f.valueType) {
    case VT_STRING:
        for (uint64_t r : sel) { double x; if (try_parse_number(items[r], &x)) { s += x; c++; } }
        return {s, c};
    case VT_DICT: {
        std::vector<double> dv;
        for (const std::string& e : f.dict) { double x; dv.push_back(try_parse_number(e, &x) ? x : NAN); }
        for (uint64_t r : sel) { const double x = dv.at((uint8_t)items[r].at(0)); if (!std::isnan(x)) { s += x; c++; } }
        return {s, c};
    }
    case VT_UINT8: case VT_UINT16: case VT_UINT32: {
        uint64_t u = 0;
        for (uint64_t r : sel) u += typed_u64(items[r]);
        return {(double)u, n};
    }
    case VT_UINT64: case VT_INT64:
        for (uint64_t r : sel) s += typed_number(f.valueType, items[r]);
        return {s, n};
    case VT_FLOAT64:
        for (uint64_t r : sel) { const double x = typed_number(VT_FLOAT64, items[r]); if (!std::isnan(x)) s += x; }
        return {s, n};
    }
    return {0.0, 0};   // ipv4, iso8601
}
// getFloatValueAtRow -> ok, *x
inline bool value_at_row(const HitsField& f, const std::vector<std::string>& items, uint64_t r, double* x) {
    if (f.kind == HITS_FIELD_ABSENT) return false;
    if (f.kind == HITS_FIELD_CONST) return try_parse_float64(f.payload, x);
    switch (f.valueType) {
    case VT_STRING: return try_parse_float64(items[r], x);
    case VT_DICT: return try_parse_float64(f.dict.at((uint8_t)items[r].at(0)), x);
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: case VT_INT64: *x = typed_number(f.valueType, items[r]); return true;
    case VT_FLOAT64: *x = typed_number(VT_FLOAT64, items[r]); return !std::isnan(*x);
    }
    return false;
}

// One block: its selected rows (the oracle's bitmap words), its timestamps column as stored, its by-fields and its value fields (a value field
// named `_time` is passed as absent: isTime columns give nothing).
inline void stats_block(uint64_t rows, const uint64_t* words, sv ts_data, int ts_mt, int64_t min_ts, int64_t max_ts, const std::vector<HitsField>& by,
                        const std::vector<HitsField>& vals, int64_t step, int64_t offset, int calendar, StatsResult& res) {
    std::vector<uint64_t> sel;
    for (uint64_t i = 0; i < rows; i++) if (words[i / 64] >> (i % 64) & 1) sel.push_back(i);
    if (sel.empty()) return;
    if (!ts_mt) throw std::runtime_error("the block has no timestamps");
    std::vector<std::vector<std::string>> texts;
    for (const HitsField& f : by) texts.push_back(field_texts(f, rows));
    std::vector<int64_t> ts;
    const int64_t lo = truncate_timestamp(min_ts, step, offset, calendar), hi = truncate_timestamp(max_ts, step, offset, calendar);
    if (lo != hi) ts = unmarshal_int64_array(ts_data, (uint8_t)ts_mt, min_ts, rows);
    std::vector<std::pair<int64_t, std::vector<std::string>>> keys;
    for (uint64_t r : sel) {
        std::vector<std::string> key;
        for (auto& t : texts) key.push_back(t[r]);
        keys.emplace_back(lo == hi ? lo : truncate_timestamp(ts[r], step, offset, calendar), std::move(key));
    }
    bool one = true;
    for (auto& k : keys) one = one && k == keys[0];
    if (one) {
        auto it = res.try_emplace(keys[0], vals.size()).first;
        it->second.rows += sel.size();
        for (size_t f = 0; f < vals.size(); f++) { const auto [x, c] = sum_values(vals[f], rows, sel); it->second.add(f, x, c); }
        return;
    }
    std::vector<std::vector<std::string>> items;
    for (const HitsField& f : vals) items.push_back(f.kind == HITS_FIELD_VALUES ? stored_items(f, rows) : std::vector<std::string>());
    for (size_t i = 0; i < sel.size(); i++) {
        auto it = res.try_emplace(keys[i], vals.size()).first;
        it->second.rows++;
        for (size_t f = 0; f < vals.size(); f++) { double x; if (value_at_row(vals[f], items[f], sel[i], &x)) it->second.add(f, x, 1); }
    }
}

}  // namespace vlo
