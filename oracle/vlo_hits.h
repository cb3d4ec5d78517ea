// ORACLE -- TEST INFRASTRUCTURE ONLY (see vlo_util.h header).
//
// CPU restatement of `stats by (_time:step offset off, f1, ...) count()`, the aggregation /select/logsql/hits appends to a query
// (app/vlselect/logsql/logsql.go:116-219, lib/logstorage/parser.go:407-445), over oracle blocks: the oracle filter's bitmap, the oracle's
// timestamps decode of the stored timestamps column, the values as blockResultColumn.getValues reads them from the stored values block, and
// truncateTimestamp (lib/logstorage/block_result.go:818-848) with a civil calendar of its own (walking years and months, not a closed formula).
// Built into oracle/liboracle_hits.so (vlo_hits_api.cpp, oracle/build_hits.sh), bound by oracle/vlohits.py.
#pragma once
#include <map>
#include "vlo_block.h"

namespace vlo {

enum { HITS_PLAIN = 0, HITS_WEEK = 1, HITS_MONTH = 2, HITS_YEAR = 3 };
static const int64_t kDayNs = 86400LL * 1000000000LL;

inline bool leap_year(int64_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }
inline int64_t year_days(int64_t y) { return leap_year(y) ? 366 : 365; }
inline int64_t month_days(int64_t y, int m) { static const int d[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31}; return d[m - 1] + (m == 2 && leap_year(y)); }

// first day (days since 1970-01-01) of the month / year that holds day `days`
inline int64_t first_day_of(int64_t days, bool year_only) {
    int64_t y = 1970, start = 0;   // start = first day of year y
    while (days < start) { y--; start -= year_days(y); }
    while (days >= start + year_days(y)) { start += year_days(y); y++; }
    if (year_only) return start;
    for (int m = 1; m <= 12; m++) {
        if (days < start + month_days(y, m)) return start;
        start += month_days(y, m);
    }
    throw std::runtime_error("civil calendar walk fell off the year");
}

// Go's int64 arithmetic wraps: sums and products on uint64
inline int64_t truncate_timestamp(int64_t ts, int64_t bucket_size, int64_t bucket_offset, int calendar) {
    if (bucket_size <= 0) bucket_size = 1;   // getBucketedTimestampValues :763-766
    uint64_t off = (uint64_t)bucket_offset;
    if (calendar == HITS_WEEK) off += (uint64_t)(4 * kDayNs);   // weeks start on Monday
    const int64_t t = (int64_t)((uint64_t)ts - off);
    int64_t res;
    if (calendar == HITS_MONTH || calendar == HITS_YEAR) {
        // time.Unix(0, t).UTC(): the day is the floor of t / day; time.Date(y, m, 1, ...).UnixNano() wraps like int64
        int64_t days = t / kDayNs;
        if (t % kDayNs < 0) days--;
        const int64_t first = first_day_of(days, calendar == HITS_YEAR);
        res = (int64_t)((uint64_t)first * 86400ULL * 1000000000ULL);
    } else {
        int64_t r = t % bucket_size;
        if (r < 0) r += bucket_size;
        res = (int64_t)((uint64_t)t - (uint64_t)r);
    }
    return (int64_t)((uint64_t)res + off);
}

struct HitsResult {
    std::map<std::pair<int64_t, std::vector<std::string>>, uint64_t> groups;   // (bucket, key texts) -> rows; std::string compares bytes unsigned
    uint64_t rows = 0;
    uint64_t blocks_decoded = 0;   // blocks with selected rows whose min and max timestamps fall into different buckets
};

// One by-field of one block, as the block stores it: absent, const, or a values column (valuesBlock as stored + valueType + dict)
enum { HITS_FIELD_ABSENT = 0, HITS_FIELD_CONST = 1, HITS_FIELD_VALUES = 2 };
struct HitsField { int kind = HITS_FIELD_ABSENT; uint8_t valueType = VT_STRING; std::string payload; std::vector<std::string> dict; };

// the value of the field in every row of the block, as blockResultColumn.getValues yields it
inline std::vector<std::string> field_texts(const HitsField& f, uint64_t rows) {
    if (f.kind == HITS_FIELD_ABSENT) return std::vector<std::string>(rows, std::string());
    if (f.kind == HITS_FIELD_CONST) return std::vector<std::string>(rows, f.payload);
    const DecodedStringsBlock d = decode_values_block_stage(f.payload);
    const std::vector<sv> items = unmarshal_strings(d, rows);
    std::vector<std::string> out; out.reserve(rows);
    for (sv v : items) {
        if (f.valueType == VT_DICT) {
            if (v.size() != 1 || (uint8_t)v[0] >= f.dict.size()) throw std::runtime_error("bad dict value");
            out.push_back(f.dict[(uint8_t)v[0]]);
        } else out.push_back(encoded_to_string(f.valueType, v));
    }
    return out;
}

// One block: its selected rows (the oracle's bitmap words), its timestamps column as stored (marshal type 0 = none) and its by-fields.
inline void hits_stats_block(uint64_t rows, const uint64_t* words, sv ts_data, int ts_mt, int64_t min_ts, int64_t max_ts, const std::vector<HitsField>& by,
                             int64_t step, int64_t offset, int calendar, HitsResult& res) {
    std::vector<uint64_t> sel;
    for (uint64_t i = 0; i < rows; i++) if (words[i / 64] >> (i % 64) & 1) sel.push_back(i);
    if (sel.empty()) return;
    if (!ts_mt) throw std::runtime_error("the block has no timestamps");
    std::vector<std::vector<std::string>> texts;
    for (const HitsField& f : by) texts.push_back(field_texts(f, rows));
    const int64_t lo = truncate_timestamp(min_ts, step, offset, calendar), hi = truncate_timestamp(max_ts, step, offset, calendar);
    std::vector<int64_t> ts;
    if (lo != hi) { ts = unmarshal_int64_array(ts_data, (uint8_t)ts_mt, min_ts, rows); res.blocks_decoded++; }   // getTimestamps
    for (uint64_t r : sel) {
        std::vector<std::string> key;
        for (auto& t : texts) key.push_back(t[r]);
        res.groups[{lo == hi ? lo : truncate_timestamp(ts[r], step, offset, calendar), std::move(key)}]++;
    }
    res.rows += sel.size();
}

}  // namespace vlo
