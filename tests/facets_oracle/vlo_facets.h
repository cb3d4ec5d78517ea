// TEST INFRASTRUCTURE ONLY: the CPU restatement of `| facets` (lib/logstorage/pipe_facets.go:162-420, hits_map.go:85-115) that the facets tests
// compare the device and tests/facets_model.py with.  One pipeFacetsProcessorShard with concurrency 1 over oracle blocks, then its flush.  The
// blocks come as the oracle stores them (the oracle filter's bitmap words, the stored timestamps column, each field's const value or values
// block); values and timestamps are decoded with the oracle's own routines (oracle/vlo_util.h, vlo_timestamps.h, vlo_block.h) and `_time` is
// formatted by a calendar walk of its own, not by the engine's formatter.  Built by tests/facets_oracle/build.sh into liboracle_facets.so.
#pragma once
#include <algorithm>
#include <map>
#include <tuple>
#include "vlo_hits.h"

namespace vlo {

enum { FACETS_FIELD_TIME = 3 };                       // after HITS_FIELD_ABSENT / _CONST / _VALUES
enum { FACET_U64 = 0, FACET_NEG = 1, FACET_STR = 2 };   // hitsMapAdaptive's u64, negative64 and strings maps

struct FacetKey {
    int cls; uint64_t num; std::string text;
    bool operator<(const FacetKey& o) const { return std::tie(cls, num, text) < std::tie(o.cls, o.num, o.text); }
    std::string str() const {   // appendTopEntryFacets: marshalUint64String / marshalInt64String / the bytes
        if (cls == FACET_STR) return text;
        return cls == FACET_U64 ? std::to_string(num) : std::to_string((int64_t)num);
    }
};
struct FacetFieldHits { bool mustIgnore = false; std::map<FacetKey, uint64_t> m; };

inline int uint64_string_len(uint64_t n) {   // uint64StringLen: exact below 10^10, 20 from there on
    int k = 1;
    for (uint64_t p = 10; k < 10 && n >= p; p *= 10) k++;
    return n >= 10000000000ULL ? 20 : k;
}
inline int int64_string_len(int64_t n) {
    if (n >= 0) return uint64_string_len((uint64_t)n);
    return n == INT64_MIN ? 21 : 1 + uint64_string_len((uint64_t)(-n));
}

// marshalTimestampRFC3339NanoString in UTC, by walking years and months from 1970
inline std::string rfc3339_nano(int64_t ts) {
    int64_t secs = ts / 1000000000LL, frac = ts % 1000000000LL;
    if (frac < 0) { frac += 1000000000LL; secs--; }
    int64_t days = secs / 86400, sod = secs % 86400;
    if (sod < 0) { sod += 86400; days--; }
    int64_t y = 1970;
    while (days < 0) { y--; days += year_days(y); }
    while (days >= year_days(y)) { days -= year_days(y); y++; }
    int m = 1;
    while (days >= month_days(y, m)) { days -= month_days(y, m); m++; }
    char buf[64];
    snprintf(buf, sizeof buf, "%04lld-%02d-%02lldT%02lld:%02lld:%02lld", (long long)y, m, (long long)days + 1, (long long)(sod / 3600), (long long)(sod / 60 % 60),
             (long long)(sod % 60));
    std::string s = buf;
    if (frac) {
        snprintf(buf, sizeof buf, ".%09lld", (long long)frac);
        std::string f = buf;
        while (f.back() == '0') f.pop_back();
        s += f;
    }
    return s + "Z";
}

struct FacetsShard {
    uint64_t maxValuesPerField, maxValueLen;
    std::map<std::string, FacetFieldHits> m;
    uint64_t rowsTotal = 0, blocksDecoded = 0;

    void ignore(FacetFieldHits& f) { f.m.clear(); f.mustIgnore = true; }
    void add(FacetFieldHits& f, FacetKey k, uint64_t hits) { f.m[std::move(k)] += hits; }
    void update_generic(FacetFieldHits& f, sv v, uint64_t hits) {   // updateStateGeneric + hitsMapAdaptive.updateStateGeneric
        if (v.empty()) return;
        if (v.size() > maxValueLen) { ignore(f); return; }
        uint64_t n; int64_t i;
        if (try_parse_uint64(v, &n)) add(f, {FACET_U64, n, ""}, hits);
        else if (v[0] == '-' && try_parse_int64(v, &i)) add(f, {FACET_NEG, (uint64_t)i, ""}, hits);
        else add(f, {FACET_STR, 0, std::string(v)}, hits);
    }
    void update_uint64(FacetFieldHits& f, uint64_t n) {
        if (maxValueLen <= 20 && (uint64_t)uint64_string_len(n) > maxValueLen) { ignore(f); return; }
        add(f, {FACET_U64, n, ""}, 1);
    }
    void update_int64(FacetFieldHits& f, int64_t n) {
        if (maxValueLen <= 21 && (uint64_t)int64_string_len(n) > maxValueLen) { ignore(f); return; }
        add(f, {n >= 0 ? FACET_U64 : FACET_NEG, (uint64_t)n, ""}, 1);
    }

    // writeBlock: the fields of one block (kind HITS_FIELD_* or FACETS_FIELD_TIME), its selected rows as bitmap words, its timestamps column
    void block(uint64_t rows, const uint64_t* words, const std::vector<std::string>& names, const std::vector<HitsField>& fields, const std::vector<int>& is_time,
               sv ts_data, int ts_mt, int64_t min_ts, int64_t max_ts) {
        std::vector<uint64_t> sel;
        for (uint64_t i = 0; i < rows; i++) if (words[i / 64] >> (i % 64) & 1) sel.push_back(i);
        if (sel.empty()) return;
        std::vector<int64_t> ts;   // blockResult reads the timestamps of every block with selected rows when `_time` is a column
        if (std::find(is_time.begin(), is_time.end(), 1) != is_time.end()) {
            if (!ts_mt) throw std::runtime_error("the block has no timestamps");
            if (min_ts == max_ts) ts.assign(rows, min_ts);
            else { ts = unmarshal_int64_array(ts_data, (uint8_t)ts_mt, min_ts, rows); blocksDecoded++; }
        }
        for (size_t k = 0; k < fields.size(); k++) {
            if (!is_time[k] && fields[k].kind == HITS_FIELD_ABSENT) continue;
            FacetFieldHits& f = m[names[k]];
            if (f.mustIgnore) continue;
            if (f.m.size() > maxValuesPerField) { ignore(f); continue; }
            if (is_time[k]) {
                for (uint64_t r : sel) update_generic(f, rfc3339_nano(ts[r]), 1);
                continue;
            }
            const HitsField& c = fields[k];
            if (c.kind == HITS_FIELD_CONST) { update_generic(f, c.payload, sel.size()); continue; }
            const DecodedStringsBlock d = decode_values_block_stage(c.payload);
            const std::vector<sv> items = unmarshal_strings(d, rows);
            switch (c.valueType) {
            case VT_DICT: {   // forEachDictValueWithHits: only entries with selected rows
                std::vector<uint64_t> hits(c.dict.size(), 0);
                for (uint64_t r : sel) {
                    if (items[r].size() != 1 || (uint8_t)items[r][0] >= c.dict.size()) throw std::runtime_error("bad dict value");
                    hits[(uint8_t)items[r][0]]++;
                }
                for (size_t i = 0; i < c.dict.size(); i++) if (hits[i]) update_generic(f, c.dict[i], hits[i]);
                break;
            }
            case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64:
                for (uint64_t r : sel) { uint64_t n = 0; for (char ch : items[r]) n = n << 8 | (uint8_t)ch; update_uint64(f, n); }
                break;
            case VT_INT64:
                for (uint64_t r : sel) { uint64_t n = 0; for (char ch : items[r]) n = n << 8 | (uint8_t)ch; update_int64(f, unzigzag(n)); }
                break;
            default:
                for (uint64_t r : sel) update_generic(f, encoded_to_string(c.valueType, items[r]), 1);
            }
        }
        rowsTotal += sel.size();
    }

    bool dropped(const FacetFieldHits& f) const { return f.mustIgnore || f.m.size() > maxValuesPerField; }
    // the entries of a field by hits descending, then text, then class (the reference's sort.Slice leaves such ties unordered)
    std::vector<std::pair<FacetKey, uint64_t>> entries(const FacetFieldHits& f) const {
        std::vector<std::pair<FacetKey, uint64_t>> v(f.m.begin(), f.m.end());
        std::sort(v.begin(), v.end(), [](const auto& a, const auto& b) {
            if (a.second != b.second) return a.second > b.second;
            const int c = a.first.str().compare(b.first.str());
            return c ? c < 0 : a.first.cls < b.first.cls;
        });
        return v;
    }
    // flush: the fields in name order, without dropped fields and (unless keepConstFields) fields whose one entry covers every row, at most
    // `limit` entries each
    std::vector<std::tuple<std::string, std::string, uint64_t>> flush(uint64_t limit, bool keepConstFields) const {
        std::vector<std::tuple<std::string, std::string, uint64_t>> out;
        for (auto& [name, f] : m) {
            if (dropped(f)) continue;
            auto v = entries(f);
            if (v.size() == 1 && v[0].second == rowsTotal && !keepConstFields) continue;
            for (size_t i = 0; i < v.size() && i < limit; i++) out.emplace_back(name, v[i].first.str(), v[i].second);
        }
        return out;
    }
};

}  // namespace vlo
