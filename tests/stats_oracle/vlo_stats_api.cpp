// TEST INFRASTRUCTURE ONLY: C API of the sum / avg restatement (vlo_stats.h) for tests/vlostats.py.
#include "vlo_stats.h"

using namespace vlo;

namespace {
thread_local std::string g_err;
template <class F> int guard(F&& f) {
    try { f(); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
struct Stats {
    int64_t step, offset; int calendar; uint32_t nby, nv;
    std::vector<HitsField> fields;   // by-fields, then value fields, of the block being added
    StatsResult res;
};
void put_u64(std::string& o, uint64_t v) { o.append((const char*)&v, 8); }
void put_f64(std::string& o, double v) { o.append((const char*)&v, 8); }
}  // namespace

extern "C" {

const char* vlos_last_error() { return g_err.c_str(); }
void* vlos_new(int64_t step, int64_t offset, int calendar, uint32_t nby, uint32_t nv) { return new Stats{step, offset, calendar, nby, nv, std::vector<HitsField>(nby + nv), {}}; }
void vlos_free(void* h) { delete (Stats*)h; }
// field f (by-fields first, then value fields) of the next block: kind HITS_FIELD_*; payload = the const value or the values block as stored
int vlos_field(void* h, uint32_t f, int kind, int value_type, const uint8_t* payload, uint64_t len, const uint8_t* dict_blob, const uint64_t* dict_offs, uint32_t dict_len) {
    return guard([&] {
        Stats& S = *(Stats*)h;
        if (f >= S.fields.size()) throw std::runtime_error("field index out of range");
        HitsField& x = S.fields[f];
        x.kind = kind; x.valueType = (uint8_t)value_type; x.payload.assign((const char*)payload, len); x.dict.clear();
        for (uint32_t k = 0; k < dict_len; k++) x.dict.emplace_back((const char*)dict_blob + dict_offs[k], dict_offs[k + 1] - dict_offs[k]);
    });
}
int vlos_block(void* h, uint64_t rows, const uint64_t* words, const uint8_t* ts, uint64_t ts_len, int ts_mt, int64_t min_ts, int64_t max_ts) {
    return guard([&] {
        Stats& S = *(Stats*)h;
        const std::vector<HitsField> by(S.fields.begin(), S.fields.begin() + S.nby), vals(S.fields.begin() + S.nby, S.fields.end());
        stats_block(rows, words, sv((const char*)ts, ts_len), ts_mt, min_ts, max_ts, by, vals, S.step, S.offset, S.calendar, S.res);
        for (HitsField& x : S.fields) x = HitsField();
    });
}
// out = u64 groups, then per group (by bucket, then texts): i64 bucket, u64 rows, per by-field u64 length + bytes, per value field f64 sum,
// u64 count, f64 sum |x|, u8 integers only.  Returns the bytes needed (nothing written when that is more than cap).
int64_t vlos_result(void* h, uint8_t* out, uint64_t cap) {
    const Stats& S = *(Stats*)h;
    std::string o;
    put_u64(o, S.res.size());
    for (auto& [k, g] : S.res) {
        put_u64(o, (uint64_t)k.first); put_u64(o, g.rows);
        for (const std::string& t : k.second) { put_u64(o, t.size()); o += t; }
        for (uint32_t f = 0; f < S.nv; f++) { put_f64(o, g.sum[f]); put_u64(o, g.count[f]); put_f64(o, g.abs[f]); o.push_back((char)g.ints[f]); }
    }
    if (o.size() <= cap) memcpy(out, o.data(), o.size());
    return (int64_t)o.size();
}
// the oracle's tryParseFloat64 (non-exact) and tryParseNumber: 1 when s is a number
int vlos_try_parse_float64(const char* s, uint64_t n, double* out) { return try_parse_float64(sv(s, n), out); }
int vlos_try_parse_number(const char* s, uint64_t n, double* out) { return try_parse_number(sv(s, n), out); }

}  // extern "C"
