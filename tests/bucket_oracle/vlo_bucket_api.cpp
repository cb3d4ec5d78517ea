// TEST INFRASTRUCTURE ONLY: C API of the bucketed by-fields restatement (vlo_bucket.h) for tests/vlobucket.py.
#include "vlo_bucket.h"

using namespace vlo;

namespace {
thread_local std::string g_err;
template <class F> int guard(F&& f) {
    try { f(); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
struct Bucketed {
    int64_t step, offset; int calendar; uint32_t nby, nv;
    std::vector<ByBucket> buckets;
    std::vector<ByColumn> by;        // of the block being added
    std::vector<HitsField> vals;
    StatsResult res;
};
void put_u64(std::string& o, uint64_t v) { o.append((const char*)&v, 8); }
}  // namespace

extern "C" {

const char* vlob_last_error() { return g_err.c_str(); }
// getBucketedValue(s) -> its length into out (nothing written when more than cap), -2 when the engine turns the bucket down
int64_t vlob_bucket_text(double size, double offset, int calendar, const char* s, uint64_t n, char* out, uint64_t cap) {
    ByBucket b; b.size = size; b.offset = offset; b.calendar = calendar; b.enabled = true;
    if (!b.rejected().empty()) return -2;
    const std::string t = get_bucketed_value(sv(s, n), b);
    if (t.size() <= cap) memcpy(out, t.data(), t.size());
    return (int64_t)t.size();
}
void* vlob_new(int64_t step, int64_t offset, int calendar, uint32_t nby, uint32_t nv) {
    return new Bucketed{step, offset, calendar, nby, nv, std::vector<ByBucket>(nby), std::vector<ByColumn>(nby), std::vector<HitsField>(nv), {}};
}
void vlob_free(void* h) { delete (Bucketed*)h; }
int vlob_bucket(void* h, uint32_t f, double size, double offset, int calendar, int enabled) {
    return guard([&] {
        Bucketed& S = *(Bucketed*)h;
        if (f >= S.nby) throw std::runtime_error("by-field index out of range");
        ByBucket& b = S.buckets[f];
        b.size = size; b.offset = offset; b.calendar = calendar; b.enabled = enabled != 0;
        if (b.enabled && !b.rejected().empty()) throw std::runtime_error("bucket rejected: " + b.rejected());
    });
}
// field f (by-fields first, then value fields) of the next block: kind HITS_FIELD_*; payload = the const value or the values block as stored;
// min / max = the column header's minValue / maxValue
int vlob_field(void* h, uint32_t f, int kind, int value_type, const uint8_t* payload, uint64_t len, const uint8_t* dict_blob, const uint64_t* dict_offs, uint32_t dict_len,
               uint64_t min_value, uint64_t max_value) {
    return guard([&] {
        Bucketed& S = *(Bucketed*)h;
        if (f >= S.nby + S.nv) throw std::runtime_error("field index out of range");
        HitsField& x = f < S.nby ? S.by[f].f : S.vals[f - S.nby];
        x.kind = kind; x.valueType = (uint8_t)value_type; x.payload.assign((const char*)payload, len); x.dict.clear();
        for (uint32_t k = 0; k < dict_len; k++) x.dict.emplace_back((const char*)dict_blob + dict_offs[k], dict_offs[k + 1] - dict_offs[k]);
        if (f < S.nby) { S.by[f].min_value = min_value; S.by[f].max_value = max_value; }
    });
}
int vlob_block(void* h, uint64_t rows, const uint64_t* words, const uint8_t* ts, uint64_t ts_len, int ts_mt, int64_t min_ts, int64_t max_ts) {
    return guard([&] {
        Bucketed& S = *(Bucketed*)h;
        bucketed_stats_block(rows, words, sv((const char*)ts, ts_len), ts_mt, min_ts, max_ts, S.by, S.buckets, S.vals, S.step, S.offset, S.calendar, S.res);
        for (ByColumn& x : S.by) x = ByColumn();
        for (HitsField& x : S.vals) x = HitsField();
    });
}
// out = u64 groups, then per group (by bucket, then texts): i64 bucket, u64 rows, per by-field u64 length + bytes, per value field f64 sum,
// u64 count, f64 sum |x|, u8 integers only.  Returns the bytes needed (nothing written when that is more than cap).
int64_t vlob_result(void* h, uint8_t* out, uint64_t cap) {
    const Bucketed& S = *(Bucketed*)h;
    std::string o;
    put_u64(o, S.res.size());
    for (auto& [k, g] : S.res) {
        put_u64(o, (uint64_t)k.first); put_u64(o, g.rows);
        for (const std::string& t : k.second) { put_u64(o, t.size()); o += t; }
        for (uint32_t f = 0; f < S.nv; f++) { o.append((const char*)&g.sum[f], 8); put_u64(o, g.count[f]); o.append((const char*)&g.abs[f], 8); o.push_back((char)g.ints[f]); }
    }
    if (o.size() <= cap) memcpy(out, o.data(), o.size());
    return (int64_t)o.size();
}

}  // extern "C"
