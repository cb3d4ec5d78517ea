// TEST INFRASTRUCTURE ONLY: C API of the histogram restatement (vlo_vmrange.h) for tests/vlovmrange.py.
#include "vlo_vmrange.h"

using namespace vlo;

namespace {
thread_local std::string g_err;
template <class F> int guard(F&& f) {
    try { f(); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
struct Vmr {
    int64_t step, offset; int calendar; uint32_t nby, nv;
    std::vector<ByBucket> buckets;
    std::vector<ByColumn> by;        // of the block being added
    std::vector<HitsField> vals;
    VmrResult res;
};
void put_u64(std::string& o, uint64_t v) { o.append((const char*)&v, 8); }
}  // namespace

extern "C" {

const char* vlov_last_error() { return g_err.c_str(); }
int vlov_index(double v) { return vmrange_index(v); }
// tryParseNumber(s) -> ok, *out
int vlov_parse_number(const char* s, uint64_t n, double* out) { return try_parse_number(sv(s, n), out) ? 1 : 0; }
void* vlov_new(int64_t step, int64_t offset, int calendar, uint32_t nby, uint32_t nv) {
    return new Vmr{step, offset, calendar, nby, nv, std::vector<ByBucket>(nby), std::vector<ByColumn>(nby), std::vector<HitsField>(nv), {}};
}
void vlov_free(void* h) { delete (Vmr*)h; }
int vlov_bucket(void* h, uint32_t f, double size, double offset, int calendar, int enabled) {
    return guard([&] {
        Vmr& S = *(Vmr*)h;
        if (f >= S.nby) throw std::runtime_error("by-field index out of range");
        ByBucket& b = S.buckets[f];
        b.size = size; b.offset = offset; b.calendar = calendar; b.enabled = enabled != 0;
        if (b.enabled && !b.rejected().empty()) throw std::runtime_error("bucket rejected: " + b.rejected());
    });
}
// as vlob_field (tests/bucket_oracle/vlo_bucket_api.cpp)
int vlov_field(void* h, uint32_t f, int kind, int value_type, const uint8_t* payload, uint64_t len, const uint8_t* dict_blob, const uint64_t* dict_offs, uint32_t dict_len,
               uint64_t min_value, uint64_t max_value) {
    return guard([&] {
        Vmr& S = *(Vmr*)h;
        if (f >= S.nby + S.nv) throw std::runtime_error("field index out of range");
        HitsField& x = f < S.nby ? S.by[f].f : S.vals[f - S.nby];
        x.kind = kind; x.valueType = (uint8_t)value_type; x.payload.assign((const char*)payload, len); x.dict.clear();
        for (uint32_t k = 0; k < dict_len; k++) x.dict.emplace_back((const char*)dict_blob + dict_offs[k], dict_offs[k + 1] - dict_offs[k]);
        if (f < S.nby) { S.by[f].min_value = min_value; S.by[f].max_value = max_value; }
    });
}
int vlov_block(void* h, uint64_t rows, const uint64_t* words, const uint8_t* ts, uint64_t ts_len, int ts_mt, int64_t min_ts, int64_t max_ts) {
    return guard([&] {
        Vmr& S = *(Vmr*)h;
        vmrange_block(rows, words, sv((const char*)ts, ts_len), ts_mt, min_ts, max_ts, S.by, S.buckets, S.vals, S.step, S.offset, S.calendar, S.res);
        for (ByColumn& x : S.by) x = ByColumn();
        for (HitsField& x : S.vals) x = HitsField();
    });
}
// out = u64 groups, then per group: i64 bucket, u64 rows, per by-field u64 length + bytes, per value field u64 entries then (u64 index, u64 hits)
// each.  Returns the bytes needed (nothing written when that is more than cap).
int64_t vlov_result(void* h, uint8_t* out, uint64_t cap) {
    const Vmr& S = *(Vmr*)h;
    std::string o;
    put_u64(o, S.res.size());
    for (auto& [k, g] : S.res) {
        put_u64(o, (uint64_t)k.first); put_u64(o, g.rows);
        for (const std::string& t : k.second) { put_u64(o, t.size()); o += t; }
        for (const auto& m : g.hits) { put_u64(o, m.size()); for (auto& [i, c] : m) { put_u64(o, (uint64_t)i); put_u64(o, c); } }
    }
    if (o.size() <= cap) memcpy(out, o.data(), o.size());
    return (int64_t)o.size();
}

}  // extern "C"
