// TEST INFRASTRUCTURE ONLY: C API of the facets restatement (vlo_facets.h) for tests/vlofacets.py.
#include "vlo_facets.h"

using namespace vlo;

namespace {
thread_local std::string g_err;
template <class F> int guard(F&& f) {
    try { f(); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
struct Facets {
    FacetsShard shard;
    std::vector<std::string> names;
    std::vector<HitsField> fields;   // of the block being added
    std::vector<int> is_time;
};
void put_u64(std::string& o, uint64_t v) { o.append((const char*)&v, 8); }
int64_t copy_out(const std::string& o, uint8_t* out, uint64_t cap) {
    if (o.size() <= cap) memcpy(out, o.data(), o.size());
    return (int64_t)o.size();
}
}  // namespace

extern "C" {

const char* vlof_last_error() { return g_err.c_str(); }

// max_values_per_field / max_value_len: 0 = the endpoint's defaults (1000 / 128)
void* vlof_new(uint64_t max_values, uint64_t max_len, uint32_t nfields) {
    Facets* h = new Facets{{max_values ? max_values : 1000, max_len ? max_len : 128, {}}, std::vector<std::string>(nfields), std::vector<HitsField>(nfields),
                           std::vector<int>(nfields, 0)};
    return h;
}
void vlof_free(void* h) { delete (Facets*)h; }

// field f: its name and whether it is `_time`
int vlof_name(void* h, uint32_t f, const char* name, uint64_t len, int is_time) {
    return guard([&] {
        Facets& F = *(Facets*)h;
        if (f >= F.names.size()) throw std::runtime_error("field index out of range");
        F.names[f].assign(name, len); F.is_time[f] = is_time;
    });
}
// field f of the next block: kind HITS_FIELD_*; payload = the const value or the values block as stored; dict: packed entries
int vlof_field(void* h, uint32_t f, int kind, int value_type, const uint8_t* payload, uint64_t len, const uint8_t* dict_blob, const uint64_t* dict_offs, uint32_t dict_len) {
    return guard([&] {
        Facets& F = *(Facets*)h;
        if (f >= F.fields.size()) throw std::runtime_error("field index out of range");
        HitsField& x = F.fields[f];
        x.kind = kind; x.valueType = (uint8_t)value_type; x.payload.assign((const char*)payload, len); x.dict.clear();
        for (uint32_t k = 0; k < dict_len; k++) x.dict.emplace_back((const char*)dict_blob + dict_offs[k], dict_offs[k + 1] - dict_offs[k]);
    });
}
// the block whose fields were just given: rows, the oracle's bitmap words, the timestamps column (ts_mt = 0: none)
int vlof_block(void* h, uint64_t rows, const uint64_t* words, const uint8_t* ts, uint64_t ts_len, int ts_mt, int64_t min_ts, int64_t max_ts) {
    return guard([&] {
        Facets& F = *(Facets*)h;
        F.shard.block(rows, words, F.names, F.fields, F.is_time, sv((const char*)ts, ts_len), ts_mt, min_ts, max_ts);
        for (HitsField& x : F.fields) x = HitsField();
    });
}
// out = u64 selected rows, u64 blocks decoded, then per field: u8 dropped, u64 entries, per entry (hits descending, then text, then class):
// u8 class, u64 hits, u64 length + text.  Returns the bytes needed (nothing written when that is more than cap).
int64_t vlof_state(void* h, uint8_t* out, uint64_t cap) {
    const Facets& F = *(Facets*)h;
    std::string o;
    put_u64(o, F.shard.rowsTotal); put_u64(o, F.shard.blocksDecoded);
    for (const std::string& name : F.names) {
        auto it = F.shard.m.find(name);
        const bool drop = it != F.shard.m.end() && F.shard.dropped(it->second);
        o.push_back((char)drop);
        if (drop || it == F.shard.m.end()) { put_u64(o, 0); continue; }
        auto v = F.shard.entries(it->second);
        put_u64(o, v.size());
        for (auto& [k, hits] : v) { o.push_back((char)k.cls); put_u64(o, hits); const std::string t = k.str(); put_u64(o, t.size()); o += t; }
    }
    return copy_out(o, out, cap);
}
// out = u64 rows, per row: u64 length + field name, u64 length + value, u64 hits (flush with the given limit and keep_const_fields)
int64_t vlof_flush(void* h, uint64_t limit, int keep_const_fields, uint8_t* out, uint64_t cap) {
    const Facets& F = *(Facets*)h;
    const auto rows = F.shard.flush(limit, keep_const_fields != 0);
    std::string o;
    put_u64(o, rows.size());
    for (auto& [name, text, hits] : rows) { put_u64(o, name.size()); o += name; put_u64(o, text.size()); o += text; put_u64(o, hits); }
    return copy_out(o, out, cap);
}

}  // extern "C"
