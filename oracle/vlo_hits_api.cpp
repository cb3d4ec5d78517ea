// ORACLE -- TEST INFRASTRUCTURE ONLY (see vlo_util.h header).
//
// C API of the hits-aggregation restatement (vlo_hits.h) for tests/ and tools/ via oracle/vlohits.py.  The blocks arrive as the oracle
// stores them (bitmap words of the oracle's own search, the timestamps column, the by-fields' const values or values blocks), so this
// library shares no objects with liboracle.so.
#include "vlo_hits.h"

using namespace vlo;

namespace {
thread_local std::string g_err;
template <class F> int guard(F&& f) {
    try { f(); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
struct Hits {
    int64_t step, offset; int calendar;
    uint32_t nby;
    HitsResult res;
    std::vector<HitsField> fields;   // of the block being added
};
}  // namespace

extern "C" {

const char* vloh_last_error() { return g_err.c_str(); }

int64_t vloh_truncate_timestamp(int64_t ts, int64_t step, int64_t offset, int calendar) { return truncate_timestamp(ts, step, offset, calendar); }

void* vloh_new(int64_t step, int64_t offset, int calendar, uint32_t nby) { return new Hits{step, offset, calendar, nby, {}, std::vector<HitsField>(nby)}; }
void vloh_free(void* h) { delete (Hits*)h; }

// by-field f of the next block: kind HITS_FIELD_*; payload = the const value or the values block as stored; dict: packed entries
int vloh_field(void* h, uint32_t f, int kind, int value_type, const uint8_t* payload, uint64_t len, const uint8_t* dict_blob, const uint64_t* dict_offs, uint32_t dict_len) {
    return guard([&] {
        Hits& H = *(Hits*)h;
        if (f >= H.nby) throw std::runtime_error("by-field index out of range");
        HitsField& x = H.fields[f];
        x.kind = kind; x.valueType = (uint8_t)value_type; x.payload.assign((const char*)payload, len); x.dict.clear();
        for (uint32_t k = 0; k < dict_len; k++) x.dict.emplace_back((const char*)dict_blob + dict_offs[k], dict_offs[k + 1] - dict_offs[k]);
    });
}

// the block whose by-fields were just given: rows, the oracle's bitmap words, the timestamps column (ts_mt = 0: none)
int vloh_block(void* h, uint64_t rows, const uint64_t* words, const uint8_t* ts, uint64_t ts_len, int ts_mt, int64_t min_ts, int64_t max_ts) {
    return guard([&] {
        Hits& H = *(Hits*)h;
        hits_stats_block(rows, words, sv((const char*)ts, ts_len), ts_mt, min_ts, max_ts, H.fields, H.step, H.offset, H.calendar, H.res);
        for (HitsField& x : H.fields) x = HitsField();
    });
}

// out = u64 groups, u64 selected rows, u64 blocks decoded, then per group (sorted by bucket, then by the texts): i64 bucket, u64 count,
// per by-field u64 length + bytes.  Returns the bytes needed (nothing written when that is more than cap).
int64_t vloh_result(void* h, uint8_t* out, uint64_t cap) {
    const HitsResult& res = ((Hits*)h)->res;
    std::string o;
    auto u64 = [&](uint64_t v) { o.append((const char*)&v, 8); };
    u64(res.groups.size()); u64(res.rows); u64(res.blocks_decoded);
    for (auto& g : res.groups) {
        u64((uint64_t)g.first.first); u64(g.second);
        for (auto& t : g.first.second) { u64(t.size()); o += t; }
    }
    if (o.size() <= cap) memcpy(out, o.data(), o.size());
    return (int64_t)o.size();
}

}  // extern "C"
