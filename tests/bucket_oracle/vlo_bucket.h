// TEST INFRASTRUCTURE ONLY: a C++ restatement of bucketed by-fields, `stats by (_time:step, f:size offset off, ...) count(), sum(v), avg(v)`,
// from the reference Go: byStatsField.hasBucketConfig (lib/logstorage/pipe_stats.go:1522), newValuesBucketedForColumn and everything it calls
// (lib/logstorage/block_result.go:703-1764: the header fast paths of the typed kinds, truncateUint64 / Int64 / Float64 / Uint32,
// getBucketedValue), marshalDurationString and marshalTimestampRFC3339NanoString (values_encoder.go), decimal.FromFloat (VictoriaMetrics
// lib/decimal) and math.Pow10, with Go's float -> integer conversions on amd64.  Per block as pipeStatsProcessorShard.writeBlock feeds it
// (pipe_stats.go:552-626, 700-730), on top of the oracle's value decode (oracle/vlo_hits.h) and the sums restatement (tests/stats_oracle).
#pragma once
#include <cmath>
#include "../stats_oracle/vlo_stats.h"

namespace vlo {

// ---- Go conversions on amd64 and math.Pow10 --------------------------------------------------------------------------------------------------
inline uint64_t go_uint64_of_float(double f) {   // the compiler's branch at 2^63: uint64(x) = int64(x) below it, int64(x - 2^63) | 2^63 above
    const double cutoff = 9223372036854775808.0;
    if (f < cutoff) return (uint64_t)go_int64_of_float(f);
    return (uint64_t)go_int64_of_float(f - cutoff) | (1ULL << 63);
}
inline uint32_t go_uint32_of_float(double f) { return (uint32_t)(uint64_t)go_int64_of_float(f); }   // CVTTSD2SQ, then the low 32 bits
inline int32_t go_int32_of_float(double f) {                                                         // CVTTSD2SL
    if (!(f == f) || f >= 2147483648.0 || f <= -2147483649.0) return INT32_MIN;
    return (int32_t)f;
}
inline double math_pow10(int n) {
    static const double tab[] = {1e00, 1e01, 1e02, 1e03, 1e04, 1e05, 1e06, 1e07, 1e08, 1e09, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15,
                                 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31};
    static const double postab32[] = {1e00, 1e32, 1e64, 1e96, 1e128, 1e160, 1e192, 1e224, 1e256, 1e288};
    static const double negtab32[] = {1e-00, 1e-32, 1e-64, 1e-96, 1e-128, 1e-160, 1e-192, 1e-224, 1e-256, 1e-288, 1e-320};
    if (0 <= n && n <= 308) return postab32[(unsigned)n / 32] * tab[(unsigned)n % 32];
    if (-323 <= n && n <= 0) return negtab32[(unsigned)-n / 32] / tab[(unsigned)-n % 32];
    return n > 0 ? INFINITY : 0;
}
// decimal.FromFloat(f) for a finite f > 0: (v, e) with f ~ v * 10^e
inline std::pair<int64_t, int> decimal_from_float(double f) {
    uint64_t u = go_uint64_of_float(f);
    if ((double)u == f) {   // positiveFloatToDecimal's integer path, getDecimalAndScale
        if (u < (1ULL << 55) && u % 10 != 0) return {(int64_t)u, 0};
        int scale = 0;
        while (u >= (1ULL << 55)) { u /= 10; scale++; }
        if (u % 10 != 0) return {(int64_t)u, scale};
        u /= 10; scale++;
        while (u != 0 && u % 10 == 0) { u /= 10; scale++; }
        return {(int64_t)u, scale};
    }
    int scale = 0;   // positiveFloatToDecimalSlow
    double prec = 1e12;
    if (f > 1e6 || f < 1e-6) {
        if (f > 1e6) prec = 1e15;
        int exp;
        (void)std::frexp(f, &exp);
        if (exp < -1022) exp = -1022; else if (exp > 1023) exp = 1023;
        const double ln2_ln10 = 0.301029995663981195213738894724493026768189881462108541310;   // the untyped constant math.Ln2 / math.Ln10
        scale = (int16_t)((double)exp * ln2_ln10);
        f *= math_pow10(-scale);
    }
    while (f < prec) {
        double x;
        const double frac = std::modf(f, &x);
        if (frac * prec < x) { f = x; break; }
        if ((1 - frac) * prec < x) { f = x + 1; break; }
        f *= 100;
        scale -= 2;
    }
    u = go_uint64_of_float(f);
    if (u % 10 != 0) return {(int64_t)u, scale};
    return {(int64_t)(u / 10), scale + 1};
}

// ---- the truncations and the two formatters the buckets add ------------------------------------------------------------------------------------
inline uint64_t truncate_uint64(uint64_t n, uint64_t size, uint64_t off) {
    if (off == 0) return n - n % size;
    if (off > n) return 0;
    n -= off; n -= n % size; n += off;
    return n;
}
inline uint32_t truncate_uint32(uint32_t n, uint32_t size, uint32_t off) {
    if (off == 0) return n - n % size;
    if (off > n) return 0;
    n -= off; n -= n % size; n += off;
    return n;
}
inline int64_t go_mod(int64_t a, int64_t b) { return b == -1 ? 0 : a % b; }   // Go: MinInt64 % -1 == 0
inline int64_t wrap_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
inline int64_t wrap_sub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
inline int64_t truncate_int64(int64_t n, int64_t size, int64_t off) {
    if (off == 0) { int64_t r = go_mod(n, size); if (r < 0) r = wrap_add(r, size); return wrap_sub(n, r); }
    n = wrap_sub(n, off);
    int64_t r = go_mod(n, size);
    if (r < 0) r = wrap_add(r, size);
    n = wrap_sub(n, r);
    return wrap_add(n, off);
}
inline double truncate_float64(double f, double p10, int64_t size_p10, double off) {
    if (off == 0) {
        int64_t fp = go_int64_of_float(std::floor(f * p10));
        fp = wrap_sub(fp, go_mod(fp, size_p10));
        return (double)fp / p10;
    }
    f -= off;
    int64_t fp = go_int64_of_float(std::floor(f * p10));
    fp = wrap_sub(fp, go_mod(fp, size_p10));
    f = (double)fp / p10;
    return f + off;
}
inline void marshal_duration_string(std::string& dst, int64_t nsecs) {
    const int64_t S = 1000000000LL;
    if (nsecs == 0) { dst.push_back('0'); return; }
    if (nsecs < 0) { dst.push_back('-'); nsecs = wrap_sub(0, nsecs); }
    const bool float_secs = nsecs >= S;
    const int64_t W = 7 * 24 * 3600 * S, D = 24 * 3600 * S, H = 3600 * S, M = 60 * S;
    if (nsecs >= W) { const int64_t w = nsecs / W; nsecs -= w * W; marshal_uint64_string(dst, (uint64_t)w); dst.push_back('w'); }
    if (nsecs >= D) { const int64_t d = nsecs / D; nsecs -= d * D; marshal_uint64_string(dst, (uint8_t)d); dst.push_back('d'); }
    if (nsecs >= H) { const int64_t h = nsecs / H; nsecs -= h * H; marshal_uint64_string(dst, (uint8_t)h); dst.push_back('h'); }
    if (nsecs >= M) { const int64_t m = nsecs / M; nsecs -= m * M; marshal_uint64_string(dst, (uint8_t)m); dst.push_back('m'); }
    if (nsecs >= S) {
        if (float_secs) { marshal_float64_string(dst, (double)nsecs / 1e9); dst.push_back('s'); return; }
        const int64_t s = nsecs / S; nsecs -= s * S; marshal_uint64_string(dst, (uint8_t)s); dst.push_back('s');
    }
    if (nsecs >= 1000000) { const int64_t ms = nsecs / 1000000; nsecs -= ms * 1000000; marshal_uint64_string(dst, (uint16_t)ms); dst += "ms"; }
    if (nsecs >= 1000) { const int64_t us = nsecs / 1000; nsecs -= us * 1000; marshal_uint64_string(dst, (uint16_t)us); dst += "\xC2\xB5s"; }
    if (nsecs > 0) { marshal_uint64_string(dst, (uint16_t)nsecs); dst += "ns"; }
}
inline void marshal_timestamp_rfc3339nano_string(std::string& dst, int64_t nsecs) {   // time.RFC3339Nano in UTC: trailing zeros of the fraction dropped
    std::string iso;
    marshal_timestamp_iso8601_string(iso, nsecs);
    dst.append(iso, 0, 19);
    int64_t frac = nsecs % 1000000000LL;
    if (frac < 0) frac += 1000000000LL;
    if (frac) {
        char b[16];
        snprintf(b, sizeof b, ".%09lld", (long long)frac);
        std::string f(b);
        while (f.back() == '0') f.pop_back();
        dst += f;
    }
    dst.push_back('Z');
}

// ---- one by-field bucket ---------------------------------------------------------------------------------------------------------------------
struct ByBucket {
    double size = 0, offset = 0; int calendar = HITS_PLAIN; bool enabled = false;
    // (p10, bucketSizeP10) of the float truncation, as getBucketedFloat64Values / getBucketedValue compute them
    std::pair<double, int64_t> float_params() const {
        const double s = size <= 0 ? 1 : size;
        const int e = decimal_from_float(s).second;
        const double p10 = math_pow10(-e);
        return {p10, go_int64_of_float(s * p10)};
    }
    // why the engine turns this bucket down: what the reference cannot compute (NaN / Inf never come out of tryParseBucketSize; a zero
    // bucketSizeP10 is an integer divide by zero in truncateFloat64)
    std::string rejected() const {
        if (!std::isfinite(size) || !std::isfinite(offset)) return "not finite";
        if (calendar < 0 || calendar > HITS_YEAR) return "calendar";
        if (float_params().second == 0) return "bucketSizeP10 == 0";
        return "";
    }
    int64_t i64_size() const { const int64_t n = go_int64_of_float(size); return n <= 0 ? 1 : n; }
};

// getBucketedValue
inline std::string get_bucketed_value(sv s, const ByBucket& bf) {
    if (s.empty()) return std::string();
    const char c = s[0];
    if ((c < '0' || c > '9') && c != '-') return std::string(s);
    std::string out;
    int64_t n; double f; uint32_t ip;
    if (try_parse_int64(s, &n)) { marshal_int64_string(out, truncate_int64(n, bf.i64_size(), go_int64_of_float(bf.offset))); return out; }
    if (try_parse_float64(s, &f)) {
        const auto [p10, sp10] = bf.float_params();
        marshal_float64_string(out, truncate_float64(f, p10, sp10, bf.offset));
        return out;
    }
    if (try_parse_timestamp_rfc3339nano(s, &n)) {
        marshal_timestamp_rfc3339nano_string(out, truncate_timestamp(n, bf.i64_size(), go_int64_of_float(bf.offset), bf.calendar));
        return out;
    }
    if (try_parse_ipv4(s, &ip)) {
        uint32_t size = go_uint32_of_float(bf.size);
        if (size == 0) size = 1;
        marshal_ipv4_string(out, truncate_uint32(ip, size, (uint32_t)go_int32_of_float(bf.offset)));
        return out;
    }
    if (try_parse_duration(s, &n)) { marshal_duration_string(out, truncate_int64(n, bf.i64_size(), go_int64_of_float(bf.offset))); return out; }
    return std::string(s);
}

// newValuesBucketedForColumn for one by-field of one block: a field the block lacks is "" (getConstValues of an empty column)
struct ByColumn { HitsField f; uint64_t min_value = 0, max_value = 0; };
inline std::vector<std::string> bucketed_texts(const ByColumn& col, uint64_t rows, const ByBucket& bf) {
    const HitsField& f = col.f;
    if (!bf.enabled) return field_texts(f, rows);
    if (f.kind == HITS_FIELD_ABSENT) return std::vector<std::string>(rows);
    if (f.kind == HITS_FIELD_CONST) return std::vector<std::string>(rows, get_bucketed_value(f.payload, bf));
    std::vector<std::string> out;
    if (f.valueType == VT_STRING) {
        for (const std::string& s : field_texts(f, rows)) out.push_back(get_bucketed_value(s, bf));
        return out;
    }
    if (f.valueType == VT_DICT) {
        std::vector<std::string> db;
        for (const std::string& e : f.dict) db.push_back(get_bucketed_value(e, bf));
        for (const std::string& v : stored_items(f, rows)) out.push_back(db.at((uint8_t)v.at(0)));
        return out;
    }
    const std::vector<std::string> items = stored_items(f, rows);
    std::string s;
    switch (f.valueType) {
    case VT_UINT8: case VT_UINT16: case VT_UINT32: case VT_UINT64: {
        uint64_t size = go_uint64_of_float(bf.size);
        if (size <= 0) size = 1;
        const uint64_t off = (uint64_t)go_int64_of_float(bf.offset);
        const uint64_t lo = truncate_uint64((uint64_t)(int64_t)col.min_value, size, off), hi = truncate_uint64((uint64_t)(int64_t)col.max_value, size, off);
        if (lo == hi) { marshal_uint64_string(s, lo); return std::vector<std::string>(rows, s); }
        for (const std::string& v : items) { s.clear(); marshal_uint64_string(s, truncate_uint64(typed_u64(v), size, off)); out.push_back(s); }
        return out;
    }
    case VT_INT64: {
        int64_t size = go_int64_of_float(bf.size);
        if (size == 0) size = 1;
        const int64_t off = go_int64_of_float(bf.offset);
        const int64_t lo = truncate_int64((int64_t)col.min_value, size, off), hi = truncate_int64((int64_t)col.max_value, size, off);
        if (lo == hi) { marshal_int64_string(s, lo); return std::vector<std::string>(rows, s); }
        for (const std::string& v : items) { s.clear(); marshal_int64_string(s, truncate_int64(unzigzag(typed_u64(v)), size, off)); out.push_back(s); }
        return out;
    }
    case VT_FLOAT64: {
        const auto [p10, sp10] = bf.float_params();
        double mn, mx;
        memcpy(&mn, &col.min_value, 8); memcpy(&mx, &col.max_value, 8);
        const double lo = truncate_float64(mn, p10, sp10, bf.offset), hi = truncate_float64(mx, p10, sp10, bf.offset);
        if (lo == hi) { marshal_float64_string(s, lo); return std::vector<std::string>(rows, s); }
        for (const std::string& v : items) { s.clear(); marshal_float64_string(s, truncate_float64(typed_number(VT_FLOAT64, v), p10, sp10, bf.offset)); out.push_back(s); }
        return out;
    }
    case VT_IPV4: {
        uint32_t size = go_uint32_of_float(bf.size);
        if (size <= 0) size = 1;
        const uint32_t off = (uint32_t)go_int32_of_float(bf.offset);
        const uint32_t lo = truncate_uint32((uint32_t)(int32_t)col.min_value, size, off), hi = truncate_uint32((uint32_t)(int32_t)col.max_value, size, off);
        if (lo == hi) { marshal_ipv4_string(s, lo); return std::vector<std::string>(rows, s); }
        for (const std::string& v : items) { s.clear(); marshal_ipv4_string(s, truncate_uint32((uint32_t)typed_u64(v), size, off)); out.push_back(s); }
        return out;
    }
    case VT_ISO8601: {
        const int64_t size = bf.i64_size(), off = go_int64_of_float(bf.offset);
        const int64_t lo = truncate_timestamp((int64_t)col.min_value, size, off, bf.calendar), hi = truncate_timestamp((int64_t)col.max_value, size, off, bf.calendar);
        if (lo == hi) { marshal_timestamp_iso8601_string(s, lo); return std::vector<std::string>(rows, s); }
        for (const std::string& v : items) { s.clear(); marshal_timestamp_iso8601_string(s, truncate_timestamp((int64_t)typed_u64(v), size, off, bf.calendar)); out.push_back(s); }
        return out;
    }
    }
    throw std::runtime_error("unknown value type");
}

// stats_block with bucketed by-fields (vals empty: the count alone)
inline void bucketed_stats_block(uint64_t rows, const uint64_t* words, sv ts_data, int ts_mt, int64_t min_ts, int64_t max_ts, const std::vector<ByColumn>& by,
                                 const std::vector<ByBucket>& buckets, const std::vector<HitsField>& vals, int64_t step, int64_t offset, int calendar, StatsResult& res) {
    std::vector<uint64_t> sel;
    for (uint64_t i = 0; i < rows; i++) if (words[i / 64] >> (i % 64) & 1) sel.push_back(i);
    if (sel.empty()) return;
    if (!ts_mt) throw std::runtime_error("the block has no timestamps");
    std::vector<std::vector<std::string>> texts;
    for (size_t f = 0; f < by.size(); f++) texts.push_back(bucketed_texts(by[f], rows, buckets[f]));
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
    if (one) {   // the key of every selected row is the same: sumValues
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
