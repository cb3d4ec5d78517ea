// Host+device primitives of the scan engine: Go-exact UTF-8 decoding, token-rune classification, XXH64,
// matchPhrase / matchPrefix, number -> string formatting.  Everything here is used by the CUDA kernels (vl_engine.cu)
// and by the host-side program compiler (vl_program.cpp).
//
// Reference semantics (file:line relative to the VictoriaLogs tree):
//   isTokenChar / isTokenRune            lib/logstorage/tokenizer.go:128-148
//   matchPhrase / getPhrasePos           lib/logstorage/filter_phrase.go:211-270
//   matchPrefix                          lib/logstorage/filter_prefix.go:318-352
//   XXH64 (cespare/xxhash v2.3.0)        call sites lib/logstorage/bloomfilter.go:136,138,164
//   marshal*String                       lib/logstorage/values_encoder.go:1367-1422
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define VL_HD __host__ __device__ __forceinline__
#define VL_HDN static __host__ __device__
#else
#define VL_HD inline
#define VL_HDN inline
#endif

namespace vl {

#include "unicode_tables.inc"
#ifdef __CUDACC__
// device copy of the token ranges (5.6 KB, only touched for non-ASCII neighbours of a match candidate)
static __device__ const unsigned int D_TOKEN_RANGES[VL_TOKEN_RANGES_COUNT][2] = { VL_TOKEN_RANGES_INIT };
#endif

static const int32_t kRuneError = 0xFFFD;

// utf8.DecodeRune (Go stdlib): invalid encodings yield (RuneError, 1); empty input (RuneError, 0)
VL_HD int32_t decode_rune(const uint8_t* p, uint32_t n, int* size) {
    if (n < 1) { *size = 0; return kRuneError; }
    uint32_t p0 = p[0];
    if (p0 < 0x80) { *size = 1; return (int32_t)p0; }
    int sz; uint32_t lo = 0x80, hi = 0xBF;
    if (p0 < 0xC2) { *size = 1; return kRuneError; }
    else if (p0 <= 0xDF) sz = 2;
    else if (p0 == 0xE0) { sz = 3; lo = 0xA0; }
    else if (p0 == 0xED) { sz = 3; hi = 0x9F; }
    else if (p0 <= 0xEF) sz = 3;
    else if (p0 == 0xF0) { sz = 4; lo = 0x90; }
    else if (p0 <= 0xF3) sz = 4;
    else if (p0 == 0xF4) { sz = 4; hi = 0x8F; }
    else { *size = 1; return kRuneError; }
    if ((int)n < sz) { *size = 1; return kRuneError; }
    uint32_t b1 = p[1];
    if (b1 < lo || hi < b1) { *size = 1; return kRuneError; }
    if (sz == 2) { *size = 2; return (int32_t)(((p0 & 0x1F) << 6) | (b1 & 0x3F)); }
    uint32_t b2 = p[2];
    if (b2 < 0x80 || 0xBF < b2) { *size = 1; return kRuneError; }
    if (sz == 3) { *size = 3; return (int32_t)(((p0 & 0x0F) << 12) | ((b1 & 0x3F) << 6) | (b2 & 0x3F)); }
    uint32_t b3 = p[3];
    if (b3 < 0x80 || 0xBF < b3) { *size = 1; return kRuneError; }
    *size = 4;
    return (int32_t)(((p0 & 0x07) << 18) | ((b1 & 0x3F) << 12) | ((b2 & 0x3F) << 6) | (b3 & 0x3F));
}

// utf8.DecodeLastRune
VL_HD int32_t decode_last_rune(const uint8_t* p, uint32_t n, int* size) {
    if (n == 0) { *size = 0; return kRuneError; }
    int end = (int)n, start = end - 1;
    uint32_t r = p[start];
    if (r < 0x80) { *size = 1; return (int32_t)r; }
    int lim = end - 4; if (lim < 0) lim = 0;
    for (start--; start >= lim; start--) if ((p[start] & 0xC0) != 0x80) break;
    if (start < 0) start = 0;
    int sz;
    int32_t rr = decode_rune(p + start, (uint32_t)(end - start), &sz);
    if (start + sz != end) { *size = 1; return kRuneError; }
    *size = sz;
    return rr;
}

VL_HD bool is_token_char(uint32_t c) {
    return (c - 'a' < 26u) || (c - 'A' < 26u) || (c - '0' < 10u) || c == '_';
}
VL_HD bool is_token_rune(int32_t r) {
    if (r < 0x80) return r >= 0 && is_token_char((uint32_t)r);
    int lo = 0, hi = VL_TOKEN_RANGES_COUNT - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
#ifdef __CUDA_ARCH__
        unsigned a = D_TOKEN_RANGES[mid][0], b = D_TOKEN_RANGES[mid][1];
#else
        unsigned a = VL_TOKEN_RANGES[mid][0], b = VL_TOKEN_RANGES[mid][1];
#endif
        if ((uint32_t)r < a) hi = mid - 1; else if ((uint32_t)r > b) lo = mid + 1; else return true;
    }
    return false;
}

// ---- XXH64 (seed 0) ------------------------------------------------------------------------------------------------
#define VL_P1 11400714785074694791ULL
#define VL_P2 14029467366897019727ULL
#define VL_P3 1609587929392839161ULL
#define VL_P4 9650029242287828579ULL
#define VL_P5 2870177450012600261ULL
VL_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
VL_HD uint64_t ld_le64(const uint8_t* p) { uint64_t v = 0; for (int i = 7; i >= 0; i--) v = (v << 8) | p[i]; return v; }
VL_HD uint32_t ld_le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
VL_HD uint64_t xxh_round(uint64_t acc, uint64_t in) { acc += in * VL_P2; acc = rotl64(acc, 31); return acc * VL_P1; }
VL_HD uint64_t xxh_merge(uint64_t acc, uint64_t v) { v = xxh_round(0, v); acc ^= v; return acc * VL_P1 + VL_P4; }
VL_HDN uint64_t xxh64(const uint8_t* p, uint32_t n) {
    const uint8_t* end = p + n;
    uint64_t h;
    if (n >= 32) {
        uint64_t v1 = VL_P1 + VL_P2, v2 = VL_P2, v3 = 0, v4 = 0ULL - VL_P1;
        do {
            v1 = xxh_round(v1, ld_le64(p)); v2 = xxh_round(v2, ld_le64(p + 8));
            v3 = xxh_round(v3, ld_le64(p + 16)); v4 = xxh_round(v4, ld_le64(p + 24));
            p += 32;
        } while (p + 32 <= end);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xxh_merge(h, v1); h = xxh_merge(h, v2); h = xxh_merge(h, v3); h = xxh_merge(h, v4);
    } else h = VL_P5;
    h += (uint64_t)n;
    while (p + 8 <= end) { h ^= xxh_round(0, ld_le64(p)); h = rotl64(h, 27) * VL_P1 + VL_P4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)ld_le32(p) * VL_P1; h = rotl64(h, 23) * VL_P2 + VL_P3; p += 4; }
    while (p < end) { h ^= (uint64_t)(*p) * VL_P5; h = rotl64(h, 11) * VL_P1; p++; }
    h ^= h >> 33; h *= VL_P2; h ^= h >> 29; h *= VL_P3; h ^= h >> 32;
    return h;
}
// XXH64 of the 8 little-endian bytes of v: the bloom probe chain h_i = XXH64(LE8(h0 + i)) (bloomfilter.go:133-141)
VL_HD uint64_t xxh64_u64(uint64_t v) {
    uint64_t h = VL_P5 + 8;
    h ^= xxh_round(0, v); h = rotl64(h, 27) * VL_P1 + VL_P4;
    h ^= h >> 33; h *= VL_P2; h ^= h >> 29; h *= VL_P3; h ^= h >> 32;
    return h;
}

// ---- substring search + phrase/prefix predicates over byte spans ---------------------------------------------------------
// index of needle in s[from:], or -1 (strings.Index)
VL_HDN int find_bytes(const uint8_t* s, uint32_t n, const uint8_t* nd, uint32_t m, uint32_t from) {
    if (m == 0) return from <= n ? (int)from : -1;
    if (m > n) return -1;
    uint8_t c0 = nd[0];
    for (uint32_t i = from; i + m <= n; i++) {
        if (s[i] != c0) continue;
        uint32_t k = 1;
        while (k < m && s[i + k] == nd[k]) k++;
        if (k == m) return (int)i;
    }
    return -1;
}

// boundary check for an occurrence at [pos, pos+m) inside the string [0, n)  (filter_phrase.go:247-266)
VL_HD bool phrase_boundaries_ok(const uint8_t* s, uint32_t n, uint32_t pos, uint32_t m, bool startsWithToken, bool endsWithToken) {
    int sz;
    if (startsWithToken && pos > 0) {
        int32_t r = s[pos - 1];
        if (r >= 0x80) r = decode_last_rune(s, pos, &sz);
        if (r == kRuneError || is_token_rune(r)) return false;
    }
    if (endsWithToken && pos + m < n) {
        int32_t r = s[pos + m];
        if (r >= 0x80) r = decode_rune(s + pos + m, n - pos - m, &sz);
        if (r == kRuneError || is_token_rune(r)) return false;
    }
    return true;
}
VL_HD bool needle_starts_with_token(const uint8_t* nd, uint32_t m) {
    if (m == 0) return false;
    int sz; int32_t r = nd[0];
    if (r >= 0x80) r = decode_rune(nd, m, &sz);
    return is_token_rune(r);
}
VL_HD bool needle_ends_with_token(const uint8_t* nd, uint32_t m) {
    if (m == 0) return false;
    int sz; int32_t r = nd[m - 1];
    if (r >= 0x80) r = decode_last_rune(nd, m, &sz);
    return is_token_rune(r);
}
VL_HDN bool match_phrase(const uint8_t* s, uint32_t n, const uint8_t* nd, uint32_t m) {
    if (m == 0) return n == 0;
    if (m > n) return false;
    bool st = needle_starts_with_token(nd, m), en = needle_ends_with_token(nd, m);
    uint32_t pos = 0;
    for (;;) {
        int k = find_bytes(s, n, nd, m, pos);
        if (k < 0) return false;
        if (phrase_boundaries_ok(s, n, (uint32_t)k, m, st, en)) return true;
        pos = (uint32_t)k + 1;
    }
}
VL_HDN bool match_prefix(const uint8_t* s, uint32_t n, const uint8_t* nd, uint32_t m) {
    if (m == 0) return n > 0;
    if (m > n) return false;
    bool st = needle_starts_with_token(nd, m);
    uint32_t pos = 0;
    for (;;) {
        int k = find_bytes(s, n, nd, m, pos);
        if (k < 0) return false;
        if (phrase_boundaries_ok(s, n, (uint32_t)k, m, st, false)) return true;
        pos = (uint32_t)k + 1;
    }
}
VL_HD bool bytes_equal(const uint8_t* a, uint32_t n, const uint8_t* b, uint32_t m) {
    if (n != m) return false;
    for (uint32_t i = 0; i < n; i++) if (a[i] != b[i]) return false;
    return true;
}

// ---- big-endian loads ------------------------------------------------------------------------------------------------
VL_HD uint32_t ld_be16(const uint8_t* p) { return ((uint32_t)p[0] << 8) | p[1]; }
VL_HD uint32_t ld_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
VL_HD uint64_t ld_be64(const uint8_t* p) { return ((uint64_t)ld_be32(p) << 32) | ld_be32(p + 4); }

// ---- number -> string (values_encoder.go:1367-1422); each returns the length written into buf (>= 32 bytes) -------------
VL_HD int fmt_u64(uint8_t* buf, uint64_t v) {
    uint8_t tmp[20]; int n = 0;
    do { tmp[n++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
    for (int i = 0; i < n; i++) buf[i] = tmp[n - 1 - i];
    return n;
}
VL_HD int fmt_i64(uint8_t* buf, int64_t v) {
    if (v < 0) { buf[0] = '-'; return 1 + fmt_u64(buf + 1, (uint64_t)0 - (uint64_t)v); }
    return fmt_u64(buf, (uint64_t)v);
}
VL_HD int fmt_ipv4(uint8_t* buf, uint32_t ip) {
    int n = 0;
    n += fmt_u64(buf + n, ip >> 24); buf[n++] = '.';
    n += fmt_u64(buf + n, (ip >> 16) & 0xFF); buf[n++] = '.';
    n += fmt_u64(buf + n, (ip >> 8) & 0xFF); buf[n++] = '.';
    n += fmt_u64(buf + n, ip & 0xFF);
    return n;
}
VL_HD void fmt_pad(uint8_t* buf, uint32_t v, int width) { for (int i = width - 1; i >= 0; i--) { buf[i] = (uint8_t)('0' + v % 10); v /= 10; } }
// time.Unix(0,ns).UTC().AppendFormat("2006-01-02T15:04:05.000Z")  (years outside 0..9999 cannot occur: |ns| < 2^63)
VL_HDN int fmt_iso8601(uint8_t* buf, int64_t nsecs) {
    int64_t secs = nsecs / 1000000000LL, rem = nsecs % 1000000000LL;
    if (rem < 0) { rem += 1000000000LL; secs -= 1; }
    int64_t days = secs / 86400, sod = secs % 86400;
    if (sod < 0) { sod += 86400; days -= 1; }
    int64_t z = days + 719468;
    int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    uint32_t doe = (uint32_t)(z - era * 146097);
    uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    int64_t y = (int64_t)yoe + era * 400;
    uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    uint32_t mp = (5 * doy + 2) / 153;
    uint32_t d = doy - (153 * mp + 2) / 5 + 1;
    uint32_t m = mp < 10 ? mp + 3 : mp - 9;
    y += (m <= 2);
    fmt_pad(buf, (uint32_t)y, 4); buf[4] = '-'; fmt_pad(buf + 5, m, 2); buf[7] = '-'; fmt_pad(buf + 8, d, 2); buf[10] = 'T';
    fmt_pad(buf + 11, (uint32_t)(sod / 3600), 2); buf[13] = ':'; fmt_pad(buf + 14, (uint32_t)((sod / 60) % 60), 2); buf[16] = ':';
    fmt_pad(buf + 17, (uint32_t)(sod % 60), 2); buf[19] = '.'; fmt_pad(buf + 20, (uint32_t)(rem / 1000000LL), 3); buf[23] = 'Z';
    return 24;
}
// marshalTimestampRFC3339NanoString in UTC: "2006-01-02T15:04:05" (fmt_iso8601's first 19 bytes), the fraction without its trailing zeros, "Z"
VL_HDN int fmt_rfc3339nano(uint8_t* buf, int64_t nsecs) {
    fmt_iso8601(buf, nsecs);
    int n = 19;
    int64_t frac = nsecs % 1000000000LL;
    if (frac < 0) frac += 1000000000LL;
    if (frac) {
        buf[n++] = '.'; fmt_pad(buf + n, (uint32_t)frac, 9); n += 9;
        while (buf[n - 1] == '0') n--;
    }
    buf[n++] = 'Z';
    return n;
}

// ---- predicates of the range / length filters ------------------------------------------------------------------------------------------
// utf8.RuneCountInString (matchLenRange, filter_len_range.go:333-336): every invalid byte counts as one rune
VL_HDN uint64_t rune_count(const uint8_t* s, uint32_t n) {
    uint64_t c = 0;
    for (uint32_t i = 0; i < n;) { if (s[i] < 0x80) { i++; c++; continue; } int w; decode_rune(s + i, n - i, &w); i += (uint32_t)w; c++; }
    return c;
}
// Go string comparison: bytewise, the shorter string first on a tie (-1, 0, 1)
VL_HDN int bytes_cmp(const uint8_t* a, uint32_t n, const uint8_t* b, uint32_t m) {
    uint32_t k = n < m ? n : m;
    for (uint32_t i = 0; i < k; i++) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return n == m ? 0 : n < m ? -1 : 1;
}
// tryParseIPv4 (values_encoder.go:675-730) over tryParseDateUint64 (:588-619), whose two-character fast path checks the first digit only
VL_HDN bool parse_date_u64_hd(const uint8_t* s, uint32_t n, uint64_t* out) {
    if (n == 0 || n > 9) return false;
    if (n == 2) { if (s[0] < '0' || s[0] > '9') return false; *out = 10ull * (uint8_t)(s[0] - '0') + (uint8_t)(s[1] - (uint8_t)'0'); return true; }
    uint64_t v = 0;
    for (uint32_t i = 0; i < n; i++) { if (s[i] < '0' || s[i] > '9') return false; v = v * 10 + (uint64_t)(s[i] - '0'); }
    *out = v; return true;
}
VL_HDN bool parse_ipv4_hd(const uint8_t* s, uint32_t n, uint32_t* out) {
    if (n < 7 || n > 15) return false;
    uint32_t dots = 0; for (uint32_t i = 0; i < n; i++) dots += s[i] == '.';
    if (dots != 3) return false;
    uint32_t ip = 0, pos = 0;
    for (int k = 0; k < 4; k++) {
        uint32_t e = pos;
        if (k < 3) { while (s[e] != '.') e++; if (e == pos || e - pos > 3) return false; } else e = n;
        uint64_t v;
        if (!parse_date_u64_hd(s + pos, e - pos, &v) || v > 255) return false;
        ip = (ip << 8) | (uint32_t)v;
        pos = e + 1;
    }
    *out = ip; return true;
}

// the per-value predicate of the filter kinds 9..12 (include/vlscan.h); a = needle, b = second needle (string_range: maxValue)
VL_HDN bool range_predicate(int kind, const uint8_t* s, uint32_t n, const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn, uint64_t aux0, uint64_t aux1) {
    switch (kind) {
    case 9: return n >= an && bytes_equal(s, an, a, an);                                   // matchExactPrefix filter_exact_prefix.go:275-277
    case 10: { uint64_t c = rune_count(s, n); return c >= aux0 && c <= aux1; }             // matchLenRange filter_len_range.go:333-336
    case 11: return bytes_cmp(s, n, a, an) >= 0 && bytes_cmp(s, n, b, bn) < 0;             // matchStringRange filter_string_range.go:226-230
    case 12: { uint32_t ip; return parse_ipv4_hd(s, n, &ip) && ip >= aux0 && ip <= aux1; }  // matchIPv4Range filter_ipv4_range.go:167-173
    }
    return false;
}

// ---- float64 -> shortest decimal text: strconv.AppendFloat(dst, f, 'f', -1, 64) (marshalFloat64String, values_encoder.go:1397-1399) ----
// Shortest digits that round-trip (Ryu, Adams 2018: the same digit string Go's shortest formatter produces), printed in fixed notation
// without exponent.  Tables generated by tools/gen_ryu_tables.py.  Returns the length (<= 344 bytes incl. sign).
#include "ryu_tables.inc"
static const uint64_t H_RYU_POW5_INV_SPLIT[342][2] = { VL_RYU_POW5_INV_SPLIT_INIT };
static const uint64_t H_RYU_POW5_SPLIT[326][2] = { VL_RYU_POW5_SPLIT_INIT };
#ifdef __CUDACC__
static __device__ const uint64_t D_RYU_POW5_INV_SPLIT[342][2] = { VL_RYU_POW5_INV_SPLIT_INIT };
static __device__ const uint64_t D_RYU_POW5_SPLIT[326][2] = { VL_RYU_POW5_SPLIT_INIT };
#endif
#define VL_FMT_F64_MAX 352

VL_HD uint64_t umul128(uint64_t a, uint64_t b, uint64_t* hi) {
#ifdef __CUDA_ARCH__
    *hi = __umul64hi(a, b); return a * b;
#else
    unsigned __int128 p = (unsigned __int128)a * b; *hi = (uint64_t)(p >> 64); return (uint64_t)p;
#endif
}
VL_HD uint64_t ryu_mul_shift64(uint64_t m, uint64_t mul0, uint64_t mul1, int j) {
    uint64_t hi0, hi2;
    (void)umul128(m, mul0, &hi0);
    uint64_t lo2 = umul128(m, mul1, &hi2);
    uint64_t sum = hi0 + lo2;
    if (sum < hi0) hi2++;
    int dist = j - 64;
    return dist == 0 ? sum : (hi2 << (64 - dist)) | (sum >> dist);
}
VL_HD uint32_t ryu_pow5_factor(uint64_t v) { uint32_t c = 0; for (;;) { uint64_t q = v / 5; if (v - 5 * q != 0) break; v = q; c++; } return c; }
VL_HD uint32_t ryu_pow5bits(int32_t e) { return (uint32_t)(((e * 1217359) >> 19) + 1); }
VL_HD uint32_t ryu_log10_pow2(int32_t e) { return (uint32_t)((e * 78913) >> 18); }
VL_HD uint32_t ryu_log10_pow5(int32_t e) { return (uint32_t)((e * 732923) >> 20); }

// shortest decimal: value == digits * 10^exp10 (digits has no sign; value != 0, finite)
VL_HDN void ryu_d2d(uint64_t mant, uint32_t expo, uint64_t* digits, int32_t* exp10) {
    int32_t e2; uint64_t m2;
    if (expo == 0) { e2 = 1 - 1023 - 52 - 2; m2 = mant; } else { e2 = (int32_t)expo - 1023 - 52 - 2; m2 = (1ull << 52) | mant; }
    const bool acceptBounds = (m2 & 1) == 0;
    const uint64_t mv = 4 * m2;
    const uint32_t mmShift = mant != 0 || expo <= 1;
    uint64_t vr, vp, vm; int32_t e10;
    bool vmTZ = false, vrTZ = false;
    if (e2 >= 0) {
        const uint32_t q = ryu_log10_pow2(e2) - (e2 > 3);
        e10 = (int32_t)q;
        const int32_t k = VL_RYU_POW5_INV_BITCOUNT + (int32_t)ryu_pow5bits((int32_t)q) - 1;
        const int32_t i = -e2 + (int32_t)q + k;
#ifdef __CUDA_ARCH__
        const uint64_t m0 = D_RYU_POW5_INV_SPLIT[q][0], m1 = D_RYU_POW5_INV_SPLIT[q][1];
#else
        const uint64_t m0 = H_RYU_POW5_INV_SPLIT[q][0], m1 = H_RYU_POW5_INV_SPLIT[q][1];
#endif
        vr = ryu_mul_shift64(4 * m2, m0, m1, i); vp = ryu_mul_shift64(4 * m2 + 2, m0, m1, i); vm = ryu_mul_shift64(4 * m2 - 1 - mmShift, m0, m1, i);
        if (q <= 21) {
            const uint32_t mvMod5 = (uint32_t)(mv % 5);
            if (mvMod5 == 0) vrTZ = ryu_pow5_factor(mv) >= q;
            else if (acceptBounds) vmTZ = ryu_pow5_factor(mv - 1 - mmShift) >= q;
            else vp -= ryu_pow5_factor(mv + 2) >= q;
        }
    } else {
        const uint32_t q = ryu_log10_pow5(-e2) - (-e2 > 1);
        e10 = (int32_t)q + e2;
        const int32_t i = -e2 - (int32_t)q;
        const int32_t k = (int32_t)ryu_pow5bits(i) - VL_RYU_POW5_BITCOUNT;
        const int32_t j = (int32_t)q - k;
#ifdef __CUDA_ARCH__
        const uint64_t m0 = D_RYU_POW5_SPLIT[i][0], m1 = D_RYU_POW5_SPLIT[i][1];
#else
        const uint64_t m0 = H_RYU_POW5_SPLIT[i][0], m1 = H_RYU_POW5_SPLIT[i][1];
#endif
        vr = ryu_mul_shift64(4 * m2, m0, m1, j); vp = ryu_mul_shift64(4 * m2 + 2, m0, m1, j); vm = ryu_mul_shift64(4 * m2 - 1 - mmShift, m0, m1, j);
        if (q <= 1) {
            vrTZ = true;
            if (acceptBounds) vmTZ = mmShift == 1; else --vp;
        } else if (q < 63) vrTZ = (mv & ((1ull << q) - 1)) == 0;
    }
    int32_t removed = 0; uint32_t last = 0; uint64_t out;
    if (vmTZ || vrTZ) {
        while (vp / 10 > vm / 10) { vmTZ &= vm % 10 == 0; vrTZ &= last == 0; last = (uint32_t)(vr % 10); vr /= 10; vp /= 10; vm /= 10; removed++; }
        if (vmTZ) while (vm % 10 == 0) { vrTZ &= last == 0; last = (uint32_t)(vr % 10); vr /= 10; vp /= 10; vm /= 10; removed++; }
        if (vrTZ && last == 5 && vr % 2 == 0) last = 4;   // round even when exactly halfway
        out = vr + ((vr == vm && (!acceptBounds || !vmTZ)) || last >= 5);
    } else {
        bool roundUp = false;
        while (vp / 10 > vm / 10) { roundUp = vr % 10 >= 5; vr /= 10; vp /= 10; vm /= 10; removed++; }
        out = vr + (vr == vm || roundUp);
    }
    *digits = out; *exp10 = e10 + removed;
}

VL_HDN int fmt_f64(uint8_t* buf, uint64_t bits) {
    const bool neg = bits >> 63;
    const uint64_t mant = bits & ((1ull << 52) - 1);
    const uint32_t expo = (uint32_t)((bits >> 52) & 0x7FF);
    int n = 0;
    if (expo == 0x7FF) {   // strconv: "NaN", "+Inf", "-Inf"
        const char* s = mant ? "NaN" : (neg ? "-Inf" : "+Inf");
        while (s[n]) { buf[n] = (uint8_t)s[n]; n++; }
        return n;
    }
    if (neg) buf[n++] = '-';
    if (expo == 0 && mant == 0) { buf[n++] = '0'; return n; }
    uint64_t dig; int32_t e10;
    ryu_d2d(mant, expo, &dig, &e10);
    uint8_t d[20]; int nd = 0;
    while (dig) { d[nd++] = (uint8_t)('0' + dig % 10); dig /= 10; }   // least significant first
    if (e10 >= 0) {
        for (int i = nd - 1; i >= 0; i--) buf[n++] = d[i];
        for (int i = 0; i < e10; i++) buf[n++] = '0';
    } else {
        int point = nd + e10;   // digits before the decimal point
        if (point > 0) {
            for (int i = nd - 1; i >= 0; i--) { if (nd - 1 - i == point) buf[n++] = '.'; buf[n++] = d[i]; }
        } else {
            buf[n++] = '0'; buf[n++] = '.';
            for (int i = 0; i < -point; i++) buf[n++] = '0';
            for (int i = nd - 1; i >= 0; i--) buf[n++] = d[i];
        }
    }
    return n;
}

// ---- `_time` buckets of `stats by (_time:step offset off)`: truncateTimestamp (lib/logstorage/block_result.go:818-848) -------------------
// Go's int64 arithmetic wraps, so every sum and product here is done on uint64.  Month / year buckets go through the UTC civil date
// (truncateTimestampToMonth / ToYear :2641-2649, time.Date(...).UnixNano(), which wraps the same way near 1677 and 2262).
enum { BUCKET_PLAIN = 0, BUCKET_WEEK = 1, BUCKET_MONTH = 2, BUCKET_YEAR = 3 };
static const int64_t kNsPerDay = 86400ll * 1000000000ll;
VL_HD int64_t days_from_civil(int64_t y, uint32_t m, uint32_t d) {   // proleptic Gregorian, days since 1970-01-01
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const int64_t yoe = y - era * 400;
    const int64_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
    const int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}
VL_HD void civil_from_days(int64_t z, int64_t* y, uint32_t* m) {
    z += 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const int64_t doe = z - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const int64_t mp = (5 * doy + 2) / 153;
    *m = (uint32_t)(mp < 10 ? mp + 3 : mp - 9);
    *y = yoe + era * 400 + (*m <= 2);
}
// step <= 0 counts as 1 (getBucketedTimestampValues :763-766); `calendar` is BUCKET_*
VL_HD int64_t truncate_timestamp(int64_t ts, int64_t step, int64_t offset, uint32_t calendar) {
    if (step <= 0) step = 1;
    uint64_t off = (uint64_t)offset;
    if (calendar == BUCKET_WEEK) off += 4ull * (uint64_t)kNsPerDay;   // weeks start on Monday
    const uint64_t t = (uint64_t)ts - off;
    const int64_t st = (int64_t)t;
    if (calendar == BUCKET_MONTH || calendar == BUCKET_YEAR) {
        int64_t days = st / kNsPerDay;
        if (st % kNsPerDay < 0) days--;
        int64_t y; uint32_t m;
        civil_from_days(days, &y, &m);
        const int64_t first = days_from_civil(y, calendar == BUCKET_YEAR ? 1 : m, 1);
        return (int64_t)((uint64_t)first * (uint64_t)kNsPerDay + off);
    }
    int64_t r = st % step;
    if (r < 0) r += step;
    return (int64_t)(t - (uint64_t)r + off);
}

}  // namespace vl
