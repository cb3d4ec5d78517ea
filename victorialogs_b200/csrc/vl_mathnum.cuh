// parseMathNumber on the device (and, as the same source, on the host for CPU tests): the value -> float64 conversion behind range(), le_field()
// and lt_field() on string-like values (lib/logstorage/pipe_math.go:1066-1080).  What it is made of:
//   tryParseNumber, isLikelyNumber              lib/logstorage/block_result.go:2710-2752
//   isNumberPrefix                              lib/logstorage/parser.go:3077-3097
//   tryParseFloat64Prefix / tryParseFloat64     lib/logstorage/values_encoder.go:761-850
//   tryParseBytes, addInt64NoOverflow           lib/logstorage/values_encoder.go:855-974
//   tryParseDuration                            lib/logstorage/values_encoder.go:990-1061
//   TryParseTimestampRFC3339Nano, parseTimezoneOffset, tryParseHHMM   lib/logstorage/values_encoder.go:340-423
//   tryParseIPv4, tryParseDateUint64, tryParseUint64, tryParseTimestampSecs   lib/logstorage/values_encoder.go:466-730
// and, from Go's standard library (not under the reference tree; restated from its documented behaviour): strconv.ParseFloat(s, 64) - decimal and
// hexadecimal floats, "inf" / "infinity", `_` separators under the base-prefix rule - and strconv.ParseInt(s, 0, 64).  Decimal -> double is
// exact: the digits go through a big-decimal that is shifted by powers of two until the 53-bit mantissa can be read off and rounded half to even
// (the algorithm of strconv's decimal.go, without its shortcut tables).  No allocation, no recursion; one value in, one double out.
// A timestamp without `Z` or a numeric offset takes the process' local zone in the reference; like the oracle this code uses UTC.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "vl_hd.cuh"

#ifdef __CUDACC__
#define VLM_HD static __host__ __device__
#else
#define VLM_HD static inline
#endif

namespace vl {
namespace mn {

struct Span { const uint8_t* p; uint32_t n; };
VLM_HD Span sub(Span s, uint32_t from) { return Span{s.p + from, s.n - from}; }
VLM_HD Span head(Span s, uint32_t len) { return Span{s.p, len}; }
VLM_HD bool has_prefix(Span s, const char* lit, uint32_t ln) { if (s.n < ln) return false; for (uint32_t i = 0; i < ln; i++) if (s.p[i] != (uint8_t)lit[i]) return false; return true; }
VLM_HD int find_byte(Span s, uint8_t c) { for (uint32_t i = 0; i < s.n; i++) if (s.p[i] == c) return (int)i; return -1; }
VLM_HD uint32_t count_byte(Span s, uint8_t c) { uint32_t k = 0; for (uint32_t i = 0; i < s.n; i++) k += s.p[i] == c; return k; }

// tryParseUint64 values_encoder.go:553-585
VLM_HD bool parse_u64(Span s, uint64_t* out) {
    if (s.n == 0 || s.n > 26) return false;
    if (s.n > 1 && s.p[0] == '0') return false;
    uint64_t n = 0;
    for (uint32_t i = 0; i < s.n; i++) {
        const uint8_t c = s.p[i];
        if (c == '_') continue;
        if (c < '0' || c > '9') return false;
        if (n > 0xFFFFFFFFFFFFFFFFull / 10) return false;
        n *= 10;
        const uint64_t n1 = n + (uint64_t)(c - '0');
        if (n1 < n) return false;
        n = n1;
    }
    *out = n;
    return true;
}
// tryParseDateUint64 :588-619 (the two-character fast path checks only its first digit: byte arithmetic wraps)
VLM_HD bool parse_date_u64(Span s, uint64_t* out) {
    if (s.n == 0 || s.n > 9) return false;
    if (s.n == 2) { if (s.p[0] < '0' || s.p[0] > '9') return false; *out = 10ull * (uint8_t)(s.p[0] - '0') + (uint8_t)(s.p[1] - (uint8_t)'0'); return true; }
    uint64_t n = 0;
    for (uint32_t i = 0; i < s.n; i++) { if (s.p[i] < '0' || s.p[i] > '9') return false; n = n * 10 + (uint64_t)(s.p[i] - '0'); }
    *out = n;
    return true;
}
VLM_HD double pow10_neg(int n) {   // math.Pow10(n) for n in [-31, 0]: exact literals
    const double t[32] = {1e0, 1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7, 1e-8, 1e-9, 1e-10, 1e-11, 1e-12, 1e-13, 1e-14, 1e-15, 1e-16,
                          1e-17, 1e-18, 1e-19, 1e-20, 1e-21, 1e-22, 1e-23, 1e-24, 1e-25, 1e-26, 1e-27, 1e-28, 1e-29, 1e-30, 1e-31};
    return (n <= 0 && n >= -31) ? t[-n] : 0.0;
}
// tryParseFloat64Internal :788-850; exact = true adds the 2^53 bound on plain integers
VLM_HD bool parse_f64_internal(Span s, bool exact, double* out) {
    if (s.n == 0 || s.n > 27) return false;
    const bool minus = s.p[0] == '-';
    if (minus) s = sub(s, 1);
    const int dot = find_byte(s, '.');
    if (dot < 0) {
        uint64_t v;
        if (!parse_u64(s, &v)) return false;
        if (exact && v >= (1ull << 53)) return false;
        const double f = (double)v;
        *out = minus ? -f : f;
        return true;
    }
    if (dot == 0 || (uint32_t)dot == s.n - 1) return false;
    const Span si = head(s, (uint32_t)dot), sf = sub(s, (uint32_t)dot + 1);
    uint64_t ni;
    if (!parse_u64(si, &ni)) return false;
    uint32_t k = 0;
    while (k + 1 < sf.n && sf.p[k] == '0') k++;
    uint64_t nf;
    if (!parse_u64(sub(sf, k), &nf)) return false;
    const int us = (int)count_byte(sf, '_');
    const double f = fma((double)nf, pow10_neg(us - (int)sf.n), (double)ni);
    *out = minus ? -f : f;
    return true;
}
// tryParseFloat64Prefix :762-773
VLM_HD bool parse_f64_prefix(Span s, double* f, Span* tail) {
    uint32_t i = 0;
    while (i < s.n && ((s.p[i] >= '0' && s.p[i] <= '9') || s.p[i] == '.' || s.p[i] == '_')) i++;
    if (i == 0) return false;
    if (!parse_f64_internal(head(s, i), false, f)) return false;
    *tail = sub(s, i);
    return true;
}
VLM_HD int64_t int64_of_float(double f) {   // int64(f) as amd64 computes it (CVTTSD2SQ: out of range and NaN -> 0x8000000000000000)
    if (!(f == f) || f >= 9223372036854775808.0 || f < -9223372036854775808.0) return (int64_t)0x8000000000000000ull;
    return (int64_t)f;
}
VLM_HD int64_t add_no_overflow(int64_t n, double f) {   // addInt64NoOverflow :968-974
    const int64_t x = int64_of_float(f);
    if (n < 0 || x < 0 || x > 0x7FFFFFFFFFFFFFFFll - n) return 0x7FFFFFFFFFFFFFFFll;
    return n + x;
}
// tryParseDuration :990-1061
VLM_HD bool parse_duration(Span s, int64_t* out) {
    if (s.n == 0) return false;
    const bool minus = s.p[0] == '-';
    if (minus) s = sub(s, 1);
    int64_t nsecs = 0;
    while (s.n) {
        double f; Span tail;
        if (!parse_f64_prefix(s, &f, &tail)) return false;
        s = tail;
        if (s.n == 0) return false;
        if (s.n >= 3 && s.p[0] == 0xC2 && s.p[1] == 0xB5 && s.p[2] == 's') { nsecs = add_no_overflow(nsecs, f * 1e3); s = sub(s, 3); continue; }   // "µs"
        if (s.n >= 2) {
            if (s.p[0] == 'm' && s.p[1] == 's') { nsecs = add_no_overflow(nsecs, f * 1e6); s = sub(s, 2); continue; }
            if (s.p[0] == 'n' && s.p[1] == 's') { nsecs = add_no_overflow(nsecs, f); s = sub(s, 2); continue; }
        }
        double unit;
        switch (s.p[0]) {
        case 'y': unit = 365 * 24 * 3600e9; break; case 'w': unit = 7 * 24 * 3600e9; break; case 'd': unit = 24 * 3600e9; break;
        case 'h': unit = 3600e9; break; case 'm': unit = 60e9; break; case 's': unit = 1e9; break;
        default: return false;
        }
        nsecs = add_no_overflow(nsecs, f * unit); s = sub(s, 1);
    }
    *out = minus ? -nsecs : nsecs;
    return true;
}
// tryParseBytes :855-966
VLM_HD bool parse_bytes(Span s, int64_t* out) {
    if (s.n == 0) return false;
    const bool minus = s.p[0] == '-';
    if (minus) s = sub(s, 1);
    int64_t n = 0;
    while (s.n) {
        double f; Span tail;
        if (!parse_f64_prefix(s, &f, &tail)) return false;
        if (tail.n == 0 && f != floor(f)) return false;   // no fractional numbers without a suffix
        s = tail;
        if (s.n == 0) { n = add_no_overflow(n, f); continue; }
        double mul = 0; uint32_t ln = 0;
        const uint8_t c0 = s.p[0], c1 = s.n > 1 ? s.p[1] : 0, c2 = s.n > 2 ? s.p[2] : 0;
        const double bin = c0 == 'K' ? 1024.0 : c0 == 'M' ? 1048576.0 : c0 == 'G' ? 1073741824.0 : c0 == 'T' ? 1099511627776.0 : 0.0;
        const double dec = c0 == 'K' ? 1e3 : c0 == 'M' ? 1e6 : c0 == 'G' ? 1e9 : c0 == 'T' ? 1e12 : 0.0;
        if (bin != 0.0 && c1 == 'i' && c2 == 'B') { mul = bin; ln = 3; }
        else if (bin != 0.0 && c1 == 'i') { mul = bin; ln = 2; }
        else if (dec != 0.0 && c1 == 'B') { mul = dec; ln = 2; }
        else if (c0 == 'B') { mul = 1.0; ln = 1; }
        else if (dec != 0.0) { mul = dec; ln = 1; }
        else return false;
        n = add_no_overflow(n, f * mul); s = sub(s, ln);
    }
    *out = minus ? -n : n;
    return true;
}
// isNumberPrefix parser.go:3077-3097, isLikelyNumber block_result.go:2739-2752
VLM_HD bool is_number_prefix(Span s) {
    if (s.n == 0) return false;
    if (s.p[0] == '-' || s.p[0] == '+') { s = sub(s, 1); if (s.n == 0) return false; }
    if (s.n == 3 && (s.p[0] | 0x20) == 'i' && (s.p[1] | 0x20) == 'n' && (s.p[2] | 0x20) == 'f') return true;
    if (s.p[0] == '.') { s = sub(s, 1); if (s.n == 0) return false; }
    return s.p[0] >= '0' && s.p[0] <= '9';
}
VLM_HD bool is_likely_number(Span s) {
    if (!is_number_prefix(s)) return false;
    if (count_byte(s, '.') > 1) return false;                                 // likely an IP address
    if (find_byte(s, ':') >= 0 || count_byte(s, '-') > 2) return false;       // likely a timestamp
    return true;
}
// strconv underscoreOK: `_` only between digits or right after a base prefix
VLM_HD bool underscores_ok(Span s) {
    char saw = '^'; uint32_t i = 0;
    if (s.n && (s.p[0] == '-' || s.p[0] == '+')) i = 1;
    bool hex = false;
    if (s.n - i >= 2 && s.p[i] == '0' && ((s.p[i + 1] | 0x20) == 'b' || (s.p[i + 1] | 0x20) == 'o' || (s.p[i + 1] | 0x20) == 'x')) { hex = (s.p[i + 1] | 0x20) == 'x'; i += 2; saw = '0'; }
    for (; i < s.n; i++) {
        const uint8_t c = s.p[i];
        if ((c >= '0' && c <= '9') || (hex && (c | 0x20) >= 'a' && (c | 0x20) <= 'f')) { saw = '0'; continue; }
        if (c == '_') { if (saw != '0') return false; saw = '_'; continue; }
        if (saw == '_') return false;
        saw = '!';
    }
    return saw != '_';
}

// ---- exact decimal -> double: strconv's decimal (decimal.go) without its shortcut tables -------------------------------------------------------------
struct BigDec { uint8_t d[840]; int nd, dp; bool trunc; };   // value = 0.d[0]d[1]... x 10^dp; digits beyond 800 are dropped, `trunc` remembers a non-zero one
VLM_HD void bd_trim(BigDec& a) { while (a.nd > 0 && a.d[a.nd - 1] == 0) a.nd--; if (a.nd == 0) a.dp = 0; }
VLM_HD void bd_right_shift(BigDec& a, unsigned k) {   // a /= 2^k, k <= 60
    int r = 0, w = 0; uint64_t n = 0;
    for (; (n >> k) == 0; r++) {
        if (r >= a.nd) { if (n == 0) { a.nd = 0; return; } while ((n >> k) == 0) { n *= 10; r++; } break; }
        n = n * 10 + a.d[r];
    }
    a.dp -= r - 1;
    const uint64_t mask = (1ull << k) - 1;
    for (; r < a.nd; r++) { const uint64_t dig = n >> k; n &= mask; a.d[w++] = (uint8_t)dig; n = n * 10 + a.d[r]; }
    while (n > 0) { const uint64_t dig = n >> k; n &= mask; if (w < 800) a.d[w++] = (uint8_t)dig; else if (dig > 0) a.trunc = true; n *= 10; }
    a.nd = w;
    bd_trim(a);
}
VLM_HD void bd_left_shift(BigDec& a, unsigned k) {   // a *= 2^k, k <= 60: right to left with carry, into a copy shifted by the most digits 2^60 can add (19)
    const int delta = 19;
    uint64_t n = 0;
    int w = a.nd + delta;
    for (int r = a.nd - 1; r >= 0; r--) {
        n += (uint64_t)a.d[r] << k;
        const uint64_t q = n / 10, rem = n - 10 * q;
        w--;
        if (w < 800) a.d[w] = (uint8_t)rem; else if (rem) a.trunc = true;
        n = q;
    }
    while (n > 0) { const uint64_t q = n / 10, rem = n - 10 * q; w--; if (w < 800) a.d[w] = (uint8_t)rem; else if (rem) a.trunc = true; n = q; }
    // digits now sit at [w, nd + delta): move them to the front
    const int total = a.nd + delta - w, keep = total < 800 ? total : 800;
    for (int i = 0; i < keep; i++) a.d[i] = a.d[w + i];
    a.dp += total - a.nd;
    a.nd = keep;
    bd_trim(a);
}
VLM_HD void bd_shift(BigDec& a, int k) {
    if (a.nd == 0) return;
    while (k > 60) { bd_left_shift(a, 60); k -= 60; }
    if (k > 0) bd_left_shift(a, (unsigned)k);
    while (k < -60) { bd_right_shift(a, 60); k += 60; }
    if (k < 0) bd_right_shift(a, (unsigned)-k);
}
VLM_HD uint64_t bd_rounded_integer(const BigDec& a) {   // the integer part, rounded half to even (strconv decimal.RoundedInteger)
    if (a.dp > 20) return 0xFFFFFFFFFFFFFFFFull;
    uint64_t n = 0; int i = 0;
    for (; i < a.dp && i < a.nd; i++) n = n * 10 + a.d[i];
    for (; i < a.dp; i++) n *= 10;
    // shouldRoundUp(a, dp)
    bool up = false;
    if (a.dp >= 0 && a.dp < a.nd) {
        if (a.d[a.dp] == 5 && a.dp + 1 == a.nd) up = a.trunc || (a.dp > 0 && (a.d[a.dp - 1] & 1));   // exactly halfway: to even (unless digits were dropped)
        else up = a.d[a.dp] >= 5;
    }
    return up ? n + 1 : n;
}
// digits (ascii, no sign) with an optional '.', decimal exponent e10 added on top -> the nearest double; *range = the value overflows
VLM_HD double bd_to_double(const uint8_t* digs, uint32_t n, int e10, bool* range) {
    BigDec a; a.nd = 0; a.dp = 0; a.trunc = false;
    // strconv readFloat: leading zeros are skipped (each moves the point left), the point position is the number of significant digits in
    // front of it, at most 800 digits are kept and a dropped non-zero digit is remembered
    int nd_all = 0, dp = 0; bool sawdot = false;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t c = digs[i];
        if (c == '_') continue;
        if (c == '.') { sawdot = true; dp = nd_all; continue; }
        if (c == '0' && nd_all == 0) { dp--; continue; }
        nd_all++;
        if (a.nd < 800) a.d[a.nd++] = (uint8_t)(c - '0'); else if (c != '0') a.trunc = true;
    }
    if (!sawdot) dp = nd_all;
    a.dp = dp + e10;
    bd_trim(a);
    *range = false;
    if (a.nd == 0) return 0.0;
    if (a.dp > 310) { *range = true; return INFINITY; }
    if (a.dp < -330) return 0.0;
    const int powtab[9] = {1, 3, 6, 9, 13, 16, 19, 23, 26};
    int exp = 0;
    while (a.dp > 0) { const int sft = a.dp >= 9 ? 27 : powtab[a.dp]; bd_shift(a, -sft); exp += sft; }
    while (a.dp < 0 || (a.dp == 0 && a.d[0] < 5)) { const int sft = -a.dp >= 9 ? 27 : powtab[-a.dp]; bd_shift(a, sft); exp -= sft; }
    exp--;   // the value is now in [1, 2) x 2^exp
    const int bias = -1023;
    if (exp < bias + 1) { const int sft = bias + 1 - exp; bd_shift(a, -sft); exp += sft; }
    if (exp - bias >= 2047) { *range = true; return INFINITY; }
    bd_shift(a, 53);
    uint64_t mant = bd_rounded_integer(a);
    if (mant == (2ull << 52)) { mant >>= 1; exp++; if (exp - bias >= 2047) { *range = true; return INFINITY; } }
    if ((mant & (1ull << 52)) == 0) exp = bias;   // denormal
    const uint64_t bits = (mant & ((1ull << 52) - 1)) | ((uint64_t)(exp - bias) << 52);
    double f; memcpy(&f, &bits, 8);
    return f;
}
// strconv.ParseFloat(s, 64) for strings that passed isLikelyNumber
VLM_HD bool go_parse_float(Span s, double* out) {
    if (s.n == 0 || s.n > 4096) return false;
    if (find_byte(s, '_') >= 0 && !underscores_ok(s)) return false;
    uint32_t i = 0; bool neg = false;
    if (s.p[0] == '+' || s.p[0] == '-') { neg = s.p[0] == '-'; i = 1; }
    const Span u = sub(s, i);
    {   // inf / infinity, any case
        const char* w = "infinity"; bool m3 = u.n == 3, m8 = u.n == 8;
        for (uint32_t k = 0; k < u.n && k < 8; k++) if ((u.p[k] | 0x20) != (uint8_t)w[k]) { m3 = m8 = false; break; }
        if (m3 || m8) { *out = neg ? -INFINITY : INFINITY; return true; }
    }
    if (u.n >= 2 && u.p[0] == '0' && (u.p[1] | 0x20) == 'x') {
        // hexadecimal: 0x h* [. h*] p [+-] d+ ; at least one hex digit, the exponent is mandatory
        uint64_t mant = 0; int exp2 = 0; bool any = false, dot = false, sticky = false; uint32_t k = 2;
        for (; k < u.n; k++) {
            const uint8_t c = u.p[k];
            if (c == '_') continue;
            if (c == '.') { if (dot) return false; dot = true; continue; }
            const int dgt = (c >= '0' && c <= '9') ? c - '0' : ((c | 0x20) >= 'a' && (c | 0x20) <= 'f') ? (c | 0x20) - 'a' + 10 : -1;
            if (dgt < 0) break;
            any = true;
            if (mant >> 60) { sticky |= dgt != 0; if (!dot) exp2 += 4; }   // no room: the digit only moves the exponent / the sticky bit
            else { mant = (mant << 4) | (uint64_t)dgt; if (dot) exp2 -= 4; }
        }
        if (!any || k >= u.n || (u.p[k] | 0x20) != 'p') return false;
        k++;
        bool eneg = false;
        if (k < u.n && (u.p[k] == '+' || u.p[k] == '-')) { eneg = u.p[k] == '-'; k++; }
        if (k >= u.n) return false;
        int e = 0;
        for (; k < u.n; k++) { const uint8_t c = u.p[k]; if (c == '_') continue; if (c < '0' || c > '9') return false; if (e < 100000) e = e * 10 + (c - '0'); }
        exp2 += eneg ? -e : e;
        if (mant == 0) { *out = neg ? -0.0 : 0.0; return true; }
        // normalise to 64 bits, then round to 53 with sticky, handling denormals
        while (!(mant >> 63)) { mant <<= 1; exp2--; }
        int ex = exp2 + 63;                     // value = 1.xxx * 2^ex
        int drop = 11;                          // bits to drop for a normal number
        if (ex < -1022) drop += -1022 - ex;     // denormal: drop more
        if (ex > 1023) return false;            // out of range
        uint64_t m;
        if (drop > 64) m = 0;                                                                              // less than half of the smallest denormal
        else if (drop == 64) { const bool half = mant >> 63, rest = (mant << 1) != 0 || sticky; m = (half && rest) ? 1 : 0; }   // exactly half rounds to even: 0
        else {
            m = mant >> drop;
            const uint64_t rem = mant & ((1ull << drop) - 1), halfbit = 1ull << (drop - 1);
            if (rem > halfbit || (rem == halfbit && (sticky || (m & 1)))) m++;
        }
        uint64_t bits;
        if (ex < -1022) bits = m;   // denormal (m may have rounded up into the smallest normal: the bit pattern is right as it is)
        else { if (m >> 53) { m >>= 1; ex++; if (ex > 1023) return false; } bits = (m & ((1ull << 52) - 1)) | ((uint64_t)(ex + 1023) << 52); }
        double f; memcpy(&f, &bits, 8);
        *out = neg ? -f : f;
        return true;
    }
    // decimal: d* [. d*] [e [+-] d+], at least one digit
    uint32_t k = 0; bool any = false, dot = false;
    for (; k < u.n; k++) {
        const uint8_t c = u.p[k];
        if (c == '_') continue;
        if (c == '.') { if (dot) return false; dot = true; continue; }
        if (c < '0' || c > '9') break;
        any = true;
    }
    if (!any) return false;
    const uint32_t mant_len = k;
    int e10 = 0;
    if (k < u.n) {
        if ((u.p[k] | 0x20) != 'e') return false;
        k++;
        bool eneg = false;
        if (k < u.n && (u.p[k] == '+' || u.p[k] == '-')) { eneg = u.p[k] == '-'; k++; }
        if (k >= u.n) return false;
        for (; k < u.n; k++) { const uint8_t c = u.p[k]; if (c == '_') continue; if (c < '0' || c > '9') return false; if (e10 < 10000) e10 = e10 * 10 + (c - '0'); }
        if (eneg) e10 = -e10;
    }
    bool range = false;
    const double f = bd_to_double(u.p, mant_len, e10, &range);
    if (range) return false;   // ParseFloat reports a range error: not a number for tryParseNumber
    *out = neg ? -f : f;
    return true;
}
// strconv.ParseInt(s, 0, 64)
VLM_HD bool go_parse_int0(Span s, int64_t* out) {
    if (s.n == 0) return false;
    if (find_byte(s, '_') >= 0 && !underscores_ok(s)) return false;
    bool neg = false;
    if (s.p[0] == '+' || s.p[0] == '-') { neg = s.p[0] == '-'; s = sub(s, 1); }
    if (s.n == 0) return false;
    unsigned base = 10;
    if (s.p[0] == '0' && s.n >= 2) {
        const uint8_t pch = s.p[1] | 0x20;
        if (pch == 'x') { base = 16; s = sub(s, 2); } else if (pch == 'b') { base = 2; s = sub(s, 2); } else if (pch == 'o') { base = 8; s = sub(s, 2); } else { base = 8; s = sub(s, 1); }
        if (s.n == 0) return false;
    }
    uint64_t v = 0; bool any = false;
    const uint64_t lim = 1ull << 63;
    for (uint32_t i = 0; i < s.n; i++) {
        const uint8_t c = s.p[i];
        if (c == '_') continue;
        const unsigned d = (c >= '0' && c <= '9') ? (unsigned)(c - '0') : ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') ? (unsigned)((c | 0x20) - 'a' + 10) : 99u;
        if (d >= base) return false;
        if (v > (lim - d) / base) return false;   // v * base + d would exceed 2^63
        v = v * base + d; any = true;
    }
    if (!any) return false;
    if (!neg && v > lim - 1) return false;
    *out = neg ? (int64_t)(0 - v) : (int64_t)v;
    return true;
}
// tryParseNumber block_result.go:2710-2737
VLM_HD bool parse_number(Span s, double* out) {
    if (s.n == 0) return false;
    if (parse_f64_internal(s, false, out)) return true;
    int64_t n;
    if (parse_duration(s, &n)) { *out = (double)n; return true; }
    if (parse_bytes(s, &n)) { *out = (double)n; return true; }
    if (is_likely_number(s)) {
        if (go_parse_float(s, out)) return true;
        if (go_parse_int0(s, &n)) { *out = (double)n; return true; }
    }
    return false;
}
// time.Date(...).Unix() for UTC with Go's normalisation of out-of-range fields
VLM_HD int64_t date_unix(int64_t year, int64_t month, int64_t day, int64_t hour, int64_t min, int64_t sec) {
    int64_t m = month - 1;
    { if (m < 0) { int64_t k = (-m - 1) / 12 + 1; year -= k; m += k * 12; } if (m >= 12) { int64_t k = m / 12; year += k; m -= k * 12; } }
    { if (sec < 0) { int64_t k = (-sec - 1) / 60 + 1; min -= k; sec += k * 60; } if (sec >= 60) { int64_t k = sec / 60; min += k; sec -= k * 60; } }
    { if (min < 0) { int64_t k = (-min - 1) / 60 + 1; hour -= k; min += k * 60; } if (min >= 60) { int64_t k = min / 60; hour += k; min -= k * 60; } }
    { if (hour < 0) { int64_t k = (-hour - 1) / 24 + 1; day -= k; hour += k * 24; } if (hour >= 24) { int64_t k = hour / 24; day += k; hour -= k * 24; } }
    int64_t y = year; const unsigned mth = (unsigned)(m + 1);
    y -= mth <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const unsigned yoe = (unsigned)(y - era * 400);
    const unsigned doy = (153 * (mth + (mth > 2 ? -3 : 9)) + 2) / 5;
    const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    const int64_t days = era * 146097 + (int64_t)doe - 719468 + (day - 1);
    return days * 86400 + hour * 3600 + min * 60 + sec;
}
// tryParseTimestampSecs :466-551; consumes "YYYY-MM-DDTHH:MM:SS" from the front of *s
VLM_HD bool parse_timestamp_secs(Span* sp, int64_t* secs) {
    Span s = *sp; uint64_t n;
    if (s.n < 19) return false;
    if (s.p[4] != '-' || !parse_date_u64(head(s, 4), &n) || n < 1677 || n > 2262) return false;
    const int64_t year = (int64_t)n; s = sub(s, 5);
    if (s.p[2] != '-' || !parse_date_u64(head(s, 2), &n)) return false;
    const int64_t month = (int64_t)n; s = sub(s, 3);
    if ((s.p[2] != 'T' && s.p[2] != ' ') || !parse_date_u64(head(s, 2), &n)) return false;
    const int64_t day = (int64_t)n; s = sub(s, 3);
    if (s.p[2] != ':' || !parse_date_u64(head(s, 2), &n)) return false;
    const int64_t hour = (int64_t)n; s = sub(s, 3);
    if (s.p[2] != ':' || !parse_date_u64(head(s, 2), &n)) return false;
    const int64_t minute = (int64_t)n; s = sub(s, 3);
    if (!parse_date_u64(head(s, 2), &n)) return false;
    const int64_t second = (int64_t)n; s = sub(s, 2);
    const int64_t v = date_unix(year, month, day, hour, minute, second);
    if (v < -9223372036LL || v >= 9223372036LL) return false;
    *secs = v; *sp = s;
    return true;
}
// TryParseTimestampRFC3339Nano :340-381 (local zone == UTC)
VLM_HD bool parse_rfc3339nano(Span s, int64_t* out) {
    if (s.n < 19) return false;
    int64_t secs;
    if (!parse_timestamp_secs(&s, &secs)) return false;
    int64_t nsecs = secs * 1000000000LL;
    if (s.n && s.p[s.n - 1] == 'Z') s.n--;
    else {
        int at = -1;
        for (int i = (int)s.n - 1; i >= 0; i--) if (s.p[i] == '+' || s.p[i] == '-') { at = i; break; }
        if (at >= 0) {
            const Span off = sub(s, (uint32_t)at + 1);
            const bool minus = s.p[at] == '-';
            if (off.n != 5 || off.p[2] != ':') return false;
            uint64_t hh, mm;
            if (!parse_date_u64(head(off, 2), &hh) || hh > 24) return false;
            if (!parse_date_u64(sub(off, 3), &mm) || mm > 60) return false;
            const int64_t o = (int64_t)hh * 3600000000000LL + (int64_t)mm * 60000000000LL;
            nsecs -= minus ? -o : o;
            s.n = (uint32_t)at;
        }
    }
    if (s.n == 0) { *out = nsecs; return true; }
    if (s.p[0] == '.') s = sub(s, 1);
    const uint32_t digits = s.n;
    if (digits > 9) return false;
    uint64_t frac;
    if (!parse_date_u64(s, &frac)) return false;
    for (uint32_t i = digits; i < 9; i++) frac *= 10;
    *out = nsecs + (int64_t)frac;
    return true;
}
// tryParseIPv4 :675-730
VLM_HD bool parse_ipv4(Span s, uint32_t* out) {
    if (s.n < 7 || s.n > 15 || count_byte(s, '.') != 3) return false;
    uint32_t ip = 0;
    for (int k = 0; k < 3; k++) {
        const int n = find_byte(s, '.');
        if (n <= 0 || n > 3) return false;
        uint64_t v;
        if (!parse_date_u64(head(s, (uint32_t)n), &v) || v > 255) return false;
        ip = (ip << 8) | (uint32_t)v;
        s = sub(s, (uint32_t)n + 1);
    }
    uint64_t v;
    if (!parse_date_u64(s, &v) || v > 255) return false;
    *out = (ip << 8) | (uint32_t)v;
    return true;
}
// parseMathNumber pipe_math.go:1066-1080; NaN when the value is none of the forms
VLM_HD double parse_math_number(const uint8_t* p, uint32_t n) {
    const Span s{p, n};
    double f;
    if (parse_number(s, &f)) return f;
    int64_t ns;
    if (parse_rfc3339nano(s, &ns)) return (double)ns;
    uint32_t ip;
    if (parse_ipv4(s, &ip)) return (double)ip;
    uint64_t bits = 0x7FF8000000000001ull;   // math.NaN()
    memcpy(&f, &bits, 8);
    return f;
}
// tryParseInt64 values_encoder.go:622-645 (the facets key a '-' text by the same rule, vl_agg.cuh facet_text_key)
VLM_HD bool parse_i64(Span s, int64_t* out) {
    if (s.n == 0) return false;
    const bool minus = s.p[0] == '-';
    if (minus) s = sub(s, 1);
    uint64_t n;
    if (!parse_u64(s, &n)) return false;
    if (n >= (1ull << 63) && !(minus && n == (1ull << 63))) return false;
    *out = (int64_t)(minus ? 0 - n : n);
    return true;
}

}  // namespace mn

// ---- bucketed by-fields: `stats by (f:size offset off)` (getBucketedValue and the truncations, lib/logstorage/block_result.go:935-1764) --------
// The query's bucketSize and bucketOffset as every value kind reads them, converted once on the host (vlscan_hits_stats) by Go's float -> integer
// rules on amd64.  The float steps of trunc_f64 are separate IEEE operations on the device too: a fused multiply-add would round differently.
struct BucketSpec {
    uint32_t enabled, calendar;     // calendar: BUCKET_* (bucketSizeStr "week" / "month" / "year")
    uint64_t u64_size, u64_off;     // uint64(size) with 0 -> 1, uint64(int64(offset)): uint8..uint64 values
    int64_t i64_size, i64_off;      // int64(size) with <= 0 -> 1, int64(offset): integer and duration texts, timestamps
    int64_t i64_col_size;           // int64(size) with only 0 -> 1: int64 values (getBucketedInt64Values)
    uint32_t u32_size, u32_off;     // uint32(size) with 0 -> 1, uint32(int32(offset)): IPv4 values and texts
    double offset, p10;             // bucketOffset; math.Pow10(-e), e the exponent of decimal.FromFloat(size) (size <= 0 -> 1)
    int64_t size_p10;               // int64(size * p10), never 0 (the reference would divide by it)
};
#ifdef __CUDA_ARCH__
#define VLB_MUL(a, b) __dmul_rn(a, b)
#define VLB_ADD(a, b) __dadd_rn(a, b)
#define VLB_SUB(a, b) __dsub_rn(a, b)
#define VLB_DIV(a, b) __ddiv_rn(a, b)
#else
#define VLB_MUL(a, b) ((a) * (b))
#define VLB_ADD(a, b) ((a) + (b))
#define VLB_SUB(a, b) ((a) - (b))
#define VLB_DIV(a, b) ((a) / (b))
#endif
// truncateUint64 :1237-1249, truncateUint32 :1540-1553
VLM_HD uint64_t trunc_u64(uint64_t n, uint64_t size, uint64_t off) {
    if (off == 0) return n - n % size;
    if (off > n) return 0;
    n -= off;
    return n - n % size + off;
}
VLM_HD uint32_t trunc_u32(uint32_t n, uint32_t size, uint32_t off) { return (uint32_t)trunc_u64(n, size, off); }
// truncateInt64 :1333-1351, with Go's wrapping int64 arithmetic (and x % -1 == 0, where C leaves INT64_MIN % -1 undefined)
VLM_HD int64_t trunc_i64(int64_t n, int64_t size, int64_t off) {
    const uint64_t t = (uint64_t)n - (uint64_t)off;
    int64_t r = size == -1 ? 0 : (int64_t)t % size;
    if (r < 0) r = (int64_t)((uint64_t)r + (uint64_t)size);
    return (int64_t)(t - (uint64_t)r + (uint64_t)off);
}
// truncateFloat64 :1438-1456
VLM_HD double trunc_f64(double f, const BucketSpec& bk) {
    if (bk.offset != 0) f = VLB_SUB(f, bk.offset);
    int64_t fp = mn::int64_of_float(floor(VLB_MUL(f, bk.p10)));
    fp = (int64_t)((uint64_t)fp - (uint64_t)(fp % bk.size_p10));   // size_p10 is > 0 or INT64_MIN
    const double g = VLB_DIV((double)fp, bk.p10);
    return bk.offset != 0 ? VLB_ADD(g, bk.offset) : g;
}
VLM_HD uint64_t f64_bits(double f) { uint64_t u; memcpy(&u, &f, 8); return u; }
VLM_HD double f64_of_bits(uint64_t u) { double f; memcpy(&f, &u, 8); return f; }
// marshalDurationString values_encoder.go:1063-1126 (-nsecs wraps like Go's: INT64_MIN prints as "-")
VLM_HD int fmt_duration(uint8_t* buf, int64_t nsecs) {
    if (nsecs == 0) { buf[0] = '0'; return 1; }
    int n = 0;
    if (nsecs < 0) { buf[n++] = '-'; nsecs = (int64_t)(0 - (uint64_t)nsecs); }
    const int64_t S = 1000000000LL, W = 7 * 86400 * S, D = 86400 * S, H = 3600 * S, M = 60 * S;
    const bool float_secs = nsecs >= S;
    const int64_t units[4] = {W, D, H, M};
    const char names[4] = {'w', 'd', 'h', 'm'};
    for (int k = 0; k < 4; k++)
        if (nsecs >= units[k]) { const int64_t q = nsecs / units[k]; nsecs -= q * units[k]; n += fmt_u64(buf + n, (uint64_t)q); buf[n++] = (uint8_t)names[k]; }
    if (nsecs >= S) {
        if (float_secs) { n += fmt_f64(buf + n, f64_bits(VLB_DIV((double)nsecs, 1e9))); buf[n++] = 's'; return n; }
        n += fmt_u64(buf + n, (uint64_t)(nsecs / S)); buf[n++] = 's'; nsecs %= S;
    }
    if (nsecs >= 1000000) { n += fmt_u64(buf + n, (uint64_t)(nsecs / 1000000)); buf[n++] = 'm'; buf[n++] = 's'; nsecs %= 1000000; }
    if (nsecs >= 1000) { n += fmt_u64(buf + n, (uint64_t)(nsecs / 1000)); buf[n++] = 0xC2; buf[n++] = 0xB5; buf[n++] = 's'; nsecs %= 1000; }
    if (nsecs > 0) { n += fmt_u64(buf + n, (uint64_t)nsecs); buf[n++] = 'n'; buf[n++] = 's'; }
    return n;
}
// getBucketedValue :1666-1764: the bucket of a text, written into buf (VL_FMT_F64_MAX bytes), or the text itself when it has none.  Returns the
// length; *out = buf or s.
VLM_HD uint32_t bucket_text(const BucketSpec& bk, const uint8_t* s, uint32_t n, uint8_t* buf, const uint8_t** out) {
    *out = s;
    if (n == 0 || ((s[0] < '0' || s[0] > '9') && s[0] != '-')) return n;
    const mn::Span sp{s, n};
    int64_t i; double f; uint32_t ip; int k;
    if (mn::parse_i64(sp, &i)) k = fmt_i64(buf, trunc_i64(i, bk.i64_size, bk.i64_off));
    else if (mn::parse_f64_internal(sp, false, &f)) k = fmt_f64(buf, f64_bits(trunc_f64(f, bk)));
    else if (mn::parse_rfc3339nano(sp, &i)) k = fmt_rfc3339nano(buf, truncate_timestamp(i, bk.i64_size, bk.i64_off, bk.calendar));
    else if (mn::parse_ipv4(sp, &ip)) k = fmt_ipv4(buf, trunc_u32(ip, bk.u32_size, bk.u32_off));
    else if (mn::parse_duration(sp, &i)) k = fmt_duration(buf, trunc_i64(i, bk.i64_size, bk.i64_off));
    else return n;
    *out = buf;
    return (uint32_t)k;
}

}  // namespace vl
