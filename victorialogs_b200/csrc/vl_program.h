// Host-side program compiler: serialised filter tree (include/vlscan.h) -> leaves, AND/OR bloom pre-pass entries,
// typed needles, regex automata.  Mirrors what the Go filters derive lazily (sync.Once) on first use:
//   filterPhrase.initTokens  lib/logstorage/filter_phrase.go:52-55      filterPrefix.initTokens  filter_prefix.go:49-52
//   filterExact.initTokens   filter_exact.go:43-46                      filterRegexp.initTokens  filter_regexp.go:44-51
//   inValues.initTokensHashesAny / typed sets   in_values.go:104-346   getCommonTokensFor{And,Or}Filters  filter_and.go:122-187, filter_or.go:126-193
#pragma once
#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>
#include "vl_hd.cuh"
#include "vl_anycase.cuh"
#include "vl_regex.h"
#include "vl_types.h"

namespace vl {

// ---- host helpers -------------------------------------------------------------------------------------------------
template <class F> inline void host_each_token(const std::string& s, F&& f) {   // tokenizer.go:34-117
    const uint8_t* p = (const uint8_t*)s.data(); uint32_t n = (uint32_t)s.size();
    bool ascii = true; for (uint32_t i = 0; i < n; i++) if (p[i] >= 0x80) { ascii = false; break; }
    uint32_t i = 0;
    while (i < n) {
        int w = 1;
        // skip non-token runes
        while (i < n) { int32_t r = ascii ? p[i] : decode_rune(p + i, n - i, &w); if (is_token_rune(r)) break; i += ascii ? 1 : w; }
        if (i >= n) break;
        uint32_t st = i;
        while (i < n) { int32_t r = ascii ? p[i] : decode_rune(p + i, n - i, &w); if (!is_token_rune(r)) break; i += ascii ? 1 : w; }
        f(s.substr(st, i - st));
    }
}
inline std::vector<std::string> host_tokenize(const std::vector<std::string>& a) {   // tokenizeStrings tokenizer.go:12-24
    std::vector<std::string> out; std::unordered_set<std::string> seen;
    for (size_t k = 0; k < a.size(); k++) {
        if (k > 0 && a[k] == a[k - 1]) continue;
        host_each_token(a[k], [&](std::string t) { if (seen.insert(t).second) out.push_back(std::move(t)); });
    }
    return out;
}
inline std::string host_strip_last_token(std::string s) {   // getTokensSkipLast filter_prefix.go:354-363
    for (;;) { int w; int32_t r = decode_last_rune((const uint8_t*)s.data(), (uint32_t)s.size(), &w); if (!is_token_rune(r)) break; s.resize(s.size() - w); }
    return s;
}
inline std::string host_strip_first_last_token(std::string s) {   // skipFirstLastToken filter_regexp.go:53-69
    size_t b = 0;
    for (;;) { int w; int32_t r = decode_rune((const uint8_t*)s.data() + b, (uint32_t)(s.size() - b), &w); if (!is_token_rune(r)) break; b += w; }
    s.erase(0, b);
    return host_strip_last_token(s);
}
inline void host_token_hashes(const std::vector<std::string>& toks, std::vector<uint64_t>& out) {   // appendTokensHashes bloomfilter.go:126-144
    for (auto& t : toks) { uint64_t h = xxh64((const uint8_t*)t.data(), (uint32_t)t.size()); for (int i = 0; i < 6; i++) out.push_back(xxh64_u64(h + i)); }
}

// strings.ToLower / strings.ToUpper (Go: rune by rune through unicode.ToLower / ToUpper; an invalid byte becomes U+FFFD)
inline std::string host_map_case(const std::string& s, bool upper) {
    std::string out;
    const uint8_t* p = (const uint8_t*)s.data(); uint32_t n = (uint32_t)s.size();
    for (uint32_t i = 0; i < n;) {
        int w; int32_t r = decode_rune(p + i, n - i, &w); i += (uint32_t)w;
        r = upper ? to_upper_rune_host(r) : to_lower_rune(r);
        uint8_t enc[4]; int e = encode_rune(enc, r);
        out.append((const char*)enc, (size_t)e);
    }
    return out;
}

// values_encoder.go:553-585
inline bool parse_u64(const std::string& s, uint64_t* out) {
    if (s.empty() || s.size() > 26) return false;
    if (s.size() > 1 && s[0] == '0') return false;
    uint64_t n = 0;
    for (char c : s) {
        if (c == '_') continue;
        if (c < '0' || c > '9') return false;
        if (n > UINT64_MAX / 10) return false;
        n *= 10; uint64_t d = (uint64_t)(c - '0');
        if (n + d < n) return false;
        n += d;
    }
    *out = n; return true;
}
inline bool parse_date_u64(const std::string& s, uint64_t* out) {   // tryParseDateUint64 :588-619 (2-digit fast path checks only the first digit)
    if (s.empty() || s.size() > 9) return false;
    if (s.size() == 2) { if (s[0] < '0' || s[0] > '9') return false; *out = 10ull * (uint8_t)(s[0] - '0') + (uint8_t)((uint8_t)s[1] - (uint8_t)'0'); return true; }
    uint64_t n = 0;
    for (char c : s) { if (c < '0' || c > '9') return false; n = n * 10 + (uint64_t)(c - '0'); }
    *out = n; return true;
}
inline bool parse_i64(std::string s, int64_t* out) {   // :622-645
    if (s.empty()) return false;
    bool neg = s[0] == '-'; if (neg) s.erase(0, 1);
    uint64_t n; if (!parse_u64(s, &n)) return false;
    if (n >= (1ull << 63)) { if (neg && n == (1ull << 63)) { *out = INT64_MIN; return true; } return false; }
    *out = neg ? -(int64_t)n : (int64_t)n; return true;
}
inline bool parse_ipv4(std::string s, uint32_t* out) {   // :675-730
    if (s.size() < 7 || s.size() > 15 || std::count(s.begin(), s.end(), '.') != 3) return false;
    uint32_t ip = 0;
    for (int k = 0; k < 4; k++) {
        size_t n = k < 3 ? s.find('.') : s.size();
        if (k < 3 && (n == std::string::npos || n == 0 || n > 3)) return false;
        uint64_t v; if (!parse_date_u64(s.substr(0, n), &v) || v > 255) return false;
        ip = (ip << 8) | (uint32_t)v;
        if (k < 3) s.erase(0, n + 1);
    }
    *out = ip; return true;
}
inline double host_pow10_neg(int n) {   // math.Pow10 for n in [-31, 0]
    static const double t[] = {1e0, 1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7, 1e-8, 1e-9, 1e-10, 1e-11, 1e-12, 1e-13, 1e-14, 1e-15, 1e-16,
                               1e-17, 1e-18, 1e-19, 1e-20, 1e-21, 1e-22, 1e-23, 1e-24, 1e-25, 1e-26, 1e-27, 1e-28, 1e-29, 1e-30, 1e-31};
    return (n <= 0 && n >= -31) ? t[-n] : std::pow(10.0, n);
}
inline bool parse_f64_exact(std::string s, double* out) {   // tryParseFloat64Internal(isExact=true) :788-850
    if (s.empty() || s.size() > 27) return false;
    bool neg = s[0] == '-'; if (neg) s.erase(0, 1);
    size_t dot = s.find('.');
    if (dot == std::string::npos) {
        uint64_t v; if (!parse_u64(s, &v) || v >= (1ull << 53)) return false;
        *out = neg ? -(double)v : (double)v; return true;
    }
    if (dot == 0 || dot == s.size() - 1) return false;
    std::string ip = s.substr(0, dot), fp = s.substr(dot + 1);
    uint64_t ni; if (!parse_u64(ip, &ni)) return false;
    size_t z = 0; while (z + 1 < fp.size() && fp[z] == '0') z++;
    uint64_t nf; if (!parse_u64(fp.substr(z), &nf)) return false;
    int us = (int)std::count(fp.begin(), fp.end(), '_');
    double f = std::fma((double)nf, host_pow10_neg(us - (int)fp.size()), (double)ni);
    *out = neg ? -f : f; return true;
}
inline int64_t host_days_from_civil(int64_t y, unsigned m, unsigned d) {
    y -= m <= 2; int64_t era = (y >= 0 ? y : y - 399) / 400; unsigned yoe = (unsigned)(y - era * 400);
    unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1; unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}
inline bool parse_iso8601(const std::string& s, int64_t* out) {   // tryParseTimestampISO8601 :428-464 + tryParseTimestampSecs :466-551
    if (s.size() != 24) return false;
    uint64_t Y, M, D, h, mi, se, ms;
    if (s[4] != '-' || !parse_date_u64(s.substr(0, 4), &Y) || Y < 1677 || Y > 2262) return false;
    if (s[7] != '-' || !parse_date_u64(s.substr(5, 2), &M)) return false;
    if ((s[10] != 'T' && s[10] != ' ') || !parse_date_u64(s.substr(8, 2), &D)) return false;
    if (s[13] != ':' || !parse_date_u64(s.substr(11, 2), &h)) return false;
    if (s[16] != ':' || !parse_date_u64(s.substr(14, 2), &mi)) return false;
    if (!parse_date_u64(s.substr(17, 2), &se)) return false;
    // time.Date normalisation: month, then sec->min->hour->day carries
    int64_t year = (int64_t)Y, mon = (int64_t)M - 1, day = (int64_t)D, hour = (int64_t)h, min = (int64_t)mi, sec = (int64_t)se;
    auto norm = [](int64_t& hi, int64_t& lo, int64_t base) { if (lo < 0) { int64_t n = (-lo - 1) / base + 1; hi -= n; lo += n * base; } if (lo >= base) { int64_t n = lo / base; hi += n; lo -= n * base; } };
    norm(year, mon, 12); norm(min, sec, 60); norm(hour, min, 60); norm(day, hour, 24);
    int64_t secs = (host_days_from_civil(year, (unsigned)(mon + 1), 1) + day - 1) * 86400 + hour * 3600 + min * 60 + sec;
    if (secs < -9223372036LL || secs >= 9223372036LL) return false;
    if (s[19] != '.' || s[23] != 'Z' || !parse_date_u64(s.substr(20, 3), &ms)) return false;
    *out = secs * 1000000000LL + (int64_t)ms * 1000000LL; return true;
}
inline uint64_t host_zigzag(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }

// ---- filter of the row-agnostic substring scan (k_substr_scan, vl_kernels.cuh) ----------------------------------------------------------
// An occurrence of the needle that starts at byte r of an aligned 4-byte word leaves c0 = min(4 - r, L) needle bytes in that word and
// c1 = min(4, L - (4 - r)) in the next one.  Per r the kernel tests ONE aligned word: the one that carries more needle bytes (the first on a tie).
// pat / msk: its bytes and which of them count (little-endian word); delta: occurrence start - address of that word.  Every occurrence is found
// by exactly the pattern of its r; everything a pattern finds is verified at (word address + delta[r]).  Returns whether some mask is partial
// (needles of >= 7 bytes: never).  nd16 = the first 16 needle bytes as little-endian words, zero padded.
inline bool fill_scan_patterns(const uint8_t* nd, uint32_t L, uint32_t pat[4], uint32_t msk[4], int32_t delta[4], uint32_t nd16[4]) {
    bool masked = false;
    for (uint32_t r = 0; r < 4; r++) {
        const uint32_t c0 = std::min<uint32_t>(4 - r, L), c1 = L > 4 - r ? std::min<uint32_t>(4, L - (4 - r)) : 0;
        uint32_t p = 0, m = 0;
        if (c1 > c0) { for (uint32_t i = 0; i < c1; i++) { p |= (uint32_t)nd[4 - r + i] << (8 * i); m |= 0xFFu << (8 * i); } delta[r] = -(int32_t)(4 - r); }
        else { for (uint32_t i = 0; i < c0; i++) { p |= (uint32_t)nd[i] << (8 * (r + i)); m |= 0xFFu << (8 * (r + i)); } delta[r] = (int32_t)r; }
        pat[r] = p; msk[r] = m;
        if (m != 0xFFFFFFFFu) masked = true;
    }
    for (int k = 0; k < 4; k++) nd16[k] = 0;
    for (uint32_t i = 0; i < std::min<uint32_t>(L, 16); i++) nd16[i >> 2] |= (uint32_t)nd[i] << (8 * (i & 3));
    return masked;
}

// ---- program ------------------------------------------------------------------------------------------------------
struct PNode { int kind = F_NOOP; int leaf = -1; std::vector<int> kids; int prepass_begin = 0, prepass_count = 0; };

struct Program {
    std::vector<std::string> fields;
    std::vector<PNode> nodes; int root = -1;
    std::vector<DevLeaf> leaves;
    std::vector<std::vector<std::string>> leaf_tokens;
    std::vector<DevPrepass> prepass;
    std::vector<DevRegex> regexes;
    std::vector<CompiledRegex> host_regexes;
    std::vector<uint8_t> blob;
    std::vector<uint64_t> u64s;
    std::vector<uint32_t> u32s;
    // device images, one per device ordinal (owned by the engine)
    mutable std::mutex mu;
    mutable std::map<int, void*> dev_images;

    int field_id(const std::string& name) {
        std::string c = name.empty() ? "_msg" : name;   // getCanonicalColumnName
        for (size_t i = 0; i < fields.size(); i++) if (fields[i] == c) return (int)i;
        fields.push_back(c); return (int)fields.size() - 1;
    }
    uint32_t put_bytes(const void* p, size_t n, size_t align = 1) {
        while (blob.size() % align) blob.push_back(0);
        uint32_t off = (uint32_t)blob.size();
        blob.insert(blob.end(), (const uint8_t*)p, (const uint8_t*)p + n);
        return off;
    }
    uint32_t put_hashes(const std::vector<uint64_t>& h) { uint32_t off = (uint32_t)u64s.size(); u64s.insert(u64s.end(), h.begin(), h.end()); return off; }
    // packed string list: u32 offsets[n+1] (relative) then the bytes; returns {offs_off, blob_off}
    std::pair<uint32_t, uint32_t> put_strings(const std::vector<std::string>& v) {
        std::vector<uint32_t> offs(v.size() + 1, 0);
        std::string cat;
        for (size_t i = 0; i < v.size(); i++) { cat += v[i]; offs[i + 1] = (uint32_t)cat.size(); }
        uint32_t oo = put_bytes(offs.data(), offs.size() * 4, 4);
        uint32_t bo = put_bytes(cat.data(), cat.size());
        return {oo, bo};
    }
};

class ProgramBuilder {
    const uint8_t* p_; size_t n_, i_ = 0;
    Program& P;
    struct FT { std::string field; std::vector<std::string> tokens; };   // fieldTokens
    std::vector<std::vector<FT>> node_ft_;   // per node (AND/OR): by-field tokens
    std::vector<bool> node_ft_done_;

    uint64_t varuint() {
        uint64_t v = 0; int sh = 0;
        for (int k = 0; k < 10; k++) { if (i_ >= n_) throw ProgError("truncated filter tree"); uint8_t b = p_[i_++]; v |= (uint64_t)(b & 0x7F) << sh; if (b < 0x80) return v; sh += 7; }
        throw ProgError("bad varuint in filter tree");
    }
    std::string bytes() { uint64_t l = varuint(); if (l > n_ - i_) throw ProgError("truncated filter tree"); std::string s((const char*)p_ + i_, l); i_ += l; return s; }

    void typed_needles(DevLeaf& L, const std::string& s) {
        uint64_t u = 0; int64_t i = 0; double f = 0; uint32_t ip = 0; int64_t ts = 0;
        bool uok = parse_u64(s, &u);
        for (int vt : {VT_UINT8, VT_UINT16, VT_UINT32, VT_UINT64}) { L.typed[vt].ok = uok; L.typed[vt].val = uok ? u : 0; }
        if (parse_i64(s, &i)) { L.typed[VT_INT64].ok = 1; L.typed[VT_INT64].val = host_zigzag(i); L.typed[VT_INT64].sval = i; }
        if (parse_f64_exact(s, &f)) { L.typed[VT_FLOAT64].ok = 1; memcpy(&L.typed[VT_FLOAT64].val, &f, 8); }
        if (parse_ipv4(s, &ip)) { L.typed[VT_IPV4].ok = 1; L.typed[VT_IPV4].val = ip; }
        if (parse_iso8601(s, &ts)) { L.typed[VT_ISO8601].ok = 1; L.typed[VT_ISO8601].val = (uint64_t)ts; L.typed[VT_ISO8601].sval = ts; }
    }
    int new_leaf(int kind, const std::string& field, const std::string& needle, const std::vector<std::string>& tokens) {
        DevLeaf L; memset(&L, 0, sizeof L);
        L.kind = (uint8_t)kind; L.field = P.field_id(field); L.regex = -1;
        L.needle_off = P.put_bytes(needle.data(), needle.size()); L.needle_len = (uint32_t)needle.size();
        L.starts_tok = needle_starts_with_token((const uint8_t*)needle.data(), (uint32_t)needle.size());
        L.ends_tok = needle_ends_with_token((const uint8_t*)needle.data(), (uint32_t)needle.size());
        std::vector<uint64_t> h; host_token_hashes(tokens, h);
        L.hashes_off = P.put_hashes(h); L.nhashes = (uint32_t)h.size();
        // string-column strategy: phrase / prefix with a non-empty needle stream the payload through the substring scan
        L.str_strategy = STR_ROW; L.scan_needle_off = L.needle_off; L.scan_needle_len = L.needle_len;
        if ((kind == F_PHRASE || kind == F_PREFIX) && !needle.empty()) { L.str_strategy = STR_SCAN; L.scan_mode = kind == F_PHRASE ? SCAN_PHRASE : SCAN_PREFIX; }
        P.leaves.push_back(L); P.leaf_tokens.push_back(tokens);
        return (int)P.leaves.size() - 1;
    }
    // regexp leaves: "find the literal, then verify" shapes of regexutil.Regex.MatchString (regex.go:86-212) use the scan
    void regex_strategy(DevLeaf& L, const DevRegex& R) {
        auto scan = [&](int mode, uint32_t off, uint32_t len) { L.str_strategy = STR_SCAN; L.scan_mode = (uint8_t)mode; L.scan_needle_off = off; L.scan_needle_len = len; };
        L.str_strategy = STR_ROW;
        if (R.only_prefix) { if (R.prefix_len == 0) L.str_strategy = STR_ALL; else scan(SCAN_CONTAINS, R.prefix_off, R.prefix_len); }
        else if (R.prefix_len > 0) {
            if (R.dot_star) scan(SCAN_CONTAINS, R.prefix_off, R.prefix_len);
            else if (R.dot_plus) scan(SCAN_RX_DOTPLUS, R.prefix_off, R.prefix_len);
            else if (R.sub_kind == 2) L.str_strategy = STR_ROW;   // substrDotPlus first-occurrence rule (regex.go:181-185)
            // `PREFIX.*LITERAL` (dot-all): equivalent to "LITERAL occurs somewhere behind an occurrence of PREFIX".  Scan for the longer of the
            // two literals (rarer in the data, and from 7 bytes on every occurrence covers a whole aligned word) and verify the other one.
            else if (R.tail_len > R.prefix_len) scan(SCAN_RX_TAIL, R.tail_off, R.tail_len);
            else scan(SCAN_RX_SUFFIX, R.prefix_off, R.prefix_len);
        } else {
            if (R.dot_star) L.str_strategy = STR_ALL;
            else if (R.sub_kind == 1) scan(SCAN_CONTAINS, R.sub_off, R.sub_len);
        }
    }
    int depth_ = 0;
    int node() {
        if (i_ >= n_) throw ProgError("truncated filter tree");
        if (P.nodes.size() > 100000) throw ProgError("filter tree too large");
        // the compiler, the token merging and the scan interpreter recurse once per level, and the interpreter holds a bitmap register per level
        if (++depth_ > 64) throw ProgError("filter tree nests too deeply (more than 64 levels)");
        struct Leave { int& d; ~Leave() { d--; } } leave{depth_};
        int kind = p_[i_++];
        int id = (int)P.nodes.size(); P.nodes.emplace_back(); node_ft_.emplace_back(); node_ft_done_.push_back(false);
        P.nodes[id].kind = kind;
        switch (kind) {
        case F_NOOP: break;
        case F_PHRASE: {
            std::string f = bytes(), s = bytes();
            int l = new_leaf(kind, f, s, host_tokenize({s}));
            DevLeaf& L = P.leaves[l]; typed_needles(L, s);
            L.f64_phrase_gate = L.typed[VT_FLOAT64].ok || s == "." || s == "+" || s == "-";
            size_t d = s.find('.'); L.f64_exact_form = d != std::string::npos && d > 0 && d < s.size() - 1;
            P.nodes[id].leaf = l; break;
        }
        case F_PREFIX: {
            std::string f = bytes(), s = bytes();
            int l = new_leaf(kind, f, s, host_tokenize({host_strip_last_token(s)}));
            DevLeaf& L = P.leaves[l]; typed_needles(L, s);
            L.f64_prefix_gate = L.typed[VT_FLOAT64].ok || s == "." || s == "+" || s == "-" || (!s.empty() && (s[0] == 'e' || s[0] == 'E'));
            P.nodes[id].leaf = l; break;
        }
        case F_EXACT: {
            std::string f = bytes(), s = bytes();
            int l = new_leaf(kind, f, s, host_tokenize({s}));
            typed_needles(P.leaves[l], s);
            P.nodes[id].leaf = l; break;
        }
        case F_IN: {
            std::string f = bytes(); uint64_t cnt = varuint();
            if (cnt > (1u << 22)) throw ProgError("too many in() values");
            std::vector<std::string> vals; for (uint64_t k = 0; k < cnt; k++) vals.push_back(bytes());
            int l = new_leaf(kind, f, "", {});
            build_in(P.leaves[l], vals);
            P.nodes[id].leaf = l; break;
        }
        case F_REGEXP: {
            std::string f = bytes(), expr = bytes();
            CompiledRegex cr;
            try { cr = compile_regex(expr); } catch (const RxError& e) { throw ProgError(e.what()); }
            std::vector<std::string> lits; for (auto& x : cr.literals) lits.push_back(host_strip_first_last_token(x));
            int l = new_leaf(kind, f, expr, host_tokenize(lits));
            P.leaves[l].regex = put_regex(cr);
            regex_strategy(P.leaves[l], P.regexes.back());
            P.nodes[id].leaf = l; break;
        }
        case F_EXACT_PREFIX: {   // filter_exact_prefix.go:13-54: tokens = getTokensSkipLast(prefix)
            std::string f = bytes(), s = bytes();
            int l = new_leaf(kind, f, s, host_tokenize({host_strip_last_token(s)}));
            DevLeaf& L = P.leaves[l]; typed_needles(L, s);
            if (!(s < "0" || s > "9")) L.gates |= GATE_DIGIT_PREFIX;
            P.nodes[id].leaf = l; break;
        }
        case F_LEN_RANGE: {      // filter_len_range.go:14-22
            std::string f = bytes(); uint64_t mn = varuint(), mx = varuint();
            int l = new_leaf(kind, f, "", {});
            DevLeaf& L = P.leaves[l]; L.aux0 = mn; L.aux1 = mx; L.always_none = mn > mx;
            P.nodes[id].leaf = l; break;
        }
        case F_STRING_RANGE: {   // filter_string_range.go:12-20; the per-type gates of :88-224 depend on the arguments only
            std::string f = bytes(), a = bytes(), b = bytes();
            int l = new_leaf(kind, f, a, {});
            uint32_t off2 = P.put_bytes(b.data(), b.size());
            DevLeaf& L = P.leaves[l]; L.needle2_off = off2; L.needle2_len = (uint32_t)b.size();
            L.always_none = a > b;
            if (!(a > "9" || b < "0")) L.gates |= GATE_SR_UINT;
            if (!((a != "-" && a > "9") || (b != "-" && b < "0"))) L.gates |= GATE_SR_INT;
            if (!(a > "9" || b < "+")) L.gates |= GATE_SR_FLOAT;
            P.nodes[id].leaf = l; break;
        }
        case F_IPV4_RANGE: {     // filter_ipv4_range.go:12-20
            std::string f = bytes(); uint64_t mn = varuint(), mx = varuint();
            if (mn > 0xFFFFFFFFull || mx > 0xFFFFFFFFull) throw ProgError("ipv4_range bounds do not fit 32 bits");
            int l = new_leaf(kind, f, "", {});
            DevLeaf& L = P.leaves[l]; L.aux0 = mn; L.aux1 = mx; L.always_none = mn > mx;
            P.nodes[id].leaf = l; break;
        }
        case F_VALUE_TYPE: {     // filter_value_type.go:12-15; names: valueType.String() values_encoder.go:62-89
            std::string f = bytes(), t = bytes();
            int l = new_leaf(kind, f, t, {});
            static const std::pair<const char*, int> names[] = {{"const", VTYPE_CONST}, {"string", VT_STRING}, {"dict", VT_DICT}, {"uint8", VT_UINT8}, {"uint16", VT_UINT16},
                {"uint32", VT_UINT32}, {"uint64", VT_UINT64}, {"int64", VT_INT64}, {"float64", VT_FLOAT64}, {"ipv4", VT_IPV4}, {"iso8601", VT_ISO8601}};
            uint64_t code = VTYPE_NO_SUCH;
            for (auto& nm : names) if (t == nm.first) code = (uint64_t)nm.second;
            P.leaves[l].aux0 = code;
            P.nodes[id].leaf = l; break;
        }
        case F_ANY_CASE_PHRASE: case F_ANY_CASE_PREFIX: {   // filter_any_case_phrase.go:14-53, filter_any_case_prefix.go:14-65
            std::string f = bytes(), s = bytes();
            const bool pre = kind == F_ANY_CASE_PREFIX;
            const std::string lower = host_map_case(s, false), upper = host_map_case(s, true);
            // initTokens: the tokens of the phrase AS WRITTEN (prefix: without its last token); they are probed on typed columns only
            std::vector<std::string> tokens = host_tokenize({pre ? host_strip_last_token(s) : s});
            int l = new_leaf(kind, f, lower, tokens);
            DevLeaf& L = P.leaves[l];
            L.starts_tok = needle_starts_with_token((const uint8_t*)lower.data(), (uint32_t)lower.size());
            L.ends_tok = needle_ends_with_token((const uint8_t*)lower.data(), (uint32_t)lower.size());
            typed_needles(L, lower);
            { DevLeaf U; memset(&U, 0, sizeof U); typed_needles(U, upper); L.typed[VT_ISO8601] = U.typed[VT_ISO8601]; }   // iso8601 columns see the upper-cased phrase
            L.needle2_off = P.put_bytes(upper.data(), upper.size()); L.needle2_len = (uint32_t)upper.size();
            std::vector<std::string> up; for (auto& t : tokens) up.push_back(host_map_case(t, true));
            std::vector<uint64_t> h2; host_token_hashes(up, h2);
            L.hashes2_off = P.put_hashes(h2); L.nhashes2 = (uint32_t)h2.size();
            if (pre) L.f64_prefix_gate = L.typed[VT_FLOAT64].ok || lower == "." || lower == "+" || lower == "-" || (!lower.empty() && (lower[0] == 'e' || lower[0] == 'E'));
            else { L.f64_phrase_gate = L.typed[VT_FLOAT64].ok || lower == "." || lower == "+" || lower == "-"; size_t d = lower.find('.'); L.f64_exact_form = d != std::string::npos && d > 0 && d < lower.size() - 1; }
            L.str_strategy = STR_ROW;   // case folding happens per value (any_case_match): no literal to scan for
            P.leaf_tokens[l].clear();   // not among the kinds whose tokens feed the AND / OR pre-pass (filter_and.go:140-166)
            P.nodes[id].leaf = l; break;
        }
        case F_SEQUENCE: case F_CONTAINS_ALL: case F_CONTAINS_ANY: {
            std::string f = bytes(); uint64_t cnt = varuint();
            if (cnt > (1u << 22)) throw ProgError("too many values");
            std::vector<std::string> vals; for (uint64_t k = 0; k < cnt; k++) vals.push_back(bytes());
            if (kind == F_SEQUENCE) {   // filter_sequence.go:12-67: empty phrases are dropped; no phrase left = matches everything
                std::vector<std::string> ph; for (auto& v : vals) if (!v.empty()) ph.push_back(v);
                if (ph.empty()) { P.field_id(f); P.nodes[id].kind = F_NOOP; break; }
                int l = new_leaf(kind, f, ph[0], host_tokenize(ph));
                DevLeaf& L = P.leaves[l];
                typed_needles(L, ph[0]);   // typed columns: a single phrase is matched as an exact value (:213-258)
                put_list(L, ph);
                P.nodes[id].leaf = l; break;
            }
            // contains_all / contains_any share inValues with in(): string set, typed sets, common tokens + per-value token sets
            bool has_empty = false; for (auto& v : vals) has_empty |= v.empty();
            if (kind == F_CONTAINS_ALL && (vals.empty() || (vals.size() == 1 && vals[0].empty()))) { P.field_id(f); P.nodes[id].kind = F_NOOP; break; }   // filter_contains_all.go:92-96
            if (kind == F_CONTAINS_ANY && has_empty) { P.field_id(f); P.nodes[id].kind = F_NOOP; break; }                                                  // filter_contains_any.go:84-92
            int l = new_leaf(kind, f, "", {});
            build_in(P.leaves[l], vals, kind == F_CONTAINS_ANY);
            DevLeaf& L = P.leaves[l];
            put_list(L, vals);
            if (kind == F_CONTAINS_ANY) L.always_none = vals.empty();
            else {
                // getTokensHashesAll in_values.go:94-102: the tokens of all values together; aux0 = number of distinct non-empty values (:80-88)
                std::vector<uint64_t> h; host_token_hashes(host_tokenize(vals), h);
                L.hashes_off = P.put_hashes(h); L.nhashes = (uint32_t)h.size();
                std::unordered_set<std::string> uniq; for (auto& v : vals) if (!v.empty()) uniq.insert(v);
                L.aux0 = uniq.size();
            }
            P.leaf_tokens[l].clear();
            P.nodes[id].leaf = l; break;
        }
        case F_RANGE: {   // filter_range.go:14-24: [minValue, maxValue] as float64, both ends inclusive
            std::string f = bytes();
            if (n_ - i_ < 16) throw ProgError("truncated filter tree");
            uint64_t a = 0, b = 0;
            for (int k = 0; k < 8; k++) { a |= (uint64_t)p_[i_ + k] << (8 * k); b |= (uint64_t)p_[i_ + 8 + k] << (8 * k); }
            i_ += 16;
            double mn, mx; memcpy(&mn, &a, 8); memcpy(&mx, &b, 8);
            int l = new_leaf(kind, f, "", {});
            DevLeaf& L = P.leaves[l];
            L.always_none = mn > mx;
            L.rng_fmin = a; L.rng_fmax = b;
            const double c = std::ceil(mn), fl = std::floor(mx);
            auto u64c = [](double v) -> uint64_t { return v < 0 ? 0 : v >= 18446744073709551616.0 ? UINT64_MAX : (uint64_t)v; };           // toUint64Clamp :380-388
            auto i64c = [](double v) -> int64_t { return v < -9223372036854775808.0 ? INT64_MIN : v >= 9223372036854775808.0 ? INT64_MAX : (int64_t)v; };   // toInt64Clamp :396-404
            auto u32c = [](double v) -> uint32_t { return v < 0 ? 0u : v > 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)v; };                    // toUint32Clamp :412-420
            L.rng_ulo = u64c(c); L.rng_uhi = u64c(fl); L.rng_ilo = i64c(c); L.rng_ihi = i64c(fl); L.rng_iplo = u32c(c); L.rng_iphi = u32c(fl);
            L.str_strategy = STR_ROW;
            P.leaf_tokens[l].clear();
            P.nodes[id].leaf = l; break;
        }
        case F_EQ_FIELD: case F_LE_FIELD: {   // filter_eq_field.go:14-22, filter_le_field.go:14-24
            std::string f = bytes(), o = bytes();
            uint32_t excl = 0;
            if (kind == F_LE_FIELD) { if (i_ >= n_) throw ProgError("truncated filter tree"); excl = p_[i_++] ? 1 : 0; }
            const int fa = P.field_id(f), fb = P.field_id(o);
            if (fa == fb) {   // the same field on both sides: eq_field / le_field match every row, lt_field none
                if (kind == F_LE_FIELD && excl) { int l = new_leaf(kind, f, "", {}); DevLeaf& L = P.leaves[l]; L.field2 = fb; L.pair_excl = 1; L.always_none = 1; P.leaf_tokens[l].clear(); P.nodes[id].leaf = l; }
                else P.nodes[id].kind = F_NOOP;
                break;
            }
            int l = new_leaf(kind, f, "", {});
            DevLeaf& L = P.leaves[l];
            L.field2 = fb; L.pair_excl = excl; L.str_strategy = STR_ROW;
            P.leaf_tokens[l].clear();
            P.nodes[id].leaf = l; break;
        }
        case F_TIME: {   // filter_time.go:14-23: [minTimestamp, maxTimestamp] in nanoseconds, both ends inclusive; no field (the block's timestamps column)
            if (n_ - i_ < 16) throw ProgError("truncated filter tree");
            uint64_t mn = 0, mx = 0;
            for (int k = 0; k < 8; k++) { mn |= (uint64_t)p_[i_ + k] << (8 * k); mx |= (uint64_t)p_[i_ + 8 + k] << (8 * k); }
            i_ += 16;
            DevLeaf L; memset(&L, 0, sizeof L);
            L.kind = F_TIME; L.field = -1; L.regex = -1; L.aux0 = mn; L.aux1 = mx; L.always_none = (int64_t)mn > (int64_t)mx; L.str_strategy = STR_ROW;
            P.leaves.push_back(L); P.leaf_tokens.push_back({});
            P.nodes[id].leaf = (int)P.leaves.size() - 1; break;
        }
        case F_AND: case F_OR: { uint64_t c = varuint(); if (c > 100000) throw ProgError("too many children"); for (uint64_t k = 0; k < c; k++) { int ch = node(); P.nodes[id].kids.push_back(ch); } break; }
        case F_NOT: { int ch = node(); P.nodes[id].kids.push_back(ch); break; }
        default: throw ProgError("unknown filter kind " + std::to_string(kind));
        }
        return id;
    }
    void put_list(DevLeaf& L, const std::vector<std::string>& v) {   // (varuint length, bytes)*: the PhraseList the value predicates walk (vl_anycase.cuh)
        std::string blob;
        for (auto& s : v) { uint64_t n = s.size(); while (n >= 0x80) { blob.push_back((char)(n | 0x80)); n >>= 7; } blob.push_back((char)n); blob += s; }
        L.list_off = P.put_bytes(blob.data(), blob.size()); L.list_len = (uint32_t)blob.size(); L.in_count = (uint32_t)v.size();
    }
    int put_regex(const CompiledRegex& cr) {
        DevRegex R; memset(&R, 0, sizeof R);
        R.prefix_off = P.put_bytes(cr.prefix.data(), cr.prefix.size()); R.prefix_len = (uint32_t)cr.prefix.size();
        const std::string& sub = !cr.substrDotStar.empty() ? cr.substrDotStar : cr.substrDotPlus;
        R.sub_off = P.put_bytes(sub.data(), sub.size()); R.sub_len = (uint32_t)sub.size();
        R.sub_kind = !cr.substrDotStar.empty() ? 1 : !cr.substrDotPlus.empty() ? 2 : 0;
        R.only_prefix = cr.isOnlyPrefix; R.dot_star = cr.isSuffixDotStar; R.dot_plus = cr.isSuffixDotPlus;
        R.nclasses = cr.suffix.nclasses; R.nstates = cr.suffix.nstates;
        R.bounds_off = P.put_bytes(cr.suffix.bounds.data(), cr.suffix.bounds.size() * 4, 4);
        R.ascii_off = P.put_bytes(cr.suffix.ascii_class, 128);
        R.trans_off = P.put_bytes(cr.suffix.trans.data(), cr.suffix.trans.size() * 2, 2);
        R.accept_off = P.put_bytes(cr.suffix.accept_end.data(), cr.suffix.accept_end.size());
        R.tail_off = P.put_bytes(cr.tailLiteral.data(), cr.tailLiteral.size()); R.tail_len = (uint32_t)cr.tailLiteral.size();
        P.regexes.push_back(R); P.host_regexes.push_back(cr);
        return (int)P.regexes.size() - 1;
    }
    void build_in(DevLeaf& L, const std::vector<std::string>& vals, bool keep_all_sets = false) {
        // string set (deduplicated; order irrelevant)
        std::vector<std::string> uniq; { std::unordered_set<std::string> seen; for (auto& v : vals) if (seen.insert(v).second) uniq.push_back(v); }
        L.in_count = (uint32_t)uniq.size();
        auto po = P.put_strings(uniq); L.in_offs_off = po.first; L.in_blob_off = po.second;
        for (auto& v : uniq) if (v.empty()) L.in_has_empty = 1;
        // typed sets in_values.go:141-315
        for (int vt = VT_UINT8; vt < VT_MAX; vt++) {
            std::vector<uint64_t> set;
            for (auto& v : vals) {
                uint64_t u; int64_t i; double f; uint32_t ip; int64_t ts;
                switch (vt) {
                case VT_UINT8: if (parse_u64(v, &u) && u < (1ull << 8)) set.push_back(u); break;
                case VT_UINT16: if (parse_u64(v, &u) && u < (1ull << 16)) set.push_back(u); break;
                case VT_UINT32: if (parse_u64(v, &u) && u < (1ull << 32)) set.push_back(u); break;
                case VT_UINT64: if (parse_u64(v, &u)) set.push_back(u); break;
                case VT_INT64: if (parse_i64(v, &i)) set.push_back(host_zigzag(i)); break;
                case VT_FLOAT64: if (parse_f64_exact(v, &f)) { memcpy(&u, &f, 8); set.push_back(u); } break;
                case VT_IPV4: if (parse_ipv4(v, &ip)) set.push_back(ip); break;
                case VT_ISO8601: if (parse_iso8601(v, &ts)) set.push_back((uint64_t)ts); break;
                }
            }
            std::sort(set.begin(), set.end()); set.erase(std::unique(set.begin(), set.end()), set.end());
            L.in_typed_off[vt] = P.put_hashes(set); L.in_typed_cnt[vt] = (uint32_t)set.size();
        }
        // getCommonTokensAndTokenSets in_values.go:317-371 (per ORIGINAL value, duplicates included, like the reference)
        std::vector<std::vector<std::string>> sets; for (auto& v : vals) sets.push_back(host_tokenize({v}));
        std::vector<std::string> common;
        if (!sets.empty()) {
            common = sets[0];
            for (size_t k = 1; k < sets.size() && !common.empty(); k++) {
                std::vector<std::string> d; for (auto& t : common) if (std::find(sets[k].begin(), sets[k].end(), t) != sets[k].end()) d.push_back(t);
                common.swap(d);
            }
        }
        if (!common.empty()) for (auto& s : sets) { std::vector<std::string> d; for (auto& t : s) if (std::find(common.begin(), common.end(), t) == common.end()) d.push_back(t); s.swap(d); }
        std::vector<uint64_t> ch; host_token_hashes(common, ch);
        L.hashes_off = P.put_hashes(ch); L.nhashes = (uint32_t)ch.size();
        L.in_nsets = (uint32_t)sets.size();
        L.in_skip_sets = sets.size() > 1000;   // maxTokenSetsToInit
        std::vector<uint32_t> desc;
        // (contains_any probes every value's own tokens on string columns whatever their number, filter_contains_any.go:170-189)
        if (!L.in_skip_sets || keep_all_sets) for (auto& s : sets) { std::vector<uint64_t> h; host_token_hashes(s, h); desc.push_back(P.put_hashes(h)); desc.push_back((uint32_t)h.size()); }
        L.in_sets_off = (uint32_t)P.u32s.size(); P.u32s.insert(P.u32s.end(), desc.begin(), desc.end());
        P.leaf_tokens.back() = common;
    }
    // ---- AND / OR bloom pre-pass token merging -------------------------------------------------------------------------
    bool leaf_has_tokens(int kind) const { return kind == F_PHRASE || kind == F_PREFIX || kind == F_EXACT || kind == F_REGEXP || kind == F_EXACT_PREFIX || kind == F_SEQUENCE; }
    const std::vector<FT>& by_field(int id) {
        if (node_ft_done_[id]) return node_ft_[id];
        node_ft_done_[id] = true;
        PNode& nd = P.nodes[id];
        std::vector<FT>& out = node_ft_[id];
        if (nd.kind == F_AND) {
            std::vector<std::string> names; std::map<std::string, std::vector<std::string>> m;
            auto merge = [&](const std::string& f, const std::vector<std::string>& t) { if (t.empty()) return; if (!m.count(f)) names.push_back(f); auto& v = m[f]; v.insert(v.end(), t.begin(), t.end()); };
            for (int k : nd.kids) {
                const PNode& c = P.nodes[k];
                if (leaf_has_tokens(c.kind)) merge(P.fields[P.leaves[c.leaf].field], P.leaf_tokens[c.leaf]);
                else if (c.kind == F_OR) for (auto& ft : by_field(k)) merge(ft.field, ft.tokens);
            }
            for (auto& f : names) { FT ft; ft.field = f; std::unordered_set<std::string> seen; for (auto& t : m[f]) if (seen.insert(t).second) ft.tokens.push_back(t); out.push_back(ft); }
        } else if (nd.kind == F_OR) {
            std::vector<std::string> names; std::map<std::string, std::vector<std::vector<std::string>>> m;
            auto merge = [&](const std::string& f, const std::vector<std::string>& t) { if (t.empty()) return; if (!m.count(f)) names.push_back(f); m[f].push_back(t); };
            bool ok = true;
            for (int k : nd.kids) {
                const PNode& c = P.nodes[k];
                if (leaf_has_tokens(c.kind)) merge(P.fields[P.leaves[c.leaf].field], P.leaf_tokens[c.leaf]);
                else if (c.kind == F_AND) for (auto& ft : by_field(k)) merge(ft.field, ft.tokens);
                else { ok = false; break; }
            }
            if (ok) for (auto& f : names) {
                auto& tt = m[f];
                if (tt.size() != nd.kids.size()) continue;
                std::vector<std::string> common = tt[0];
                for (size_t k = 1; k < tt.size() && !common.empty(); k++) { std::vector<std::string> d; for (auto& t : common) if (std::find(tt[k].begin(), tt[k].end(), t) != tt[k].end()) d.push_back(t); common.swap(d); }
                if (common.empty()) continue;
                out.push_back(FT{f, common});
            }
        }
        return out;
    }
public:
    ProgramBuilder(const void* tree, size_t n, Program& prog) : p_((const uint8_t*)tree), n_(n), P(prog) {}
    void build() {
        P.root = node();
        if (i_ != n_) throw ProgError("trailing bytes after the filter tree");
        for (size_t id = 0; id < P.nodes.size(); id++) {
            if (P.nodes[id].kind != F_AND && P.nodes[id].kind != F_OR) continue;
            const auto& fts = by_field((int)id);
            P.nodes[id].prepass_begin = (int)P.prepass.size(); P.nodes[id].prepass_count = (int)fts.size();
            for (auto& ft : fts) {
                DevPrepass pp; memset(&pp, 0, sizeof pp);
                pp.field = P.field_id(ft.field); pp.ntokens = (uint32_t)ft.tokens.size();
                auto po = P.put_strings(ft.tokens); pp.tok_offs_off = po.first; pp.tok_blob_off = po.second;
                std::vector<uint64_t> h; host_token_hashes(ft.tokens, h);
                pp.hashes_off = P.put_hashes(h); pp.nhashes = (uint32_t)h.size();
                P.prepass.push_back(pp);
            }
        }
        while (P.blob.size() % 16) P.blob.push_back(0);
    }
};

}  // namespace vl
