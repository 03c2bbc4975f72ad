// ORACLE — test infrastructure only. Never linked into or called from the product path.
//
// CPU restatement of the reference's CSV path (S3 CSV source):
//   line reader / splitter / sanitiser   pkg/csv/reader.go:89-324   (single-line mode: NewlinesInValue=false, :137-155)
//   row -> ChangeItem                    pkg/providers/s3/reader/registry/csv/reader_csv.go:186-343
//   per-type value rules                 reader_csv.go:345-452
//   text -> canonical Go type            pkg/abstract/changeitem/strictify/strictify.go:18-181
//        through github.com/spf13/cast v1.7.1 (go.mod:63; third party, not vendored: its string paths are
//        restated from the published source — strconv.ParseInt(trimZeroDecimal(s), 0, 0), strconv.ParseBool,
//        strconv.ParseFloat, StringToDate layout list) and pkg/util/castx/caste.go:36-52
//   default values                       pkg/abstract/change_item_builders.go:87-109
// Pinned by pkg/csv/reader_test.go cases (tests/test_csv.py); the cast string paths are UNPINNED by the reference
// (its CSV tests use plain decimal cells) — cells whose conversion depends on rarely used Go syntax the device does
// not implement (underscored literals, hex floats, non-ISO time layouts) are reported with CSV_UNSUPPORTED by both.
#pragma once
#include <cstdint>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <array>
#include "go_strconv.hpp"

namespace orc {

enum CsvErr { CSV_OK = 0, CSV_MISSING_CELL = 16, CSV_SINGLE_QUOTE = 17, CSV_BAD_INT = 18, CSV_RANGE = 19, CSV_BAD_BOOL = 20,
              CSV_BAD_TIME = 21, CSV_BAD_FLOAT = 22, CSV_UNSUPPORTED = 23, CSV_DOUBLE_QUOTE_DISABLED = 24, CSV_QUOTING_DISABLED = 25 };

struct CsvOpts {
    uint8_t delimiter = ',', quote = '"', escape = '\\';
    bool double_quote = true, strings_can_be_null = false, quoted_strings_can_be_null = false, include_missing = false;
    std::vector<std::string> null_values, true_values, false_values;
};

inline bool go_space_fwd(const uint8_t* p, size_t n, size_t& w) {   // unicode.IsSpace at p, width out
    if (!n) return false;
    uint8_t b = p[0];
    if (b == ' ' || (b >= 9 && b <= 13)) { w = 1; return true; }
    if (b == 0xC2 && n >= 2 && (p[1] == 0x85 || p[1] == 0xA0)) { w = 2; return true; }
    if (n >= 3) {
        if (b == 0xE1 && p[1] == 0x9A && p[2] == 0x80) { w = 3; return true; }
        if (b == 0xE2 && p[1] == 0x80 && ((p[2] >= 0x80 && p[2] <= 0x8A) || p[2] == 0xA8 || p[2] == 0xA9 || p[2] == 0xAF)) { w = 3; return true; }
        if (b == 0xE2 && p[1] == 0x81 && p[2] == 0x9F) { w = 3; return true; }
        if (b == 0xE3 && p[1] == 0x80 && p[2] == 0x80) { w = 3; return true; }
    }
    return false;
}
inline void go_trim_space(const uint8_t*& p, size_t& n) {
    size_t w;
    while (n && go_space_fwd(p, n, w)) { p += w; n -= w; }
    for (;;) {
        if (!n) return;
        if (go_space_fwd(p + n - 1, 1, w)) { n -= 1; continue; }
        if (n >= 2 && go_space_fwd(p + n - 2, 2, w) && w == 2) { n -= 2; continue; }
        if (n >= 3 && go_space_fwd(p + n - 3, 3, w) && w == 3) { n -= 3; continue; }
        return;
    }
}

// strconv.ParseInt(trimZeroDecimal(s), 0, 0) without underscore support. rc: 0 ok, 1 syntax/range error, 2 unsupported
inline int cast_parse_int(const uint8_t* s, size_t n, int64_t& out) {
    {   // trimZeroDecimal
        bool zero = false; size_t i = n;
        for (; i > 0; i--) { uint8_t c = s[i - 1]; if (c == '.') { if (zero) { n = i - 1; } break; } else if (c == '0') zero = true; else break; }
    }
    if (!n) return 1;
    size_t i = 0; bool neg = false;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; if (n == 1) return 1; }
    int base = 10;
    if (s[i] == '0' && i + 1 < n) {
        uint8_t c = s[i + 1] | 0x20;
        if (c == 'x') { base = 16; i += 2; } else if (c == 'b') { base = 2; i += 2; } else if (c == 'o') { base = 8; i += 2; } else { base = 8; i += 1; }
        if (i >= n) return 1;
    }
    uint64_t v = 0; const uint64_t lim = neg ? (uint64_t)1 << 63 : ((uint64_t)1 << 63) - 1;
    for (; i < n; i++) {
        uint8_t c = s[i]; int d;
        if (c == '_') return 2;
        if (c >= '0' && c <= '9') d = c - '0'; else if ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') d = (c | 0x20) - 'a' + 10; else return 1;
        if (d >= base) return 1;
        unsigned __int128 t = (unsigned __int128)v * base + d; if (t > lim) return 1;
        v = (uint64_t)t;
    }
    out = neg ? (int64_t)(0 - v) : (int64_t)v; return 0;
}
// strconv.ParseBool
inline int go_parse_bool(const uint8_t* s, size_t n, bool& out) {
    std::string t((const char*)s, n);
    if (t == "1" || t == "t" || t == "T" || t == "TRUE" || t == "true" || t == "True") { out = true; return 0; }
    if (t == "0" || t == "f" || t == "F" || t == "FALSE" || t == "false" || t == "False") { out = false; return 0; }
    return 1;
}
// decimal float text -> double: exact (Clinger fast path: <= 15 significant digits and |exp10| <= 22); rc 2 otherwise
inline int parse_float_fast(const uint8_t* s, size_t n, double& out) {
    size_t i = 0; bool neg = false;
    if (!n) return 1;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    uint64_t m = 0; int nd = 0, dp = 0; bool any = false, seen_dot = false;
    for (; i < n; i++) {
        uint8_t c = s[i];
        if (c >= '0' && c <= '9') { any = true; if (m || c != '0') { if (nd >= 19) return 2; m = m * 10 + (c - '0'); nd++; } if (seen_dot) dp--; }
        else if (c == '.' && !seen_dot) seen_dot = true;
        else break;
    }
    if (!any) return (n - i >= 3) ? 2 : 1;     // inf / nan / garbage
    int e = 0;
    if (i < n && (s[i] | 0x20) == 'e') {
        i++; bool eneg = false; if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; i++; }
        if (i >= n) return 1; int ev = 0;
        for (; i < n; i++) { if (s[i] < '0' || s[i] > '9') return 1; if (ev < 10000) ev = ev * 10 + (s[i] - '0'); }
        e = eneg ? -ev : ev;
    }
    if (i != n) return (s[i] == '_' || (s[i] | 0x20) == 'x' || (s[i] | 0x20) == 'p') ? 2 : 1;
    e += dp;
    if (m == 0) { out = neg ? -0.0 : 0.0; return 0; }
    if (nd > 15 || e < -22 || e > 22) return 2;
    static const double p10[] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    double d = (double)m; d = e < 0 ? d / p10[-e] : d * p10[e];
    out = neg ? -d : d; return 0;
}
// cast.StringToDate subset: "2006-01-02", "2006-01-02[T ]15:04:05[.frac][Z|±hh:mm|±hhmm]"; rc 2 for anything else that is not plainly garbage
inline int parse_time_iso(const uint8_t* s, size_t n, int64_t& sec, uint32_t& nsec) {
    auto dig = [&](size_t p, int k, int& v) { v = 0; for (int i = 0; i < k; i++) { if (p + i >= n || s[p + i] < '0' || s[p + i] > '9') return false; v = v * 10 + (s[p + i] - '0'); } return true; };
    int y, mo, d, hh = 0, mi = 0, ss = 0; nsec = 0; int64_t off = 0;
    if (!(dig(0, 4, y) && n >= 10 && s[4] == '-' && dig(5, 2, mo) && s[7] == '-' && dig(8, 2, d))) return 2;
    static const int dm[] = {0, 31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    if (mo < 1 || mo > 12 || d < 1 || d > dm[mo] + ((mo == 2 && leap) ? 1 : 0)) return 1;
    size_t p = 10;
    if (p < n) {
        if (s[p] != 'T' && s[p] != ' ') return 2;
        if (!(dig(p + 1, 2, hh) && p + 3 < n && s[p + 3] == ':' && dig(p + 4, 2, mi) && p + 6 < n && s[p + 6] == ':' && dig(p + 7, 2, ss))) return 2;
        if (hh > 23 || mi > 59 || ss > 59) return 1;
        p += 9;
        if (p < n && s[p] == '.') { size_t q = p + 1; uint32_t f = 0; int k = 0; while (q < n && s[q] >= '0' && s[q] <= '9') { if (k < 9) { f = f * 10 + (s[q] - '0'); k++; } q++; } if (q == p + 1) return 2; while (k < 9) { f *= 10; k++; } nsec = f; p = q; }
        if (p < n) {
            if (s[p] == 'Z' && p + 1 == n) p++;
            else if (s[p] == '+' || s[p] == '-') {
                int sign = s[p] == '-' ? -1 : 1, oh, om;
                if (dig(p + 1, 2, oh) && p + 3 < n && s[p + 3] == ':' && dig(p + 4, 2, om) && p + 6 == n) off = sign * (oh * 3600 + om * 60);
                else if (dig(p + 1, 2, oh) && dig(p + 3, 2, om) && p + 5 == n) off = sign * (oh * 3600 + om * 60);
                else return 2;
                p = n;
            } else return 2;
        }
    }
    if (p != n) return 2;
    sec = days_from_civil(y, (unsigned)mo, (unsigned)d) * 86400 + hh * 3600 + mi * 60 + ss - off;
    return 0;
}

struct CsvCol { int32_t tf; int32_t path; };   // path: field index in the row, < 0 = default value (reader_csv.go:291-297)

struct CsvColOut { std::vector<uint8_t> values, heap, aux; std::vector<uint32_t> offs{0}; };

struct CsvResult { std::vector<CsvColOut> cols; std::vector<tf_rowerr> errs; uint64_t rows = 0, lines = 0, consumed = 0; };

inline bool in_list(const std::vector<std::string>& l, const uint8_t* p, size_t n) { for (auto& x : l) if (x.size() == n && std::memcmp(x.data(), p, n) == 0) return true; return false; }

inline int width_tf(int tf) {
    switch (tf) { case TF_INT8: case TF_UINT8: case TF_BOOLEAN: return 1; case TF_INT16: case TF_UINT16: return 2; case TF_INT32: case TF_UINT32: case TF_FLOAT: return 4;
                  case TF_BYTES: case TF_UTF8: case TF_ANY: return 0; default: return 8; }
}

// One cell -> canonical value bytes (getCorrespondingValue reader_csv.go:345-362 then strictifyValue strictify.go:46-157)
inline int csv_convert(const CsvOpts& o, int tf, const std::string& cell, uint8_t val[8], uint32_t& nsec, std::string& sval) {
    const uint8_t* p = (const uint8_t*)cell.data(); size_t n = cell.size();
    std::memset(val, 0, 8); nsec = 0;
    auto is_null = [&]() {        // parseNullValues reader_csv.go:384-405
        if (o.quoted_strings_can_be_null) {
            const uint8_t* q = p; size_t m = n;
            if (m >= 2 && ((q[0] == '"' && q[m - 1] == '"') || (q[0] == '\'' && q[m - 1] == '\''))) { q++; m -= 2; }
            else if (m == 1 && (q[0] == '"' || q[0] == '\'')) { /* HasPrefix && HasSuffix on a 1-char string: TrimPrefix then TrimSuffix of the rest */ q++; m = 0; }
            return in_list(o.null_values, q, m);
        }
        return o.strings_can_be_null && in_list(o.null_values, p, n);
    };
    switch (tf) {
    case TF_BOOLEAN: {            // parseBooleanValue :430-452, then cast.ToBoolE
        bool b;
        if (o.strings_can_be_null && in_list(o.null_values, p, n)) b = false;
        else if (in_list(o.true_values, p, n)) b = true;
        else if (in_list(o.false_values, p, n)) b = false;
        else if (go_parse_bool(p, n, b)) return CSV_BAD_BOOL;
        val[0] = b; return 0;
    }
    case TF_TIMESTAMP: {          // parseTimestampValue :418-426 (base-10 ParseInt), else cast.ToTimeE(string)
        bool num = n > 0; size_t i = (n && (p[0] == '+' || p[0] == '-')) ? 1 : 0; if (i == n) num = false;
        for (size_t k = i; k < n && num; k++) if (p[k] < '0' || p[k] > '9') num = false;
        int64_t sec;
        if (num) {
            unsigned __int128 v = 0; for (size_t k = i; k < n; k++) { v = v * 10 + (p[k] - '0'); if (v > ((unsigned __int128)1 << 63)) break; }
            const bool neg = p[0] == '-';
            if (v > ((unsigned __int128)1 << 63) - (neg ? 0 : 1)) num = false; else sec = neg ? (int64_t)(0 - (uint64_t)v) : (int64_t)v;
        }
        if (!num) { int rc = parse_time_iso(p, n, sec, nsec); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_TIME; }
        std::memcpy(val, &sec, 8); return 0;
    }
    case TF_DATE: case TF_DATETIME: {   // parseDateValue :409-416 (no TimestampParsers configured) -> cast.ToTimeE(string)
        int64_t sec; int rc = parse_time_iso(p, n, sec, nsec); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_TIME;
        std::memcpy(val, &sec, 8); return 0;
    }
    case TF_FLOAT: case TF_DOUBLE: {    // parseFloatValue (DecimalPoint unset) -> cast.ToFloat32E / castx.ToJSONNumberE -> Float64()
        double d; int rc = parse_float_fast(p, n, d); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_FLOAT;
        // cast.ToFloat32E(string) is strconv.ParseFloat(s, 32): one rounding to binary32 (glibc strtof), not float32(float64)
        if (tf == TF_FLOAT) { float f = std::strtof(cell.c_str(), nullptr); std::memcpy(val, &f, 4); } else std::memcpy(val, &d, 8);
        return 0;
    }
    default: break;
    }
    // default branch: parseNullValues :384-405 -> DefaultValue (change_item_builders.go:87-109) or the cell text
    const bool null = is_null();
    switch (tf) {
    case TF_UTF8: case TF_BYTES: sval = null ? "" : cell; return 0;
    case TF_ANY: sval = null ? "{}" : cell; return null ? -1 /* JSON value, tag 0 */ : 0;
    case TF_INTERVAL: { if (null) return 0; return CSV_UNSUPPORTED; }   // cast.ToDurationE(string): time.ParseDuration
    default: {
        if (null) return 0;         // Restore(col, float64(0)) -> typed zero
        int64_t v; int rc = cast_parse_int(p, n, v); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_INT;
        int64_t lo, hi; bool uns = false;
        switch (tf) {
        case TF_INT8: lo = -128; hi = 127; break; case TF_INT16: lo = -32768; hi = 32767; break;
        case TF_INT32: lo = INT32_MIN; hi = INT32_MAX; break; case TF_INT64: lo = INT64_MIN; hi = INT64_MAX; break;
        case TF_UINT8: uns = true; lo = 0; hi = 255; break; case TF_UINT16: uns = true; lo = 0; hi = 65535; break;
        case TF_UINT32: uns = true; lo = 0; hi = 4294967295LL; break; default: uns = true; lo = 0; hi = INT64_MAX; break;
        }
        if (uns && v < 0) return CSV_BAD_INT;       // errNegativeNotAllowed
        if (v < lo || v > hi) return CSV_RANGE;     // StrictifyRangeError strictify.go:159-181
        std::memcpy(val, &v, 8); return 0;
    }
    }
}

// Reader.splitString + sanitizeElement (reader.go:220-324). Returns an error code or 0.
inline int csv_split(const CsvOpts& o, const uint8_t* line, size_t n, std::vector<std::string>& out, std::vector<char>& had_dq) {
    out.clear(); had_dq.clear();
    uint8_t prev = 0; bool inq = false; size_t prev_delim = 0, last_delim = 0;
    auto sanitize = [&](size_t a, size_t b, std::string& el) -> int {
        had_dq.push_back(0);
        const uint8_t* p = line + a; size_t m = b - a;
        go_trim_space(p, m);
        if (o.quote) {
            if (m == 1 && p[0] == o.quote) return CSV_SINGLE_QUOTE;                 // unquote :287-301
            if (m >= 2 && p[0] == o.quote && p[m - 1] == o.quote) { p++; m -= 2; }
            el.assign((const char*)p, m);
            const std::string pair(2, (char)o.quote);                                  // DoubleQuoteStr = quote + quote (s3 csv_config.go:141)
            bool has = el.find(pair) != std::string::npos;                             // swapToSingleQuotes :309-324: ReplaceAll(el, pair, `"`)
            if (has && !o.double_quote) return CSV_DOUBLE_QUOTE_DISABLED;
            if (has) { had_dq.back() = 1; std::string r; for (size_t i = 0; i < el.size(); i++) { if (el.compare(i, 2, pair) == 0) { r += '"'; i++; } else r += el[i]; } el.swap(r); }
        } else el.assign((const char*)p, m);
        return 0;
    };
    for (size_t i = 0; i < n; i++) {
        const uint8_t c = line[i];
        if (o.escape && o.escape == prev && inq) { prev = c; continue; }
        if (o.quote && c == o.quote) { inq = !inq; prev = c; continue; }
        if (c == o.delimiter && !inq) {
            last_delim = i; std::string el; int rc = sanitize(prev_delim, last_delim, el); if (rc) return rc;
            out.push_back(el); prev_delim = last_delim + 1;
        }
        prev = c;
    }
    std::string el; int rc = sanitize(last_delim + 1 <= n ? last_delim + 1 : n, n, el);     // NOTE line[lastDelimPosition+1:] with lastDelimPosition == 0 when no delimiter was seen
    if (rc) return rc;
    out.push_back(el);
    return 0;
}

inline CsvResult csv_parse(const uint8_t* buf, size_t len, const std::vector<CsvCol>& schema, const CsvOpts& o, uint64_t skip_lines) {
    CsvResult R; R.cols.resize(schema.size());
    size_t pos = 0; uint64_t line_no = 0; std::vector<std::string> cells; std::vector<char> had_dq;
    while (pos < len) {
        const uint8_t* nl = (const uint8_t*)std::memchr(buf + pos, '\n', len - pos);
        if (!nl) break;                                                   // incomplete last line is dropped (reader.go:162-165)
        const size_t end = (size_t)(nl - buf) + 1;
        const uint8_t* line = buf + pos; const size_t n = end - pos; pos = end; R.consumed = end;
        const uint64_t ln = line_no++;
        if (ln < skip_lines) continue;
        int err = 0;
        if (!o.quote && std::memchr(line, '"', n)) err = CSV_QUOTING_DISABLED;     // readAndDecodeLine :185-187, before the split
        else if (n == 1) { cells.clear(); had_dq.clear(); }                   // "\n": ReadLine returns no entries (:141-145)
        else err = csv_split(o, line, n, cells, had_dq);
        std::vector<std::array<uint8_t, 8>> vals(schema.size()); std::vector<uint32_t> ns(schema.size(), 0); std::vector<std::string> sv(schema.size()); std::vector<int> tag(schema.size(), 1);
        // constructCI (reader_csv.go:266-343) visits every column first: a missing cell outranks conversion errors,
        // which Strictify (strictify.go:18-44) then reports for the first failing column in schema order.
        for (size_t c = 0; c < schema.size() && !err; c++)
            if (schema[c].path >= 0 && (size_t)schema[c].path >= cells.size() && !o.include_missing) err = CSV_MISSING_CELL;
        for (size_t c = 0; c < schema.size() && !err; c++) {
            const CsvCol& col = schema[c];
            if (col.path < 0 || (size_t)col.path >= cells.size()) {   // abstract.DefaultValue
                std::memset(vals[c].data(), 0, 8);
                if (col.tf == TF_ANY) { sv[c] = "{}"; tag[c] = 0; }
                continue;
            }
            if (had_dq[col.path] && width_tf(col.tf)) { err = CSV_UNSUPPORTED; break; }    // device limitation mirrored: `""` inside a non-text cell
            int rc = csv_convert(o, col.tf, cells[col.path], vals[c].data(), ns[c], sv[c]);
            if (rc == -1) { tag[c] = 0; rc = 0; }
            err = rc;
        }
        if (err) { R.errs.push_back(tf_rowerr{(uint32_t)(ln - skip_lines), (uint16_t)err, 0}); continue; }
        for (size_t c = 0; c < schema.size(); c++) {
            CsvColOut& oc = R.cols[c]; const int w = width_tf(schema[c].tf);
            if (w) oc.values.insert(oc.values.end(), vals[c].data(), vals[c].data() + w);
            else { oc.heap.insert(oc.heap.end(), sv[c].begin(), sv[c].end()); oc.offs.push_back((uint32_t)oc.heap.size()); }
            if (schema[c].tf == TF_DATE || schema[c].tf == TF_DATETIME || schema[c].tf == TF_TIMESTAMP) { const uint8_t* q = (const uint8_t*)&ns[c]; oc.aux.insert(oc.aux.end(), q, q + 4); }
            if (schema[c].tf == TF_ANY) oc.aux.push_back((uint8_t)tag[c]);
        }
        R.rows++;
    }
    R.lines = line_no > skip_lines ? line_no - skip_lines : 0;
    return R;
}

}  // namespace orc
