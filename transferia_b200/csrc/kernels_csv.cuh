// CSV -> typed columns on the device.
//   reference: pkg/csv/reader.go:89-324 (ReadLine / splitString / sanitizeElement, single-line mode),
//              pkg/providers/s3/reader/registry/csv/reader_csv.go:266-452 (constructCI, per-type value rules),
//              pkg/abstract/changeitem/strictify/strictify.go:46-181 (text -> canonical type via spf13/cast),
//              pkg/abstract/change_item_builders.go:87-109 (DefaultValue).
// In single-line mode the quote state resets at every '\n' (reader.go:137-155), so lines are independent:
//   k_csv_count_nl / k_csv_line_index   newline index (count per 8 KiB block, scan, positions)
//   k_csv_pass1   one thread per line: the reference's split state machine (escape-inside-quotes, quote toggle,
//                 delimiter outside quotes, the `line[lastDelim+1:]` last-element rule), TrimSpace, unquote, the collapse of
//                 a doubled quote character (DoubleQuoteStr = quote + quote) into `"`; fixed-width cells are converted and stored column-major (coalesced across lines),
//                 text cells leave (start, length) spans
//   k_csv_offsets per text column: exclusive scan of lengths -> uint32 offsets
//   k_csv_pass2   copy text cells into the column heaps
// The result is an ordinary HBM-resident tf_batch that the transformer / encode chain consumes directly.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"

namespace tfk {

enum CsvErr : int { CSV_MISSING_CELL = 16, CSV_SINGLE_QUOTE = 17, CSV_BAD_INT = 18, CSV_RANGE = 19, CSV_BAD_BOOL = 20,
                    CSV_BAD_TIME = 21, CSV_BAD_FLOAT = 22, CSV_UNSUPPORTED = 23, CSV_DOUBLE_QUOTE_DISABLED = 24,
                    CSV_QUOTING_DISABLED = 25 };

#define CSV_NL_BLOCK 8192

struct CsvCfg {
    uint8_t delimiter, quote, escape, double_quote, strings_can_be_null, quoted_strings_can_be_null, include_missing, pad;
    // value lists live in one blob: [n:u32][off:u32 x (n+1)][bytes]
    uint32_t null_list, true_list, false_list;     // offsets into the blob, 0xffffffff = empty
};

struct CsvColDev {
    int32_t tf; int32_t path;        // path < 0: default value
    int32_t w;                       // fixed width, 0 = text
    int32_t slot;                    // index among text columns (w == 0), else -1
    uint8_t* values;                 // [nrows * w] staging, column-major
    uint32_t* aux32;                 // time columns: nanoseconds
    uint8_t* aux8;                   // any columns: tag (1 = Go string)
};

struct CsvArgs {
    const uint8_t* text; uint64_t len;
    const uint32_t* line_end;        // position after each '\n'
    uint64_t nlines, skip;           // data rows = nlines - skip
    CsvCfg cfg; const uint8_t* blob;
    const CsvColDev* cols; int ncols;
    const int16_t* field_col; int nfields;       // first schema column that reads field f, -1 none
    const int16_t* next_same;                    // next schema column with the same path, -1 none
    uint32_t* span_start; uint32_t* span_len;    // [nslots][nrows]; len bit31 = contains a doubled quote (collapse on copy)
    uint32_t* span_raw;                          // [nslots][nrows]; the uncollapsed length of a bit31 span (set only for those)
    uint8_t* err;                                // [nrows] CSV_* code
};

// `endbits` (JSON parser): bit p set = byte p is the last byte of a message, which ends a line like '\n' does
__device__ __forceinline__ bool csv_line_end(const uint8_t* text, const uint32_t* endbits, uint64_t p) { return text[p] == '\n' || (endbits && ((endbits[p >> 5] >> (p & 31)) & 1)); }

#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(256) k_csv_count_nl(const uint8_t* text, uint64_t len, uint32_t* blk_cnt, const uint32_t* endbits) {
    __shared__ uint32_t sm[33];
    const uint64_t b0 = (uint64_t)blockIdx.x * CSV_NL_BLOCK;
    uint32_t c = 0;
    for (uint32_t k = 0; k < CSV_NL_BLOCK / 256; k++) { const uint64_t p = b0 + (uint64_t)threadIdx.x * (CSV_NL_BLOCK / 256) + k; if (p < len && csv_line_end(text, endbits, p)) c++; }
    uint32_t tot; block_excl_scan(c, &tot, sm);
    if (threadIdx.x == 0) blk_cnt[blockIdx.x] = tot;
}
#endif  // TF_KERNELS_CSV

#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(256) k_csv_line_index(const uint8_t* text, uint64_t len, const uint32_t* blk_off, uint32_t* line_end, const uint32_t* endbits) {
    __shared__ uint32_t sm[33];
    const uint64_t b0 = (uint64_t)blockIdx.x * CSV_NL_BLOCK;
    const uint64_t t0 = b0 + (uint64_t)threadIdx.x * (CSV_NL_BLOCK / 256);
    uint32_t c = 0;
    for (uint32_t k = 0; k < CSV_NL_BLOCK / 256; k++) { const uint64_t p = t0 + k; if (p < len && csv_line_end(text, endbits, p)) c++; }
    uint32_t tot; uint32_t ex = block_excl_scan(c, &tot, sm);
    uint32_t w = blk_off[blockIdx.x] + ex;
    for (uint32_t k = 0; k < CSV_NL_BLOCK / 256; k++) { const uint64_t p = t0 + k; if (p < len && csv_line_end(text, endbits, p)) line_end[w++] = (uint32_t)(p + 1); }
}
#endif  // TF_KERNELS_CSV

// Var-width columns may arrive with uint8 / uint16 LENGTHS instead of uint32 offsets (tf_col.flags TF_COL_LENS8 / 16: a quarter / half
// of the offset bytes over PCIe); widened here, then scanned into offsets by the three kernels above.
struct LensSrc { const uint8_t* p; int32_t width, pad; };
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(256) k_widen_lens(const LensSrc* src, uint64_t nrows, uint32_t* out /* [nslots][nrows] */) {
    const LensSrc ls = src[blockIdx.y];
    uint32_t* o = out + (size_t)blockIdx.y * nrows;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (uint64_t)gridDim.x * blockDim.x)
        o[r] = ls.width == 1 ? (uint32_t)ls.p[r] : (uint32_t)((const uint16_t*)ls.p)[r];
}
#endif  // TF_KERNELS_CSV

// ---- text -> value helpers (must agree with oracle/csv_oracle.hpp, which restates the Go functions)
__device__ __forceinline__ bool d_space(const uint8_t* p, uint32_t n, uint32_t& w) {   // unicode.IsSpace
    if (!n) return false;
    const uint8_t b = p[0];
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
__device__ __forceinline__ void d_trim(const uint8_t*& p, uint32_t& n) {
    uint32_t w;
    while (n && d_space(p, n, w)) { p += w; n -= w; }
    for (;;) {
        if (!n) return;
        if (d_space(p + n - 1, 1, w)) { n -= 1; continue; }
        if (n >= 2 && d_space(p + n - 2, 2, w) && w == 2) { n -= 2; continue; }
        if (n >= 3 && d_space(p + n - 3, 3, w) && w == 3) { n -= 3; continue; }
        return;
    }
}
__device__ __forceinline__ bool d_in_list(const uint8_t* blob, uint32_t list, const uint8_t* p, uint32_t n) {
    if (list == 0xffffffffu) return false;
    const uint32_t cnt = *(const uint32_t*)(blob + list); const uint32_t* off = (const uint32_t*)(blob + list + 4); const uint8_t* bytes = (const uint8_t*)(off + cnt + 1);
    for (uint32_t k = 0; k < cnt; k++) {
        const uint32_t a = off[k], b = off[k + 1];
        if (b - a != n) continue;
        uint32_t i = 0; while (i < n && bytes[a + i] == p[i]) i++;
        if (i == n) return true;
    }
    return false;
}
// strconv.ParseInt(trimZeroDecimal(s), 0, 0): rc 0 ok, 1 error, 2 unsupported (underscores)
static __device__ int d_parse_int(const uint8_t* s, uint32_t n, int64_t& out) {
    { bool zero = false; uint32_t i = n; for (; i > 0; i--) { const uint8_t c = s[i - 1]; if (c == '.') { if (zero) n = i - 1; break; } else if (c == '0') zero = true; else break; } }
    if (!n) return 1;
    uint32_t i = 0; bool neg = false;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; if (n == 1) return 1; }
    uint32_t base = 10;
    if (s[i] == '0' && i + 1 < n) {
        const uint8_t c = s[i + 1] | 0x20;
        if (c == 'x') { base = 16; i += 2; } else if (c == 'b') { base = 2; i += 2; } else if (c == 'o') { base = 8; i += 2; } else { base = 8; i += 1; }
        if (i >= n) return 1;
    }
    uint64_t v = 0; const uint64_t lim = neg ? (1ull << 63) : ((1ull << 63) - 1);
    const bool safe = n - i <= 15;             // 15 digits of any base up to 16 stay below 2^63: no overflow check (a 64-bit division) per digit
    for (; i < n; i++) {
        const uint8_t c = s[i]; uint32_t d;
        if (c == '_') return 2;
        if (c >= '0' && c <= '9') d = c - '0'; else if ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') d = (c | 0x20) - 'a' + 10; else return 1;
        if (d >= base) return 1;
        if (!safe && v > (lim - d) / base) return 1;      // v * base + d > lim
        v = v * base + d;
    }
    out = neg ? (int64_t)(0 - v) : (int64_t)v; return 0;
}
__device__ __forceinline__ bool d_eq(const uint8_t* s, uint32_t n, const char* lit) { uint32_t i = 0; for (; lit[i]; i++) if (i >= n || s[i] != (uint8_t)lit[i]) return false; return i == n; }
static __device__ int d_parse_bool(const uint8_t* s, uint32_t n, bool& out) {   // strconv.ParseBool
    if (d_eq(s, n, "1") || d_eq(s, n, "t") || d_eq(s, n, "T") || d_eq(s, n, "TRUE") || d_eq(s, n, "true") || d_eq(s, n, "True")) { out = true; return 0; }
    if (d_eq(s, n, "0") || d_eq(s, n, "f") || d_eq(s, n, "F") || d_eq(s, n, "FALSE") || d_eq(s, n, "false") || d_eq(s, n, "False")) { out = false; return 0; }
    return 1;
}
__constant__ double d_p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
// decimal text -> double, exact when <= 15 significant digits and |exp10| <= 22 (one correctly rounded IEEE op); rc 2 otherwise.
// f32 (optional): the same text rounded once to binary32, as strconv.ParseFloat(s, 32) does, not through the double
static __device__ int d_parse_float(const uint8_t* s, uint32_t n, double& out, float* f32 = nullptr) {
    uint32_t i = 0; bool neg = false;
    if (!n) return 1;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    uint64_t m = 0; int nd = 0, dp = 0; bool any = false, dot = false;
    for (; i < n; i++) {
        const uint8_t c = s[i];
        if (c >= '0' && c <= '9') { any = true; if (m || c != '0') { if (nd >= 19) return 2; m = m * 10 + (c - '0'); nd++; } if (dot) dp--; }
        else if (c == '.' && !dot) dot = true;
        else break;
    }
    if (!any) return (n - i >= 3) ? 2 : 1;
    int e = 0;
    if (i < n && (s[i] | 0x20) == 'e') {
        i++; bool eneg = false; if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; i++; }
        if (i >= n) return 1; int ev = 0;
        for (; i < n; i++) { if (s[i] < '0' || s[i] > '9') return 1; if (ev < 10000) ev = ev * 10 + (s[i] - '0'); }
        e = eneg ? -ev : ev;
    }
    if (i != n) return (s[i] == '_' || (s[i] | 0x20) == 'x' || (s[i] | 0x20) == 'p') ? 2 : 1;
    e += dp;
    if (m == 0) { out = neg ? -0.0 : 0.0; if (f32) *f32 = neg ? -0.0f : 0.0f; return 0; }
    if (nd > 15 || e < -22 || e > 22) return 2;
    const double md = (double)m, p = d_p10[e < 0 ? -e : e];
    const double d = e < 0 ? __ddiv_rn(md, p) : __dmul_rn(md, p);
    out = neg ? -d : d;
    if (f32) {
        // Rounding d again to binary32 errs only when d sits exactly on a binary32 midpoint (low 29 mantissa bits 1 << 28)
        // while m * 10^e does not. m < 2^50 and 10^|e| are exact, so one fma gives the exact residual, whose sign picks the
        // side; a zero residual is a true midpoint and ties to even. Values here lie in [1e-22, 1e37]: binary32 normals.
        float f = __double2float_rn(d);
        if ((__double_as_longlong(d) & 0x1FFFFFFFll) == (1ll << 28)) {
            const double r = e < 0 ? __fma_rn(-d, p, md) : __fma_rn(md, p, -d);       // sign of m * 10^e - d
            if (r > 0) f = __double2float_ru(d); else if (r < 0) f = __double2float_rd(d);
        }
        *f32 = neg ? -f : f;
    }
    return 0;
}
__device__ __forceinline__ int64_t d_days_from_civil(int64_t y, unsigned m, unsigned d) {
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const unsigned yoe = (unsigned)(y - era * 400);
    const unsigned doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
    const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}
static __device__ int d_parse_time(const uint8_t* s, uint32_t n, int64_t& sec, uint32_t& nsec) {
    auto dig = [&](uint32_t p, int k, int& v) { v = 0; for (int i = 0; i < k; i++) { if (p + i >= n || s[p + i] < '0' || s[p + i] > '9') return false; v = v * 10 + (s[p + i] - '0'); } return true; };
    int y, mo, d, hh = 0, mi = 0, ss = 0; nsec = 0; int64_t off = 0;
    if (!(dig(0, 4, y) && n >= 10 && s[4] == '-' && dig(5, 2, mo) && s[7] == '-' && dig(8, 2, d))) return 2;
    const int dm[13] = {0, 31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    if (mo < 1 || mo > 12 || d < 1 || d > dm[mo] + ((mo == 2 && leap) ? 1 : 0)) return 1;
    uint32_t p = 10;
    if (p < n) {
        if (s[p] != 'T' && s[p] != ' ') return 2;
        if (!(dig(p + 1, 2, hh) && p + 3 < n && s[p + 3] == ':' && dig(p + 4, 2, mi) && p + 6 < n && s[p + 6] == ':' && dig(p + 7, 2, ss))) return 2;
        if (hh > 23 || mi > 59 || ss > 59) return 1;
        p += 9;
        if (p < n && s[p] == '.') { uint32_t q = p + 1; uint32_t f = 0; int k = 0; while (q < n && s[q] >= '0' && s[q] <= '9') { if (k < 9) { f = f * 10 + (s[q] - '0'); k++; } q++; } if (q == p + 1) return 2; while (k < 9) { f *= 10; k++; } nsec = f; p = q; }
        if (p < n) {
            if (s[p] == 'Z' && p + 1 == n) p++;
            else if (s[p] == '+' || s[p] == '-') {
                const int sign = s[p] == '-' ? -1 : 1; int oh, om;
                if (dig(p + 1, 2, oh) && p + 3 < n && s[p + 3] == ':' && dig(p + 4, 2, om) && p + 6 == n) off = sign * (oh * 3600 + om * 60);
                else if (dig(p + 1, 2, oh) && dig(p + 3, 2, om) && p + 5 == n) off = sign * (oh * 3600 + om * 60);
                else return 2;
                p = n;
            } else return 2;
        }
    }
    if (p != n) return 2;
    sec = d_days_from_civil(y, (unsigned)mo, (unsigned)d) * 86400 + hh * 3600 + mi * 60 + ss - off;
    return 0;
}

__device__ __forceinline__ void csv_store_fixed(const CsvColDev& c, uint64_t row, const uint64_t v, uint32_t nsec) {
    switch (c.w) {
    case 1: c.values[row] = (uint8_t)v; break;
    case 2: ((uint16_t*)c.values)[row] = (uint16_t)v; break;
    case 4: ((uint32_t*)c.values)[row] = (uint32_t)v; break;
    default: ((uint64_t*)c.values)[row] = v; break;
    }
    if (c.aux32) c.aux32[row] = nsec;
}

// getCorrespondingValue + strictifyValue for one cell [p, p+n) (already sanitised); text cells return their span
static __device__ int csv_cell(const CsvArgs& a, const CsvColDev& c, uint64_t row, uint64_t nrows, const uint8_t* p, uint32_t n, bool has_dq) {
    const CsvCfg& o = a.cfg;
    if (has_dq && c.w) return CSV_UNSUPPORTED;       // a doubled quote inside a numeric cell: the collapsed text would have to be materialised first
    switch (c.tf) {
    case TF_BOOLEAN: {
        bool b;
        if (o.strings_can_be_null && d_in_list(a.blob, o.null_list, p, n)) b = false;
        else if (d_in_list(a.blob, o.true_list, p, n)) b = true;
        else if (d_in_list(a.blob, o.false_list, p, n)) b = false;
        else if (d_parse_bool(p, n, b)) return CSV_BAD_BOOL;
        csv_store_fixed(c, row, b ? 1 : 0, 0); return 0;
    }
    case TF_TIMESTAMP: {
        bool num = n > 0; uint32_t i = (n && (p[0] == '+' || p[0] == '-')) ? 1 : 0; if (i == n) num = false;
        for (uint32_t k = i; k < n && num; k++) if (p[k] < '0' || p[k] > '9') num = false;
        int64_t sec = 0; uint32_t nsec = 0;
        if (num) {
            const bool neg = p[0] == '-'; const uint64_t lim = neg ? (1ull << 63) : ((1ull << 63) - 1); uint64_t v = 0;
            for (uint32_t k = i; k < n; k++) { const uint32_t d = p[k] - '0'; if (v > (lim - d) / 10) { num = false; break; } v = v * 10 + d; }
            if (num) sec = neg ? (int64_t)(0 - v) : (int64_t)v;
        }
        if (!num) { const int rc = d_parse_time(p, n, sec, nsec); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_TIME; }
        csv_store_fixed(c, row, (uint64_t)sec, nsec); return 0;
    }
    case TF_DATE: case TF_DATETIME: {
        int64_t sec; uint32_t nsec; const int rc = d_parse_time(p, n, sec, nsec); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_TIME;
        csv_store_fixed(c, row, (uint64_t)sec, nsec); return 0;
    }
    case TF_FLOAT: case TF_DOUBLE: {
        double d; float f; const int rc = d_parse_float(p, n, d, c.tf == TF_FLOAT ? &f : nullptr); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_FLOAT;
        if (c.tf == TF_FLOAT) csv_store_fixed(c, row, __float_as_uint(f), 0); else csv_store_fixed(c, row, (uint64_t)__double_as_longlong(d), 0);
        return 0;
    }
    }
    bool null;
    if (o.quoted_strings_can_be_null) {
        const uint8_t* q = p; uint32_t m = n;
        if (m >= 2 && ((q[0] == '"' && q[m - 1] == '"') || (q[0] == '\'' && q[m - 1] == '\''))) { q++; m -= 2; }
        else if (m == 1 && (q[0] == '"' || q[0] == '\'')) { q++; m = 0; }
        null = d_in_list(a.blob, o.null_list, q, m);
    } else null = o.strings_can_be_null && d_in_list(a.blob, o.null_list, p, n);
    if (!c.w) {      // utf8 / string / any
        uint32_t* ss = a.span_start + (size_t)c.slot * nrows; uint32_t* sl = a.span_len + (size_t)c.slot * nrows;
        if (null) { if (c.tf == TF_ANY) { ss[row] = 0xffffffffu; sl[row] = 2; c.aux8[row] = 0; } else { ss[row] = 0; sl[row] = 0; } return 0; }
        uint32_t fl = n;
        if (has_dq) { const uint8_t q = o.quote; uint32_t k = 0; fl = 0; while (k < n) { if (p[k] == q && k + 1 < n && p[k + 1] == q) k += 2; else k++; fl++; } }
        ss[row] = (uint32_t)(p - a.text); sl[row] = fl | (has_dq ? 0x80000000u : 0u);
        if (has_dq) a.span_raw[(size_t)c.slot * nrows + row] = n;
        if (c.tf == TF_ANY) c.aux8[row] = 1;
        return 0;
    }
    if (c.tf == TF_INTERVAL) { if (null) { csv_store_fixed(c, row, 0, 0); return 0; } return CSV_UNSUPPORTED; }
    if (null) { csv_store_fixed(c, row, 0, 0); return 0; }
    int64_t v; const int rc = d_parse_int(p, n, v); if (rc) return rc == 2 ? CSV_UNSUPPORTED : CSV_BAD_INT;
    int64_t lo, hi; bool uns = false;
    switch (c.tf) {
    case TF_INT8: lo = -128; hi = 127; break; case TF_INT16: lo = -32768; hi = 32767; break;
    case TF_INT32: lo = -2147483648LL; hi = 2147483647LL; break; case TF_INT64: lo = (int64_t)(1ull << 63); hi = 0x7fffffffffffffffLL; break;
    case TF_UINT8: uns = true; lo = 0; hi = 255; break; case TF_UINT16: uns = true; lo = 0; hi = 65535; break;
    case TF_UINT32: uns = true; lo = 0; hi = 4294967295LL; break; default: uns = true; lo = 0; hi = 0x7fffffffffffffffLL; break;
    }
    if (uns && v < 0) return CSV_BAD_INT;
    if (v < lo || v > hi) return CSV_RANGE;
    csv_store_fixed(c, row, (uint64_t)v, 0); return 0;
}

__device__ __forceinline__ void csv_default(const CsvArgs& a, const CsvColDev& c, uint64_t row, uint64_t nrows) {   // abstract.DefaultValue
    if (c.w) { csv_store_fixed(c, row, 0, 0); return; }
    uint32_t* ss = a.span_start + (size_t)c.slot * nrows; uint32_t* sl = a.span_len + (size_t)c.slot * nrows;
    if (c.tf == TF_ANY) { ss[row] = 0xffffffffu; sl[row] = 2; c.aux8[row] = 0; } else { ss[row] = 0; sl[row] = 0; }
}

// One row, start to end, by one thread: the reference's split loop as written (pkg/csv/reader.go:229-261). The warp-parallel kernel below
// falls back to it for lines with more delimiters than its table holds.
static __device__ void csv_row_sequential(const CsvArgs& a, uint64_t row, uint64_t nrows) {
    const uint64_t ln = row + a.skip;
    const uint32_t ls = ln ? a.line_end[ln - 1] : 0, le = a.line_end[ln];
    const uint8_t* line = a.text + ls; const uint32_t n = le - ls;
    const CsvCfg& o = a.cfg;
    int err = 0; int nf = 0;                      // split-level error (aborts the line); fields seen
    int conv_err = 0, conv_col = 0x7fffffff;      // conversion error of the FIRST schema column that fails (strictify walks columns in order)
    // one sanitised element -> every schema column that reads field f
    auto element = [&](uint32_t ea, uint32_t eb, int f) {
        const uint8_t* p = line + ea; uint32_t m = eb - ea;
        d_trim(p, m);
        bool has_dq = false;
        if (o.quote) {
            if (m == 1 && p[0] == o.quote) { err = CSV_SINGLE_QUOTE; return; }
            if (m >= 2 && p[0] == o.quote && p[m - 1] == o.quote) { p++; m -= 2; }
            for (uint32_t k = 0; k + 1 < m; k++) if (p[k] == o.quote && p[k + 1] == o.quote) { has_dq = true; break; }
            if (has_dq && !o.double_quote) { err = CSV_DOUBLE_QUOTE_DISABLED; return; }
        }
        if (f < a.nfields) for (int c = a.field_col[f]; c >= 0; c = a.next_same[c]) {
            const int rc = csv_cell(a, a.cols[c], row, nrows, p, m, has_dq);
            if (rc && c < conv_col) { conv_col = c; conv_err = rc; }
        }
    };
    if (!o.quote) for (uint32_t i = 0; i < n; i++) if (line[i] == '"') { err = CSV_QUOTING_DISABLED; break; }      // readAndDecodeLine (reader.go:185-187), before the split
    if (n > 1 && !err) {
        uint8_t prev = 0; bool inq = false; uint32_t prev_delim = 0, last_delim = 0;
        for (uint32_t i = 0; i < n && !err; i++) {
            const uint8_t c = line[i];
            if (o.escape && o.escape == prev && inq) { prev = c; continue; }
            if (o.quote && c == o.quote) { inq = !inq; prev = c; continue; }
            if (c == o.delimiter && !inq) { last_delim = i; element(prev_delim, last_delim, nf); nf++; prev_delim = last_delim + 1; }
            prev = c;
        }
        if (!err) { element(last_delim + 1 <= n ? last_delim + 1 : n, n, nf); nf++; }    // line[lastDelimPosition+1:], lastDelimPosition == 0 without delimiters
    }
    // columns whose field is missing, or that take the default value (reader_csv.go:291-313). constructCI runs over
    // every column before Strictify does, so a missing cell outranks any conversion error.
    for (int c = 0; c < a.ncols && !err; c++) {
        const CsvColDev& cd = a.cols[c];
        if (cd.path < 0) csv_default(a, cd, row, nrows);
        else if (cd.path >= nf) { if (o.include_missing) csv_default(a, cd, row, nrows); else err = CSV_MISSING_CELL; }
    }
    if (!err) err = conv_err;
    if (err) {   // an error row is dropped later; give its cells harmless contents
        for (int c = 0; c < a.ncols; c++) { const CsvColDev& cd = a.cols[c]; if (!cd.w) { a.span_start[(size_t)cd.slot * nrows + row] = 0; a.span_len[(size_t)cd.slot * nrows + row] = 0; if (cd.aux8) cd.aux8[row] = 0; } else csv_store_fixed(cd, row, 0, 0); }
    }
    a.err[row] = (uint8_t)err;
}

// Warp-parallel tokeniser: one warp per line. The line is read 32 bytes at a time (coalesced); ballots give the quote / delimiter bitmaps of
// the slab; the in-quote state of every byte comes from bit counts over the quote bitmap — a quote that follows the escape character
// leaves the state "inside" whatever it was (reader.go:236-243: inside quotes it is skipped, outside it opens a quote), every other quote
// toggles it — so no lane walks the line; delimiters outside quotes get their ordinal from a popc prefix and land in a shared-memory
// table. Then the lanes take the line's elements 32 at a time: trim, unquote, typed parse (csv_cell) — the field-level work of a
// 99-column row runs 32 wide instead of serially.
#define CSV_WARPS 8
#define CSV_MAXF 512
// rows [row0, row1), one warp per line; s_dpos [CSV_WARPS][CSV_MAXF], s_fq [CSV_WARPS][CSV_MAXF / 32 + 1] (bit f: element f contains a quote character)
static __device__ void csv_rows_by_warp(const CsvArgs& a, uint64_t row0, uint64_t row1, uint32_t (*s_dpos)[CSV_MAXF], uint32_t (*s_fq)[CSV_MAXF / 32 + 1]) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, below = (1u << lane) - 1;
    const uint64_t nrows = a.nlines - a.skip;
    const CsvCfg& o = a.cfg;
    for (uint64_t row = row0 + warp; row < row1; row += CSV_WARPS) {
        const uint64_t ln = row + a.skip;
        const uint32_t ls = ln ? a.line_end[ln - 1] : 0, le = a.line_end[ln];
        const uint8_t* line = a.text + ls; const uint32_t n = le - ls;
        // ---- tokenise
        uint32_t nd = 0, dq = 0;         // dq: a '"' on a line read without a quote character
        if (lane <= CSV_MAXF / 32) s_fq[warp][lane] = 0;
        __syncwarp();
        if (n > 1) {
            uint32_t inq_carry = 0; uint32_t prevc = 0;
            for (uint32_t base = 0; base < n; base += 32) {
                const uint32_t i = base + lane; const bool in = i < n;
                const uint32_t c = in ? line[i] : 0u;
                if (!o.quote) dq |= __ballot_sync(0xffffffffu, c == '"');
                const uint32_t up = __shfl_up_sync(0xffffffffu, c, 1); const uint32_t prev = lane ? up : prevc;
                const bool isq = in && o.quote && c == o.quote;
                const uint32_t qm = __ballot_sync(0xffffffffu, isq);
                const uint32_t eqm = __ballot_sync(0xffffffffu, isq && o.escape && prev == o.escape);
                const uint32_t nm = qm & ~eqm;
                uint32_t inq;
                const uint32_t eqb = eqm & below;
                if (eqb) { const uint32_t h = 31 - __clz(eqb); inq = 1u ^ (__popc(nm & below & ~((2u << h) - 1)) & 1u); }
                else inq = inq_carry ^ (__popc(nm & below) & 1u);
                const bool isd = in && c == o.delimiter && !isq && !inq;
                const uint32_t dm = __ballot_sync(0xffffffffu, isd);
                if (isd) { const uint32_t k = nd + __popc(dm & below); if (k < CSV_MAXF) s_dpos[warp][k] = i; }
                if (isq) { const uint32_t fo = nd + __popc(dm & below); if (fo <= CSV_MAXF) atomicOr(&s_fq[warp][fo >> 5], 1u << (fo & 31)); }
                nd += __popc(dm);
                if (eqm) { const uint32_t h = 31 - __clz(eqm); inq_carry = 1u ^ (__popc(nm & ~((2u << h) - 1)) & 1u); }
                else inq_carry ^= __popc(nm) & 1u;
                prevc = __shfl_sync(0xffffffffu, c, 31);
            }
        }
        __syncwarp();
        if (nd > CSV_MAXF && !dq) { if (lane == 0) csv_row_sequential(a, row, nrows); __syncwarp(); continue; }      // more delimiters than the table holds
        const uint32_t nf = n > 1 && !dq ? nd + 1 : 0;
        // ---- elements, 32 at a time
        uint32_t err_key = 0xffffffffu, conv_key = 0xffffffffu;      // (field << 8) | code of the first split-level error; (column << 8) | code of the first conversion error
        for (uint32_t f = lane; f < nf; f += 32) {
            const uint32_t ea = f ? s_dpos[warp][f - 1] + 1 : (nd ? 0u : 1u);      // without any delimiter the element is line[1:] (lastDelimPosition stays 0, reader.go:255-259)
            const uint32_t eb = f < nd ? s_dpos[warp][f] : n;
            const uint8_t* p = line + (ea <= n ? ea : n); uint32_t m = eb - (ea <= n ? ea : n);
            if (m && !(p[0] > 0x20 && p[0] < 0x80 && p[m - 1] > 0x20 && p[m - 1] < 0x80)) d_trim(p, m);      // (every space TrimSpace knows starts <= 0x20 or >= 0x80)
            bool has_dq = false; int e = 0;
            if (o.quote && ((s_fq[warp][f >> 5] >> (f & 31)) & 1)) {
                if (m == 1 && p[0] == o.quote) e = CSV_SINGLE_QUOTE;
                else {
                    if (m >= 2 && p[0] == o.quote && p[m - 1] == o.quote) { p++; m -= 2; }
                    for (uint32_t k = 0; k + 1 < m; k++) if (p[k] == o.quote && p[k + 1] == o.quote) { has_dq = true; break; }
                    if (has_dq && !o.double_quote) e = CSV_DOUBLE_QUOTE_DISABLED;
                }
            }
            if (e) { const uint32_t key = (f << 8) | (uint32_t)e; if (key < err_key) err_key = key; continue; }
            if ((int)f < a.nfields) for (int c = a.field_col[f]; c >= 0; c = a.next_same[c]) {
                const int rc = csv_cell(a, a.cols[c], row, nrows, p, m, has_dq);
                if (rc) { const uint32_t key = ((uint32_t)c << 8) | (uint32_t)rc; if (key < conv_key) conv_key = key; }
            }
        }
        err_key = __reduce_min_sync(0xffffffffu, err_key); conv_key = __reduce_min_sync(0xffffffffu, conv_key);
        int err = dq ? CSV_QUOTING_DISABLED : err_key == 0xffffffffu ? 0 : (int)(err_key & 0xff);      // (raised before the split: outranks the rest)
        // columns whose field is missing, or that take the default value (reader_csv.go:291-313). constructCI runs over
        // every column before Strictify does, so a missing cell outranks any conversion error.
        bool missing = false;
        if (!err) for (int c = (int)lane; c < a.ncols; c += 32) {
            const CsvColDev& cd = a.cols[c];
            if (cd.path < 0) csv_default(a, cd, row, nrows);
            else if ((uint32_t)cd.path >= nf) { if (o.include_missing) csv_default(a, cd, row, nrows); else missing = true; }
        }
        if (!err && __any_sync(0xffffffffu, missing)) err = CSV_MISSING_CELL;
        if (!err && conv_key != 0xffffffffu) err = (int)(conv_key & 0xff);
        if (err) {   // an error row is dropped later; give its cells harmless contents
            __syncwarp();
            for (int c = (int)lane; c < a.ncols; c += 32) { const CsvColDev& cd = a.cols[c]; if (!cd.w) { a.span_start[(size_t)cd.slot * nrows + row] = 0; a.span_len[(size_t)cd.slot * nrows + row] = 0; if (cd.aux8) cd.aux8[row] = 0; } else csv_store_fixed(cd, row, 0, 0); }
        }
        if (lane == 0) a.err[row] = (uint8_t)err;
        __syncwarp();
    }
}

// The main kernel: a CTA takes 32 consecutive lines. Their bytes are one contiguous stretch of the text, staged in shared memory with
// coalesced loads; the warps tokenise them (4 lines each, the ballot scheme above) into a table of element boundaries; then LANE = LINE
// and the warps stride over the ELEMENTS: all 32 lanes parse the same column of 32 different rows — the same cell type, so no divergence
// over types, and 32 consecutive rows of one column are stored together (coalesced). Tiles longer than the staging buffer and tables
// with more than CSV_TF fields take the warp-per-line path.
#define CSV_TILE_ROWS 32
#define CSV_TILE_BYTES 28672
#define CSV_TF 250            /* element boundaries kept per line */
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(32 * CSV_WARPS, 4) k_csv_pass1(CsvArgs a) {
    __shared__ __align__(16) uint8_t s_tile[CSV_TILE_BYTES + 16];      // (the warp-per-line tables alias it)
    __shared__ uint16_t s_end[CSV_TILE_ROWS][CSV_TF + 2];              // position (relative to the line) of the first CSV_TF delimiters
    __shared__ uint32_t s_fqt[CSV_TILE_ROWS][(CSV_TF + 32) / 32];      // bit f: element f of the line contains a quote character
    __shared__ uint32_t s_nd[CSV_TILE_ROWS], s_errk[CSV_TILE_ROWS], s_convk[CSV_TILE_ROWS], s_miss[CSV_TILE_ROWS], s_ls[CSV_TILE_ROWS + 1];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, below = (1u << lane) - 1;
    const uint64_t nrows = a.nlines - a.skip;
    const CsvCfg& o = a.cfg;
    for (uint64_t row0 = (uint64_t)blockIdx.x * CSV_TILE_ROWS; row0 < nrows; row0 += (uint64_t)gridDim.x * CSV_TILE_ROWS) {
        const uint32_t nr = (uint32_t)(nrows - row0 < CSV_TILE_ROWS ? nrows - row0 : CSV_TILE_ROWS);
        const uint64_t ln0 = row0 + a.skip;
        const uint32_t g0 = ln0 ? a.line_end[ln0 - 1] : 0, g1 = a.line_end[ln0 + nr - 1];
        __syncthreads();
        if (g1 - g0 > CSV_TILE_BYTES || a.nfields > CSV_TF) {      // long lines / wide tables: one warp per line, straight from global memory
            csv_rows_by_warp(a, row0, row0 + nr, (uint32_t (*)[CSV_MAXF])s_tile, (uint32_t (*)[CSV_MAXF / 32 + 1])(s_tile + sizeof(uint32_t) * CSV_WARPS * CSV_MAXF));
            continue;
        }
        // ---- stage the tile
        {
            const uint32_t mis = (uint32_t)((uintptr_t)(a.text + g0) & 15);       // 16-byte chunks of the text, aligned in global memory
            const uint8_t* gb = a.text + g0 - mis; const uint32_t nchunk = (mis + (g1 - g0) + 15) >> 4;
            const int64_t gs = (int64_t)g0 - (int64_t)mis;      // text offset of s_tile[0]: negative in the first tile of a text that starts misaligned
            for (uint32_t c = threadIdx.x; c < nchunk; c += blockDim.x) {
                const uint32_t off = c * 16; const int64_t t = gs + off;
                // the tile is kept at the same misalignment: s_tile[mis + k] = text[g0 + k]; bytes outside [0, len) of the text are zeros
                if (t >= 0 && t + 16 <= (int64_t)a.len) *(int4*)(s_tile + off) = __ldg((const int4*)(gb + off));
                else for (uint32_t b = 0; b < 16; b++) s_tile[off + b] = (t + b >= 0 && t + b < (int64_t)a.len) ? gb[off + b] : 0;
            }
            if (threadIdx.x <= nr) s_ls[threadIdx.x] = (threadIdx.x ? a.line_end[ln0 + threadIdx.x - 1] : g0) - g0 + mis;
            if (threadIdx.x < CSV_TILE_ROWS) { s_errk[threadIdx.x] = 0xffffffffu; s_convk[threadIdx.x] = 0xffffffffu; s_miss[threadIdx.x] = 0; s_nd[threadIdx.x] = 0; }
            for (uint32_t k = threadIdx.x; k < CSV_TILE_ROWS * ((CSV_TF + 32) / 32); k += blockDim.x) (&s_fqt[0][0])[k] = 0;
        }
        __syncthreads();
        // ---- tokenise: warp w takes lines w, w + 8, ...
        for (uint32_t r = warp; r < nr; r += CSV_WARPS) {
            const uint8_t* line = s_tile + s_ls[r]; const uint32_t n = s_ls[r + 1] - s_ls[r];
            uint32_t nd = 0, dq = 0;        // dq: a '"' on a line read without a quote character
            if (n > 1) {
                uint32_t inq_carry = 0, prevc = 0;
                for (uint32_t base = 0; base < n; base += 32) {
                    const uint32_t i = base + lane; const bool in = i < n;
                    const uint32_t c = in ? line[i] : 0u;
                    if (!o.quote) dq |= __ballot_sync(0xffffffffu, c == '"');
                    const uint32_t up = __shfl_up_sync(0xffffffffu, c, 1); const uint32_t prev = lane ? up : prevc;
                    const bool isq = in && o.quote && c == o.quote;
                    const uint32_t qm = __ballot_sync(0xffffffffu, isq);
                    const uint32_t eqm = __ballot_sync(0xffffffffu, isq && o.escape && prev == o.escape);
                    const uint32_t nm = qm & ~eqm;
                    uint32_t inq;
                    const uint32_t eqb = eqm & below;
                    if (eqb) { const uint32_t h = 31 - __clz(eqb); inq = 1u ^ (__popc(nm & below & ~((2u << h) - 1)) & 1u); }
                    else inq = inq_carry ^ (__popc(nm & below) & 1u);
                    const bool isd = in && c == o.delimiter && !isq && !inq;
                    const uint32_t dm = __ballot_sync(0xffffffffu, isd);
                    if (isd) { const uint32_t k = nd + __popc(dm & below); if (k < CSV_TF) s_end[r][k] = (uint16_t)i; }
                    if (isq) { const uint32_t fo = nd + __popc(dm & below); if (fo <= CSV_TF) atomicOr(&s_fqt[r][fo >> 5], 1u << (fo & 31)); }
                    nd += __popc(dm);
                    if (eqm) { const uint32_t h = 31 - __clz(eqm); inq_carry = 1u ^ (__popc(nm & ~((2u << h) - 1)) & 1u); }
                    else inq_carry ^= __popc(nm) & 1u;
                    prevc = __shfl_sync(0xffffffffu, c, 31);
                }
            }
            if (lane == 0) s_nd[r] = nd | (n > 1 ? 0x80000000u : 0u) | (dq ? 0x40000000u : 0u);      // (nd < 2^30: a tile holds 28672 bytes)
        }
        __syncthreads();
        // ---- elements: lane = line, the warps stride over the element index
        {
            const uint32_t r = lane; const bool live = r < nr;
            const uint32_t ndw = live ? s_nd[r] : 0; const uint32_t nd = ndw & 0x3fffffffu; const uint32_t nf = (ndw >> 31) && !(ndw & 0x40000000u) ? nd + 1 : 0;
            const uint32_t n = live ? s_ls[r + 1] - s_ls[r] : 0;
            const uint8_t* line = s_tile + (live ? s_ls[r] : 0);
            const uint64_t row = row0 + r;
            // csv_cell records text cells as offsets from a.text: give it a base that makes a tile pointer come out as the text offset
            CsvArgs at = a; at.text = line - ((uint64_t)g0 + (live ? s_ls[r] : 0) - (uint32_t)((uintptr_t)(a.text + g0) & 15));
            uint32_t nf_max = nf;
#pragma unroll
            for (int d = 16; d; d >>= 1) { const uint32_t v = __shfl_xor_sync(0xffffffffu, nf_max, d); nf_max = v > nf_max ? v : nf_max; }
            uint32_t err_key = 0xffffffffu, conv_key = 0xffffffffu;
            for (uint32_t f = warp; f < nf_max; f += CSV_WARPS) {
                if (f >= nf) continue;
                if (nd > CSV_TF && f >= CSV_TF) continue;                 // boundaries beyond the table: only lines of a wider table than the schema reads (checked below)
                const uint32_t ea0 = f ? (uint32_t)s_end[r][f - 1] + 1 : (nd ? 0u : 1u);      // without any delimiter the element is line[1:] (reader.go:255-259)
                const uint32_t ea = ea0 <= n ? ea0 : n, eb = f < nd ? s_end[r][f] : n;
                const uint8_t* p = line + ea; uint32_t m = eb - ea;
                if (m && !(p[0] > 0x20 && p[0] < 0x80 && p[m - 1] > 0x20 && p[m - 1] < 0x80)) d_trim(p, m);      // (every space TrimSpace knows starts <= 0x20 or >= 0x80)
                bool has_dq = false; int e = 0;
                if (o.quote && ((s_fqt[r][f >> 5] >> (f & 31)) & 1)) {
                    if (m == 1 && p[0] == o.quote) e = CSV_SINGLE_QUOTE;
                    else {
                        if (m >= 2 && p[0] == o.quote && p[m - 1] == o.quote) { p++; m -= 2; }
                        for (uint32_t k = 0; k + 1 < m; k++) if (p[k] == o.quote && p[k + 1] == o.quote) { has_dq = true; break; }
                        if (has_dq && !o.double_quote) e = CSV_DOUBLE_QUOTE_DISABLED;
                    }
                }
                if (e) { const uint32_t key = (f << 8) | (uint32_t)e; if (key < err_key) err_key = key; continue; }
                if ((int)f < a.nfields) for (int c = a.field_col[f]; c >= 0; c = a.next_same[c]) {
                    const int rc = csv_cell(at, a.cols[c], row, nrows, p, m, has_dq);
                    if (rc) { const uint32_t key = ((uint32_t)c << 8) | (uint32_t)rc; if (key < conv_key) conv_key = key; }
                }
            }
            if (live) { if (err_key != 0xffffffffu) atomicMin(&s_errk[r], err_key); if (conv_key != 0xffffffffu) atomicMin(&s_convk[r], conv_key); }
            // columns whose field is missing, or that take the default value (reader_csv.go:291-313)
            if (live) for (int c = (int)warp; c < a.ncols; c += CSV_WARPS) {
                const CsvColDev& cd = a.cols[c];
                if (cd.path < 0) csv_default(a, cd, row, nrows);
                else if ((uint32_t)cd.path >= nf) { if (o.include_missing) csv_default(a, cd, row, nrows); else s_miss[r] = 1; }
            }
        }
        __syncthreads();
        // ---- the row's verdict: a split-level error of the first element that has one, else a missing cell (constructCI runs over every
        // column before Strictify does), else the conversion error of the first schema column that fails
        {
            const uint32_t r = lane; const bool live = r < nr;
            int err = 0;
            if (live) {
                const uint32_t ndw = s_nd[r];
                if (ndw & 0x40000000u) err = CSV_QUOTING_DISABLED;         // raised before the split: outranks every other error of the line
                else if ((ndw & 0x3fffffffu) > CSV_TF) err = -1;           // more delimiters than the table holds: redo this line sequentially
                else if (s_errk[r] != 0xffffffffu) err = (int)(s_errk[r] & 0xff);
                else if (s_miss[r]) err = CSV_MISSING_CELL;
                else if (s_convk[r] != 0xffffffffu) err = (int)(s_convk[r] & 0xff);
            }
            if (warp == 0 && live && err == -1) { csv_row_sequential(a, row0 + r, nrows); }
            if (err > 0) for (int c = (int)warp; c < a.ncols; c += CSV_WARPS) {      // an error row is dropped later; give its cells harmless contents
                const CsvColDev& cd = a.cols[c]; const uint64_t row = row0 + r;
                if (!cd.w) { a.span_start[(size_t)cd.slot * nrows + row] = 0; a.span_len[(size_t)cd.slot * nrows + row] = 0; if (cd.aux8) cd.aux8[row] = 0; } else csv_store_fixed(cd, row, 0, 0);
            }
            if (warp == 0 && live && err >= 0) a.err[row0 + r] = (uint8_t)err;
        }
    }
}
#endif  // TF_KERNELS_CSV

// per text column: offsets[r] = sum of lengths of rows < r. One CTA per column walks its rows in chunks.
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(1024) k_csv_offsets(const uint32_t* span_len, uint64_t nrows, uint32_t* offsets /* [nslots][nrows+1] */, uint64_t* col_total) {
    __shared__ uint32_t sm[33];
    const uint32_t* len = span_len + (size_t)blockIdx.x * nrows; uint32_t* off = offsets + (size_t)blockIdx.x * (nrows + 1);
    uint64_t carry = 0;
    for (uint64_t base = 0; base < nrows; base += blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        const uint32_t v = i < nrows ? (len[i] & 0x7fffffffu) : 0;
        uint32_t tot; const uint32_t ex = block_excl_scan(v, &tot, sm);
        if (i < nrows) off[i] = (uint32_t)(carry + ex);
        carry += tot;
    }
    if (threadIdx.x == 0) { off[nrows] = (uint32_t)carry; col_total[blockIdx.x] = carry; }
}
#endif  // TF_KERNELS_CSV

// The same scan over many CTAs: chunk sums, a scan of the chunk sums per column, then the offsets (3 short launches instead
// of one CTA per column walking every row).
#define CSV_OFF_CHUNK 4096
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(1024) k_offsets_sum(const uint32_t* span_len, uint64_t nrows, uint32_t nchunks, uint64_t* chunk_sum /* [nslots][nchunks] */) {
    __shared__ uint32_t sm[33];
    const uint32_t* len = span_len + (size_t)blockIdx.y * nrows;
    const uint64_t base = (uint64_t)blockIdx.x * CSV_OFF_CHUNK;
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < CSV_OFF_CHUNK / 1024; k++) { const uint64_t i = base + (uint64_t)k * 1024 + threadIdx.x; if (i < nrows) v += len[i] & 0x7fffffffu; }
    uint32_t tot; block_excl_scan(v, &tot, sm);
    if (threadIdx.x == 0) chunk_sum[(size_t)blockIdx.y * nchunks + blockIdx.x] = tot;
}
#endif  // TF_KERNELS_CSV
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(32) k_offsets_chunks(uint64_t* chunk_sum, uint32_t nchunks, uint64_t* col_total) {     // in place: exclusive scan per column, one warp
    uint64_t* cs = chunk_sum + (size_t)blockIdx.x * nchunks;
    const uint32_t lane = threadIdx.x;
    uint64_t carry = 0;
    for (uint32_t base = 0; base < nchunks; base += 32) {
        const uint32_t i = base + lane;
        const uint64_t v = i < nchunks ? cs[i] : 0;
        uint64_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint64_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += o; }
        if (i < nchunks) cs[i] = carry + inc - v;
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) col_total[blockIdx.x] = carry;
}
#endif  // TF_KERNELS_CSV
#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(1024) k_offsets_write(const uint32_t* span_len, uint64_t nrows, uint32_t nchunks, const uint64_t* chunk_base, const uint64_t* col_total, uint32_t* offsets /* [nslots][nrows+1] */) {
    __shared__ uint32_t sm[33];
    const uint32_t* len = span_len + (size_t)blockIdx.y * nrows; uint32_t* off = offsets + (size_t)blockIdx.y * (nrows + 1);
    const uint64_t base = (uint64_t)blockIdx.x * CSV_OFF_CHUNK + (uint64_t)threadIdx.x * (CSV_OFF_CHUNK / 1024);      // 4 consecutive rows per thread
    uint32_t v[CSV_OFF_CHUNK / 1024]; uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < CSV_OFF_CHUNK / 1024; k++) { const uint64_t i = base + k; v[k] = i < nrows ? (len[i] & 0x7fffffffu) : 0; sum += v[k]; }
    uint32_t tot; uint32_t ex = block_excl_scan(sum, &tot, sm);
    uint64_t run = chunk_base[(size_t)blockIdx.y * nchunks + blockIdx.x] + ex;
#pragma unroll
    for (int k = 0; k < CSV_OFF_CHUNK / 1024; k++) { const uint64_t i = base + k; if (i < nrows) off[i] = (uint32_t)run; run += v[k]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) off[nrows] = (uint32_t)col_total[blockIdx.y];
}
#endif  // TF_KERNELS_CSV

struct CsvCopyArgs { const uint8_t* text; const uint32_t* span_start; const uint32_t* span_len; const uint32_t* span_raw; const uint32_t* offsets; uint8_t* heap;
                     const uint64_t* col_base; uint64_t nrows; uint8_t quote; };      // a doubled quote character in a flagged span is copied as one '"' (swapToSingleQuotes)

#ifdef TF_KERNELS_CSV
__global__ void __launch_bounds__(256) k_csv_pass2(CsvCopyArgs a) {
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= a.nrows) return;
    const uint32_t slot = blockIdx.y;
    const uint32_t st = a.span_start[(size_t)slot * a.nrows + row], lf = a.span_len[(size_t)slot * a.nrows + row];
    const uint32_t L = lf & 0x7fffffffu;
    if (!L) return;
    uint8_t* o = a.heap + a.col_base[slot] + a.offsets[(size_t)slot * (a.nrows + 1) + row];
    if (st == 0xffffffffu) { o[0] = '{'; o[1] = '}'; return; }
    const uint8_t* s = a.text + st;
    if (lf & 0x80000000u) {      // (a pair may not take the byte after the span: that can be the quote unquote stripped)
        const uint8_t q = a.quote; const uint32_t R = a.span_raw[(size_t)slot * a.nrows + row]; uint32_t k = 0;
        for (uint32_t w = 0; w < L; w++) { const bool pair = k + 1 < R && s[k] == q && s[k + 1] == q; o[w] = pair ? '"' : s[k]; k += pair ? 2 : 1; }
    }
    else for (uint32_t k = 0; k < L; k++) o[k] = s[k];
}
#endif  // TF_KERNELS_CSV

}  // namespace tfk
