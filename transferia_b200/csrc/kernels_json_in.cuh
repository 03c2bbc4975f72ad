// Generic JSON parser on the device: message bytes -> typed columns of the parser's result schema.
//   reference: pkg/parsers/generic/generic_parser.go  doGenericParser :519-555 (lines), Unmarshal :672-730 (fastjson + typed
//              extraction by the declared column type), ParseVal :888-1123, makeChangeItem :297-404, aux columns :115-164
//              github.com/valyala/fastjson v1.6.4 (go.mod:70; parser.go, fastfloat/parse.go) for the token rules.
// The CPU restatement these kernels must agree with byte for byte is oracle/json_oracle.hpp.
//   k_json_mark_msgs      bit per byte position that ends a message (a message end terminates a line like '\n')
//   k_csv_count_nl / k_csv_line_index (kernels_csv.cuh, with the bitmap)   line index
//   k_json_count_nonempty / k_json_rank / k_json_msg_first   rank of each line among the non-empty ones -> `_idx`, error rows
//   k_json_pass1          one thread per line: fastjson grammar scan, root members matched to columns (last wins),
//                         per field typed conversion, fixed cells stored column-major, text cells sized, validity by ballot
//   k_csv_offsets         per text column exclusive scan of the lengths
//   k_json_pass2          text cells written: unescaped strings, compacted raw values, base64, canonical `any` / `_rest`
// The staged columns are an ordinary HBM-resident tf_batch consumed by the transformer / encode chain.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "kernels_fmt.cuh"
#include "kernels_csv.cuh"
#include "el_tables.cuh"
#include <math_constants.h>

namespace tfk {

enum JsnErr : int { JSN_PARSE = 32, JSN_SKIP = 33, JSN_NIL_REQUIRED = 34, JSN_PARSEVAL = 35, JSN_HOST = 36, JSN_EMPTY = 37 };
enum JsnType : uint32_t { JT_ABSENT = 0, JT_NULL = 1, JT_OBJECT = 2, JT_ARRAY = 3, JT_STRING = 4, JT_NUMBER = 5, JT_TRUE = 6, JT_FALSE = 7 };
#define JSN_MAX_DEPTH 300      /* fastjson MaxDepth */
#define JSN_DEV_DEPTH 24       /* open containers the canonical `any` re-emission tracks; deeper values -> JSN_HOST */
#define JSN_MAX_COLS 128
#define JSN_NUMBUF 96          /* longest string cell converted to a number on the device; longer -> JSN_HOST */

struct JsnColDev {
    int32_t tf, w, slot;                 // slot: index among text columns, else -1
    uint8_t key, required, pad0, pad1;
    uint32_t name_off, name_len;         // into the names blob
    uint8_t* values; uint32_t* aux32; uint8_t* aux8; uint32_t* validity;
};

struct JsnArgs {
    const uint8_t* text; uint64_t len;
    const uint32_t* line_end; uint64_t nlines;
    const uint64_t* msg_end; const uint64_t* msg_offset; const int64_t* msg_wsec; const uint32_t* msg_wnsec; uint32_t nmsgs;
    const uint32_t* rank; const uint32_t* msg_rank0;
    const JsnColDev* cols; int ncols, nfields; const uint8_t* names;
    uint8_t add_rest, add_dedupe, null_keys_allowed, use_numbers, unpack_b64, pad[3];
    uint32_t part_off, part_len;
    uint32_t* span_start; uint32_t* span_len;      // [nfields][nlines]: value offset in text, length | JsnType << 28
    uint32_t* out_len;                             // [nslots][nlines]
    uint8_t* err; uint8_t* errcol;
};

// ------------------------------------------------------------------ line helpers
__global__ void k_json_mark_msgs(const uint64_t* msg_end, uint32_t nmsgs, uint32_t* bits);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(256) k_json_mark_msgs(const uint64_t* msg_end, uint32_t nmsgs, uint32_t* bits) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= nmsgs) return;
    const uint64_t e = msg_end[m], b = m ? msg_end[m - 1] : 0;
    if (e > b) atomicOr(&bits[(e - 1) >> 5], 1u << ((e - 1) & 31));
}
#endif  // TF_KERNELS_JSON_IN
__device__ __forceinline__ void jsn_line(const uint8_t* text, const uint32_t* line_end, uint64_t L, uint32_t& ls, uint32_t& n) {
    ls = L ? line_end[L - 1] : 0; uint32_t le = line_end[L];
    if (le > ls && text[le - 1] == '\n') le--;
    if (le > ls && text[le - 1] == '\r') le--;            // bufio.ScanLines dropCR
    n = le - ls;
}
__global__ void k_json_count_nonempty(const uint8_t* text, const uint32_t* line_end, uint64_t nlines, uint32_t* blk_cnt);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(128) k_json_count_nonempty(const uint8_t* text, const uint32_t* line_end, uint64_t nlines, uint32_t* blk_cnt) {
    __shared__ uint32_t sm[33];
    const uint64_t L = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t f = 0; if (L < nlines) { uint32_t ls, n; jsn_line(text, line_end, L, ls, n); f = n ? 1 : 0; }
    uint32_t tot; block_excl_scan(f, &tot, sm);
    if (threadIdx.x == 0) blk_cnt[blockIdx.x] = tot;
}
#endif  // TF_KERNELS_JSON_IN
__global__ void k_json_rank(const uint8_t* text, const uint32_t* line_end, uint64_t nlines, const uint32_t* blk_off, uint32_t* rank);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(128) k_json_rank(const uint8_t* text, const uint32_t* line_end, uint64_t nlines, const uint32_t* blk_off, uint32_t* rank) {
    __shared__ uint32_t sm[33];
    const uint64_t L = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t f = 0; if (L < nlines) { uint32_t ls, n; jsn_line(text, line_end, L, ls, n); f = n ? 1 : 0; }
    uint32_t tot; const uint32_t ex = block_excl_scan(f, &tot, sm);
    if (L < nlines) { rank[L] = blk_off[blockIdx.x] + ex; if (L == nlines - 1) rank[nlines] = blk_off[blockIdx.x] + ex + f; }
}
#endif  // TF_KERNELS_JSON_IN
// rank of the first line of every message: _idx counts the non-empty lines of its own message from 1 (:526-531)
__global__ void k_json_msg_first(const uint64_t* msg_end, uint32_t nmsgs, const uint32_t* line_end, uint64_t nlines, const uint32_t* rank, uint32_t* msg_rank0);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(256) k_json_msg_first(const uint64_t* msg_end, uint32_t nmsgs, const uint32_t* line_end, uint64_t nlines, const uint32_t* rank, uint32_t* msg_rank0) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= nmsgs) return;
    const uint64_t start = m ? msg_end[m - 1] : 0;
    uint64_t lo = 0, hi = nlines;                          // number of lines ending at or before `start`
    while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if ((uint64_t)line_end[mid] <= start) lo = mid + 1; else hi = mid; }
    msg_rank0[m] = rank[lo];
}
#endif  // TF_KERNELS_JSON_IN

// ------------------------------------------------------------------ byte sources
__device__ __forceinline__ bool jsn_ws(uint8_t c) { return c == 0x20 || c == 0x0A || c == 0x09 || c == 0x0D; }
__device__ __forceinline__ bool jsn_numch(uint8_t c) { return (c >= '0' && c <= '9') || c == '.' || c == '-' || c == 'e' || c == 'E' || c == '+'; }
__device__ __forceinline__ bool jsn_fold3(const uint8_t* s, const char* lit) { return (s[0] | 0x20) == lit[0] && (s[1] | 0x20) == lit[1] && (s[2] | 0x20) == lit[2]; }
__device__ __forceinline__ bool jsn_hex4(const uint8_t* s, uint32_t& x) {
    x = 0;
    for (int i = 0; i < 4; i++) { const uint8_t c = s[i]; uint32_t d; if (c >= '0' && c <= '9') d = c - '0'; else if ((c | 0x20) >= 'a' && (c | 0x20) <= 'f') d = (c | 0x20) - 'a' + 10; else return false; x = x * 16 + d; }
    return true;
}

// fastjson unescapeStringBestEffort as a byte stream over the raw string body
struct Dec {
    const uint8_t* s; uint32_t n, p; uint8_t q[6]; uint8_t qn, qp;
    __device__ Dec(const uint8_t* s_, uint32_t n_) : s(s_), n(n_), p(0), qn(0), qp(0) {}
    __device__ int rune(uint32_t r) {                      // string(rune(r)): first byte returned, the rest queued
        if (r < 0x80) return (int)r;
        qp = 0;
        if (r < 0x800) { q[0] = (uint8_t)(0x80 | (r & 0x3F)); qn = 1; return (int)(0xC0 | (r >> 6)); }
        if (r < 0x10000) { q[0] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); q[1] = (uint8_t)(0x80 | (r & 0x3F)); qn = 2; return (int)(0xE0 | (r >> 12)); }
        q[0] = (uint8_t)(0x80 | ((r >> 12) & 0x3F)); q[1] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); q[2] = (uint8_t)(0x80 | (r & 0x3F)); qn = 3; return (int)(0xF0 | (r >> 18));
    }
    __device__ int next() {
        if (qp < qn) return q[qp++];
        if (p >= n) return -1;
        const uint8_t c = s[p++];
        if (c != '\\') return c;
        if (p >= n) return -1;
        const uint8_t ch = s[p++];
        switch (ch) {
        case '"': return '"'; case '\\': return '\\'; case '/': return '/';
        case 'b': return 8; case 'f': return 12; case 'n': return 10; case 'r': return 13; case 't': return 9;
        case 'u': {
            uint32_t x;
            if (n - p < 4 || !jsn_hex4(s + p, x)) { q[0] = 'u'; qn = 1; qp = 0; return '\\'; }
            const uint8_t* xs = s + p; p += 4;
            if (x < 0xD800 || x > 0xDFFF) return rune(x);
            uint32_t x1;
            if (n - p < 6 || s[p] != '\\' || s[p + 1] != 'u' || !jsn_hex4(s + p + 2, x1)) { q[0] = 'u'; q[1] = xs[0]; q[2] = xs[1]; q[3] = xs[2]; q[4] = xs[3]; qn = 5; qp = 0; return '\\'; }
            p += 6;
            return rune((x < 0xDC00 && x1 >= 0xDC00 && x1 < 0xE000) ? ((((x - 0xD800) << 10) | (x1 - 0xDC00)) + 0x10000) : 0xFFFDu);
        }
        default: q[0] = ch; qn = 1; qp = 0; return '\\';
        }
    }
};
// The Go string a non-null value becomes before ParseVal's string branch: the unescaped string, or Value.String() of
// anything else = the raw token with the whitespace outside strings removed (nested strings / keys stay raw)
struct Src {
    Dec d; const uint8_t* s; uint32_t p, n; bool str, ins, esc;
    __device__ Src(const uint8_t* v, uint32_t len, uint32_t t) : d(v + 1, t == JT_STRING ? len - 2 : 0), s(v), p(0), n(len), str(t == JT_STRING), ins(false), esc(false) {}
    __device__ int next() {
        if (str) return d.next();
        while (p < n) {
            const uint8_t c = s[p++];
            if (ins) { if (esc) esc = false; else if (c == '\\') esc = true; else if (c == '"') ins = false; return c; }
            if (jsn_ws(c)) continue;
            if (c == '"') ins = true;
            return c;
        }
        return -1;
    }
};

// ------------------------------------------------------------------ strconv on the device (mirrors oracle/json_oracle.hpp)
#define D_GO_NAN __longlong_as_double(0x7FF8000000000001ll)      /* math.NaN() */
static __device__ bool d_underscore_ok(const uint8_t* s, uint32_t n) {
    char i = '^'; uint32_t p = 0;
    if (n && (s[0] == '-' || s[0] == '+')) p = 1;
    bool hex = false;
    if (n - p >= 2 && s[p] == '0' && ((s[p + 1] | 0x20) == 'b' || (s[p + 1] | 0x20) == 'o' || (s[p + 1] | 0x20) == 'x')) { i = '0'; hex = (s[p + 1] | 0x20) == 'x'; p += 2; }
    for (; p < n; p++) {
        const uint8_t c = s[p];
        if ((c >= '0' && c <= '9') || (hex && (c | 0x20) >= 'a' && (c | 0x20) <= 'f')) { i = '0'; continue; }
        if (c == '_') { if (i != '0') return false; i = '_'; continue; }
        if (i == '_') return false;
        i = '!';
    }
    return i != '_';
}
// strconv.ParseUint(s, base, bits); base 0 = by prefix with underscores. rc 0 ok, 1 syntax, 2 range
static __device__ int d_go_parse_uint(const uint8_t* s0, uint32_t n0, int base, int bits, uint64_t& out) {
    if (!n0) return 1;
    const uint8_t* s = s0; uint32_t n = n0; const bool base0 = base == 0;
    if (base == 0) {
        base = 10;
        if (s[0] == '0') {
            if (n >= 3 && (s[1] | 0x20) == 'b') { base = 2; s += 2; n -= 2; }
            else if (n >= 3 && (s[1] | 0x20) == 'o') { base = 8; s += 2; n -= 2; }
            else if (n >= 3 && (s[1] | 0x20) == 'x') { base = 16; s += 2; n -= 2; }
            else { base = 8; s += 1; n -= 1; }
        }
    }
    const uint64_t maxv = bits == 64 ? ~0ull : ((1ull << bits) - 1);
    bool underscores = false, range = false; uint64_t v = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t c = s[i]; uint32_t d;
        if (c == '_' && base0) { underscores = true; continue; }
        if (c >= '0' && c <= '9') d = c - '0'; else if ((c | 0x20) >= 'a' && (c | 0x20) <= 'z') d = (c | 0x20) - 'a' + 10; else return 1;
        if (d >= (uint32_t)base) return 1;
        if (!range) { if (v > (maxv - d) / (uint32_t)base) range = true; else v = v * (uint32_t)base + d; }
    }
    if (underscores && !d_underscore_ok(s0, n0)) return 1;
    if (range) { out = maxv; return 2; }
    out = v; return 0;
}
static __device__ int d_go_parse_int(const uint8_t* s, uint32_t n, int base, int bits, int64_t& out) {
    if (!n) return 1;
    const uint8_t* s0 = s; const uint32_t n0 = n; bool neg = false;
    if (s[0] == '+') { s++; n--; } else if (s[0] == '-') { neg = true; s++; n--; }
    uint64_t un; const int rc = d_go_parse_uint(s, n, base, 64, un);
    if (rc == 1) return 1;
    if (base == 0) { bool us = false; for (uint32_t i = 0; i < n; i++) if (s[i] == '_') us = true; if (us && !d_underscore_ok(s0, n0)) return 1; }
    const uint64_t cutoff = 1ull << (bits - 1);
    if (rc == 2) return 2;
    if (!neg && un >= cutoff) return 2;
    if (neg && un > cutoff) return 2;
    out = neg ? (int64_t)(0 - un) : (int64_t)un; return 0;
}

// Eisel-Lemire (the algorithm strconv.ParseFloat uses after its exact path; scripts/el_proto.py checks this port against
// CPython's correctly rounded float()). false = not decided here.
static __device__ bool d_eisel_lemire(uint64_t man, int exp10, bool neg, uint64_t& bits) {
    if (man == 0) { bits = neg ? 0x8000000000000000ull : 0; return true; }
    if (exp10 < EL_QMIN || exp10 > EL_QMAX) return false;
    const int clz = __clzll((long long)man);
    man <<= clz;
    uint64_t ret_exp2 = (uint64_t)(((217706 * exp10) >> 16) + 64 + 1023) - (uint64_t)clz;
    const uint64_t tlo = d_el_pow10[exp10 - EL_QMIN][0], thi = d_el_pow10[exp10 - EL_QMIN][1];
    uint64_t xhi = __umul64hi(man, thi), xlo = man * thi;
    if ((xhi & 0x1FF) == 0x1FF && xlo + man < man) {
        const uint64_t yhi = __umul64hi(man, tlo), ylo = man * tlo;
        uint64_t mhi = xhi; const uint64_t mlo = xlo + yhi;
        if (mlo < xlo) mhi++;
        if ((mhi & 0x1FF) == 0x1FF && mlo + 1 == 0 && ylo + man < man) return false;
        xhi = mhi; xlo = mlo;
    }
    const uint64_t msb = xhi >> 63;
    uint64_t mant = xhi >> (msb + 9);
    ret_exp2 -= 1 ^ msb;
    if (xlo == 0 && (xhi & 0x1FF) == 0 && (mant & 3) == 1) return false;
    mant += mant & 1; mant >>= 1;
    if (mant >> 53) { mant >>= 1; ret_exp2 += 1; }
    if (ret_exp2 - 1 >= 0x7FF - 1) return false;
    bits = (ret_exp2 << 52) | (mant & 0x000FFFFFFFFFFFFFull);
    if (neg) bits |= 0x8000000000000000ull;
    return true;
}
// strconv.ParseFloat(s, 64). rc 0 ok, 1 syntax, 2 range (out = +-Inf), 3 needs the host (hex, underscores, undecided rounding)
static __device__ int d_go_parse_float(const uint8_t* s, uint32_t n, double& out) {
    if (!n) return 1;
    {   // special()
        const uint8_t* t = s; uint32_t m = n; bool neg = false, sign = false;
        if (t[0] == '+' || t[0] == '-') { neg = t[0] == '-'; t++; m--; sign = true; }
        if ((m == 3 && jsn_fold3(t, "inf")) || (m == 8 && jsn_fold3(t, "inf") && jsn_fold3(t + 3, "ini") && (t[6] | 0x20) == 't' && (t[7] | 0x20) == 'y')) { out = neg ? -CUDART_INF : CUDART_INF; return 0; }
        if (!sign && m == 3 && jsn_fold3(t, "nan")) { out = D_GO_NAN; return 0; }
    }
    uint32_t i = 0; bool neg = false;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    if (i + 2 < n && s[i] == '0' && (s[i + 1] | 0x20) == 'x') {       // hex float: mantissa digits, then a mandatory p exponent
        uint32_t k = i + 2; bool dig = false, dot = false;
        for (; k < n; k++) { const uint8_t c = s[k]; if (c == '_') return 3; if (c == '.') { if (dot) break; dot = true; continue; } if ((c >= '0' && c <= '9') || ((c | 0x20) >= 'a' && (c | 0x20) <= 'f')) { dig = true; continue; } break; }
        if (!dig || k >= n || (s[k] | 0x20) != 'p') return 1;
        return 3;
    }
    uint64_t man = 0; int nd = 0, ndm = 0, dp = 0; bool sawdot = false, sawdigits = false, trunc = false;
    for (; i < n; i++) {
        const uint8_t c = s[i];
        if (c == '_') return 3;                             // 1_000.5 is legal Go float syntax (underscoreOK); rare, left to the host
        if (c == '.') { if (sawdot) break; sawdot = true; dp = nd; continue; }
        if (c >= '0' && c <= '9') {
            sawdigits = true;
            if (c == '0' && nd == 0) { dp--; continue; }
            nd++;
            if (ndm < 19) { man = man * 10 + (c - '0'); ndm++; } else if (c != '0') trunc = true;
            continue;
        }
        break;
    }
    if (!sawdigits) return 1;
    if (!sawdot) dp = nd;
    if (i < n && (s[i] | 0x20) == 'e') {
        i++; if (i >= n) return 1;
        int es = 1; if (s[i] == '+') i++; else if (s[i] == '-') { es = -1; i++; }
        if (i >= n || s[i] < '0' || s[i] > '9') return 1;
        int e = 0;
        for (; i < n && ((s[i] >= '0' && s[i] <= '9') || s[i] == '_'); i++) { if (s[i] == '_') return 3; if (e < 10000) e = e * 10 + (s[i] - '0'); }
        dp += e * es;
    }
    if (i != n) return 1;
    if (man == 0) { out = neg ? -0.0 : 0.0; return 0; }
    const int exp = dp - ndm;
    if (!trunc && (man >> 53) == 0) {                       // atof64exact
        double f = __ull2double_rn(man);
        if (exp == 0) { out = neg ? -f : f; return 0; }
        if (exp > 0 && exp <= 15 + 22) {
            int e2 = exp; bool ok = true;
            if (e2 > 22) { f = __dmul_rn(f, d_p10[e2 - 22]); e2 = 22; if (f > 1e15 || f < -1e15) ok = false; }
            if (ok) { f = __dmul_rn(f, d_p10[e2]); out = neg ? -f : f; return 0; }
        } else if (exp < 0 && exp >= -22) { f = __ddiv_rn(f, d_p10[-exp]); out = neg ? -f : f; return 0; }
    }
    if (!trunc && exp >= 0 && exp <= 19) {                     // an integer below 2^64: the u64 -> f64 conversion rounds to nearest even exactly
        uint64_t m = man; bool fits = true;                     // (Eisel-Lemire gives up on exact half-way integers such as 2^53 + 1)
        for (int k = 0; k < exp; k++) { if (__umul64hi(m, 10ull)) { fits = false; break; } m *= 10ull; }
        if (fits) { const double f = __ull2double_rn(m); out = neg ? -f : f; return 0; }
    }
    uint64_t b0, b1;
    if (d_eisel_lemire(man, exp, neg, b0)) {
        if (!trunc) { out = __longlong_as_double((long long)b0); return 0; }
        if (d_eisel_lemire(man + 1, exp, neg, b1) && b0 == b1) { out = __longlong_as_double((long long)b0); return 0; }
    }
    if (dp > 310) { out = neg ? -CUDART_INF : CUDART_INF; return 2; }      // decimal.floatBits overflow
    if (dp < -330) { out = neg ? -0.0 : 0.0; return 0; }                   // underflow to zero
    return 3;
}

// ------------------------------------------------------------------ fastjson/fastfloat number getters
static __device__ uint64_t d_ff_uint64(const uint8_t* s, uint32_t n) {
    if (!n) return 0;
    uint32_t i = 0; uint64_t d = 0;
    while (i < n && s[i] >= '0' && s[i] <= '9') { d = d * 10 + (uint64_t)(s[i] - '0'); i++; if (i > 18) { uint64_t dd; return d_go_parse_uint(s, n, 10, 64, dd) == 0 ? dd : 0; } }
    if (i == 0 || i < n) return 0;
    return d;
}
static __device__ int64_t d_ff_int64(const uint8_t* s, uint32_t n) {
    if (!n) return 0;
    uint32_t i = 0; const bool minus = s[0] == '-';
    if (minus) { i++; if (i >= n) return 0; }
    uint64_t d = 0; const uint32_t j = i;
    while (i < n && s[i] >= '0' && s[i] <= '9') { d = d * 10 + (uint64_t)(s[i] - '0'); i++; if (i > 18) { int64_t dd; return d_go_parse_int(s, n, 10, 64, dd) == 0 ? dd : 0; } }
    if (i <= j || i < n) return 0;
    return minus ? -(int64_t)d : (int64_t)d;
}
__device__ const double d_pow10tab[32] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31};
__device__ const double d_pow10pos32[10] = {1e0, 1e32, 1e64, 1e96, 1e128, 1e160, 1e192, 1e224, 1e256, 1e288};
__device__ const double d_pow10neg32[11] = {1e-0, 1e-32, 1e-64, 1e-96, 1e-128, 1e-160, 1e-192, 1e-224, 1e-256, 1e-288, 1e-320};
__device__ __forceinline__ double d_go_pow10(int n) {     // math.Pow10
    if (0 <= n && n <= 308) return __dmul_rn(d_pow10pos32[n / 32], d_pow10tab[n % 32]);
    if (-323 <= n && n <= 0) return __ddiv_rn(d_pow10neg32[(-n) / 32], d_pow10tab[(-n) % 32]);
    return n > 0 ? CUDART_INF : 0.0;
}
// fastfloat.ParseBestEffort. rc 0 ok, JSN_HOST when the strconv fall-back cannot be decided on the device
static __device__ int d_ff_best(const uint8_t* s, uint32_t n, double& out) {
    out = 0;
    auto slow = [&]() -> int { double f; const int rc = d_go_parse_float(s, n, f); if (rc == 3) return JSN_HOST; out = rc == 1 ? 0.0 : f; return 0; };
    if (!n) return 0;
    uint32_t i = 0; const bool minus = s[0] == '-';
    if (minus) { i++; if (i >= n) return 0; }
    if (s[i] == '.' && (i + 1 >= n || s[i + 1] < '0' || s[i + 1] > '9')) return 0;
    uint64_t d = 0; const uint32_t j = i;
    while (i < n && s[i] >= '0' && s[i] <= '9') { d = d * 10 + (uint64_t)(s[i] - '0'); i++; if (i > 18) return slow(); }
    if (i <= j && s[i] != '.') {
        const uint8_t* t = s + i; uint32_t m = n - i; if (m && t[0] == '+') { t++; m--; }
        if ((m == 3 && jsn_fold3(t, "inf")) || (m == 8 && jsn_fold3(t, "inf") && jsn_fold3(t + 3, "ini") && (t[6] | 0x20) == 't' && (t[7] | 0x20) == 'y')) { out = minus ? -CUDART_INF : CUDART_INF; return 0; }
        if (m == 3 && jsn_fold3(t, "nan")) { out = D_GO_NAN; return 0; }
        return 0;
    }
    double f = __ull2double_rn(d);
    if (i >= n) { out = minus ? -f : f; return 0; }
    if (s[i] == '.') {
        i++;
        if (i >= n) { out = f; return 0; }
        const uint32_t k = i;
        while (i < n && s[i] >= '0' && s[i] <= '9') { d = d * 10 + (uint64_t)(s[i] - '0'); i++; if (i - j >= 17) return slow(); }
        f = __ddiv_rn(__ull2double_rn(d), d_go_pow10((int)(i - k)));
        if (i >= n) { out = minus ? -f : f; return 0; }
    }
    if (s[i] == 'e' || s[i] == 'E') {
        i++; if (i >= n) return 0;
        bool em = false;
        if (s[i] == '+' || s[i] == '-') { em = s[i] == '-'; i++; if (i >= n) return 0; }
        int exp = 0; const uint32_t j2 = i;
        while (i < n && s[i] >= '0' && s[i] <= '9') { exp = exp * 10 + (s[i] - '0'); i++; if (exp > 300) return slow(); }
        if (i <= j2) return 0;
        if (em) exp = -exp;
        f = __dmul_rn(f, d_go_pow10(exp));
        if (i >= n) { out = minus ? -f : f; return 0; }
    }
    return 0;
}
__device__ __forceinline__ int64_t d_f64_to_i64(double f) { if (!(f >= -9223372036854775808.0 && f < 9223372036854775808.0)) return (int64_t)0x8000000000000000ull; return __double2ll_rz(f); }   // amd64 CVTTSD2SQ
static __device__ bool d_valid_json_number(const uint8_t* s, uint32_t n) {      // encoding/json isValidNumber
    uint32_t i = 0; if (!n) return false;
    if (s[i] == '-') { i++; if (i == n) return false; }
    if (s[i] == '0') i++; else if (s[i] >= '1' && s[i] <= '9') { while (i < n && s[i] >= '0' && s[i] <= '9') i++; } else return false;
    if (i + 1 < n && s[i] == '.' && s[i + 1] >= '0' && s[i + 1] <= '9') { i += 2; while (i < n && s[i] >= '0' && s[i] <= '9') i++; }
    if (i + 1 < n && (s[i] == 'e' || s[i] == 'E')) { i++; if (s[i] == '+' || s[i] == '-') { i++; if (i == n) return false; } while (i < n && s[i] >= '0' && s[i] <= '9') i++; }
    return i == n;
}

// ------------------------------------------------------------------ fastjson grammar scan
// skips one already validated value starting at p, returns the position after it
static __device__ uint32_t jsn_skip_value(const uint8_t* s, uint32_t p, uint32_t n, uint32_t& t) {
    const uint8_t c = s[p];
    if (c == '"') { p++; while (p < n) { if (s[p] == '\\') { p += 2; continue; } if (s[p] == '"') break; p++; } t = JT_STRING; return p + 1; }
    if (c == '{' || c == '[') {
        t = c == '{' ? JT_OBJECT : JT_ARRAY; int depth = 0;
        while (p < n) {
            const uint8_t x = s[p];
            if (x == '"') { p++; while (p < n) { if (s[p] == '\\') { p += 2; continue; } if (s[p] == '"') break; p++; } p++; continue; }
            if (x == '{' || x == '[') depth++; else if (x == '}' || x == ']') { depth--; if (!depth) return p + 1; }
            p++;
        }
        return p;
    }
    if (c == 't') { t = JT_TRUE; return p + 4; }
    if (c == 'f') { t = JT_FALSE; return p + 5; }
    if (c == 'n') { if (p + 1 < n && s[p + 1] == 'u') { t = JT_NULL; return p + 4; } t = JT_NUMBER; return p + 3; }
    uint32_t i = p; while (i < n && jsn_numch(s[i])) i++;
    if (i < n && (i == p || (i == p + 1 && (s[p] == '-' || s[p] == '+'))) && n - i >= 3 && (jsn_fold3(s + i, "inf") || jsn_fold3(s + i, "nan"))) i += 3;
    t = JT_NUMBER; return i;
}
// Parser.Parse over one line; on_member(key_off, key_len, val_off, val_end, type) for every member of a root object, in order.
// returns 0 ok / 1 error; root_obj says whether the root value was an object
template <typename F> __device__ int jsn_scan(const uint8_t* s, uint32_t n, bool& root_obj, F&& on_member) {
    uint32_t p = 0; while (p < n && jsn_ws(s[p])) p++;
    uint32_t stk[10]; for (int i = 0; i < 10; i++) stk[i] = 0;
    int depth = 0; root_obj = false;
    uint32_t koff = 0, klen = 0, voff = 0, vtype = 0;
    int st = 0;      // 0 value, 1 key, 2 after value
    for (;;) {
        if (st == 0) {
            if (p >= n) return 1;
            if (depth + 1 > JSN_MAX_DEPTH) return 1;
            const uint8_t c = s[p]; uint32_t t;
            const bool member = depth == 1 && root_obj;
            if (member) voff = p;
            if (c == '{' || c == '[') {
                const bool obj = c == '{';
                if (member) vtype = obj ? JT_OBJECT : JT_ARRAY;
                p++; while (p < n && jsn_ws(s[p])) p++;
                if (p >= n) return 1;
                if (depth == 0) root_obj = obj;
                if (s[p] == (obj ? '}' : ']')) { p++; st = 2; continue; }
                if (obj) stk[depth >> 5] |= 1u << (depth & 31); else stk[depth >> 5] &= ~(1u << (depth & 31));
                depth++; st = obj ? 1 : 0; continue;
            }
            if (c == '"') { p++; while (p < n) { if (s[p] == '\\') { p += 2; continue; } if (s[p] == '"') break; p++; } if (p >= n) return 1; p++; t = JT_STRING; }
            else if (c == 't') { if (n - p < 4 || s[p + 1] != 'r' || s[p + 2] != 'u' || s[p + 3] != 'e') return 1; p += 4; t = JT_TRUE; }
            else if (c == 'f') { if (n - p < 5 || s[p + 1] != 'a' || s[p + 2] != 'l' || s[p + 3] != 's' || s[p + 4] != 'e') return 1; p += 5; t = JT_FALSE; }
            else if (c == 'n') {
                if (n - p >= 4 && s[p + 1] == 'u' && s[p + 2] == 'l' && s[p + 3] == 'l') { p += 4; t = JT_NULL; }
                else if (n - p >= 3 && jsn_fold3(s + p, "nan")) { p += 3; t = JT_NUMBER; }
                else return 1;
            } else {
                uint32_t i = p; while (i < n && jsn_numch(s[i])) i++;
                if (i < n && (i == p || (i == p + 1 && (s[p] == '-' || s[p] == '+')))) { if (n - i >= 3 && (jsn_fold3(s + i, "inf") || jsn_fold3(s + i, "nan"))) i += 3; else return 1; }
                p = i; t = JT_NUMBER;
            }
            if (member) vtype = t;
            st = 2; continue;
        }
        if (st == 1) {
            while (p < n && jsn_ws(s[p])) p++;
            if (p >= n || s[p] != '"') return 1;
            p++; const uint32_t k0 = p;
            while (p < n) { if (s[p] == '\\') { p += 2; continue; } if (s[p] == '"') break; p++; }
            if (p >= n) return 1;
            if (depth == 1 && root_obj) { koff = k0; klen = p - k0; }
            p++; while (p < n && jsn_ws(s[p])) p++;
            if (p >= n || s[p] != ':') return 1;
            p++; while (p < n && jsn_ws(s[p])) p++;
            st = 0; continue;
        }
        if (depth == 1 && root_obj) on_member(koff, klen, voff, p, vtype);
        if (depth == 0) break;
        while (p < n && jsn_ws(s[p])) p++;
        if (p >= n) return 1;
        const bool top_obj = (stk[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1;
        if (s[p] == ',') { p++; if (top_obj) st = 1; else { while (p < n && jsn_ws(s[p])) p++; st = 0; } continue; }
        if (s[p] == (top_obj ? '}' : ']')) { p++; depth--; if (depth == 0) break; st = 2; if (depth == 1 && root_obj) { /* nested container closed: member complete */ } continue; }
        return 1;
    }
    while (p < n && jsn_ws(s[p])) p++;
    return p == n ? 0 : 1;
}

// ------------------------------------------------------------------ keys
static __device__ bool jsn_key_is(const uint8_t* k, uint32_t klen, const uint8_t* name, uint32_t nlen) {
    bool esc = false; for (uint32_t i = 0; i < klen; i++) if (k[i] == '\\') { esc = true; break; }
    if (!esc) { if (klen != nlen) return false; for (uint32_t i = 0; i < klen; i++) if (k[i] != name[i]) return false; return true; }
    Dec d(k, klen); uint32_t i = 0;
    for (;;) { const int c = d.next(); if (c < 0) return i == nlen; if (i >= nlen || name[i] != (uint8_t)c) return false; i++; }
}
static __device__ int jsn_key_cmp(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {      // strings.Compare of the unescaped keys
    Dec da(a, an), db(b, bn);
    for (;;) { const int x = da.next(), y = db.next(); if (x < 0 && y < 0) return 0; if (x != y) return x < y ? -1 : 1; }
}
// Column name lengths and first bytes in shared memory (filled by jsn_stage_names at kernel start): the per-key column loop reads these
// instead of the descriptors in global memory.
__device__ __forceinline__ uint16_t* jsn_name_keys() { __shared__ uint16_t keys[JSN_MAX_COLS]; return keys; }   // name_len (capped at 255) | first byte << 8
__device__ __forceinline__ void jsn_stage_names(const JsnArgs& a) {
    uint16_t* nk = jsn_name_keys();
    for (int c = threadIdx.x; c < a.ncols && c < JSN_MAX_COLS; c += blockDim.x) {
        const uint32_t nl = a.cols[c].name_len;
        nk[c] = (uint16_t)((nl < 255 ? nl : 255) | ((nl ? a.names[a.cols[c].name_off] : 0) << 8));
    }
    __syncthreads();
}
// The column a root member's key names: the LAST column of that name wins (the map Unmarshal fills is read by column name). The key is
// scanned for escapes once; the common case then costs one length test per column and a byte compare only where the length fits.
static __device__ int jsn_find_col(const JsnArgs& a, const uint8_t* k, uint32_t klen) {
    bool esc = false; for (uint32_t i = 0; i < klen; i++) if (k[i] == '\\') { esc = true; break; }
    int hit = -1;
    if (esc) { for (int c = 0; c < a.ncols; c++) if (jsn_key_is(k, klen, a.names + a.cols[c].name_off, a.cols[c].name_len)) hit = c; return hit; }
    const uint16_t* nk = jsn_name_keys();
    const uint16_t want = (uint16_t)((klen < 255 ? klen : 255) | ((klen ? k[0] : 0) << 8));
    for (int c = 0; c < a.ncols; c++) {
        if (nk[c] != want) continue;                              // length and first byte in one shared-memory compare
        if (a.cols[c].name_len != klen) continue;                 // (names of 255 bytes and more share a length class)
        const uint8_t* nm = a.names + a.cols[c].name_off;
        bool eq = true; for (uint32_t i = 1; i < klen; i++) if (k[i] != nm[i]) { eq = false; break; }
        if (eq) hit = c;
    }
    return hit;
}

// ------------------------------------------------------------------ emitters (CountSink / MemSink)
// encoding/json appendString (escapeHTML on) over a byte source
template <typename Sink, typename S> __device__ void jsn_quote(Sink& sk, S& src) {
    const char* hex = "0123456789abcdef";
    sk.put('"');
    uint8_t w[4]; int wn = 0; bool eof = false;
    for (;;) {
        while (wn < 4 && !eof) { const int c = src.next(); if (c < 0) eof = true; else w[wn++] = (uint8_t)c; }
        if (!wn) break;
        const uint8_t b = w[0]; int use = 1;
        if (b < 0x80) {
            if (b >= 0x20 && b != '"' && b != '\\' && b != '<' && b != '>' && b != '&') sk.put(b);
            else {
                sk.put('\\');
                switch (b) {
                case '\\': case '"': sk.put(b); break;
                case '\b': sk.put('b'); break; case '\f': sk.put('f'); break; case '\n': sk.put('n'); break; case '\r': sk.put('r'); break; case '\t': sk.put('t'); break;
                default: sk.put('u'); sk.put('0'); sk.put('0'); sk.put((uint8_t)hex[b >> 4]); sk.put((uint8_t)hex[b & 15]);
                }
            }
        } else {
            uint32_t r = 0xFFFD; int width = 1;
            if (b >= 0xC2 && b <= 0xDF && wn >= 2 && (w[1] & 0xC0) == 0x80) { r = ((b & 0x1Fu) << 6) | (w[1] & 0x3Fu); width = 2; }
            else if (b >= 0xE0 && b <= 0xEF && wn >= 3 && (w[1] & 0xC0) == 0x80 && (w[2] & 0xC0) == 0x80) {
                const uint32_t t = ((b & 0x0Fu) << 12) | ((w[1] & 0x3Fu) << 6) | (w[2] & 0x3Fu);
                if (t >= 0x800 && !(t >= 0xD800 && t <= 0xDFFF)) { r = t; width = 3; }
            } else if (b >= 0xF0 && b <= 0xF4 && wn >= 4 && (w[1] & 0xC0) == 0x80 && (w[2] & 0xC0) == 0x80 && (w[3] & 0xC0) == 0x80) {
                const uint32_t t = ((b & 0x07u) << 18) | ((w[1] & 0x3Fu) << 12) | ((w[2] & 0x3Fu) << 6) | (w[3] & 0x3Fu);
                if (t >= 0x10000 && t <= 0x10FFFF) { r = t; width = 4; }
            }
            if (r == 0xFFFD && width == 1) fmt_lit(sk, "\\ufffd");
            else if (r == 0x2028 || r == 0x2029) { fmt_lit(sk, "\\u202"); sk.put((uint8_t)hex[r & 0xF]); use = width; }
            else { for (int k = 0; k < width; k++) sk.put(w[k]); use = width; }
        }
        for (int k = use; k < wn; k++) w[k - use] = w[k];
        wn -= use;
    }
    sk.put('"');
}

template <typename Sink> __device__ int jsn_emit_scalar(Sink& sk, const uint8_t* s, uint32_t off, uint32_t end, uint32_t t, bool use_numbers) {
    switch (t) {
    case JT_STRING: { Dec d(s + off + 1, end - off - 2); jsn_quote(sk, d); return 0; }
    case JT_TRUE: fmt_lit(sk, "true"); return 0;
    case JT_FALSE: fmt_lit(sk, "false"); return 0;
    case JT_NULL: fmt_lit(sk, "null"); return 0;
    default:
        if (use_numbers) { if (!d_valid_json_number(s + off, end - off)) return JSN_HOST; for (uint32_t k = off; k < end; k++) sk.put(s[k]); return 0; }
        double f; if (d_ff_best(s + off, end - off, f)) return JSN_HOST;
        if (isnan(f) || isinf(f)) return JSN_HOST;
        fmt_float_bits(sk, (uint64_t)__double_as_longlong(f), false, FM_JSON); return 0;
    }
}

struct JFrame { uint32_t beg, end, cur, last_off, last_len, flags; };     // flags: 1 object, 2 something emitted, 4 has last key, 8 filter known columns

// json.Marshal of wrapIntoEmptyInterface(value) (:603-633): objects become maps (sorted keys, last duplicate wins), numbers
// float64 or json.Number. `filter` (root object of `_rest`) drops the members whose key is a declared field.
template <typename Sink> __device__ int jsn_emit_canon(Sink& sk, const JsnArgs& a, const uint8_t* s, uint32_t off, uint32_t end, uint32_t t, bool filter) {
    const bool un = a.use_numbers;
    if (t != JT_OBJECT && t != JT_ARRAY) return jsn_emit_scalar(sk, s, off, end, t, un);
    JFrame fr[JSN_DEV_DEPTH]; int sp = 0;
    auto open = [&](uint32_t o, uint32_t e, uint32_t ty, bool flt) { JFrame& f = fr[sp++]; f.beg = o + 1; f.end = e - 1; f.cur = o + 1; f.last_off = 0; f.last_len = 0; f.flags = (ty == JT_OBJECT ? 1u : 0u) | (flt ? 8u : 0u); sk.put(ty == JT_OBJECT ? '{' : '['); };
    open(off, end, t, filter);
    while (sp > 0) {
        JFrame& f = fr[sp - 1];
        uint32_t v0 = 0, v1 = 0, vt = 0; bool have = false;
        if (f.flags & 1) {                                   // next key in sorted order
            uint32_t p = f.beg, bk = 0, bl = 0;
            for (;;) {
                while (p < f.end && jsn_ws(s[p])) p++;
                if (p >= f.end) break;
                const uint32_t k0 = p + 1; uint32_t q = k0;
                while (q < f.end) { if (s[q] == '\\') { q += 2; continue; } if (s[q] == '"') break; q++; }
                const uint32_t kl = q - k0; p = q + 1;
                while (p < f.end && jsn_ws(s[p])) p++;
                p++;                                          // ':'
                while (p < f.end && jsn_ws(s[p])) p++;
                const uint32_t a0 = p; uint32_t ty; p = jsn_skip_value(s, p, f.end, ty); const uint32_t a1 = p;
                while (p < f.end && jsn_ws(s[p])) p++;
                if (p < f.end && s[p] == ',') p++;
                if ((f.flags & 8)) { const int c = jsn_find_col(a, s + k0, kl); if (c >= 0 && c < a.nfields) continue; }
                if ((f.flags & 4) && jsn_key_cmp(s + k0, kl, s + f.last_off, f.last_len) <= 0) continue;
                if (!have || jsn_key_cmp(s + k0, kl, s + bk, bl) <= 0) { have = true; bk = k0; bl = kl; v0 = a0; v1 = a1; vt = ty; }
            }
            if (!have) { sk.put('}'); sp--; continue; }
            if (f.flags & 2) sk.put(',');
            f.flags |= 2 | 4; f.last_off = bk; f.last_len = bl;
            { Dec d(s + bk, bl); jsn_quote(sk, d); }
            sk.put(':');
        } else {
            uint32_t p = f.cur;
            while (p < f.end && jsn_ws(s[p])) p++;
            if (p >= f.end) { sk.put(']'); sp--; continue; }
            v0 = p; p = jsn_skip_value(s, p, f.end, vt); v1 = p;
            while (p < f.end && jsn_ws(s[p])) p++;
            if (p < f.end && s[p] == ',') p++;
            f.cur = p;
            if (f.flags & 2) sk.put(',');
            f.flags |= 2;
        }
        if (vt == JT_OBJECT || vt == JT_ARRAY) { if (sp >= JSN_DEV_DEPTH) return JSN_HOST; open(v0, v1, vt, false); }
        else { const int rc = jsn_emit_scalar(sk, s, v0, v1, vt, un); if (rc) return rc; }
    }
    return 0;
}

// encoding/base64 StdEncoding.DecodeString over a byte source; rc 0 ok, 1 CorruptInputError
template <typename Sink, typename S> __device__ int jsn_base64(Sink& sk, S& src) {
    auto dv = [](int c) -> int { if (c >= 'A' && c <= 'Z') return c - 'A'; if (c >= 'a' && c <= 'z') return c - 'a' + 26; if (c >= '0' && c <= '9') return c - '0' + 52; if (c == '+') return 62; if (c == '/') return 63; return -1; };
    bool end = false; int pend = -2;                         // one byte of look-ahead
    auto get = [&]() -> int { if (pend != -2) { const int c = pend; pend = -2; return c; } return src.next(); };
    while (!end) {
        int db[4] = {0, 0, 0, 0}; int j = 0, dlen = 4;
        while (j < 4) {
            const int c = get();
            if (c < 0) { if (j == 0) return 0; return 1; }
            const int v = dv(c);
            if (v >= 0) { db[j++] = v; continue; }
            if (c == '\n' || c == '\r') continue;
            if (c != '=') return 1;
            if (j < 2) return 1;
            if (j == 2) { int x; do { x = get(); } while (x == '\n' || x == '\r'); if (x != '=') return 1; }
            int x; do { x = get(); } while (x == '\n' || x == '\r');
            if (x >= 0) return 1;
            dlen = j; end = true; break;
        }
        const uint32_t val = (uint32_t)db[0] << 18 | (uint32_t)db[1] << 12 | (uint32_t)db[2] << 6 | (uint32_t)db[3];
        sk.put((uint8_t)(val >> 16)); if (dlen >= 3) sk.put((uint8_t)(val >> 8)); if (dlen == 4) sk.put((uint8_t)val);
    }
    return 0;
}

// the text cell of one var-width field from its recorded span; rc 0 / JSN_PARSEVAL / JSN_HOST. tag: `any` holds a Go string
template <typename Sink> __device__ int jsn_emit_text(Sink& sk, const JsnArgs& a, const JsnColDev& cd, const uint8_t* s, uint32_t off, uint32_t len, uint32_t t, uint8_t& tag) {
    tag = 0;
    if (cd.tf == TF_ANY) {
        if (t == JT_STRING) {                                // ParseVal :1084-1092: `\\` -> `\`, then a JSON re-parse the device leaves to the host
            Dec d(s + off + 1, len - 2); tag = 1; bool first = true; int hold = -1;
            for (;;) {
                int c = hold >= 0 ? hold : d.next(); hold = -1;
                if (c < 0) break;
                if (c == '\\') { const int c2 = d.next(); if (c2 != '\\') hold = c2 < 0 ? -1 : c2; if (c2 < 0) { sk.put('\\'); break; } }
                if (first) { if (jsn_ws((uint8_t)c)) { sk.put((uint8_t)c); continue; } if (c == '{' || c == 'n') return JSN_HOST; first = false; }
                sk.put((uint8_t)c);
            }
            return 0;
        }
        return jsn_emit_canon(sk, a, s, off, off + len, t, false);
    }
    Src src(s + off, len, t);
    if (cd.tf == TF_BYTES && a.unpack_b64) return jsn_base64(sk, src) ? JSN_PARSEVAL : 0;
    for (;;) { const int c = src.next(); if (c < 0) break; sk.put((uint8_t)c); }
    return 0;
}

__device__ __forceinline__ void jsn_store(const JsnColDev& c, uint64_t row, uint64_t v, uint32_t nsec) {
    switch (c.w) {
    case 1: c.values[row] = (uint8_t)v; break;
    case 2: ((uint16_t*)c.values)[row] = (uint16_t)v; break;
    case 4: ((uint32_t*)c.values)[row] = (uint32_t)v; break;
    default: ((uint64_t*)c.values)[row] = v; break;
    }
    if (c.aux32) c.aux32[row] = nsec;
}
__device__ __forceinline__ int jsn_bits(int tf) { switch (tf) { case TF_INT8: case TF_UINT8: return 8; case TF_INT16: case TF_UINT16: return 16; case TF_INT32: case TF_UINT32: return 32; default: return 64; } }
__device__ __forceinline__ bool jsn_is_int(int tf) { return tf == TF_INT8 || tf == TF_INT16 || tf == TF_INT32 || tf == TF_INT64; }
__device__ __forceinline__ bool jsn_is_uint(int tf) { return tf == TF_UINT8 || tf == TF_UINT16 || tf == TF_UINT32 || tf == TF_UINT64; }

// Unmarshal's typed extraction + ParseVal for a fixed-width field. rc 0 (null set when the cell is nil) / JSN_PARSEVAL / JSN_HOST
static __device__ int jsn_fixed_cell(const JsnArgs& a, const JsnColDev& cd, const uint8_t* s, uint32_t off, uint32_t len, uint32_t t, uint64_t& v, bool& null) {
    v = 0; null = false;
    const int tf = cd.tf;
    if (t == JT_ABSENT || t == JT_NULL) { null = true; return 0; }
    if (t == JT_STRING) {
        if (tf == TF_DATETIME) return JSN_HOST;                                   // araddon/dateparse
        uint8_t buf[JSN_NUMBUF]; uint32_t n = 0; Dec d(s + off + 1, len - 2);
        for (;;) { const int c = d.next(); if (c < 0) break; if (n >= JSN_NUMBUF) return JSN_HOST; buf[n++] = (uint8_t)c; }
        if (tf == TF_DOUBLE) { double f; const int rc = d_go_parse_float(buf, n, f); if (rc == 3) return JSN_HOST; if (rc) return JSN_PARSEVAL; v = (uint64_t)__double_as_longlong(f); return 0; }
        if (tf == TF_BOOLEAN) { bool b; if (d_parse_bool(buf, n, b)) return JSN_PARSEVAL; v = b; return 0; }
        if (jsn_is_int(tf)) { int64_t x; if (d_go_parse_int(buf, n, 0, jsn_bits(tf), x)) return JSN_PARSEVAL; v = (uint64_t)x; return 0; }
        uint64_t x; if (d_go_parse_uint(buf, n, 0, jsn_bits(tf), x)) return JSN_PARSEVAL; v = x; return 0;
    }
    const bool num = t == JT_NUMBER;
    if (tf == TF_DATETIME) {
        if (!num) return JSN_PARSEVAL;                                           // bool / map / slice: "unable extract timestamp"
        if (a.use_numbers) { int64_t x; if (d_go_parse_int(s + off, len, 10, 64, x)) return JSN_PARSEVAL; v = (uint64_t)x; return 0; }
        double f; if (d_ff_best(s + off, len, f)) return JSN_HOST;
        v = (uint64_t)d_f64_to_i64(fabs(f)); return 0;
    }
    if (tf == TF_DOUBLE) { double f = 0; if (num && d_ff_best(s + off, len, f)) return JSN_HOST; v = (uint64_t)__double_as_longlong(f); return 0; }
    if (tf == TF_BOOLEAN) { v = t == JT_TRUE; return 0; }
    if (jsn_is_int(tf)) { const int64_t x = num ? d_ff_int64(s + off, len) : 0; switch (jsn_bits(tf)) { case 8: v = (uint64_t)(int64_t)(int8_t)x; break; case 16: v = (uint64_t)(int64_t)(int16_t)x; break; case 32: v = (uint64_t)(int64_t)(int32_t)x; break; default: v = (uint64_t)x; } return 0; }
    v = num ? d_ff_uint64(s + off, len) : 0; return 0;                             // jsn_store truncates to the column width
}

// The lines of one CTA are a contiguous span of the input. One thread per line walks its own line byte by byte, so straight from
// global memory every load instruction of a warp touches 32 different cache lines; the CTA therefore first copies its span into
// shared memory with coalesced 16-byte loads (when it fits) and the per-line code reads that copy through the same offsets.
#define JSN_STAGE 40960
__device__ __forceinline__ const uint8_t* jsn_stage_span(const JsnArgs& a, uint8_t* stage) {
    const uint64_t L0 = (uint64_t)blockIdx.x * blockDim.x;
    if (L0 >= a.nlines) return a.text;
    const uint64_t Le = (L0 + blockDim.x < a.nlines) ? L0 + blockDim.x : a.nlines;
    const uint32_t lo = L0 ? a.line_end[L0 - 1] : 0, hi = a.line_end[Le - 1];
    const uint32_t lo16 = lo & ~15u;
    if (hi - lo16 > JSN_STAGE || ((uintptr_t)a.text & 15)) return a.text;           // uniform over the CTA
    const uint32_t full = (uint32_t)(((a.len < hi ? a.len : hi) - lo16) & ~15ull);    // whole 16-byte chunks inside the buffer
    for (uint32_t i = threadIdx.x * 16; i < full; i += blockDim.x * 16) *(int4*)(stage + i) = __ldg((const int4*)(a.text + lo16 + i));
    for (uint32_t i = full + threadIdx.x; lo16 + i < hi; i += blockDim.x) stage[i] = a.text[lo16 + i];
    __syncthreads();
    return stage - lo16;
}

// ------------------------------------------------------------------ pass 1
__global__ void k_json_pass1(JsnArgs a);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(128) k_json_pass1(JsnArgs a) {
    extern __shared__ __align__(16) uint8_t jsn_stage[];
    jsn_stage_names(a);
    const uint8_t* const text = jsn_stage_span(a, jsn_stage);
    const uint64_t L = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = L < a.nlines;
    uint32_t vb[JSN_MAX_COLS / 32]; for (int i = 0; i < JSN_MAX_COLS / 32; i++) vb[i] = 0;
    int err = 0, ecol = 0;
    if (active) {
        uint32_t ls, n; jsn_line(text, a.line_end, L, ls, n);
        const uint8_t* s = text + ls;
        const int nf = a.nfields;
        if (!n) err = JSN_EMPTY;
        uint32_t nmembers = 0; bool host = false;
        if (!err) {
            bool root_obj = false;
            const int rc = jsn_scan(s, n, root_obj, [&](uint32_t koff, uint32_t klen, uint32_t voff, uint32_t vend, uint32_t vt) {
                nmembers++;
                const int c = jsn_find_col(a, s + koff, klen);
                if (c >= 0 && c < nf) {
                    if (vend - voff >= (1u << 28)) host = true;
                    a.span_start[(size_t)c * a.nlines + L] = ls + voff; a.span_len[(size_t)c * a.nlines + L] = (vend - voff) | (vt << 28);
                } else if (c >= nf) host = true;              // a key named like an aux column takes that column's type in Unmarshal (:690): left to the host
            });
            if (rc) err = JSN_PARSE; else if (!root_obj || !nmembers) err = JSN_SKIP; else if (host) { err = JSN_HOST; ecol = nf; }
        }
        for (int f = 0; f < nf && !err; f++) {
            const JsnColDev& cd = a.cols[f];
            const uint32_t off = a.span_start[(size_t)f * a.nlines + L], sl = a.span_len[(size_t)f * a.nlines + L];
            const uint32_t t = sl >> 28, len = sl & 0x0FFFFFFFu;
            bool null = false; int rc = 0;
            if (cd.w) {
                uint64_t v; rc = jsn_fixed_cell(a, cd, text, off, len, t, v, null);
                if (!rc) jsn_store(cd, L, null ? 0 : v, 0);
            } else {
                if (t == JT_ABSENT || t == JT_NULL) null = true;
                else { CountSink cs{0}; uint8_t tag; rc = jsn_emit_text(cs, a, cd, text, off, len, t, tag); if (!rc) { a.out_len[(size_t)cd.slot * a.nlines + L] = cs.n; if (cd.aux8) cd.aux8[L] = tag; } }
                if (null) { a.out_len[(size_t)cd.slot * a.nlines + L] = 0; if (cd.aux8) cd.aux8[L] = 0; }
            }
            if (rc == JSN_HOST) { err = JSN_HOST; ecol = f; break; }
            if (rc) {                                        // ParseVal error :361-366
                if ((!a.null_keys_allowed && cd.key) || cd.required) { err = JSN_PARSEVAL; ecol = f; break; }
                null = true;
                if (cd.w) jsn_store(cd, L, 0, 0); else { a.out_len[(size_t)cd.slot * a.nlines + L] = 0; if (cd.aux8) cd.aux8[L] = 0; }
                a.span_len[(size_t)f * a.nlines + L] = 0;    // pass 2 writes nothing
            }
            if (null && (cd.key || cd.required) && !a.null_keys_allowed) { err = JSN_NIL_REQUIRED; ecol = f; break; }
            if (!null) vb[f >> 5] |= 1u << (f & 31);
        }
        int c = nf;
        if (!err && a.add_rest) {
            const JsnColDev& cd = a.cols[c];
            uint32_t b = 0; while (b < n && jsn_ws(s[b])) b++;
            uint32_t e = n; while (e > b && jsn_ws(s[e - 1])) e--;
            CountSink cs{0}; const int rc = jsn_emit_canon(cs, a, s, b, e, JT_OBJECT, true);
            if (rc) { err = JSN_HOST; ecol = c; } else { a.out_len[(size_t)cd.slot * a.nlines + L] = cs.n; cd.aux8[L] = 0; vb[c >> 5] |= 1u << (c & 31); }
        }
        if (a.add_rest) c++;
        if (!err && a.add_dedupe) {
            uint32_t lo = 0, hi = a.nmsgs;                   // message of this line: first m with msg_end[m] > line start
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a.msg_end[mid] <= (uint64_t)ls) lo = mid + 1; else hi = mid; }
            const uint32_t m = lo < a.nmsgs ? lo : a.nmsgs - 1;
            jsn_store(a.cols[c], L, (uint64_t)a.msg_wsec[m], a.msg_wnsec[m]);
            a.out_len[(size_t)a.cols[c + 1].slot * a.nlines + L] = a.part_len;
            jsn_store(a.cols[c + 2], L, a.msg_offset[m], 0);
            jsn_store(a.cols[c + 3], L, (uint64_t)(a.rank[L] - a.msg_rank0[m] + 1), 0);
            for (int k = 0; k < 4; k++) vb[(c + k) >> 5] |= 1u << ((c + k) & 31);
        }
        if (err) {      // the row is dropped downstream; give its cells harmless contents
            for (int k = 0; k < a.ncols; k++) { const JsnColDev& cd = a.cols[k]; if (cd.w) jsn_store(cd, L, 0, 0); else { a.out_len[(size_t)cd.slot * a.nlines + L] = 0; if (cd.aux8) cd.aux8[L] = 0; } }
            for (int i = 0; i < JSN_MAX_COLS / 32; i++) vb[i] = 0;
        }
        a.err[L] = (uint8_t)err; a.errcol[L] = (uint8_t)ecol;
    }
    for (int c = 0; c < a.ncols; c++) {
        const uint32_t word = __ballot_sync(0xffffffffu, active && ((vb[c >> 5] >> (c & 31)) & 1));
        if ((threadIdx.x & 31) == 0 && active) a.cols[c].validity[L >> 5] = word;
    }
}
#endif  // TF_KERNELS_JSON_IN

// ------------------------------------------------------------------ pass 2: text cells
struct JsnWriteArgs { JsnArgs a; const uint32_t* offsets; uint8_t* heap; const uint64_t* col_base; };

__global__ void k_json_pass2(JsnWriteArgs w);
#ifdef TF_KERNELS_JSON_IN
__global__ void __launch_bounds__(128) k_json_pass2(JsnWriteArgs w) {
    extern __shared__ __align__(16) uint8_t jsn_stage[];
    const JsnArgs& a = w.a;
    jsn_stage_names(a);
    const uint8_t* const text = jsn_stage_span(a, jsn_stage);
    const uint64_t L = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (L >= a.nlines || a.err[L]) return;
    const int nf = a.nfields;
    for (int f = 0; f < nf; f++) {
        const JsnColDev& cd = a.cols[f];
        if (cd.w) continue;
        const uint32_t sl = a.span_len[(size_t)f * a.nlines + L]; const uint32_t t = sl >> 28, len = sl & 0x0FFFFFFFu;
        if (t == JT_ABSENT || t == JT_NULL) continue;
        MemSink ms{w.heap + w.col_base[cd.slot] + w.offsets[(size_t)cd.slot * (a.nlines + 1) + L]}; uint8_t tag;      // (short cells: a word-gathering sink measured slower here)
        jsn_emit_text(ms, a, cd, text, a.span_start[(size_t)f * a.nlines + L], len, t, tag);
    }
    int c = nf;
    if (a.add_rest) {
        const JsnColDev& cd = a.cols[c];
        uint32_t ls, n; jsn_line(text, a.line_end, L, ls, n); const uint8_t* s = text + ls;
        uint32_t b = 0; while (b < n && jsn_ws(s[b])) b++;
        uint32_t e = n; while (e > b && jsn_ws(s[e - 1])) e--;
        MemSink ms{w.heap + w.col_base[cd.slot] + w.offsets[(size_t)cd.slot * (a.nlines + 1) + L]};
        jsn_emit_canon(ms, a, s, b, e, JT_OBJECT, true);
        c++;
    }
    if (a.add_dedupe) {
        const JsnColDev& cd = a.cols[c + 1];
        uint8_t* o = w.heap + w.col_base[cd.slot] + w.offsets[(size_t)cd.slot * (a.nlines + 1) + L];
        for (uint32_t k = 0; k < a.part_len; k++) o[k] = a.names[a.part_off + k];
    }
}
#endif  // TF_KERNELS_JSON_IN

}  // namespace tfk
