// Debezium parser on the device: queue messages (schema + payload envelope, or schema-registry frames) -> typed columns.
//   reference: pkg/parsers/registry/debezium/engine/parser.go:34-98 (DoOne / DoBuf), pkg/debezium/unpacker/include_schema.go:13-25,
//              pkg/debezium/common/debezium_schema.go:31-66 (Payload / Source decoding with encoding/json, UseNumber),
//              pkg/debezium/receiver.go:142-220 (receive), receiver_engine.go:143-330 (extractVal / convertVal),
//              pkg/debezium/common/field_receiver_default.go:15-330 (default receivers), typeutil/helpers.go:972-998.
// The CPU restatement these kernels must agree with is oracle/debezium_oracle.hpp.
//   k_dbz_pass1   one thread per message: strict encoding/json validation of the envelope, payload / source / after members
//                 located (duplicates as encoding/json resolves them), op -> kind, per field typed extraction by the
//                 default receiver of its Kafka Connect type; fixed cells stored, text cells sized, validity by ballot
//   k_csv_offsets per text column exclusive scan of the lengths (kernels_csv.cuh)
//   k_dbz_pass2   text cells written: unquoted strings, base64 payloads, Decimal text, Point text
#pragma once
#include "kernels_json_in.cuh"

namespace tfk {

enum DbzErr : int { DBZ_UNPARSED = 48, DBZ_HOST = 49, DBZ_OTHER_SCHEMA = 50, DBZ_OTHER_TABLE = 51 };
enum DbzRecv : int { DR_INT8 = 1, DR_INT16, DR_INT32, DR_INT64, DR_BOOL, DR_STRING, DR_F64, DR_BYTES, DR_DECIMAL, DR_POINT, DR_VSD };
#define DBZ_MAX_DEPTH 256      /* encoding/json allows 10000 nested containers; deeper than this -> DBZ_HOST */
#define DBZ_MAX_NUM_BYTES 32   /* Decimal / VariableScaleDecimal magnitudes up to 256 bits are converted on the device */

struct DbzColDev {
    int32_t recv, scale, tf, w, slot; uint8_t key, pad[3];
    uint32_t name_off, name_len;
    uint8_t* values; uint32_t* validity;
};
struct DbzArgs {
    const uint8_t* text; const uint64_t* msg_end; uint64_t nmsgs;
    const DbzColDev* cols; int ncols; const uint8_t* names;
    const uint8_t* schema_text; uint32_t schema_len; uint32_t schema_id; uint8_t use_sr, check_table, pad[2];
    uint32_t tbl_schema_off, tbl_schema_len, tbl_name_off, tbl_name_len;
    uint32_t* span_start; uint32_t* span_len;      // [ncols][nmsgs]
    uint32_t* out_len;                             // [nslots][nmsgs]
    uint8_t* kinds; uint32_t* tx_id; uint64_t* lsn; uint64_t* commit_time;
    uint8_t* err; uint8_t* errcol;
};

// ------------------------------------------------------------------ encoding/json grammar (checkValid)
// validates ONE value starting at s[p] (after optional whitespace); returns 0 ok / 1 syntax error / 2 too deep; p ends after the
// value. odd_key is set when an object key holds a backslash or a non-ASCII byte (case folding / unescaping left to the host).
static __device__ int dbz_validate(const uint8_t* s, uint32_t n, uint32_t& p, bool& odd_key) {
    while (p < n && jsn_ws(s[p])) p++;
    uint32_t stk[DBZ_MAX_DEPTH / 32]; int depth = 0; int st = 0;      // st 0 value, 1 key, 2 after value
    for (;;) {
        if (st == 0) {
            if (p >= n) return 1;
            const uint8_t c = s[p];
            if (c == '{' || c == '[') {
                const bool obj = c == '{';
                p++; while (p < n && jsn_ws(s[p])) p++;
                if (p >= n) return 1;
                if (s[p] == (obj ? '}' : ']')) { p++; st = 2; continue; }
                if (depth >= DBZ_MAX_DEPTH) return 2;
                if (obj) stk[depth >> 5] |= 1u << (depth & 31); else stk[depth >> 5] &= ~(1u << (depth & 31));
                depth++; st = obj ? 1 : 0; continue;
            }
            if (c == '"') {
                p++;
                for (;;) {
                    if (p >= n) return 1;
                    const uint8_t x = s[p];
                    if (x == '"') break;
                    if (x < 0x20) return 1;
                    if (x == '\\') {
                        if (p + 1 >= n) return 1;
                        const uint8_t e = s[p + 1];
                        if (e == 'u') { uint32_t h; if (n - p < 6 || !jsn_hex4(s + p + 2, h)) return 1; p += 6; continue; }
                        if (e != '"' && e != '\\' && e != '/' && e != 'b' && e != 'f' && e != 'n' && e != 'r' && e != 't') return 1;
                        p += 2; continue;
                    }
                    p++;
                }
                p++;
            } else if (c == 't') { if (n - p < 4 || s[p + 1] != 'r' || s[p + 2] != 'u' || s[p + 3] != 'e') return 1; p += 4; }
            else if (c == 'f') { if (n - p < 5 || s[p + 1] != 'a' || s[p + 2] != 'l' || s[p + 3] != 's' || s[p + 4] != 'e') return 1; p += 5; }
            else if (c == 'n') { if (n - p < 4 || s[p + 1] != 'u' || s[p + 2] != 'l' || s[p + 3] != 'l') return 1; p += 4; }
            else { uint32_t q = p; while (q < n && jsn_numch(s[q])) q++; if (!d_valid_json_number(s + p, q - p)) return 1; p = q; }
            st = 2; continue;
        }
        if (st == 1) {
            while (p < n && jsn_ws(s[p])) p++;
            if (p >= n || s[p] != '"') return 1;
            p++;
            for (;;) {
                if (p >= n) return 1;
                const uint8_t x = s[p];
                if (x == '"') break;
                if (x < 0x20) return 1;
                if (x >= 0x80) odd_key = true;
                if (x == '\\') {
                    odd_key = true;
                    if (p + 1 >= n) return 1;
                    const uint8_t e = s[p + 1];
                    if (e == 'u') { uint32_t h; if (n - p < 6 || !jsn_hex4(s + p + 2, h)) return 1; p += 6; continue; }
                    if (e != '"' && e != '\\' && e != '/' && e != 'b' && e != 'f' && e != 'n' && e != 'r' && e != 't') return 1;
                    p += 2; continue;
                }
                p++;
            }
            p++; while (p < n && jsn_ws(s[p])) p++;
            if (p >= n || s[p] != ':') return 1;
            p++; while (p < n && jsn_ws(s[p])) p++;
            st = 0; continue;
        }
        if (depth == 0) return 0;
        while (p < n && jsn_ws(s[p])) p++;
        if (p >= n) return 1;
        const bool top_obj = (stk[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1;
        if (s[p] == ',') { p++; if (top_obj) st = 1; else { while (p < n && jsn_ws(s[p])) p++; st = 0; } continue; }
        if (s[p] == (top_obj ? '}' : ']')) { p++; depth--; st = 2; continue; }
        return 1;
    }
}

// members of an already validated object [off, end) (the braces included): f(key_off, key_len, val_off, val_end, type)
template <typename F> __device__ void dbz_members(const uint8_t* s, uint32_t off, uint32_t end, F&& f) {
    uint32_t p = off + 1; const uint32_t e = end - 1;
    for (;;) {
        while (p < e && jsn_ws(s[p])) p++;
        if (p >= e) return;
        const uint32_t k0 = p + 1; uint32_t q = k0;
        while (q < e) { if (s[q] == '\\') { q += 2; continue; } if (s[q] == '"') break; q++; }
        p = q + 1;
        while (p < e && jsn_ws(s[p])) p++;
        p++;
        while (p < e && jsn_ws(s[p])) p++;
        const uint32_t v0 = p; uint32_t t; p = jsn_skip_value(s, p, e, t);
        f(k0, q - k0, v0, p, t);
        while (p < e && jsn_ws(s[p])) p++;
        if (p < e && s[p] == ',') p++;
    }
}
__device__ __forceinline__ bool dbz_key_eq(const uint8_t* k, uint32_t kl, const char* name) { uint32_t i = 0; for (; name[i]; i++) if (i >= kl || k[i] != (uint8_t)name[i]) return false; return i == kl; }
__device__ __forceinline__ bool dbz_key_fold(const uint8_t* k, uint32_t kl, const char* name) {
    uint32_t i = 0;
    for (; name[i]; i++) { if (i >= kl) return false; uint8_t a = k[i], b = (uint8_t)name[i]; if (a >= 'A' && a <= 'Z') a += 32; if (b >= 'A' && b <= 'Z') b += 32; if (a != b) return false; }
    return i == kl;
}
__device__ __forceinline__ bool dbz_key_is_bytes(const uint8_t* k, uint32_t kl, const uint8_t* name, uint32_t nl) { if (kl != nl) return false; for (uint32_t i = 0; i < kl; i++) if (k[i] != name[i]) return false; return true; }

// encoding/json unquote of a validated string body as a byte stream: escapes resolved, a lone / unpaired \u surrogate and every
// byte of an invalid UTF-8 sequence become U+FFFD
struct GoDec {
    const uint8_t* s; uint32_t n, p; uint8_t q[4]; uint8_t qn, qp;
    __device__ GoDec(const uint8_t* s_, uint32_t n_) : s(s_), n(n_), p(0), qn(0), qp(0) {}
    __device__ int rune(uint32_t r) {
        if (r < 0x80) return (int)r;
        qp = 0;
        if (r < 0x800) { q[0] = (uint8_t)(0x80 | (r & 0x3F)); qn = 1; return (int)(0xC0 | (r >> 6)); }
        if (r < 0x10000) { q[0] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); q[1] = (uint8_t)(0x80 | (r & 0x3F)); qn = 2; return (int)(0xE0 | (r >> 12)); }
        q[0] = (uint8_t)(0x80 | ((r >> 12) & 0x3F)); q[1] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); q[2] = (uint8_t)(0x80 | (r & 0x3F)); qn = 3; return (int)(0xF0 | (r >> 18));
    }
    __device__ int next() {
        if (qp < qn) return q[qp++];
        if (p >= n) return -1;
        const uint8_t c = s[p];
        if (c < 0x80 && c != '\\') { p++; return c; }
        if (c == '\\') {
            const uint8_t e = s[p + 1];
            if (e != 'u') { p += 2; switch (e) { case 'b': return 8; case 'f': return 12; case 'n': return 10; case 'r': return 13; case 't': return 9; default: return e; } }
            uint32_t x; jsn_hex4(s + p + 2, x); p += 6;
            if (x >= 0xD800 && x < 0xDC00) { uint32_t y; if (n - p >= 6 && s[p] == '\\' && s[p + 1] == 'u' && jsn_hex4(s + p + 2, y) && y >= 0xDC00 && y < 0xE000) { p += 6; return rune((((x - 0xD800) << 10) | (y - 0xDC00)) + 0x10000); } return rune(0xFFFD); }
            if (x >= 0xDC00 && x < 0xE000) return rune(0xFFFD);
            return rune(x);
        }
        const uint32_t rem = n - p; uint32_t w = 0;
        if (c >= 0xC2 && c <= 0xDF && rem >= 2 && (s[p + 1] & 0xC0) == 0x80) w = 2;
        else if (c >= 0xE0 && c <= 0xEF && rem >= 3 && (s[p + 1] & 0xC0) == 0x80 && (s[p + 2] & 0xC0) == 0x80) { const uint32_t t = ((c & 0x0Fu) << 12) | ((s[p + 1] & 0x3Fu) << 6) | (s[p + 2] & 0x3Fu); if (t >= 0x800 && !(t >= 0xD800 && t <= 0xDFFF)) w = 3; }
        else if (c >= 0xF0 && c <= 0xF4 && rem >= 4 && (s[p + 1] & 0xC0) == 0x80 && (s[p + 2] & 0xC0) == 0x80 && (s[p + 3] & 0xC0) == 0x80) { const uint32_t t = ((c & 0x07u) << 18) | ((s[p + 1] & 0x3Fu) << 12) | ((s[p + 2] & 0x3Fu) << 6) | (s[p + 3] & 0x3Fu); if (t >= 0x10000 && t <= 0x10FFFF) w = 4; }
        if (!w) { p++; return rune(0xFFFD); }
        for (uint32_t k = 1; k < w; k++) q[k - 1] = s[p + k];
        qn = (uint8_t)(w - 1); qp = 0; p += w; return c;
    }
};
// the Go string of a value that may be a JSON string or a json.Number (extractVal :240-251)
struct DbzStr {
    GoDec d; const uint8_t* s; uint32_t p, n; bool str;
    __device__ DbzStr(const uint8_t* v, uint32_t len, uint32_t t) : d(v + 1, t == JT_STRING ? len - 2 : 0), s(v), p(0), n(len), str(t == JT_STRING) {}
    __device__ int next() { if (str) return d.next(); return p < n ? s[p++] : -1; }
};
struct BufSink { uint8_t* b; uint32_t n, cap; bool over; __device__ __forceinline__ void put(uint8_t x) { if (n < cap) b[n++] = x; else over = true; } };

// typeutil.Base64ToNumeric: base64 text source -> decimal text. rc 0 ok, 1 error, 2 the reference panics (empty buffer /
// negative scale) or the magnitude is wider than the device converts -> host
template <typename Sink, typename S> __device__ int dbz_b64_numeric(Sink& sk, S& src, int scale) {
    uint8_t buf[DBZ_MAX_NUM_BYTES]; BufSink bs{buf, 0, DBZ_MAX_NUM_BYTES, false};
    if (jsn_base64(bs, src)) return 1;
    if (bs.over || bs.n == 0 || scale < 0 || scale > 200) return 2;
    const bool neg = buf[0] & 0x80; const uint32_t nb = bs.n;
    if (neg) { for (uint32_t i = 0; i < nb; i++) buf[i] = (uint8_t)~buf[i]; for (uint32_t i = nb; i-- > 0;) { if (++buf[i] != 0) break; } }
    uint8_t dig[80]; int nd = 0;
    for (;;) {
        uint32_t first = 0; while (first < nb && buf[first] == 0) first++;
        if (first == nb) break;
        uint32_t rem = 0;
        for (uint32_t i = first; i < nb; i++) { const uint32_t v = rem * 256 + buf[i]; buf[i] = (uint8_t)(v / 10); rem = v % 10; }
        dig[nd++] = (uint8_t)('0' + rem);
    }
    if (nd == 0) { sk.put('0'); return 0; }
    if (neg) sk.put('-');
    // digits are least significant first; the text is dig[nd-1..0] with the point `scale` places from the right
    int total = nd; int lead = 0;
    if (scale != 0 && scale > nd) { lead = scale - nd + 1; total = nd + lead; }
    for (int i = 0; i < total; i++) {
        if (scale != 0 && i == total - scale) sk.put('.');
        sk.put(i < lead ? (uint8_t)'0' : dig[nd - 1 - (i - lead)]);
    }
    return 0;
}

// Point.Do: "(%v,%v)" of vv["x"], vv["y"]. rc 0 / DBZ_UNPARSED / DBZ_HOST
template <typename Sink> __device__ int dbz_point(Sink& sk, const uint8_t* s, uint32_t off, uint32_t end) {
    uint32_t xo = 0, xe = 0, xt = JT_ABSENT, yo = 0, ye = 0, yt = JT_ABSENT;
    dbz_members(s, off, end, [&](uint32_t k0, uint32_t kl, uint32_t v0, uint32_t v1, uint32_t t) {
        if (dbz_key_eq(s + k0, kl, "x")) { xo = v0; xe = v1; xt = t; } else if (dbz_key_eq(s + k0, kl, "y")) { yo = v0; ye = v1; yt = t; } });
    if (xt == JT_ABSENT || yt == JT_ABSENT) return DBZ_UNPARSED;
    auto pv = [&](uint32_t o, uint32_t e, uint32_t t) -> bool {
        switch (t) {
        case JT_NUMBER: for (uint32_t k = o; k < e; k++) sk.put(s[k]); return true;
        case JT_STRING: { GoDec d(s + o + 1, e - o - 2); for (;;) { const int c = d.next(); if (c < 0) break; sk.put((uint8_t)c); } return true; }
        case JT_NULL: fmt_lit(sk, "<nil>"); return true;
        case JT_TRUE: fmt_lit(sk, "true"); return true; case JT_FALSE: fmt_lit(sk, "false"); return true;
        default: return false;
        }
    };
    sk.put('('); if (!pv(xo, xe, xt)) return DBZ_HOST; sk.put(','); if (!pv(yo, ye, yt)) return DBZ_HOST; sk.put(')');
    return 0;
}

__device__ __forceinline__ bool dbz_is_unavailable(const uint8_t* s, uint32_t off, uint32_t len) {
    const char* u = "\"__debezium_unavailable_value\""; if (len != 30) return false;
    for (uint32_t i = 0; i < 30; i++) if (s[off + i] != (uint8_t)u[i]) return false;
    return true;
}

// one text cell (DR_STRING / DR_BYTES / DR_DECIMAL / DR_POINT) from its value span
template <typename Sink> __device__ int dbz_emit_text(Sink& sk, const DbzColDev& cd, const uint8_t* s, uint32_t off, uint32_t len, uint32_t t) {
    if (cd.recv == DR_POINT) { if (t != JT_OBJECT) return DBZ_HOST; return dbz_point(sk, s, off, off + len); }
    if (t != JT_STRING && t != JT_NUMBER) return DBZ_UNPARSED;                 // "assert no one value extracted"
    DbzStr src(s + off, len, t);
    if (cd.recv == DR_STRING) { for (;;) { const int c = src.next(); if (c < 0) break; sk.put((uint8_t)c); } return 0; }
    if (cd.recv == DR_BYTES) return jsn_base64(sk, src) ? DBZ_UNPARSED : 0;
    const int rc = dbz_b64_numeric(sk, src, cd.scale); return rc == 2 ? DBZ_HOST : rc ? DBZ_UNPARSED : 0;
}

// a JSON number literal into an unsigned struct field (encoding/json: strconv.ParseUint, then the width check)
__device__ __forceinline__ bool dbz_lit_uint(const uint8_t* s, uint32_t off, uint32_t end, uint32_t t, int bits, uint64_t& out, bool& set) {
    set = false;
    if (t == JT_NULL) return true;
    if (t != JT_NUMBER) return false;
    uint64_t v; if (d_go_parse_uint(s + off, end - off, 10, 64, v)) return false;
    if (bits < 64 && (v >> bits)) return false;
    out = v; set = true; return true;
}

// The messages of one CTA are a contiguous span of the input; one thread per message walks its own message byte by byte, so the CTA
// first copies the span into shared memory with coalesced 16-byte loads (when it fits) and the per-message code reads that copy
// through the same offsets (cf. jsn_stage_span).
#define DBZ_STAGE 73728
__device__ __forceinline__ const uint8_t* dbz_stage_span(const DbzArgs& a, uint8_t* stage) {
    const uint64_t M0 = (uint64_t)blockIdx.x * blockDim.x;
    if (M0 >= a.nmsgs) return a.text;
    const uint64_t Me = (M0 + blockDim.x < a.nmsgs) ? M0 + blockDim.x : a.nmsgs;
    const uint64_t lo = M0 ? a.msg_end[M0 - 1] : 0, hi = a.msg_end[Me - 1];
    const uint64_t lo16 = lo & ~15ull;
    if (hi - lo16 > DBZ_STAGE || ((uintptr_t)a.text & 15)) return a.text;           // uniform over the CTA
    const uint32_t full = (uint32_t)((hi - lo16) & ~15ull);                         // whole 16-byte chunks inside the span
    for (uint32_t i = threadIdx.x * 16; i < full; i += blockDim.x * 16) *(int4*)(stage + i) = __ldg((const int4*)(a.text + lo16 + i));
    for (uint64_t i = full + threadIdx.x; lo16 + i < hi; i += blockDim.x) stage[i] = a.text[lo16 + i];
    __syncthreads();
    return stage - lo16;
}

__global__ void k_dbz_pass1(DbzArgs a);
#ifdef TF_KERNELS_DBZ
__global__ void __launch_bounds__(128) k_dbz_pass1(DbzArgs a) {
    extern __shared__ __align__(16) uint8_t dbz_stage[];
    const uint8_t* const text = dbz_stage_span(a, dbz_stage);      // the CTA's messages, copied to shared memory with coalesced loads when they fit
    const uint64_t M = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = M < a.nmsgs;
    uint32_t vb[JSN_MAX_COLS / 32]; for (int i = 0; i < JSN_MAX_COLS / 32; i++) vb[i] = 0;
    int err = 0, ecol = 0;
    if (active) {
        const uint64_t ms = M ? a.msg_end[M - 1] : 0; const uint32_t n = (uint32_t)(a.msg_end[M] - ms);
        const uint8_t* s = text + ms;
        uint32_t pay_off = 0, pay_end = 0, pay_t = JT_ABSENT;
        uint32_t sch_off = 0, sch_end = 0; bool have_schema = false;
        if (!n) err = DBZ_UNPARSED;                                              // "debezium parser received empty message"
        else if (a.use_sr) {
            if (s[0] != 0 || n < 5) err = DBZ_UNPARSED;
            else {
                bool more = false; for (uint32_t i = 5; i < n; i++) if (s[i] == 0) { more = true; break; }
                const uint32_t id = ((uint32_t)s[1] << 24) | ((uint32_t)s[2] << 16) | ((uint32_t)s[3] << 8) | s[4];
                if (more) err = DBZ_HOST;                                         // several events in one message: host
                else if (id != a.schema_id) err = DBZ_OTHER_SCHEMA;
                else {
                    uint32_t p = 5; bool odd = false; while (p < n && jsn_ws(s[p])) p++;
                    const uint32_t v0 = p; const int rc = dbz_validate(s, n, p, odd);
                    if (rc == 1) err = DBZ_UNPARSED; else if (rc == 2 || odd) err = DBZ_HOST;
                    else { uint32_t t; jsn_skip_value(s, v0, n, t); pay_off = v0; pay_end = p; pay_t = t; }
                }
            }
        } else {
            uint32_t p = 0; bool odd = false; while (p < n && jsn_ws(s[p])) p++;
            const uint32_t v0 = p; const int rc = dbz_validate(s, n, p, odd);
            uint32_t q = p; while (q < n && jsn_ws(s[q])) q++;
            if (rc == 1 || (rc == 0 && q != n)) err = DBZ_UNPARSED;              // json.Unmarshal: syntax error / data after the value
            else if (rc == 2) err = DBZ_HOST;
            else {
                uint32_t rt; jsn_skip_value(s, v0, n, rt);
                if (rt != JT_OBJECT) err = DBZ_UNPARSED;                           // null: both RawMessages stay empty -> EOF; others: type error
                else if (odd) err = DBZ_HOST;
                else {
                    bool folded = false;
                    dbz_members(s, v0, p, [&](uint32_t k0, uint32_t kl, uint32_t a0, uint32_t a1, uint32_t t) {
                        if (dbz_key_eq(s + k0, kl, "schema")) { sch_off = a0; sch_end = a1; have_schema = true; }
                        else if (dbz_key_eq(s + k0, kl, "payload")) { pay_off = a0; pay_end = a1; pay_t = t; }
                        else if (dbz_key_fold(s + k0, kl, "schema") || dbz_key_fold(s + k0, kl, "payload")) folded = true; });
                    if (folded) err = DBZ_HOST; else if (pay_t == JT_ABSENT) err = DBZ_UNPARSED;
                }
            }
        }
        // ---- payload struct
        bool bad = false; int kind = -1; uint32_t tx = 0; uint64_t lsn = 0, tsms = 0;
        uint32_t af_off = 0, af_end = 0, be_off = 0, be_end = 0; bool has_af = false, has_be = false;
        uint32_t tsch_o = 0, tsch_e = 0, ttab_o = 0, ttab_e = 0; bool has_tsch = false, has_ttab = false;
        if (!err) {
            uint32_t op_o = 0, op_e = 0; bool has_op = false; bool host = false;
            if (pay_t == JT_OBJECT) {
                dbz_members(s, pay_off, pay_end, [&](uint32_t k0, uint32_t kl, uint32_t v0, uint32_t v1, uint32_t t) {
                    const uint8_t* k = s + k0;
                    if (dbz_key_eq(k, kl, "op")) { if (t == JT_STRING) { op_o = v0; op_e = v1; has_op = true; } else if (t != JT_NULL) bad = true; }
                    else if (dbz_key_eq(k, kl, "after")) { if (t == JT_OBJECT) { if (has_af) host = true; af_off = v0; af_end = v1; has_af = true; } else if (t == JT_NULL) has_af = false; else bad = true; }
                    else if (dbz_key_eq(k, kl, "before")) { if (t == JT_OBJECT) { if (has_be) host = true; be_off = v0; be_end = v1; has_be = true; } else if (t == JT_NULL) has_be = false; else bad = true; }
                    else if (dbz_key_eq(k, kl, "ts_ms")) { uint64_t x; bool set; if (!dbz_lit_uint(s, v0, v1, t, 64, x, set)) bad = true; }
                    else if (dbz_key_eq(k, kl, "source")) {
                        if (t == JT_OBJECT) {
                            dbz_members(s, v0, v1, [&](uint32_t f0, uint32_t fl, uint32_t x0, uint32_t x1, uint32_t xt) {
                                const uint8_t* f = s + f0; uint64_t x; bool set;
                                if (dbz_key_eq(f, fl, "lsn")) { if (!dbz_lit_uint(s, x0, x1, xt, 64, x, set)) bad = true; else if (set) lsn = x; }
                                else if (dbz_key_eq(f, fl, "ts_ms")) { if (!dbz_lit_uint(s, x0, x1, xt, 64, x, set)) bad = true; else if (set) tsms = x; }
                                else if (dbz_key_eq(f, fl, "txId")) { if (!dbz_lit_uint(s, x0, x1, xt, 32, x, set)) bad = true; else if (set) tx = (uint32_t)x; }
                                else if (dbz_key_eq(f, fl, "xmin")) { if (xt == JT_NUMBER) { int64_t y; if (d_go_parse_int(s + x0, x1 - x0, 10, 64, y)) bad = true; } else if (xt != JT_NULL) bad = true; }
                                else if (dbz_key_eq(f, fl, "connector") || dbz_key_eq(f, fl, "db") || dbz_key_eq(f, fl, "name") || dbz_key_eq(f, fl, "schema") || dbz_key_eq(f, fl, "sequence") ||
                                         dbz_key_eq(f, fl, "snapshot") || dbz_key_eq(f, fl, "table") || dbz_key_eq(f, fl, "version")) {
                                    if (xt == JT_STRING) { if (dbz_key_eq(f, fl, "schema")) { tsch_o = x0; tsch_e = x1; has_tsch = true; } else if (dbz_key_eq(f, fl, "table")) { ttab_o = x0; ttab_e = x1; has_ttab = true; } }
                                    else if (xt != JT_NULL) bad = true;
                                } else if (dbz_key_fold(f, fl, "connector") || dbz_key_fold(f, fl, "db") || dbz_key_fold(f, fl, "lsn") || dbz_key_fold(f, fl, "name") || dbz_key_fold(f, fl, "schema") || dbz_key_fold(f, fl, "sequence") ||
                                           dbz_key_fold(f, fl, "snapshot") || dbz_key_fold(f, fl, "table") || dbz_key_fold(f, fl, "ts_ms") || dbz_key_fold(f, fl, "txId") || dbz_key_fold(f, fl, "version") || dbz_key_fold(f, fl, "xmin")) host = true; });
                        } else if (t != JT_NULL) bad = true;
                    } else if (dbz_key_eq(k, kl, "transaction")) { }
                    else if (dbz_key_fold(k, kl, "after") || dbz_key_fold(k, kl, "before") || dbz_key_fold(k, kl, "op") || dbz_key_fold(k, kl, "source") || dbz_key_fold(k, kl, "transaction") || dbz_key_fold(k, kl, "ts_ms")) host = true; });
            } else if (pay_t != JT_NULL) bad = true;
            // precedence as in the oracle: folded keys / duplicate maps first (found while walking), then type errors, then op
            if (host) err = DBZ_HOST;
            else if (bad) err = DBZ_UNPARSED;
            else {
                if (has_op) { GoDec d(s + op_o + 1, op_e - op_o - 2); const int c0 = d.next(), c1 = d.next(); if (c1 < 0) { if (c0 == 'c' || c0 == 'r') kind = TF_KIND_INSERT; else if (c0 == 'u') kind = TF_KIND_UPDATE; else if (c0 == 'd') kind = TF_KIND_DELETE; } }
                if (kind < 0) err = DBZ_UNPARSED;                                 // "unknown op"
            }
        }
        if (!err && !a.use_sr) {                                                  // the plan is keyed on the exact schema bytes (receiver.go:63-96 hashes them)
            bool same = have_schema && (sch_end - sch_off) == a.schema_len;
            if (same) for (uint32_t i = 0; i < a.schema_len; i++) if (s[sch_off + i] != a.schema_text[i]) { same = false; break; }
            if (!same) err = DBZ_OTHER_SCHEMA;
        }
        if (!err && a.check_table) {
            auto eq = [&](bool has, uint32_t o, uint32_t e, uint32_t no, uint32_t nl) -> bool {
                if (!has) return nl == 0;
                GoDec d(s + o + 1, e - o - 2); uint32_t i = 0;
                for (;;) { const int c = d.next(); if (c < 0) return i == nl; if (i >= nl || a.names[no + i] != (uint8_t)c) return false; i++; } };
            if (!eq(has_tsch, tsch_o, tsch_e, a.tbl_schema_off, a.tbl_schema_len) || !eq(has_ttab, ttab_o, ttab_e, a.tbl_name_off, a.tbl_name_len)) err = DBZ_OTHER_TABLE;
        }
        // ---- fields (receiver.go:204-217)
        if (!err) {
            const bool del = kind == TF_KIND_DELETE; const bool has = del ? has_be : has_af; const uint32_t vo = del ? be_off : af_off, ve = del ? be_end : af_end;
            if (has) dbz_members(s, vo, ve, [&](uint32_t k0, uint32_t kl, uint32_t v0, uint32_t v1, uint32_t t) {
                for (int c = 0; c < a.ncols; c++) if (dbz_key_is_bytes(s + k0, kl, a.names + a.cols[c].name_off, a.cols[c].name_len)) {
                    a.span_start[(size_t)c * a.nmsgs + M] = (uint32_t)ms + v0; a.span_len[(size_t)c * a.nmsgs + M] = (v1 - v0) | (t << 28); } });
            for (int c = 0; c < a.ncols && !err; c++) {
                const DbzColDev& cd = a.cols[c];
                const uint32_t off = a.span_start[(size_t)c * a.nmsgs + M], sl = a.span_len[(size_t)c * a.nmsgs + M];
                const uint32_t t = sl >> 28, len = sl & 0x0FFFFFFFu;
                if (t == JT_ABSENT) { err = DBZ_UNPARSED; ecol = c; break; }            // "unable to get field %s"
                if (len >= (1u << 28) - 1) { err = DBZ_HOST; ecol = c; break; }
                bool null = t == JT_NULL; int rc = 0;
                if (!null && t == JT_STRING && dbz_is_unavailable(text, off, len)) rc = DBZ_HOST;
                else if (!null) {
                    const uint8_t* v = text + off;
                    switch (cd.recv) {
                    case DR_INT8: case DR_INT16: case DR_INT32: case DR_INT64: {
                        int64_t x; if (t != JT_NUMBER || d_go_parse_int(v, len, 10, 64, x)) rc = DBZ_UNPARSED;
                        else { switch (cd.w) { case 1: cd.values[M] = (uint8_t)x; break; case 2: ((uint16_t*)cd.values)[M] = (uint16_t)x; break; case 4: ((uint32_t*)cd.values)[M] = (uint32_t)x; break; default: ((uint64_t*)cd.values)[M] = (uint64_t)x; } }
                        break;
                    }
                    case DR_BOOL: if (t != JT_TRUE && t != JT_FALSE) rc = DBZ_UNPARSED; else cd.values[M] = t == JT_TRUE; break;
                    case DR_F64: {
                        double f; if (t != JT_NUMBER) rc = DBZ_UNPARSED; else { const int pr = d_go_parse_float(v, len, f); if (pr == 3) rc = DBZ_HOST; else if (pr) rc = DBZ_UNPARSED; else ((uint64_t*)cd.values)[M] = (uint64_t)__double_as_longlong(f); }
                        break;
                    }
                    case DR_VSD: {
                        if (t != JT_OBJECT) { rc = DBZ_HOST; break; }
                        uint32_t vo2 = 0, ve2 = 0, vt2 = JT_ABSENT, so2 = 0, se2 = 0, st2 = JT_ABSENT;
                        dbz_members(text, off, off + len, [&](uint32_t k0, uint32_t kl, uint32_t x0, uint32_t x1, uint32_t xt) {
                            if (dbz_key_eq(text + k0, kl, "value")) { vo2 = x0; ve2 = x1; vt2 = xt; } else if (dbz_key_eq(text + k0, kl, "scale")) { so2 = x0; se2 = x1; st2 = xt; } });
                        if (vt2 == JT_ABSENT) { rc = DBZ_UNPARSED; break; }
                        if (vt2 != JT_STRING) { rc = DBZ_HOST; break; }
                        int64_t scale = 0;
                        if (st2 != JT_ABSENT) { if (st2 != JT_NUMBER) { rc = DBZ_HOST; break; } if (d_go_parse_int(text + so2, se2 - so2, 10, 64, scale)) { rc = DBZ_UNPARSED; break; } }
                        uint8_t nb[JSN_NUMBUF + 160]; BufSink bs{nb, 0, sizeof nb, false}; DbzStr src(text + vo2, ve2 - vo2, JT_STRING);
                        const int br = (scale < 0 || scale > 200) ? 2 : dbz_b64_numeric(bs, src, (int)scale);
                        if (br == 2 || bs.over) { rc = DBZ_HOST; break; } if (br) { rc = DBZ_UNPARSED; break; }
                        double f; const int pr = d_go_parse_float(nb, bs.n, f); if (pr) { rc = DBZ_HOST; break; }
                        ((uint64_t*)cd.values)[M] = (uint64_t)__double_as_longlong(f); break;
                    }
                    default: { CountSink cs{0}; rc = dbz_emit_text(cs, cd, text, off, len, t); if (!rc) a.out_len[(size_t)cd.slot * a.nmsgs + M] = cs.n; }
                    }
                }
                if (rc) { err = rc; ecol = c; break; }
                if (null) { if (cd.w) { switch (cd.w) { case 1: cd.values[M] = 0; break; case 2: ((uint16_t*)cd.values)[M] = 0; break; case 4: ((uint32_t*)cd.values)[M] = 0; break; default: ((uint64_t*)cd.values)[M] = 0; } } else a.out_len[(size_t)cd.slot * a.nmsgs + M] = 0; }
                else vb[c >> 5] |= 1u << (c & 31);
            }
        }
        if (err) {
            for (int c = 0; c < a.ncols; c++) { const DbzColDev& cd = a.cols[c]; if (cd.w) { switch (cd.w) { case 1: cd.values[M] = 0; break; case 2: ((uint16_t*)cd.values)[M] = 0; break; case 4: ((uint32_t*)cd.values)[M] = 0; break; default: ((uint64_t*)cd.values)[M] = 0; } } else a.out_len[(size_t)cd.slot * a.nmsgs + M] = 0; }
            for (int i = 0; i < JSN_MAX_COLS / 32; i++) vb[i] = 0;
            kind = TF_KIND_INSERT; tx = 0; lsn = 0; tsms = 0;
        }
        a.kinds[M] = (uint8_t)kind; a.tx_id[M] = tx; a.lsn[M] = lsn; a.commit_time[M] = tsms * 1000000ull;
        a.err[M] = (uint8_t)err; a.errcol[M] = (uint8_t)ecol;
    }
    for (int c = 0; c < a.ncols; c++) {
        const uint32_t word = __ballot_sync(0xffffffffu, active && ((vb[c >> 5] >> (c & 31)) & 1));
        if ((threadIdx.x & 31) == 0 && active) a.cols[c].validity[M >> 5] = word;
    }
}
#endif  // TF_KERNELS_DBZ

struct DbzWriteArgs { DbzArgs a; const uint32_t* offsets; uint8_t* heap; const uint64_t* col_base; };

__global__ void k_dbz_pass2(DbzWriteArgs w);
#ifdef TF_KERNELS_DBZ
__global__ void __launch_bounds__(128) k_dbz_pass2(DbzWriteArgs w) {
    const DbzArgs& a = w.a;
    const uint64_t M = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (M >= a.nmsgs || a.err[M]) return;
    for (int c = 0; c < a.ncols; c++) {
        const DbzColDev& cd = a.cols[c];
        if (cd.w) continue;
        const uint32_t sl = a.span_len[(size_t)c * a.nmsgs + M]; const uint32_t t = sl >> 28, len = sl & 0x0FFFFFFFu;
        if (t == JT_ABSENT || t == JT_NULL) continue;
        MemSink ms{w.heap + w.col_base[cd.slot] + w.offsets[(size_t)cd.slot * (a.nmsgs + 1) + M]};
        dbz_emit_text(ms, cd, a.text, a.span_start[(size_t)c * a.nmsgs + M], len, t);
    }
}
#endif  // TF_KERNELS_DBZ

}  // namespace tfk
