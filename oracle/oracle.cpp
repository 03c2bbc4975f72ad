// ORACLE — test infrastructure only. Never linked into or called from the product path.
// CPU restatement (row-at-a-time, boxed values) of transferia's per-batch hot path.
// Every function names the reference file:line it follows (paths relative to the
// reference repository root).  See oracle.h for the parity status.
#include "oracle.h"
#include "go_strconv.hpp"
#include "hashes.hpp"
#include "lz4_block.hpp"
#include "csv_oracle.hpp"
#include "json_oracle.hpp"
#include "debezium_oracle.hpp"
#include "cast_oracle.hpp"
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <limits>

using namespace orc;

namespace {

// ------------------------------------------------------------------ boxed values
struct Boxed {
    orc_val v;
    std::string own;     // storage when the value was produced by a transformer
    void set_string(std::string s, int kind) { own = std::move(s); v.kind = kind; v.s = (const uint8_t*)own.data(); v.slen = own.size(); }
};

inline bool col_valid(const tf_col& c, uint64_t r) { return !c.validity || ((c.validity[r >> 3] >> (r & 7)) & 1); }

// The Go dynamic type a column's value has under the typesystem contract
// pkg/abstract/typesystem/values/type_checkers.go:39-84.
void box(const tf_col& c, uint64_t r, orc_val& v) {
    std::memset(&v, 0, sizeof v);
    if (!col_valid(c, r)) { v.kind = OG_NIL; return; }
    switch (c.type) {
    case TF_INT8:  v.kind = OG_INT8;  v.i = ((const int8_t*)c.values)[r]; break;
    case TF_INT16: v.kind = OG_INT16; v.i = ((const int16_t*)c.values)[r]; break;
    case TF_INT32: v.kind = OG_INT32; v.i = ((const int32_t*)c.values)[r]; break;
    case TF_INT64: v.kind = OG_INT64; v.i = ((const int64_t*)c.values)[r]; break;
    case TF_UINT8:  v.kind = OG_UINT8;  v.u = ((const uint8_t*)c.values)[r]; break;
    case TF_UINT16: v.kind = OG_UINT16; v.u = ((const uint16_t*)c.values)[r]; break;
    case TF_UINT32: v.kind = OG_UINT32; v.u = ((const uint32_t*)c.values)[r]; break;
    case TF_UINT64: v.kind = OG_UINT64; v.u = ((const uint64_t*)c.values)[r]; break;
    case TF_FLOAT:  v.kind = OG_FLOAT32; v.f = ((const float*)c.values)[r]; v.u = ((const uint32_t*)c.values)[r]; break;   // u: the bits (float -> double quiets a signaling NaN)
    case TF_DOUBLE: v.kind = OG_FLOAT64; v.f = ((const double*)c.values)[r]; break;
    case TF_BOOLEAN: v.kind = OG_BOOL; v.i = ((const uint8_t*)c.values)[r] != 0; break;
    case TF_INTERVAL: v.kind = OG_DURATION; v.i = ((const int64_t*)c.values)[r]; break;
    case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:
        v.kind = OG_TIME; v.i = ((const int64_t*)c.values)[r]; v.nsec = c.aux ? ((const uint32_t*)c.aux)[r] : 0; break;
    case TF_BYTES: v.kind = OG_BYTES; v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; break;
    case TF_UTF8:  v.kind = OG_STRING; v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; break;
    case TF_ANY:
        v.kind = (c.aux && ((const uint8_t*)c.aux)[r] == 1) ? OG_STRING : OG_JSON;
        v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; break;
    default: v.kind = OG_NIL;
    }
}

// encoding/json string encoder with escapeHTML=true (json.Marshal default): Go 1.25 encode.go appendString
std::string go_json_quote(const uint8_t* s, size_t n) {
    static const char* hex = "0123456789abcdef";
    std::string d; d += '"';
    size_t i = 0;
    while (i < n) {
        uint8_t b = s[i];
        if (b < 0x80) {
            if (b >= 0x20 && b != '"' && b != '\\' && b != '<' && b != '>' && b != '&') { d += (char)b; i++; continue; }
            d += '\\';
            switch (b) {
            case '\\': case '"': d += (char)b; break;
            case '\b': d += 'b'; break; case '\f': d += 'f'; break; case '\n': d += 'n'; break; case '\r': d += 'r'; break; case '\t': d += 't'; break;
            default: d += "u00"; d += hex[b >> 4]; d += hex[b & 15];
            }
            i++; continue;
        }
        // decode one UTF-8 rune (Go utf8.DecodeRune semantics: invalid -> RuneError width 1)
        uint32_t r = 0xFFFD; size_t w = 1;
        if (b >= 0xC2 && b <= 0xDF && i + 1 < n && (s[i + 1] & 0xC0) == 0x80) { r = ((b & 0x1F) << 6) | (s[i + 1] & 0x3F); w = 2; }
        else if (b >= 0xE0 && b <= 0xEF && i + 2 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80) {
            uint32_t t = ((b & 0x0F) << 12) | ((s[i + 1] & 0x3F) << 6) | (s[i + 2] & 0x3F);
            if (t >= 0x800 && !(t >= 0xD800 && t <= 0xDFFF)) { r = t; w = 3; }
        } else if (b >= 0xF0 && b <= 0xF4 && i + 3 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80 && (s[i + 3] & 0xC0) == 0x80) {
            uint32_t t = ((b & 0x07) << 18) | ((s[i + 1] & 0x3F) << 12) | ((s[i + 2] & 0x3F) << 6) | (s[i + 3] & 0x3F);
            if (t >= 0x10000 && t <= 0x10FFFF) { r = t; w = 4; }
        }
        if (r == 0xFFFD && w == 1) { d += "\\ufffd"; i++; continue; }
        if (r == 0x2028 || r == 0x2029) { d += "\\u202"; d += hex[r & 0xF]; i += w; continue; }
        d.append((const char*)s + i, w); i += w;
    }
    d += '"';
    return d;
}

// fmt.Sprintf("%v", value) for the dynamic types the typesystem produces
std::string go_sprint_v(const orc_val& v) {
    switch (v.kind) {
    case OG_NIL: return "<nil>";
    case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: case OG_INT: return fmt_i64(v.i);
    case OG_UINT8: case OG_UINT16: case OG_UINT32: case OG_UINT64: case OG_UINT: return fmt_u64(v.u);
    case OG_FLOAT32: return fmt_f32((float)v.f, FMT_G_V);
    case OG_FLOAT64: return fmt_f64(v.f, FMT_G_V);
    case OG_BOOL: return v.i ? "true" : "false";
    case OG_STRING: case OG_JSON: return std::string((const char*)v.s, v.slen);
    case OG_BYTES: {   // %v of []byte: [1 2 3]
        std::string s = "[";
        for (uint64_t i = 0; i < v.slen; i++) { if (i) s += ' '; s += fmt_u64(v.s[i]); }
        return s + "]";
    }
    case OG_DURATION: return fmt_duration(v.i);
    case OG_TIME: {    // time.Time.String(): "2006-01-02 15:04:05.999999999 -0700 MST" (UTC)
        std::string r = fmt_rfc3339nano_utc(v.i, v.nsec);
        r[r.find('T')] = ' '; r.pop_back(); return r + " +0000 UTC";
    }
    }
    return "";
}

// to_string.SerializeToString: pkg/transformer/registry/to_string/to_string.go:145-171 (skipUTCConversion=false)
std::string serialize_to_string(const orc_val& v, int32_t yt) {
    switch (yt) {
    case TF_BYTES: if (v.kind == OG_BYTES) return std::string((const char*)v.s, v.slen); break;   // :151-155
    case TF_ANY:                                                                                   // :156-160 json.Marshal(value)
        if (v.kind == OG_NIL) return "null";
        if (v.kind == OG_STRING) return go_json_quote(v.s, v.slen);
        if (v.kind == OG_JSON) return std::string((const char*)v.s, v.slen);
        if (v.kind == OG_BOOL) return v.i ? "true" : "false";
        if (v.kind == OG_FLOAT64) return fmt_f64(v.f, FMT_JSON);
        if (v.kind == OG_FLOAT32) return fmt_f32((float)v.f, FMT_JSON);
        if (v.kind >= OG_INT8 && v.kind <= OG_UINT64) return go_sprint_v(v);
        break;
    case TF_DATE: if (v.kind == OG_TIME) return fmt_date_only(v.i); break;                         // :161-164
    case TF_DATETIME: case TF_TIMESTAMP: if (v.kind == OG_TIME) return fmt_rfc3339nano_utc(v.i, v.nsec); break;  // :165-168
    }
    return go_sprint_v(v);                                                                         // :170
}

// ------------------------------------------------------------------ filter_rows
// toInt64E: pkg/transformer/registry/filter_rows/util.go:47-79
// returns 0 ok, 1 not-int, 2 overflow
int to_int64e(const orc_val& v, int64_t& out) {
    switch (v.kind) {
    case OG_INT: case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: out = v.i; return 0;
    case OG_UINT: case OG_UINT8: case OG_UINT16: case OG_UINT32: out = (int64_t)v.u; return 0;
    case OG_UINT64: if (v.u > (uint64_t)std::numeric_limits<int64_t>::max()) return 2; out = (int64_t)v.u; return 0;
    default: return 1;
    }
}
// spf13/cast v1.7.1 ToFloat64E (filter_rows.go:201)
bool to_float64e(const orc_val& v, double& out) {
    switch (v.kind) {
    case OG_FLOAT64: case OG_FLOAT32: out = v.f; return true;
    case OG_INT: case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: out = (double)v.i; return true;
    case OG_UINT: case OG_UINT8: case OG_UINT16: case OG_UINT32: case OG_UINT64: out = (double)v.u; return true;
    case OG_BOOL: out = v.i ? 1 : 0; return true;
    case OG_NIL: out = 0; return true;
    case OG_STRING: {   // strconv.ParseFloat(s, 64)
        if (v.slen == 0 || v.slen > 400) return false;
        std::string s((const char*)v.s, v.slen);
        for (char c : s) if (!(std::isdigit((unsigned char)c) || c == '.' || c == 'e' || c == 'E' || c == '+' || c == '-' || c == '_' )) {
            // Go also accepts inf/nan/hex floats; not reachable from typed columns
            return false;
        }
        char* end = nullptr; double d = std::strtod(s.c_str(), &end);
        if (end != s.c_str() + s.size()) return false;
        out = d; return true;
    }
    default: return false;   // time.Time, []byte, json text, Duration(int64 kind via fmt.Stringer? no: cast handles time.Duration? -> not numeric here)
    }
}

template <typename T> bool ordered(T a, T b, int op, bool& res) {   // matchOrderedValue filter_rows.go:367-383
    switch (op) {
    case OP_EQ: res = a == b; return true; case OP_NE: res = a != b; return true;
    case OP_LT: res = a < b; return true;  case OP_LE: res = a <= b; return true;
    case OP_GT: res = a > b; return true;  case OP_GE: res = a >= b; return true;
    }
    return false;
}
int cmp_bytes(const uint8_t* a, size_t an, const uint8_t* b, size_t bn) {
    size_t m = an < bn ? an : bn; int c = m ? std::memcmp(a, b, m) : 0;
    if (c) return c < 0 ? -1 : 1;
    return an < bn ? -1 : (an > bn ? 1 : 0);
}
bool contains_bytes(const uint8_t* h, size_t hn, const uint8_t* n, size_t nn) {
    if (nn == 0) return true;
    if (nn > hn) return false;
    for (size_t i = 0; i + nn <= hn; i++) if (std::memcmp(h + i, n, nn) == 0) return true;
    return false;
}

// matchValue: pkg/transformer/registry/filter_rows/filter_rows.go:180-365
int match_value(const orc_val& v1, const orc_term& t, bool& matched) {
    const int op = t.op; const bool is_set = (op == OP_IN || op == OP_NOTIN);
    const int base = t.vtype & 15; const bool is_list = (t.vtype & LV_LIST) != 0;
    int64_t int1 = 0; bool is_int1 = false, is_float1 = false;
    int r = to_int64e(v1, int1);
    if (r == 0) is_int1 = true; else if (r == 2) return TF_ROWERR_FILTER_OVERFLOW;          // :190-197
    double float1 = 0; bool fok = to_float64e(v1, float1);
    if (!is_int1 && fok) is_float1 = true;                                                     // :199-205
    auto in_ilist = [&](int64_t x) { for (int k = 0; k < t.nlist; k++) if (t.ilist[k] == x) return true; return false; };
    auto in_flist = [&](double x) { for (int k = 0; k < t.nlist; k++) if (t.flist[k] == x) return true; return false; };
    auto set_res = [&](bool contained) { matched = (op == OP_IN) ? contained : !contained; return 0; };
    switch (base) {
    case LV_INT:                                                                                // :213-241
        if (is_int1) {
            if (is_set) return set_res(in_ilist(int1));
            return ordered<int64_t>(int1, t.i, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        }
        if (is_float1) {
            if (is_set) { if (std::trunc(float1) == float1) return set_res(in_ilist(gocast::go_f2i64(float1))); matched = false; return 0; }   // int64(float1): amd64 CVTTSD2SQ
            return ordered<double>(float1, (double)t.i, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        }
        break;
    case LV_FLOAT:                                                                              // :243-267
        if (is_int1) {
            if (is_set) return set_res(in_flist((double)int1));
            return ordered<double>((double)int1, t.f, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        }
        if (is_float1) {
            if (is_set) return set_res(in_flist(float1));
            return ordered<double>(float1, t.f, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        }
        break;
    case LV_BOOL:                                                                               // :269-285
        if (is_list) break;   // val2.IsBool() is false for lists -> falls to default/unsupported
        if (v1.kind == OG_BOOL) return ordered<int>(v1.i ? 1 : 0, t.i ? 1 : 0, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        break;
    case LV_STRING: {                                                                           // :287-328
        const bool isb = v1.kind == OG_BYTES;
        if (!is_list && isb) {
            if (op == OP_MATCH) { matched = contains_bytes(v1.s, v1.slen, t.s, t.slen); return 0; }
            if (op == OP_NOTMATCH) { matched = !contains_bytes(v1.s, v1.slen, t.s, t.slen); return 0; }
            int c = cmp_bytes(v1.s, v1.slen, t.s, t.slen);                                      // matchBytesValue :385-401
            switch (op) {
            case OP_EQ: matched = c == 0; return 0; case OP_NE: matched = c != 0; return 0;
            case OP_LT: matched = c < 0; return 0;  case OP_LE: matched = c < 1; return 0;
            case OP_GT: matched = c > 0; return 0;  case OP_GE: matched = c > -1; return 0;
            }
            return TF_ROWERR_FILTER_TYPEPAIR;
        }
        if (isb || v1.kind == OG_STRING) {
            if (op == OP_MATCH) { matched = contains_bytes(v1.s, v1.slen, t.s, t.slen); return 0; }
            if (op == OP_NOTMATCH) { matched = !contains_bytes(v1.s, v1.slen, t.s, t.slen); return 0; }
            if (is_set) {
                bool c = false;
                for (int k = 0; k < t.nlist && !c; k++) { uint32_t a = t.soffs[k], b = t.soffs[k + 1]; c = (b - a == v1.slen) && std::memcmp(t.sheap + a, v1.s, v1.slen) == 0; }
                return set_res(c);
            }
            int c = cmp_bytes(v1.s, v1.slen, t.s, t.slen);
            switch (op) {
            case OP_EQ: matched = c == 0; return 0; case OP_NE: matched = c != 0; return 0;
            case OP_LT: matched = c < 0; return 0;  case OP_LE: matched = c <= 0; return 0;
            case OP_GT: matched = c > 0; return 0;  case OP_GE: matched = c >= 0; return 0;
            }
            return TF_ROWERR_FILTER_TYPEPAIR;
        }
        break;
    }
    case LV_TIME:                                                                               // :330-351
        if (v1.kind == OG_TIME) {
            int64_t um = v1.i * 1000000 + (int64_t)(v1.nsec / 1000);                           // time.UnixMicro()
            if (is_set) return set_res(in_ilist(um));
            return ordered<int64_t>(um, t.i, op, matched) ? 0 : TF_ROWERR_FILTER_TYPEPAIR;
        }
        break;   // string-typed dates (stringToTime, util.go:15-45) do not occur in typed columns
    case LV_NULL:                                                                               // :353-358
        if (op == OP_EQ) { matched = v1.kind == OG_NIL; return 0; }
        if (op == OP_NE) { matched = v1.kind != OG_NIL; return 0; }
        break;
    }
    return TF_ROWERR_FILTER_TYPEPAIR;                                                           // :364
}

// ------------------------------------------------------------------ ClickHouse sink
// columntypes.ToChType + Nullable(!Required): pkg/providers/clickhouse/columntypes/types.go:210-248,
// sink_table.go:196-208,229-235.  ch:-prefixed original types are not handled (fatal).
std::string ch_base_type(int32_t yt) {
    switch (yt) {
    case TF_ANY: case TF_BYTES: case TF_UTF8: return "String";
    case TF_DOUBLE: return "Float64"; case TF_FLOAT: return "Float32"; case TF_BOOLEAN: return "UInt8";
    case TF_INT8: return "Int8"; case TF_INT16: return "Int16"; case TF_INT32: return "Int32"; case TF_INT64: return "Int64";
    case TF_UINT8: return "UInt8"; case TF_UINT16: return "UInt16"; case TF_UINT32: return "UInt32"; case TF_UINT64: return "UInt64";
    case TF_DATE: return "Date"; case TF_DATETIME: return "DateTime"; case TF_TIMESTAMP: return "DateTime64(6)";
    case TF_INTERVAL: return "Int64";
    }
    return "String";
}
std::string ch_type(const orc_colschema& c, int32_t yt) {
    std::string b = ch_base_type(yt);
    return c.required ? b : "Nullable(" + b + ")";
}

const int64_t CH_MIN_DATE = 0;              // 1970-01-01  columntypes/types.go:15-18
const int64_t CH_MAX_DATE = 4291747200LL;   // 2106-01-01

struct ColBuilder {
    int32_t yt; bool nullable;
    std::vector<uint8_t> nulls, data;
    void put(const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; data.insert(data.end(), b, b + n); }
    void put_varint(uint64_t v) { while (v >= 0x80) { data.push_back((uint8_t)(v | 0x80)); v >>= 7; } data.push_back((uint8_t)v); }
    void put_str(const uint8_t* s, size_t n) { put_varint(n); put(s, n); }
};

// One value: columntypes.Restore (columntypes/types.go:74-115) -> abstract.Restore
// (pkg/abstract/restore.go:20-223) -> driver column append (clickhouse-go/v2 lib/column, third-party).
// Returns false on a value the driver would reject.
bool append_value(ColBuilder& cb, const orc_val& v) {
    const bool is_null = v.kind == OG_NIL;
    if (cb.nullable) cb.nulls.push_back(is_null ? 1 : 0);
    else if (is_null && !(cb.yt == TF_ANY || cb.yt == TF_BYTES || cb.yt == TF_UTF8)) {
        // nil into a non-Nullable column: the reference relies on insert_null_as_default / the driver's zero value
    }
    switch (cb.yt) {
    case TF_INT8: { int8_t x = is_null ? 0 : (int8_t)v.i; cb.put(&x, 1); return true; }
    case TF_INT16: { int16_t x = is_null ? 0 : (int16_t)v.i; cb.put(&x, 2); return true; }
    case TF_INT32: { int32_t x = is_null ? 0 : (int32_t)v.i; cb.put(&x, 4); return true; }
    case TF_INT64: { int64_t x = is_null ? 0 : v.i; cb.put(&x, 8); return true; }
    case TF_INTERVAL: { int64_t x = is_null ? 0 : v.i; cb.put(&x, 8); return true; }
    case TF_UINT8: { uint8_t x = is_null ? 0 : (uint8_t)v.u; cb.put(&x, 1); return true; }
    case TF_UINT16: { uint16_t x = is_null ? 0 : (uint16_t)v.u; cb.put(&x, 2); return true; }
    case TF_UINT32: { uint32_t x = is_null ? 0 : (uint32_t)v.u; cb.put(&x, 4); return true; }
    case TF_UINT64: { uint64_t x = is_null ? 0 : v.u; cb.put(&x, 8); return true; }
    case TF_BOOLEAN: { uint8_t x = is_null ? 0 : (v.i ? 1 : 0); cb.put(&x, 1); return true; }
    case TF_FLOAT: { float x = is_null ? 0 : (float)v.f; if (!is_null && v.kind == OG_FLOAT32) std::memcpy(&x, &v.u, 4); cb.put(&x, 4); return true; }   // a Go float32 keeps its bits
    case TF_DOUBLE: { double x = is_null ? 0 : v.f; cb.put(&x, 8); return true; }
    case TF_DATE: {        // applyClickhouseDateBoundaries types.go:20-29, then Date = days since epoch (u16)
        int64_t s = is_null ? 0 : v.i;
        if (!is_null) { if (s > CH_MAX_DATE || (s == CH_MAX_DATE && v.nsec > 0)) s = CH_MAX_DATE; if (s < CH_MIN_DATE) s = CH_MIN_DATE; }
        uint16_t d = (uint16_t)(s / 86400); cb.put(&d, 2); return true;
    }
    case TF_DATETIME: {    // same clamp, DateTime = u32 Unix seconds
        int64_t s = is_null ? 0 : v.i;
        if (!is_null) { if (s > CH_MAX_DATE || (s == CH_MAX_DATE && v.nsec > 0)) s = CH_MAX_DATE; if (s < CH_MIN_DATE) s = CH_MIN_DATE; }
        uint32_t x = (uint32_t)s; cb.put(&x, 4); return true;
    }
    case TF_TIMESTAMP: {   // no clamp (types.go:94 covers only date/datetime); DateTime64(6) = UnixMicro
        int64_t x = is_null ? 0 : v.i * 1000000 + (int64_t)(v.nsec / 1000); cb.put(&x, 8); return true;
    }
    case TF_BYTES: case TF_UTF8:
        if (is_null) { cb.put_varint(0); return true; }
        cb.put_str(v.s, v.slen); return true;
    case TF_ANY:           // types.go:76-91: string passes through, anything else is JSON text (marshalAny)
        if (is_null) { cb.put_varint(0); return true; }
        cb.put_str(v.s, v.slen); return true;
    }
    return false;
}

void put_uvarint(std::vector<uint8_t>& o, uint64_t v) { while (v >= 0x80) { o.push_back((uint8_t)(v | 0x80)); v >>= 7; } o.push_back((uint8_t)v); }
void put_string(std::vector<uint8_t>& o, const std::string& s) { put_uvarint(o, s.size()); o.insert(o.end(), s.begin(), s.end()); }

// ClickHouse native-protocol Data block at client revision 54460 (clickhouse-go/v2 v2.46.0
// lib/proto/block.go Encode: block info, #columns, #rows, then per column name, type,
// has-custom-serialization byte (revision >= 54454), data).
std::vector<uint8_t> native_block(const std::vector<std::string>& names, const std::vector<std::string>& types,
                                  const std::vector<ColBuilder>& cols, uint64_t nrows) {
    std::vector<uint8_t> o;
    put_uvarint(o, 1); o.push_back(0);                       // field 1: is_overflows = false
    put_uvarint(o, 2); int32_t bucket = -1; const uint8_t* b = (const uint8_t*)&bucket; o.insert(o.end(), b, b + 4);  // field 2: bucket_num = -1
    put_uvarint(o, 0);
    put_uvarint(o, names.size()); put_uvarint(o, nrows);
    for (size_t c = 0; c < names.size(); c++) {
        put_string(o, names[c]); put_string(o, types[c]); o.push_back(0);
        if (nrows == 0) continue;
        if (cols[c].nullable) o.insert(o.end(), cols[c].nulls.begin(), cols[c].nulls.end());
        o.insert(o.end(), cols[c].data.begin(), cols[c].data.end());
    }
    return o;
}

// MarshalCItoJSON: pkg/providers/clickhouse/httpuploader/marshal.go:88-253 for the value types of typed columns.
// ch_base = the target column's ClickHouse base type (columntypes.ToChType of the RESULT type), nullability aside.
void json_each_row_value(std::string& o, const orc_val& v, int32_t yt_result, const std::string& ch_base) {
    const bool is_string = ch_base == "String";
    auto quoted_raw = [&](const uint8_t* p, size_t n) {            // :127-137 / :215-223 + questionableQuoter :264-266
        o += '"';
        bool need = false; for (size_t i = 0; i < n; i++) if (p[i] == '"' || p[i] == '\\') { need = true; break; }
        if (!need) o.append((const char*)p, n);
        else for (size_t i = 0; i < n; i++) { if (p[i] == '\\' || p[i] == '"') o += '\\'; o += (char)p[i]; }
        o += '"';
    };
    switch (v.kind) {
    case OG_TIME: {                                                  // marshalTime :63-78
        if (is_string) { std::string r = fmt_rfc3339nano_utc(v.i, v.nsec); r[r.find('T')] = ' '; r.pop_back(); o += '"' + r + " +0000 UTC\""; }
        else if (ch_base.rfind("DateTime64", 0) == 0) {
            const int prec = std::atoi(ch_base.c_str() + 11);
            int64_t full = v.i * 1000000000LL + (int64_t)v.nsec;     // UnixNano
            if (prec > 0 && prec < 9) { int64_t div = 1; for (int i = 0; i < 9 - prec; i++) div *= 10; full = full / div; }
            o += fmt_i64(full);
        }
        else if (ch_base == "Date") o += '"' + fmt_date_only(v.i) + '"';
        else o += fmt_i64(v.i);
        return;
    }
    case OG_STRING: quoted_raw(v.s, v.slen); return;
    case OG_BYTES: quoted_raw(v.s, v.slen); return;
    case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: case OG_INT:
        if (is_string) o += '"'; o += fmt_i64(v.i); if (is_string) o += '"'; return;
    case OG_UINT8: case OG_UINT16: case OG_UINT32: case OG_UINT64: case OG_UINT:
        if (is_string) o += '"'; o += fmt_u64(v.u); if (is_string) o += '"'; return;
    case OG_FLOAT32: if (is_string) o += '"'; o += fmt_f32((float)v.f, FMT_F); if (is_string) o += '"'; return;
    case OG_FLOAT64: if (is_string) o += '"'; o += fmt_f64(v.f, FMT_F); if (is_string) o += '"'; return;
    case OG_BOOL:                                                    // :186-205
        if (yt_result == TF_BOOLEAN) o += v.i ? "true" : "false";
        else if (is_string) o += v.i ? "\"true\"" : "\"false\"";
        else o += v.i ? "1" : "0";
        return;
    case OG_DURATION: {                                              // default branch: json.Marshal(Duration) = integer, type != any -> quoted
        o += go_json_quote((const uint8_t*)fmt_i64(v.i).data(), fmt_i64(v.i).size()); return;
    }
    case OG_JSON:                                                    // default branch :224-243 with r = the JSON text
        if (yt_result != TF_ANY || is_string) o += go_json_quote(v.s, v.slen); else o.append((const char*)v.s, v.slen);
        return;
    }
}


// number_to_float on the JSON text of an `any` value: every json.Number becomes float64 (json.Number.Float64 = strconv.ParseFloat),
// which json.Marshal then prints in its float format; a literal that does not fit float64 stays a json.Number (its text).
std::string number_to_float_text(const uint8_t* s, size_t n) {
    std::string d; bool ins = false;
    for (size_t i = 0; i < n;) {
        const char c = (char)s[i];
        if (ins) { d += c; if (c == '\\' && i + 1 < n) { d += (char)s[i + 1]; i += 2; continue; } if (c == '"') ins = false; i++; continue; }
        if (c == '"') { ins = true; d += c; i++; continue; }
        if (c == '-' || (c >= '0' && c <= '9')) {
            size_t q = i; while (q < n && ((s[q] >= '0' && s[q] <= '9') || s[q] == '-' || s[q] == '+' || s[q] == '.' || s[q] == 'e' || s[q] == 'E')) q++;
            std::string_view lit((const char*)s + i, q - i); double f;
            if (jsn::go_parse_float(lit, f) == 0 && !std::isnan(f) && !std::isinf(f)) d += fmt_f64(f, FMT_JSON); else d += lit;
            i = q; continue;
        }
        d += c; i++;
    }
    return d;
}

// ------------------------------------------------------------------ batch serializers (pkg/serializer)
// encoding/json appendString with escapeHTML = false (json.go:56-58 SetEscapeHTML(false)): only `"`, `\`, control
// characters, invalid UTF-8 and U+2028/2029 are escaped
std::string go_json_quote_nohtml(const uint8_t* s, size_t n) {
    std::string q = go_json_quote(s, n), d; d.reserve(q.size());
    for (size_t i = 0; i < q.size();) {
        if (q[i] == '\\' && i + 1 < q.size()) {
            if (q[i + 1] == 'u' && i + 5 < q.size() && (q.compare(i + 2, 4, "003c") == 0 || q.compare(i + 2, 4, "003e") == 0 || q.compare(i + 2, 4, "0026") == 0)) {
                d += q.compare(i + 2, 4, "003c") == 0 ? '<' : q.compare(i + 2, 4, "003e") == 0 ? '>' : '&'; i += 6; continue;
            }
            d += q[i]; d += q[i + 1]; i += 2; continue;
        }
        d += q[i++];
    }
    return d;
}
// JSON text produced by json.Marshal (HTML escaping on) as a second encoder with SetEscapeHTML(false) would write the same value
std::string json_unescape_html(const uint8_t* s, size_t n) {
    std::string d; bool ins = false;
    for (size_t i = 0; i < n;) {
        const char c = (char)s[i];
        if (!ins) { if (c == '"') ins = true; d += c; i++; continue; }
        if (c == '\\' && i + 1 < n) {
            if (s[i + 1] == 'u' && i + 5 < n && (!std::memcmp(s + i + 2, "003c", 4) || !std::memcmp(s + i + 2, "003e", 4) || !std::memcmp(s + i + 2, "0026", 4))) {
                d += !std::memcmp(s + i + 2, "003c", 4) ? '<' : !std::memcmp(s + i + 2, "003e", 4) ? '>' : '&'; i += 6; continue;
            }
            d += c; d += (char)s[i + 1]; i += 2; continue;
        }
        if (c == '"') ins = false;
        d += c; i++;
    }
    return d;
}
std::string base64_std(const uint8_t* s, size_t n) {
    static const char* A = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string d;
    for (size_t i = 0; i < n; i += 3) {
        const uint32_t v = (uint32_t)s[i] << 16 | (i + 1 < n ? (uint32_t)s[i + 1] << 8 : 0) | (i + 2 < n ? s[i + 2] : 0);
        d += A[v >> 18]; d += A[(v >> 12) & 63]; d += i + 1 < n ? A[(v >> 6) & 63] : '='; d += i + 2 < n ? A[v & 63] : '=';
    }
    return d;
}
bool year_in_json_range(int64_t sec) { return sec >= -62167219200LL && sec < 253402300800LL; }   // [0000-01-01, 10000-01-01)
// toJsonValue + json.Encoder for one cell (json_format.go:32-82). false: the encoder would fail
bool ser_json_value(std::string& o, const orc_val& v, int32_t yt, bool any_as_string) {
    switch (v.kind) {
    case OG_NIL: o += "null"; return true;
    case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: case OG_INT: o += fmt_i64(v.i); return true;
    case OG_UINT8: case OG_UINT16: case OG_UINT32: case OG_UINT64: case OG_UINT: o += fmt_u64(v.u); return true;
    case OG_FLOAT32: if (std::isnan(v.f) || std::isinf(v.f)) return false; o += fmt_f32((float)v.f, FMT_JSON); return true;
    case OG_FLOAT64: if (std::isnan(v.f) || std::isinf(v.f)) return false; o += fmt_f64(v.f, FMT_F); return true;   // strictify: json.Number(FormatFloat(f,'f',-1,64)) castx/caste.go:36-60
    case OG_BOOL: o += v.i ? "true" : "false"; return true;
    case OG_STRING:
        if (yt == TF_ANY && any_as_string) { std::string j = go_json_quote(v.s, v.slen); o += go_json_quote_nohtml((const uint8_t*)j.data(), j.size()); }
        else o += go_json_quote_nohtml(v.s, v.slen);
        return true;
    case OG_BYTES: o += '"'; o += base64_std(v.s, v.slen); o += '"'; return true;
    case OG_TIME: if (!year_in_json_range(v.i)) return false; o += '"'; o += fmt_rfc3339nano_utc(v.i, v.nsec); o += '"'; return true;
    case OG_DURATION: o += fmt_i64(v.i); return true;
    case OG_JSON:
        if (any_as_string) o += go_json_quote_nohtml(v.s, v.slen); else o += json_unescape_html(v.s, v.slen);
        return true;
    }
    return false;
}
// toCsvValue (csv_format.go:32-120) -> one encoding/csv field
std::string ser_csv_cell(const orc_val& v, int32_t yt) {
    switch (v.kind) {
    case OG_NIL: return "";
    case OG_INT8: case OG_INT16: case OG_INT32: case OG_INT64: case OG_INT: return fmt_i64(v.i);
    case OG_UINT8: case OG_UINT16: case OG_UINT32: case OG_UINT64: case OG_UINT: return fmt_u64(v.u);
    case OG_FLOAT32: return fmt_f32((float)v.f, FMT_F);
    case OG_FLOAT64: return fmt_f64(v.f, FMT_F);
    case OG_BOOL: return v.i ? "true" : "false";
    case OG_STRING: if (yt == TF_ANY) return go_json_quote(v.s, v.slen);        // csv_format.go:109-116 json.Marshal(value)
                    return std::string((const char*)v.s, v.slen);
    case OG_BYTES: return base64_std(v.s, v.slen);
    case OG_TIME: { std::string r = fmt_rfc3339nano_utc(v.i, v.nsec); r[r.find('T')] = ' '; r.pop_back(); return r + " +0000 UTC"; }    // castx.ToStringE -> fmt.Stringer -> Time.String()
    case OG_DURATION: return fmt_duration(v.i);
    case OG_JSON: return std::string((const char*)v.s, v.slen);
    }
    return "";
}
void csv_write_field(std::string& o, const std::string& f) {     // encoding/csv Writer.Write, Comma ',' UseCRLF false
    bool q = false;
    if (!f.empty()) {
        if (f == "\\.") q = true;
        for (char c : f) if (c == '\n' || c == '\r' || c == '"' || c == ',') q = true;
        if (!q) { size_t w; q = go_space_fwd((const uint8_t*)f.data(), f.size(), w); }
    }
    if (!q) { o += f; return; }
    o += '"'; for (char c : f) { if (c == '"') o += "\"\""; else o += c; } o += '"';
}

void to_buf(const std::vector<uint8_t>& v, orc_buf* b) {
    if (!b) return;
    b->len = v.size(); b->data = (uint8_t*)std::malloc(v.size() ? v.size() : 1);
    if (v.size()) std::memcpy(b->data, v.data(), v.size());
}
int copy_out(const std::string& s, char* dst, int cap) { if ((int)s.size() + 1 > cap) return -1; std::memcpy(dst, s.data(), s.size()); dst[s.size()] = 0; return (int)s.size(); }

}  // namespace
std::string jsn::go_quote(const uint8_t* s, size_t n) { return go_json_quote(s, n); }

extern "C" {

void orc_free(orc_buf* b) { if (b && b->data) { std::free(b->data); b->data = nullptr; b->len = 0; } }

int orc_fmt_float64(double v, int f, char* dst, int cap) { return copy_out(fmt_f64(v, (FloatFmt)f), dst, cap); }
int orc_fmt_float32(float v, int f, char* dst, int cap) { return copy_out(fmt_f32(v, (FloatFmt)f), dst, cap); }
int orc_fmt_duration(int64_t ns, char* dst, int cap) { return copy_out(fmt_duration(ns), dst, cap); }
int orc_fmt_rfc3339nano(int64_t sec, uint32_t nsec, char* dst, int cap) { return copy_out(fmt_rfc3339nano_utc(sec, nsec), dst, cap); }
int orc_serialize_to_string(const orc_val* v, int32_t yt, char* dst, int cap) { return copy_out(serialize_to_string(*v, yt), dst, cap); }

// HmacHasher.hash: pkg/transformer/registry/mask/hmac_hasher.go:29-33
void orc_hmac_sha256_hex(const uint8_t* key, uint64_t klen, const uint8_t* msg, uint64_t mlen, char out[65]) {
    uint8_t d[32]; hmac_sha256(key, klen, msg, mlen, d); std::string h = hex_lower(d, 32); std::memcpy(out, h.data(), 64); out[64] = 0;
}
void orc_sha256(const uint8_t* msg, uint64_t mlen, uint8_t out[32]) { Sha256 s; s.init(); s.update(msg, mlen); s.final(out); }
void orc_cityhash128(const uint8_t* p, uint64_t n, uint64_t* lo, uint64_t* hi) { city::u128 h = city::hash128(p, n); *lo = h.first; *hi = h.second; }
uint64_t orc_lz4_bound(uint64_t n) { return lz4_bound(n); }
uint64_t orc_lz4_compress(const uint8_t* src, uint64_t n, uint8_t* dst) { return lz4_compress(src, n, dst); }
int64_t orc_lz4_decompress(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t rs) { size_t r = lz4_decompress(src, n, dst, rs); return r == (size_t)-1 ? -1 : (int64_t)r; }

int orc_match_value(const orc_val* v, const orc_term* t, int* matched) { bool m = false; int rc = match_value(*v, *t, m); *matched = m; return rc; }

int orc_ch_type(const orc_colschema* c, char* dst, int cap) { return copy_out(ch_type(*c, c->type), dst, cap); }

}  // extern "C" (reopened below)

namespace {
uint32_t crc32_ieee(const uint8_t* p, size_t n) {            // hash/crc32 IEEE: reflected 0xEDB88320, init and final xor 0xFFFFFFFF
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u))); }
    return ~c;
}
thread_local uint32_t g_part_id = 0; thread_local bool g_has_part = false;     // PartID the last sharder step gave the current row
// Applies the transformer steps to row r (boxed in `row`); returns false when the row is dropped or errored.
// Sink and serializer wire formats take INSERT rows only on the device path (sink_table.go:296-305 refuses the others on non-updatable
// tables, marshal.go:92-95 and the queue / batch serializers need OldKeys for them): an update / delete row that survives the chain is a
// row error (TF_ROWERR_SINK_KIND_HOST, term 0xff: not raised by a transformer) that the shim routes through the Go sink.
static bool sink_refuses_kind(const tf_batch* in, uint64_t r, tf_rowerr* errs, uint64_t& ne) {
    const int kind = in->kinds ? in->kinds[r] : TF_KIND_INSERT;
    if (kind != TF_KIND_UPDATE && kind != TF_KIND_DELETE) return false;
    errs[ne++] = tf_rowerr{(uint32_t)r, TF_ROWERR_SINK_KIND_HOST, 0xff};
    return true;
}

bool apply_steps(const tf_batch* in, uint64_t r, const orc_step* steps, int nsteps, std::vector<Boxed>& row, std::vector<int32_t>& cur_type,
                 tf_rowerr* errs, uint64_t& ne) {
    const uint32_t nc = in->ncols;
    for (uint32_t c = 0; c < nc; c++) { row[c].own.clear(); box(in->cols[c], r, row[c].v); cur_type[c] = in->cols[c].type; }   // []interface{} of this ChangeItem
    const int kind = in->kinds ? in->kinds[r] : TF_KIND_INSERT;
    g_has_part = false;
    for (int s = 0; s < nsteps; s++) {
        const orc_step& st = steps[s];
        if (st.kind == STEP_SHARDER) {                            // SharderTransformer.generatePartID sharder.go:130-145
            std::string joined;
            for (int k = 0; k < st.ncols; k++) { if (k) joined += '.'; joined += serialize_to_string(row[st.cols[k]].v, cur_type[st.cols[k]]); }
            g_part_id = crc32_ieee((const uint8_t*)joined.data(), joined.size()) % (uint32_t)st.kind_mask; g_has_part = true;
        } else if (st.kind == STEP_SKIP_EVENTS) {                        // SkipEvents.Apply skip_events.go:52-62
            if ((st.kind_mask >> kind) & 1) return false;
        } else if (st.kind == STEP_FILTER_ROWS) {                // FilterRowsTransformer.Apply filter_rows.go:99-130
            if (kind == TF_KIND_UPDATE || kind == TF_KIND_DELETE) { errs[ne++] = tf_rowerr{(uint32_t)r, TF_ROWERR_FILTER_KIND, (uint16_t)st.convert_to_bytes}; return false; }
            if (st.pass_all) continue;                            // :109-113 isNameMatching == false
            bool any = false; int err = 0;
            for (int e = 0; e < st.nexpr && !any && !err; e++) {   // matchItem :137-148 (OR), matchExpression :150-177 (AND)
                bool all = true;
                for (uint32_t k = st.expr_off[e]; k < st.expr_off[e + 1]; k++) {
                    bool m = false; int rc = match_value(row[st.terms[k].col].v, st.terms[k], m);
                    if (rc) { err = rc; break; }
                    if (!m) { all = false; break; }
                }
                if (!err && all) any = true;
            }
            if (err) { errs[ne++] = tf_rowerr{(uint32_t)r, (uint16_t)err, (uint16_t)st.convert_to_bytes}; return false; }
            if (!any) return false;
        } else if (st.kind == STEP_MASK) {                        // HmacHasher.Apply hmac_hasher.go:52-74
            for (int k = 0; k < st.ncols; k++) {
                int c = st.cols[k];
                std::string text = serialize_to_string(row[c].v, cur_type[c]);
                uint8_t d[32]; hmac_sha256(st.salt, st.salt_len, (const uint8_t*)text.data(), text.size(), d);
                row[c].set_string(hex_lower(d, 32), OG_STRING); cur_type[c] = TF_UTF8;
            }
        } else if (st.kind == STEP_TO_DATETIME) {                 // ToDateTimeTransformer.Apply / SerializeToDateTime to_datetime.go:89-151
            for (int k = 0; k < st.ncols; k++) {
                int c = st.cols[k]; orc_val& v = row[c].v; int64_t sec = 0;
                if (v.kind == OG_INT32) sec = v.i; else if (v.kind == OG_UINT32) sec = (int64_t)v.u;
                std::memset(&v, 0, sizeof v); v.kind = OG_TIME; v.i = sec; cur_type[c] = TF_DATETIME;
            }
        } else if (st.kind == STEP_NUMBER_TO_FLOAT) {             // NumberToFloatTransformer.processItem number_to_float.go:75-123
            if (kind != TF_KIND_INSERT && kind != TF_KIND_UPDATE) continue;                     // supportedKinds :21, :64
            for (int k = 0; k < st.ncols; k++) {
                int c = st.cols[k]; orc_val& v = row[c].v;
                if (cur_type[c] != TF_ANY || v.kind != OG_JSON) continue;                      // a Go string / nil inside `any` is left alone
                row[c].set_string(number_to_float_text(v.s, v.slen), OG_JSON);
            }
        } else if (st.kind == STEP_TO_STRING) {                   // ToStringTransformer.Apply to_string.go:58-97
            for (int k = 0; k < st.ncols; k++) {
                int c = st.cols[k];
                row[c].set_string(serialize_to_string(row[c].v, cur_type[c]), st.convert_to_bytes ? OG_BYTES : OG_STRING);
                cur_type[c] = st.convert_to_bytes ? TF_BYTES : TF_UTF8;
            }
        }
    }
    return true;
}
void result_types(const tf_batch* in, const orc_step* steps, int nsteps, std::vector<int32_t>& out_type, std::vector<uint32_t>& out_cols) {
    const uint32_t nc = in->ncols;
    out_type.resize(nc);
    for (uint32_t c = 0; c < nc; c++) out_type[c] = in->cols[c].type;
    for (int s = 0; s < nsteps; s++) {
        if (steps[s].kind == STEP_MASK) for (int k = 0; k < steps[s].ncols; k++) out_type[steps[s].cols[k]] = TF_UTF8;        // hmac_hasher.go:35-47
        if (steps[s].kind == STEP_TO_STRING) for (int k = 0; k < steps[s].ncols; k++) out_type[steps[s].cols[k]] = steps[s].convert_to_bytes ? TF_BYTES : TF_UTF8;  // to_string.go:66-74
        if (steps[s].kind == STEP_TO_DATETIME) for (int k = 0; k < steps[s].ncols; k++) out_type[steps[s].cols[k]] = TF_DATETIME;                                  // to_datetime.go:126-135
    }
    // filter_columns (filter_columns_transformer.go:228-236): the surviving columns, schema order kept
    bool sel = false;
    for (int s = 0; s < nsteps; s++) if (steps[s].kind == STEP_SELECT_COLS) { sel = true; out_cols.clear(); for (int k = 0; k < steps[s].ncols; k++) out_cols.push_back((uint32_t)steps[s].cols[k]); }
    if (!sel) for (uint32_t c = 0; c < nc; c++) out_cols.push_back(c);
}
int width_of(int32_t tf) {
    switch (tf) {
    case TF_INT8: case TF_UINT8: case TF_BOOLEAN: return 1;
    case TF_INT16: case TF_UINT16: return 2;
    case TF_INT32: case TF_UINT32: case TF_FLOAT: return 4;
    case TF_BYTES: case TF_UTF8: case TF_ANY: return 0;
    default: return 8;
    }
}
}  // namespace

extern "C" int orc_push_encode(const tf_batch* in, const orc_colschema* schema, const orc_step* steps, int nsteps,
                    int wire_fmt, uint64_t frame_bytes, orc_buf* out_raw, orc_buf* out_wire,
                    uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs) {
    const uint32_t nc = in->ncols;
    std::vector<int32_t> out_type; std::vector<uint32_t> out_cols;
    result_types(in, steps, nsteps, out_type, out_cols);
    const uint32_t no = (uint32_t)out_cols.size();
    std::vector<ColBuilder> cbs(no);
    std::vector<std::string> names(no), types(no);
    for (uint32_t k = 0; k < no; k++) {
        const uint32_t c = out_cols[k];
        cbs[k].yt = out_type[c]; cbs[k].nullable = !schema[c].required;
        names[k] = schema[c].name; types[k] = ch_type(schema[c], out_type[c]);
    }
    uint64_t kept = 0, ne = 0;
    std::vector<Boxed> row(nc);
    std::vector<int32_t> cur_type(nc);
    if (wire_fmt == TF_WIRE_CH_JSONEACHROW) {                     // uploadAsJSON: rows as text, no Restore (sink_table.go:289-344, httpuploader/uploader.go:62-96)
        std::string text;
        std::vector<std::string> base(no);
        for (uint32_t k = 0; k < no; k++) base[k] = ch_base_type(out_type[out_cols[k]]);
        for (uint64_t r = 0; r < in->nrows; r++) {
            if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs, ne)) continue;
            if (sink_refuses_kind(in, r, errs, ne)) continue;
            text += '{'; bool has = false;
            for (uint32_t k = 0; k < no; k++) {
                const orc_val& v = row[out_cols[k]].v;
                if (v.kind == OG_NIL) continue;                   // isNilValue -> the column is omitted (marshal.go:103-105)
                if (v.kind == OG_JSON && v.slen == 4 && std::memcmp(v.s, "null", 4) == 0) continue;   // json.Marshal gives "null": name rolled back (:229-233)
                text += '"'; text += names[k]; text += "\":";
                json_each_row_value(text, v, out_type[out_cols[k]], base[k]);
                text += ','; has = true;
            }
            if (has) text.pop_back();
            text += "}\n"; kept++;
        }
        if (rows_out) *rows_out = kept;
        if (nerrs) *nerrs = ne;
        std::vector<uint8_t> bytes(text.begin(), text.end());
        to_buf(bytes, out_raw); to_buf(bytes, out_wire);
        return 0;
    }
    if ((wire_fmt & 0xff) == TF_WIRE_SER_JSON || (wire_fmt & 0xff) == TF_WIRE_SER_CSV) {   // pkg/serializer batch serializers
        const bool csv = (wire_fmt & 0xff) == TF_WIRE_SER_CSV, nl = wire_fmt & TF_WIRE_F_CLOSING_NEWLINE, aas = wire_fmt & TF_WIRE_F_ANY_AS_STRING;
        std::vector<uint32_t> order(no); for (uint32_t k = 0; k < no; k++) order[k] = k;
        if (!csv) std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return names[a] < names[b]; });   // encoding/json sorts map keys
        std::string text;
        for (uint64_t r = 0; r < in->nrows; r++) {
            if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs, ne)) continue;
            if (sink_refuses_kind(in, r, errs, ne)) continue;
            if (csv) {
                for (uint32_t k = 0; k < no; k++) { if (k) text += ','; csv_write_field(text, ser_csv_cell(row[out_cols[k]].v, out_type[out_cols[k]])); }
                text += '\n';
            } else {
                if (kept && !nl) text += '\n';                        // separator "\n" between items, none after the last (batch.go:205-219, batch_factory.go:36-39)
                text += '{'; bool row_err = false;
                for (uint32_t j = 0; j < no; j++) {
                    const uint32_t k = order[j];
                    if (j) text += ',';
                    text += go_json_quote_nohtml((const uint8_t*)names[k].data(), names[k].size()); text += ':';
                    if (!ser_json_value(text, row[out_cols[k]].v, out_type[out_cols[k]], aas)) { text += "null"; if (!row_err) errs[ne++] = tf_rowerr{(uint32_t)r, TF_ROWERR_SER_VALUE, (uint16_t)k}; row_err = true; }
                }
                text += '}';
                if (nl) text += '\n';
            }
            kept++;
        }
        if (rows_out) *rows_out = kept;
        if (nerrs) *nerrs = ne;
        std::vector<uint8_t> bytes(text.begin(), text.end());
        to_buf(bytes, out_raw); to_buf(bytes, out_wire);
        return 0;
    }
    for (uint64_t r = 0; r < in->nrows; r++) {
        if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs, ne)) continue;
        if (sink_refuses_kind(in, r, errs, ne)) continue;
        // sink: restoreVals sink_table.go:698-704 + driver append
        for (uint32_t k = 0; k < no; k++) if (!append_value(cbs[k], row[out_cols[k]].v)) return TF_E_FATAL_UNSUPPORTED;
        kept++;
    }
    if (rows_out) *rows_out = kept;
    if (nerrs) *nerrs = ne;
    if (wire_fmt == 0) return 0;
    std::vector<uint8_t> raw = native_block(names, types, cbs, kept);
    to_buf(raw, out_raw);
    if (wire_fmt == TF_WIRE_CH_NATIVE) { to_buf(raw, out_wire); return 0; }
    if (wire_fmt == TF_WIRE_CH_NATIVE_LZ4) { to_buf(ch_compress_frames(raw.data(), raw.size(), frame_bytes), out_wire); return 0; }
    return TF_E_FATAL_UNSUPPORTED;
}

// ------------------------------------------------------------------ Debezium emitter, common (no original_type) path
// One column value as addCommon stores it (pkg/debezium/emitter_common.go:67-180) and util.JSONMarshalUnescape then writes it.
// false: addCommon or the encoder returns an error (EmitKV fails).
namespace {
// Columns with a pg: original type go through AddPg (pkg/debezium/pg/emitter.go:265-629). `form` names the branch the plan picked
// for the (original type, column type) pair; the strict columnar layout fixes the Go type of the value (int16 / int32 / int64,
// bool, float64, string, []byte, time.Time in UTC, `any` JSON).
enum { DF_COMMON = 0, DF_PG_REAL = 2, DF_PG_DOUBLE = 3, DF_PG_STRING = 4, DF_PG_JSON = 6, DF_PG_DATE = 7, DF_PG_TS_MICROS = 8, DF_PG_TS_MILLIS = 9, DF_PG_TSTZ = 10, DF_PG_INET = 11 };
bool dbz_emit_value_pg(std::string& o, const orc_val& v, int form) {
    if (v.kind == OG_NIL) { o += "null"; return true; }                                         // :266-269
    if (v.kind == OG_JSON && v.slen == 4 && !std::memcmp(v.s, "null", 4)) { o += "null"; return true; }   // a nil interface inside `any`
    switch (form) {
    case DF_PG_REAL:                                                                             // :342-356 float32(t)
        if (v.kind != OG_FLOAT64 && v.kind != OG_FLOAT32) return false;
        { const float f = (float)v.f; if (std::isnan(f) || std::isinf(f)) return false; o += fmt_f32(f, FMT_JSON); }
        return true;
    case DF_PG_DOUBLE:                                                                           // :357-370 convertFloatNanInf :180-191
        if (v.kind != OG_FLOAT64) return false;
        if (std::isnan(v.f)) o += "\"NaN\""; else if (std::isinf(v.f)) o += v.f < 0 ? "\"-Infinity\"" : "\"Infinity\""; else o += fmt_f64(v.f, FMT_JSON);
        return true;
    case DF_PG_STRING:                                                                           // colVal.(string): text, uuid, cidr, macaddr, citext, character*, int4range / int8range
        if (v.kind == OG_STRING) { o += go_json_quote_nohtml(v.s, v.slen); return true; }
        if (v.kind == OG_JSON && v.slen && v.s[0] == '"') { o += json_unescape_html(v.s, v.slen); return true; }
        return false;                                                                            // the type assertion panics in the reference
    case DF_PG_INET: {                                                                           // :401-410 strings.TrimSuffix(t, "/32")
        std::string t;
        if (v.kind == OG_STRING) t.assign((const char*)v.s, v.slen);
        else return false;                                                                       // (a JSON-quoted string inside `any` would need decoding: not produced by the pg source)
        if (t.size() >= 3 && t.compare(t.size() - 3, 3, "/32") == 0) t.resize(t.size() - 3);
        o += go_json_quote_nohtml((const uint8_t*)t.data(), t.size()); return true;
    }
    case DF_PG_JSON: {                                                                           // :377-382 string(JSONMarshalUnescape(colVal))
        std::string t;
        if (v.kind == OG_STRING) t = go_json_quote_nohtml(v.s, v.slen);
        else if (v.kind == OG_JSON) t = json_unescape_html(v.s, v.slen);
        else return false;
        o += go_json_quote_nohtml((const uint8_t*)t.data(), t.size()); return true;
    }
    case DF_PG_DATE: if (v.kind != OG_TIME) return false; o += fmt_i64(v.i / 86400); return true;            // :476-478 int(t.Unix()/(3600*24))
    case DF_PG_TS_MICROS: case DF_PG_TS_MILLIS: {                                               // :558-580 ts.Time.UnixMicro() / divider (typeutil/helpers.go:104-120)
        if (v.kind != OG_TIME) return false;
        const int64_t micro = v.i * 1000000 + (int64_t)(v.nsec / 1000);
        o += fmt_i64(form == DF_PG_TS_MILLIS ? micro / 1000 : micro); return true;
    }
    case DF_PG_TSTZ:                                                                             // :581-594 SprintfDebeziumTime typeutil/helpers.go:1107-1116
        if (v.kind != OG_TIME) return false;
        o += '"'; o += fmt_rfc3339nano_utc(v.i, v.nsec); o += '"'; return true;
    }
    return false;
}
bool dbz_emit_value(std::string& o, const orc_val& v, int32_t yt, int form = DF_COMMON) {
    if (form != DF_COMMON) return dbz_emit_value_pg(o, v, form);
    if (v.kind == OG_NIL) { o += "null"; return true; }                                         // :68-71
    const bool sint = v.kind == OG_INT8 || v.kind == OG_INT16 || v.kind == OG_INT32 || v.kind == OG_INT64 || v.kind == OG_INT;
    const bool uint = v.kind == OG_UINT8 || v.kind == OG_UINT16 || v.kind == OG_UINT32 || v.kind == OG_UINT64 || v.kind == OG_UINT;
    switch (yt) {
    case TF_INT8: case TF_INT16: case TF_INT32: case TF_INT64:                                   // :74-79 the value itself is stored
        if (!sint) return false; o += fmt_i64(v.i); return true;
    case TF_UINT8: case TF_UINT16: case TF_UINT32: case TF_UINT64:                               // :81-86 uint64(t)
        if (uint) { o += fmt_u64(v.u); return true; }
        if (sint) { o += fmt_u64((uint64_t)v.i); return true; }
        return false;
    case TF_FLOAT: case TF_DOUBLE:                                                               // :88-98
        if (v.kind == OG_FLOAT32) { if (std::isnan(v.f) || std::isinf(v.f)) return false; o += fmt_f32((float)v.f, FMT_JSON); return true; }
        if (v.kind == OG_FLOAT64) { if (std::isnan(v.f) || std::isinf(v.f)) return false; o += fmt_f64(v.f, FMT_JSON); return true; }
        return false;
    case TF_BYTES:                                                                               // :100-108
        if (v.kind != OG_STRING && v.kind != OG_BYTES) return false;
        o += '"'; o += base64_std(v.s, v.slen); o += '"'; return true;
    case TF_UTF8:                                                                                // :110-120
        if (v.kind == OG_STRING) { o += go_json_quote_nohtml(v.s, v.slen); return true; }
        if (v.kind == OG_BYTES) { o += '"'; o += base64_std(v.s, v.slen); o += '"'; return true; }   // a []byte value is marshalled as base64
        if (v.kind == OG_TIME) { o += fmt_i64(v.i / 86400); return true; }                       // mysql:date
        return false;
    case TF_BOOLEAN:                                                                             // :122-130
        if (v.kind == OG_BOOL) { o += v.i ? "true" : "false"; return true; }
        if (v.kind == OG_INT8) { o += v.i == 1 ? "true" : "false"; return true; }
        return false;
    case TF_DATETIME: case TF_TIMESTAMP:                                                         // :132-146 time.Time.MarshalJSON
        if (v.kind != OG_TIME || !year_in_json_range(v.i)) return false;
        o += '"'; o += fmt_rfc3339nano_utc(v.i, v.nsec); o += '"'; return true;
    case TF_ANY:                                                                                 // :148-160
        if (v.kind == OG_STRING) { o += go_json_quote_nohtml(v.s, v.slen); return true; }
        if (v.kind == OG_JSON) {
            if (v.slen == 4 && !std::memcmp(v.s, "null", 4)) { o += "null"; return true; }     // a nil interface: colVal == nil
            if (v.slen && v.s[0] == '"') { o += json_unescape_html(v.s, v.slen); return true; }  // a Go string
            if (v.slen && v.s[0] == '{') {                                                       // map -> string(JSONMarshalUnescape(t)) stored as a string
                const std::string t = json_unescape_html(v.s, v.slen);
                o += go_json_quote_nohtml((const uint8_t*)t.data(), t.size()); return true;
            }
        }
        return false;
    default: return false;                                                                       // :161-163 unknown input data type
    }
}
std::string dbz_pack(const std::string& payload, const char* schema, int64_t schema_id) {
    if (schema_id >= 0) {                                                                        // packer_schema_registry.go:66-76
        std::string m; m += '\0'; for (int sh = 24; sh >= 0; sh -= 8) m += (char)(((uint32_t)schema_id >> sh) & 0xff);
        return m + payload;
    }
    if (schema) return "{\"payload\":" + payload + ",\"schema\":" + schema + "}";                // packer_include_schema.go:34-38 (map keys sorted)
    return payload;                                                                              // packer_skip_schema.go:12-19
}
}  // namespace

// Emitter.EmitKV for the rows of one batch (pkg/debezium/emitter_value_converter.go:626-690; valPayload :453-512,
// buildSource :329-372, makeKey / buildKV :259-327). INSERT rows only: update / delete events read ChangeItem.OldKeys.
extern "C" int orc_debezium_emit_crud(const tf_batch* in, const tf_old_keys* old, int tombstones, const orc_colschema* schema, const uint8_t* is_key, const uint8_t* forms, const orc_step* steps, int nsteps,
                                 const tf_row_meta* meta, const orc_dbz_emit_opts* o, orc_buf* out, uint32_t* key_sizes, uint32_t* row_sizes, uint32_t* msg_sizes,
                                 uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs);
extern "C" int orc_debezium_emit(const tf_batch* in, const orc_colschema* schema, const uint8_t* is_key, const uint8_t* forms, const orc_step* steps, int nsteps,
                                 const tf_row_meta* meta, const orc_dbz_emit_opts* o, orc_buf* out, uint32_t* key_sizes, uint32_t* row_sizes,
                                 uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs) {
    return orc_debezium_emit_crud(in, nullptr, 1, schema, is_key, forms, steps, nsteps, meta, o, out, key_sizes, row_sizes, nullptr, rows_out, errs, nerrs);
}
// Emitter.emitKV for every row kind (:626-674): 1 message for insert / plain update, delete event + tombstone for delete,
// delete event + tombstone + insert event for an update whose primary key changed (ChangeItem.KeysChanged change_item.go:235-284).
extern "C" int orc_debezium_emit_crud(const tf_batch* in, const tf_old_keys* old, int tombstones, const orc_colschema* schema, const uint8_t* is_key, const uint8_t* forms, const orc_step* steps, int nsteps,
                                 const tf_row_meta* meta, const orc_dbz_emit_opts* o, orc_buf* out, uint32_t* key_sizes, uint32_t* row_sizes, uint32_t* msg_sizes,
                                 uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs) {
    const uint32_t nc = in->ncols;
    std::vector<int32_t> out_type; std::vector<uint32_t> out_cols;
    result_types(in, steps, nsteps, out_type, out_cols);
    const uint32_t no = (uint32_t)out_cols.size();
    std::vector<std::string> names(no);
    for (uint32_t k = 0; k < no; k++) names[k] = schema[out_cols[k]].name;
    std::vector<uint32_t> order(no); for (uint32_t k = 0; k < no; k++) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return names[a] < names[b]; });
    auto q = [](const char* t) { const std::string s = t ? t : ""; return go_json_quote_nohtml((const uint8_t*)s.data(), s.size()); };
    uint64_t kept = 0, ne = 0;
    std::vector<Boxed> row(nc); std::vector<int32_t> cur_type(nc);
    std::string text;
    for (uint64_t r = 0; r < in->nrows; r++) {
        const int kind = in->kinds ? in->kinds[r] : TF_KIND_INSERT;
        if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs, ne)) continue;
        bool row_err = false;
        const bool old_row = old && old->values && kind != TF_KIND_INSERT && (old->row_has ? old->row_has[r] != 0 : true);      // len(OldKeys.KeyNames) > 0
        auto present = [&](uint32_t c) { return old_row && old->present_cols && old->present_cols[c]; };
        uint32_t n_present = 0, n_pkeys = 0;
        for (uint32_t c = 0; c < nc; c++) { if (old && old->present_cols && old->present_cols[c]) n_present++; }
        for (uint32_t k = 0; k < no; k++) if (is_key[out_cols[k]]) n_pkeys++;
        auto emit = [&](std::string& t, const orc_val& v, uint32_t k) {
            if (!dbz_emit_value(t, v, out_type[out_cols[k]], forms ? forms[out_cols[k]] : 0)) { t += "null"; if (!row_err) errs[ne++] = tf_rowerr{(uint32_t)r, TF_ROWERR_SER_VALUE, (uint16_t)k}; row_err = true; }
        };
        auto obj = [&](bool keys_only) {                          // buildKV over ColumnNames / ColumnValues
            std::string t = "{"; bool first = true;
            for (uint32_t j = 0; j < no; j++) {
                const uint32_t k = order[j];
                if (keys_only && !is_key[out_cols[k]]) continue;
                if (!first) t += ','; first = false;
                t += go_json_quote_nohtml((const uint8_t*)names[k].data(), names[k].size()); t += ':';
                emit(t, row[out_cols[k]].v, k);
            }
            return t + "}";
        };
        // mode 0: makeValues over OldKeys.KeyNames (keys_only: the primary keys among them); mode 1: every column null, OldKeys on top (op "d")
        auto obj_old = [&](bool keys_only, int mode) {
            std::string t = "{"; bool first = true;
            for (uint32_t j = 0; j < no; j++) {
                const uint32_t k = order[j]; const uint32_t c = out_cols[k];
                if (keys_only && !is_key[c]) continue;
                const bool pr = present(c);
                if (mode == 0 && !pr) continue;
                if (!first) t += ','; first = false;
                t += go_json_quote_nohtml((const uint8_t*)names[k].data(), names[k].size()); t += ':';
                if (pr) { orc_val ov; box(old->values->cols[c], r, ov); emit(t, ov, k); }
                else if (o->source_type == 2) emit(t, row[c].v, k);            // mysql: `before` starts from ColumnValues (:469-477)
                else t += "null";
            }
            return t + "}";
        };
        bool changed = false;
        if (kind == TF_KIND_UPDATE)
            for (uint32_t k = 0; k < no && !changed; k++) {
                const uint32_t c = out_cols[k]; if (!is_key[c]) continue;
                const orc_val& nv = row[c].v;
                if (present(c)) {
                    orc_val ov; box(old->values->cols[c], r, ov);
                    if (ov.kind != nv.kind) changed = true;
                    else if (ov.kind == OG_NIL) changed = false;
                    else if (ov.kind == OG_STRING || ov.kind == OG_BYTES || ov.kind == OG_JSON) changed = ov.slen != nv.slen || std::memcmp(ov.s, nv.s, ov.slen) != 0;
                    else if (ov.kind == OG_FLOAT32 || ov.kind == OG_FLOAT64) changed = std::memcmp(&ov.f, &nv.f, sizeof ov.f) != 0;
                    else if (ov.kind == OG_TIME) changed = ov.i != nv.i || ov.nsec != nv.nsec;
                    else if (ov.kind >= OG_UINT8 && ov.kind <= OG_UINT64) changed = ov.u != nv.u;
                    else changed = ov.i != nv.i;
                } else changed = nv.kind != OG_NIL;
            }
        const uint64_t lsn = meta && meta->lsn ? meta->lsn[r] : 0, ct = meta && meta->commit_time ? meta->commit_time[r] : 0;
        const uint32_t id = meta && meta->id ? meta->id[r] : 0;
        const std::string snap = o->snapshot ? "\"true\"" : "\"false\"";
        std::string src = "{";
        if (o->source_type == 1) {            // pg: connector db lsn name schema snapshot table ts_ms txId version xmin
            src += "\"connector\":\"postgresql\",\"db\":" + q(o->database) + ",\"lsn\":" + fmt_u64(lsn) + ",\"name\":" + q(o->name) + ",\"schema\":" + q(o->schema) +
                   ",\"snapshot\":" + snap + ",\"table\":" + q(o->table) + ",\"ts_ms\":" + fmt_u64(ct / 1000000) + ",\"txId\":" + fmt_u64(id) + ",\"version\":" + q(o->version) + ",\"xmin\":null";
        } else if (o->source_type == 2) {     // mysql: connector db file gtid name pos query row server_id snapshot table thread ts_ms version
            char file[64]; std::snprintf(file, sizeof file, "mysql-log.%06llu", (unsigned long long)(lsn / 1000000000000ull));      // typeutil/helpers.go:1101-1105
            std::string gtid = "null";
            if (meta && meta->txid_offsets && meta->txid_heap && meta->txid_offsets[r + 1] > meta->txid_offsets[r])
                gtid = go_json_quote_nohtml(meta->txid_heap + meta->txid_offsets[r], meta->txid_offsets[r + 1] - meta->txid_offsets[r]);
            src += "\"connector\":\"mysql\",\"db\":" + q(o->schema) + ",\"file\":" + q(file) + ",\"gtid\":" + gtid + ",\"name\":" + q(o->name) + ",\"pos\":" + fmt_u64(lsn % 1000000000000ull) +
                   ",\"query\":null,\"row\":0,\"server_id\":0,\"snapshot\":" + snap + ",\"table\":" + q(o->table) + ",\"thread\":null,\"ts_ms\":" + fmt_u64(ct / 1000000) + ",\"version\":" + q(o->version);
        } else {
            src += "\"db\":" + q(o->database) + ",\"name\":" + q(o->name) + ",\"snapshot\":" + snap + ",\"table\":" + q(o->table) + ",\"ts_ms\":" + fmt_u64(ct / 1000000) + ",\"version\":" + q(o->version);
        }
        src += "}";
        int plan[3], np = 0;                                       // 0 regular, 1 delete event, 2 tombstone, 3 insert event
        if (changed) { plan[np++] = 1; if (tombstones) plan[np++] = 2; plan[np++] = 3; }
        else if (kind == TF_KIND_DELETE) { plan[np++] = 1; if (tombstones) plan[np++] = 2; }
        else plan[np++] = 0;
        const bool has_prev = old_row && n_present > n_pkeys;      // hasPreviousValues :277-285
        uint32_t total = 0;
        if (msg_sizes) msg_sizes[7 * kept] = (uint32_t)np;
        for (int m = 0; m < np; m++) {
            const int mt = plan[m];
            const bool key_from_after = mt == 3 || !old_row;      // makeKey :259-274
            const char op = mt == 1 ? 'd' : (mt == 3 ? 'c' : (kind == TF_KIND_UPDATE ? 'u' : (kind == TF_KIND_DELETE ? 'd' : (o->snapshot ? 'r' : 'c'))));
            std::string key_msg;
            if (!o->drop_keys) key_msg = dbz_pack(key_from_after ? obj(true) : obj_old(true, 0), o->key_schema, o->key_schema_id);
            if (m == 0) key_sizes[kept] = (uint32_t)key_msg.size();
            text += key_msg; total += (uint32_t)key_msg.size();
            if (mt == 2) { if (msg_sizes) { msg_sizes[7 * kept + 1 + 2 * m] = (uint32_t)key_msg.size(); msg_sizes[7 * kept + 2 + 2 * m] = 0xffffffffu; } continue; }
            const std::string after = op == 'd' ? "null" : obj(false);
            const std::string before = op == 'd' ? obj_old(false, 1) : ((op == 'u' && has_prev) ? obj_old(false, 0) : "null");
            // payloadTSMS = time.Unix(CommitTime/1e9, CommitTime%1e9) (GetPayloadTSMS :697-699); UnixNano()/1e6 in int64
            const std::string payload = "{\"after\":" + after + ",\"before\":" + before + ",\"op\":\"" + std::string(1, op) + "\",\"source\":" + src +
                                        ",\"transaction\":null,\"ts_ms\":" + fmt_i64((int64_t)ct / 1000000) + "}";
            const std::string val_msg = dbz_pack(payload, o->val_schema, o->val_schema_id);
            text += val_msg; total += (uint32_t)val_msg.size();
            if (msg_sizes) { msg_sizes[7 * kept + 1 + 2 * m] = (uint32_t)key_msg.size(); msg_sizes[7 * kept + 2 + 2 * m] = (uint32_t)val_msg.size(); }
        }
        row_sizes[kept] = total; kept++;
    }
    if (rows_out) *rows_out = kept;
    if (nerrs) *nerrs = ne;
    std::vector<uint8_t> bytes(text.begin(), text.end());
    to_buf(bytes, out);
    return 0;
}

extern "C" uint32_t orc_crc32_ieee(const uint8_t* p, uint64_t n) { return crc32_ieee(p, n); }
extern "C" int orc_shard_ids(const tf_batch* in, const orc_colschema* schema, const orc_step* steps, int nsteps, uint32_t* part_ids, uint64_t* rows_out) {
    (void)schema;
    std::vector<Boxed> row(in->ncols); std::vector<int32_t> cur_type(in->ncols);
    std::vector<tf_rowerr> errs(in->nrows + 1); uint64_t ne = 0, kept = 0;
    for (uint64_t r = 0; r < in->nrows; r++) {
        if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs.data(), ne)) continue;
        part_ids[kept++] = g_has_part ? g_part_id : 0xFFFFFFFFu;
    }
    if (rows_out) *rows_out = kept;
    return 0;
}

extern "C" int orc_push_columns(const tf_batch* in, const orc_colschema* schema, const orc_step* steps, int nsteps,
                     orc_buf* out, orc_regions* regions, int32_t* out_types, uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs) {
    (void)schema;
    const uint32_t nc = in->ncols;
    std::vector<int32_t> out_type; std::vector<uint32_t> out_cols;
    result_types(in, steps, nsteps, out_type, out_cols);
    const uint32_t no = (uint32_t)out_cols.size();
    struct CB { std::vector<uint8_t> values, valid_bits, aux, heap; std::vector<uint32_t> offs; bool has_valid, has_aux; };
    std::vector<CB> cb(no);
    std::vector<char> rewritten(nc, 0);     // mask_field / convert_to_string give the column a fresh, never-nil text value
    for (int s = 0; s < nsteps; s++) if (steps[s].kind == STEP_MASK || steps[s].kind == STEP_TO_STRING || steps[s].kind == STEP_TO_DATETIME) for (int k = 0; k < steps[s].ncols; k++) rewritten[steps[s].cols[k]] = 1;   // number_to_float keeps nil / tags: only the text changes
    for (uint32_t k = 0; k < no; k++) {
        const tf_col& ic = in->cols[out_cols[k]];
        const bool masked = rewritten[out_cols[k]] != 0;
        cb[k].has_valid = ic.validity && !masked; cb[k].has_aux = ic.aux && !masked; cb[k].offs.push_back(0);
    }
    uint64_t kept = 0, ne = 0;
    std::vector<Boxed> row(nc); std::vector<int32_t> cur_type(nc);
    for (uint64_t r = 0; r < in->nrows; r++) {
        if (!apply_steps(in, r, steps, nsteps, row, cur_type, errs, ne)) continue;
        for (uint32_t k = 0; k < no; k++) {
            const uint32_t c = out_cols[k]; const orc_val& v = row[c].v; const tf_col& ic = in->cols[c]; CB& b = cb[k];
            const int w = width_of(out_type[c]);
            if (b.has_valid) { if ((kept & 7) == 0) b.valid_bits.push_back(0); if (v.kind != OG_NIL) b.valid_bits.back() |= (uint8_t)(1u << (kept & 7)); }
            if (w) {   // the value keeps its input representation (zero for nil)
                uint8_t tmp[8] = {0};
                if (rewritten[c]) std::memcpy(tmp, &v.i, 8);          // convert_to_datetime: time.Time seconds
                else if (v.kind != OG_NIL) std::memcpy(tmp, (const uint8_t*)ic.values + (size_t)w * r, w);
                b.values.insert(b.values.end(), tmp, tmp + w);
            } else {
                if (v.kind != OG_NIL) b.heap.insert(b.heap.end(), v.s, v.s + v.slen);
                b.offs.push_back((uint32_t)b.heap.size());
            }
            if (b.has_aux) {
                if (ic.type == TF_ANY) b.aux.push_back(((const uint8_t*)ic.aux)[r]);
                else { uint32_t x = ((const uint32_t*)ic.aux)[r]; const uint8_t* q = (const uint8_t*)&x; b.aux.insert(b.aux.end(), q, q + 4); }
            }
        }
        kept++;
    }
    std::vector<uint8_t> buf;
    auto put = [&](const void* p, size_t n) -> uint64_t { while (buf.size() % 16) buf.push_back(0); uint64_t at = buf.size(); const uint8_t* q = (const uint8_t*)p; buf.insert(buf.end(), q, q + n); return at; };
    for (uint32_t k = 0; k < no; k++) {
        CB& b = cb[k]; orc_regions& g = regions[k]; const int w = width_of(out_type[out_cols[k]]);
        out_types[k] = out_type[out_cols[k]];
        g.values = w ? put(b.values.data(), b.values.size()) : ~0ull;
        g.validity = b.has_valid ? put(b.valid_bits.data(), b.valid_bits.size()) : ~0ull;
        g.aux = b.has_aux ? put(b.aux.data(), b.aux.size()) : ~0ull;
        g.offsets = w ? ~0ull : put(b.offs.data(), b.offs.size() * 4);
        g.heap = w ? ~0ull : put(b.heap.data(), b.heap.size());
        g.heap_len = w ? 0 : b.heap.size();
    }
    to_buf(buf, out);
    if (rows_out) *rows_out = kept;
    if (nerrs) *nerrs = ne;
    return 0;
}

extern "C" {

int orc_csv_parse(const uint8_t* buf, uint64_t len, const int32_t* types, const int32_t* paths, int ncols, const orc_csv_opts* o,
                  orc_buf* out, orc_regions* regions, uint64_t* rows, uint64_t* lines, uint64_t* consumed,
                  tf_rowerr* errs, uint64_t errs_cap, uint64_t* nerrs) {
    CsvOpts co; co.delimiter = o->delimiter; co.quote = o->quote; co.escape = o->escape; co.double_quote = o->double_quote;
    co.strings_can_be_null = o->strings_can_be_null; co.quoted_strings_can_be_null = o->quoted_strings_can_be_null; co.include_missing = o->include_missing;
    auto split = [](const char* s, std::vector<std::string>& v) { if (!s) return; std::string cur; for (const char* p = s;; p++) { if (*p == '\n' || *p == 0) { v.push_back(cur); cur.clear(); if (!*p) break; } else cur += *p; } };
    split(o->null_values, co.null_values); split(o->true_values, co.true_values); split(o->false_values, co.false_values);
    std::vector<CsvCol> sc(ncols);
    for (int c = 0; c < ncols; c++) { sc[c].tf = types[c]; sc[c].path = paths[c]; }
    CsvResult R = csv_parse(buf, len, sc, co, o->skip_lines);
    std::vector<uint8_t> b;
    auto put = [&](const void* p, size_t n) -> uint64_t { while (b.size() % 16) b.push_back(0); uint64_t at = b.size(); const uint8_t* q = (const uint8_t*)p; b.insert(b.end(), q, q + n); return at; };
    for (int c = 0; c < ncols; c++) {
        CsvColOut& oc = R.cols[c]; orc_regions& g = regions[c]; const int w = width_tf(types[c]);
        g.values = w ? put(oc.values.data(), oc.values.size()) : ~0ull;
        g.validity = ~0ull;
        g.aux = oc.aux.empty() && !(types[c] == TF_ANY || types[c] == TF_DATE || types[c] == TF_DATETIME || types[c] == TF_TIMESTAMP) ? ~0ull : put(oc.aux.data(), oc.aux.size());
        g.offsets = w ? ~0ull : put(oc.offs.data(), oc.offs.size() * 4);
        g.heap = w ? ~0ull : put(oc.heap.data(), oc.heap.size());
        g.heap_len = w ? 0 : oc.heap.size();
    }
    to_buf(b, out);
    *rows = R.rows; *lines = R.lines; *consumed = R.consumed;
    uint64_t ne = 0; for (auto& e : R.errs) if (ne < errs_cap) errs[ne++] = e;
    *nerrs = R.errs.size();
    return 0;
}

int orc_json_parse(const uint8_t* buf, uint64_t len, const orc_json_msg* msgs, uint64_t nmsgs,
                   const char* const* names, const int32_t* types, const uint8_t* keys, const uint8_t* required, int ncols,
                   const orc_json_opts* o, orc_buf* out, orc_regions* regions, uint64_t* rows, uint64_t* lines,
                   tf_rowerr* errs, uint64_t errs_cap, uint64_t* nerrs) {
    jsn::Opts jo; jo.add_rest = o->add_rest; jo.add_dedupe_keys = o->add_dedupe_keys; jo.null_keys_allowed = o->null_keys_allowed;
    jo.use_numbers_in_any = o->use_numbers_in_any; jo.unpack_bytes_base64 = o->unpack_bytes_base64; jo.partition = o->partition ? o->partition : "";
    std::vector<jsn::Field> fs(ncols);
    for (int c = 0; c < ncols; c++) { fs[c].name = names[c]; fs[c].tf = types[c]; fs[c].key = keys[c]; fs[c].required = required[c]; }
    std::vector<jsn::Msg> ms(nmsgs);
    for (uint64_t k = 0; k < nmsgs; k++) ms[k] = jsn::Msg{msgs[k].end, msgs[k].offset, msgs[k].write_sec, msgs[k].write_nsec};
    jsn::Result R = jsn::parse(buf, len, ms, fs, jo);
    std::vector<uint8_t> b;
    auto put = [&](const void* p, size_t n) -> uint64_t { while (b.size() % 16) b.push_back(0); uint64_t at = b.size(); const uint8_t* q = (const uint8_t*)p; b.insert(b.end(), q, q + n); return at; };
    for (int c = 0; c < ncols; c++) {
        jsn::ColOut& oc = R.cols[c]; orc_regions& g = regions[c]; const int w = jsn::width_tf(types[c]);
        g.values = w ? put(oc.values.data(), oc.values.size()) : ~0ull;
        oc.valid.resize((R.rows + 7) / 8, 0);
        g.validity = R.rows ? put(oc.valid.data(), oc.valid.size()) : ~0ull;
        const bool has_aux = types[c] == TF_ANY || types[c] == TF_DATE || types[c] == TF_DATETIME || types[c] == TF_TIMESTAMP;
        g.aux = has_aux && R.rows ? put(oc.aux.data(), oc.aux.size()) : ~0ull;
        g.offsets = w ? ~0ull : put(oc.offs.data(), oc.offs.size() * 4);
        g.heap = w ? ~0ull : put(oc.heap.data(), oc.heap.size());
        g.heap_len = w ? 0 : oc.heap.size();
    }
    to_buf(b, out);
    *rows = R.rows; *lines = R.lines;
    uint64_t ne = 0; for (auto& e : R.errs) if (ne < errs_cap) errs[ne++] = e;
    *nerrs = R.errs.size();
    return 0;
}

int orc_base64_to_numeric(const char* b64, int scale, char* dst, int cap) { std::string o; const int rc = dbz::base64_to_numeric(b64, scale, o); if (rc) return -rc; return copy_out(o, dst, cap); }

int orc_debezium_parse(const uint8_t* buf, uint64_t len, const uint64_t* msg_ends, uint64_t nmsgs, const orc_dbz_field* fields, int nfields, const orc_dbz_opts* o,
                       orc_buf* out, orc_regions* regions, int32_t* out_types, uint8_t* kinds, uint32_t* tx_ids, uint64_t* lsns, uint64_t* commit_times, uint32_t* row_msg,
                       uint64_t* rows, tf_rowerr* errs, uint64_t* nerrs) {
    dbz::Plan pl; pl.use_sr = o->use_sr; pl.schema_id = o->schema_id; pl.check_table = o->check_table;
    pl.schema_text.assign((const char*)o->schema_text, o->schema_len); pl.table_schema = o->table_schema ? o->table_schema : ""; pl.table_name = o->table_name ? o->table_name : "";
    for (int i = 0; i < nfields; i++) { dbz::Field f; f.name = fields[i].name; f.recv = fields[i].recv; f.scale = fields[i].scale; f.key = fields[i].key; pl.after.push_back(f); }
    pl.before = pl.after;
    auto tf_of = [](int recv) { switch (recv) { case dbz::R_INT8: return (int)TF_INT8; case dbz::R_INT16: return (int)TF_INT16; case dbz::R_INT32: return (int)TF_INT32; case dbz::R_INT64: return (int)TF_INT64; case dbz::R_BOOL: return (int)TF_BOOLEAN;
                                             case dbz::R_F64: case dbz::R_VSD: return (int)TF_DOUBLE; case dbz::R_BYTES: return (int)TF_BYTES; default: return (int)TF_UTF8; } };
    std::vector<jsn::ColOut> cols(nfields); uint64_t nrow = 0, ne = 0, start = 0;
    for (uint64_t m = 0; m < nmsgs; m++) {
        const uint64_t end = msg_ends[m] <= len ? msg_ends[m] : len;
        std::string_view msg((const char*)buf + start, end - start); start = end;
        int events = 0; int rc0 = 0; dbz::Row row0;
        // several events in one registry-framed message (parser.go:42-50 splits at the next 0x00): left to the host parser
        const bool multi = pl.use_sr && msg.size() >= 5 && msg[0] == 0 && msg.find('\0', 5) != std::string_view::npos;
        if (multi) { rc0 = dbz::DBZ_HOST; events = 1; }
        else dbz::do_message(pl, msg, [&](int rc, const dbz::Row& r) { if (events == 0) { rc0 = rc; row0 = r; } events++; });
        if (rc0) { errs[ne++] = tf_rowerr{(uint32_t)m, (uint16_t)rc0, (uint16_t)row0.err_col}; continue; }
        const uint64_t r = nrow++;
        kinds[r] = (uint8_t)row0.kind; tx_ids[r] = row0.tx_id; lsns[r] = row0.lsn; commit_times[r] = row0.commit_time; row_msg[r] = (uint32_t)m;
        for (int c = 0; c < nfields; c++) {
            jsn::ColOut& oc = cols[c]; const dbz::Cell& ce = row0.cells[c]; const int tf = tf_of(fields[c].recv); const int w = jsn::width_tf(tf);
            if (oc.valid.size() < r / 8 + 1) oc.valid.resize(r / 8 + 1, 0);
            if (!ce.is_null) oc.valid[r / 8] |= (uint8_t)(1u << (r % 8));
            if (w) { uint64_t v = 0; if (tf == TF_DOUBLE) std::memcpy(&v, &ce.f, 8); else v = (uint64_t)ce.i; if (ce.is_null) v = 0; for (int k = 0; k < w; k++) oc.values.push_back((uint8_t)(v >> (8 * k))); }
            else { if (!ce.is_null) oc.heap.insert(oc.heap.end(), ce.s.begin(), ce.s.end()); oc.offs.push_back((uint32_t)oc.heap.size()); }
        }
    }
    std::vector<uint8_t> b;
    auto put = [&](const void* p, size_t n) -> uint64_t { while (b.size() % 16) b.push_back(0); uint64_t at = b.size(); const uint8_t* q = (const uint8_t*)p; b.insert(b.end(), q, q + n); return at; };
    for (int c = 0; c < nfields; c++) {
        jsn::ColOut& oc = cols[c]; orc_regions& g = regions[c]; const int tf = tf_of(fields[c].recv); const int w = jsn::width_tf(tf); out_types[c] = tf;
        g.values = w ? put(oc.values.data(), oc.values.size()) : ~0ull;
        oc.valid.resize((nrow + 7) / 8, 0);
        g.validity = nrow ? put(oc.valid.data(), oc.valid.size()) : ~0ull;
        g.aux = ~0ull;
        g.offsets = w ? ~0ull : put(oc.offs.data(), oc.offs.size() * 4);
        g.heap = w ? ~0ull : put(oc.heap.data(), oc.heap.size());
        g.heap_len = w ? 0 : oc.heap.size();
    }
    to_buf(b, out); *rows = nrow; *nerrs = ne;
    return 0;
}

// BatchJSON (pkg/serializer/queue/json_batcher.go:29-66) over the lengths of the serialized items: start row of each message
int orc_queue_json_batches(const uint64_t* len_elements, uint64_t n, uint64_t max_message_size, uint64_t max_change_items, uint64_t* starts, uint64_t* n_msgs) {
    uint64_t k = 0; int64_t startIndex = 0; uint64_t sumBodies = 0;
    for (int64_t i = 0; i < (int64_t)n; i++) {
        // isJSONExtraElementViolatesConstraint :13-28
        const int64_t numNew = i - startIndex + 1; bool viol = false;
        if (max_message_size != 0) { const int64_t newLines = numNew - 1; if (sumBodies + (uint64_t)newLines + len_elements[i] > max_message_size) viol = true; }
        if (max_change_items != 0 && (uint64_t)numNew > max_change_items) viol = true;
        if (viol) {
            const int64_t numPrev = i - startIndex;
            if (numPrev == 0) { starts[k++] = (uint64_t)startIndex; startIndex = i + 1; sumBodies = 0; }
            else { starts[k++] = (uint64_t)startIndex; startIndex = i; sumBodies = len_elements[i]; }
        } else sumBodies += len_elements[i];
    }
    if ((uint64_t)startIndex != n) starts[k++] = (uint64_t)startIndex;
    starts[k] = n; *n_msgs = k; return 0;
}

// util.DeepSizeof(item.ColumnValues) (pkg/util/sizeof.go:7-110) over the canonical Go values of one row
int orc_measure(const tf_batch* in, uint64_t* per_row, uint64_t* total) {
    uint64_t sum = 0;
    for (uint64_t r = 0; r < in->nrows; r++) {
        uint64_t sz = 24;                                                // sizeofSlice: reflect.Type.Size() of []interface{}
        for (uint32_t c = 0; c < in->ncols; c++) {
            orc_val v; box(in->cols[c], r, v);
            sz += 16;                                                    // element kind Interface: + Type().Size()
            switch (v.kind) {
            case OG_NIL: break;                                          // DeepSizeof(nil): reflect.Invalid -> 0
            case OG_INT8: case OG_UINT8: case OG_BOOL: sz += 1; break;
            case OG_INT16: case OG_UINT16: sz += 2; break;
            case OG_INT32: case OG_UINT32: case OG_FLOAT32: sz += 4; break;
            case OG_INT64: case OG_UINT64: case OG_FLOAT64: case OG_DURATION: case OG_INT: case OG_UINT: sz += 8; break;
            case OG_STRING: case OG_JSON: sz += 16 + v.slen; break;      // reflect.String: Size() + Len()
            case OG_BYTES: sz += 24 + v.slen; break;                     // sizeofSlice of uint8
            case OG_TIME: sz += 24; break;                               // SizeOfStruct(time.Time): wall, ext, loc are unexported -> Type().Size() each
            }
        }
        if (per_row) per_row[r] = sz;
        sum += sz;
    }
    *total = sum; return 0;
}

int orc_ch_decode_frames(const uint8_t* wire, uint64_t n, orc_buf* raw, uint64_t* n_frames) {
    std::vector<uint8_t> r; size_t nf = 0;
    if (!ch_decompress_frames(wire, n, r, &nf)) return -1;
    to_buf(r, raw); if (n_frames) *n_frames = nf; return 0;
}

}  // extern "C"


// ---------------------------------------------------------------- typesystem casts over boxed Go values (cast_oracle.hpp), text interface for the tests
namespace {
bool goval_from_text(const char* go, const char* v, uint64_t vlen, gocast::GoVal& out) {
    using namespace gocast;
    const std::string t = go, s(v, vlen);
    out = GoVal();
    if (t == "nil") return true;
    if (t == "bool") { out.k = BOOL; out.i = s == "true"; return true; }
    if (t.rfind("int", 0) == 0) { out.k = INT; out.bits = t.size() > 3 ? std::atoi(t.c_str() + 3) : 0; out.i = (int64_t)std::strtoll(s.c_str(), nullptr, 10); return true; }
    if (t.rfind("uint", 0) == 0) { out.k = UINT; out.bits = t.size() > 4 ? std::atoi(t.c_str() + 4) : 0; out.u = (uint64_t)std::strtoull(s.c_str(), nullptr, 10); return true; }
    if (t == "float32") { out.k = F32; out.f = (double)(float)std::strtod(s.c_str(), nullptr); return true; }
    if (t == "float64") { out.k = F64; out.f = std::strtod(s.c_str(), nullptr); return true; }
    if (t == "string") { out.k = STRING; out.s = s; return true; }
    if (t == "[]byte") { out.k = BYTES; out.s = s; return true; }
    if (t == "json.Number") { out.k = JSONNUM; out.s = s; return true; }
    if (t == "map") { out.k = MAP; out.s = s; return true; }
    if (t == "time.Duration") { out.k = DURATION; out.i = (int64_t)std::strtoll(s.c_str(), nullptr, 10); return true; }
    if (t == "time.Time") { const size_t d = s.find('.'); out.k = TIME; out.i = (int64_t)std::strtoll(s.substr(0, d).c_str(), nullptr, 10); out.nsec = d == std::string::npos ? 0 : (uint32_t)std::strtoul(s.c_str() + d + 1, nullptr, 10); return true; }
    return false;
}
void goval_to_text(const gocast::GoVal& v, std::string& go, std::string& txt) {
    using namespace gocast;
    char b[64];
    switch (v.k) {
    case NIL: go = "nil"; txt = ""; break;
    case BOOL: go = "bool"; txt = v.i ? "true" : "false"; break;
    case INT: go = "int" + (v.bits ? std::to_string(v.bits) : std::string()); txt = std::to_string(v.i); break;
    case UINT: go = "uint" + (v.bits ? std::to_string(v.bits) : std::string()); txt = std::to_string(v.u); break;
    case F32: go = "float32"; std::snprintf(b, sizeof b, "%.9g", v.f); txt = b; break;
    case F64: go = "float64"; std::snprintf(b, sizeof b, "%.17g", v.f); txt = b; break;
    case STRING: go = "string"; txt = v.s; break;
    case BYTES: go = "[]byte"; txt = v.s; break;
    case JSONNUM: go = "json.Number"; txt = v.s; break;
    case MAP: go = "map"; txt = v.s; break;
    case DURATION: go = "time.Duration"; txt = std::to_string(v.i); break;
    case TIME: go = "time.Time"; std::snprintf(b, sizeof b, "%lld.%09u", (long long)v.i, v.nsec); txt = b; break;
    }
}
int put_out(const std::string& go, const std::string& txt, char* out_go, int go_cap, char* out_v, uint64_t v_cap, uint64_t* out_vlen) {
    if ((int)go.size() + 1 > go_cap || txt.size() > v_cap) return -1;
    std::memcpy(out_go, go.c_str(), go.size() + 1); std::memcpy(out_v, txt.data(), txt.size()); *out_vlen = txt.size(); return 0;
}
}  // namespace

extern "C" int orc_strictify_value(const char* go, const char* v, uint64_t vlen, int32_t tf, char* out_go, int go_cap, char* out_v, uint64_t v_cap, uint64_t* out_vlen) {
    gocast::GoVal in, out; if (!goval_from_text(go, v, vlen, in)) return -1;
    const int rc = gocast::strictify_value(in, tf, out);
    std::string g, t; goval_to_text(out, g, t);
    if (put_out(g, t, out_go, go_cap, out_v, v_cap, out_vlen)) return -1;
    return rc;
}
extern "C" int orc_restore_value(const char* go, const char* v, uint64_t vlen, const char* data_type, char* out_go, int go_cap, char* out_v, uint64_t v_cap, uint64_t* out_vlen) {
    gocast::GoVal in, out; if (!goval_from_text(go, v, vlen, in)) return -1;
    const int rc = gocast::restore_value(in, data_type, out);
    std::string g, t; goval_to_text(out, g, t);
    if (put_out(g, t, out_go, go_cap, out_v, v_cap, out_vlen)) return -1;
    return rc;
}
/* csv.Splitter: row_ends[k] = end offset of the k-th complete row; returns the row count (what follows the last end is the io.EOF remainder) */
extern "C" uint64_t orc_csv_split_rows(const uint8_t* p, uint64_t n, uint64_t* row_ends, uint64_t cap) {
    std::vector<std::string> rows; std::string rest;
    gocast::csv_split_rows(std::string((const char*)p, n), rows, rest);
    uint64_t pos = 0;
    for (size_t k = 0; k < rows.size() && k < cap; k++) { pos += rows[k].size(); row_ends[k] = pos; }
    return rows.size();
}
