// ORACLE — test infrastructure only. Never linked into or called from the product path.
//
// The typesystem casts over boxed Go values, restated function by function:
//   strictify.Strictify / strictifyValue / toSignedInt / toUnsignedInt   pkg/abstract/changeitem/strictify/strictify.go:18-181
//   abstract.Restore / maybeStringToNumeric                              pkg/abstract/restore.go:20-247
//   castx.ToJSONNumberE / ToByteSliceE / ToStringE                       pkg/util/castx/caste.go:16-106
//   csv.Splitter.ConsumeRow / updateState                                pkg/csv/splitter.go:38-85
// Third party, NOT under /root/reference: github.com/spf13/cast v1.7.1 (go.mod:63) ToIntNE / ToUintNE / ToFloat32E / ToBoolE / ToTimeE /
// ToDurationE / trimZeroDecimal — restated from its published caste.go; github.com/valyala/fastjson v1.6.4 fastfloat.Parse.
// Pinned by the reference's own unit tests: strictify_test.go:54-684, restore_test.go:14-135, splitter_test.go:14-106
// (tests/golden/cast_goldens.json, extracted by tests/golden/make_cast_goldens.py).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "csv_oracle.hpp"
#include "go_strconv.hpp"
#include "json_oracle.hpp"

namespace gocast {

enum Kind { NIL, BOOL, INT, UINT, F32, F64, STRING, BYTES, JSONNUM, TIME, DURATION, MAP };
struct GoVal {
    Kind k = NIL; int bits = 64;          // INT / UINT: 8 16 32 64, 0 = Go `int` / `uint`
    int64_t i = 0; uint64_t u = 0; double f = 0; std::string s; uint32_t nsec = 0;      // TIME: i = Unix seconds; DURATION: i = ns; MAP: s = JSON text
};
enum { OK = 0, CAST_ERR = 1, RANGE_ERR = 2, PANIC = 3, UNPINNED = 4 };      // UNPINNED: a third-party layout list this restatement does not carry (dateparse, StringToDate tail)

// Go's float -> integer conversion on amd64 (CVTTSD2SQ): out of range and NaN give the "integer indefinite" value
inline int64_t go_f2i64(double f) { if (!(f >= -9223372036854775808.0 && f < 9223372036854775808.0)) return INT64_MIN; return (int64_t)f; }
inline uint64_t go_f2u64(double f) {      // amd64: below 2^63 through CVTTSD2SQ, else subtract 2^63 first
    if (f < 9223372036854775808.0) return (uint64_t)go_f2i64(f);
    const int64_t x = go_f2i64(f - 9223372036854775808.0); return (uint64_t)x ^ 0x8000000000000000ull;
}
inline std::string trim_zero_decimal(const std::string& s) {      // cast v1.7.1 caste.go trimZeroDecimal
    bool found_zero = false;
    for (size_t i = s.size(); i > 0; i--) {
        const char c = s[i - 1];
        if (c == '.') { if (found_zero) return s.substr(0, i - 1); }
        else if (c == '0') found_zero = true;
        else return s;
    }
    return s;
}
// fastfloat.Parse(s) succeeds? (valyala/fastjson v1.6.4 fastfloat/parse.go Parse)
inline bool ff_parse_ok(const std::string& s) {
    if (s.empty()) return false;
    size_t i = 0; const bool minus = s[0] == '-';
    if (minus) { i++; if (i >= s.size()) return false; }
    if (s[i] == '.' && (i + 1 >= s.size() || s[i + 1] < '0' || s[i + 1] > '9')) return false;
    auto slow = [&]() { double f; const int rc = jsn::go_parse_float(s, f); return rc == 0 || (rc == 2); };      // ParseFloat range error still returns ±Inf: accepted
    const size_t j = i;
    while (i < s.size() && s[i] >= '0' && s[i] <= '9') { i++; if (i > 18) return slow(); }
    if (i <= j && s[i] != '.') {
        std::string t = s.substr(i); if (!t.empty() && t[0] == '+') t = t.substr(1);
        return jsn::fold_eq(t, "inf") || jsn::fold_eq(t, "infinity") || jsn::fold_eq(t, "nan");
    }
    if (i >= s.size()) return true;
    if (s[i] == '.') {
        i++; if (i >= s.size()) return true;
        const size_t k = i;
        while (i < s.size() && s[i] >= '0' && s[i] <= '9') { i++; if (i - j >= 19) return slow(); }
        if (i < k) return false;
        if (i >= s.size()) return true;
    }
    if (s[i] == 'e' || s[i] == 'E') {
        i++; if (i >= s.size()) return false;
        if (s[i] == '+' || s[i] == '-') { i++; if (i >= s.size()) return false; }
        const size_t e0 = i; int ex = 0;
        while (i < s.size() && s[i] >= '0' && s[i] <= '9') { ex = ex * 10 + (s[i] - '0'); i++; if (ex > 300) return slow(); }
        if (i <= e0) return false;
        if (i >= s.size()) return true;
    }
    return false;
}

// ---------------------------------------------------------------- spf13/cast v1.7.1
// ToInt64E and friends: the value as int64 before the final Go conversion to the target width
inline int cast_to_i64(const GoVal& v, int64_t& out) {
    switch (v.k) {
    case NIL: out = 0; return OK;
    case BOOL: out = v.i ? 1 : 0; return OK;
    case INT: out = v.i; return OK;
    case UINT: out = (int64_t)v.u; return OK;
    case F32: case F64: out = go_f2i64(v.f); return OK;
    case STRING: case JSONNUM: { int64_t x; if (jsn::go_parse_int(trim_zero_decimal(v.s), 0, 64, x)) return CAST_ERR; out = x; return OK; }      // strconv.ParseInt(trimZeroDecimal(s), 0, 0)
    default: return CAST_ERR;      // []byte, time.Time, time.Duration (no case in ToIntE for Duration: reflect kind int64 is not matched by the type switch), maps
    }
}
inline int cast_to_u64(const GoVal& v, uint64_t& out) {      // ToUint64E: negative values are refused
    switch (v.k) {
    case NIL: out = 0; return OK;
    case BOOL: out = v.i ? 1 : 0; return OK;
    case INT: if (v.i < 0) return CAST_ERR; out = (uint64_t)v.i; return OK;
    case UINT: out = v.u; return OK;
    case F32: case F64: if (v.f < 0) return CAST_ERR; out = go_f2u64(v.f); return OK;
    case STRING: case JSONNUM: {
        const std::string t = trim_zero_decimal(v.s);
        uint64_t x; if (jsn::go_parse_uint(t, 0, 64, x) == 0) { out = x; return OK; }      // v1.7.x: ParseUint for the 64-bit target (cast issue #143)
        return CAST_ERR;
    }
    default: return CAST_ERR;
    }
}
// the narrower unsigned targets go through ParseInt and refuse negatives (ToUint8E / 16 / 32)
inline int cast_to_un(const GoVal& v, int bits, uint64_t& out) {
    if (bits == 64) return cast_to_u64(v, out);
    if (v.k == STRING || v.k == JSONNUM) { int64_t x; if (jsn::go_parse_int(trim_zero_decimal(v.s), 0, 64, x)) return CAST_ERR; if (x < 0) return CAST_ERR; out = (uint64_t)x; return OK; }
    return cast_to_u64(v, out);
}
inline int cast_to_f64(const GoVal& v, double& out) {      // ToFloat64E
    switch (v.k) {
    case NIL: out = 0; return OK;
    case BOOL: out = v.i ? 1 : 0; return OK;
    case INT: out = (double)v.i; return OK;
    case UINT: out = (double)v.u; return OK;
    case F32: case F64: out = v.f; return OK;
    case STRING: case JSONNUM: { double f; const int rc = jsn::go_parse_float(v.s, f); if (rc == 1) return CAST_ERR; if (rc == 2) return UNPINNED; out = f; return OK; }
    default: return CAST_ERR;
    }
}
inline int cast_to_bool(const GoVal& v, bool& out) {      // ToBoolE
    switch (v.k) {
    case NIL: out = false; return OK;
    case BOOL: out = v.i != 0; return OK;
    case INT: out = v.i != 0; return OK;
    case UINT: out = v.u != 0; return OK;
    case F32: case F64: out = v.f != 0; return OK;
    case DURATION: out = v.i != 0; return OK;
    case STRING: { bool b; if (orc::go_parse_bool((const uint8_t*)v.s.data(), v.s.size(), b)) return CAST_ERR; out = b; return OK; }
    case JSONNUM: { int64_t x; if (cast_to_i64(v, x)) return CAST_ERR; out = x != 0; return OK; }
    default: return CAST_ERR;
    }
}

// ---------------------------------------------------------------- castx
inline int castx_to_string(const GoVal& v, std::string& out) {      // castx.ToStringE (caste.go:52-106)
    switch (v.k) {
    case NIL: out = ""; return OK;
    case BOOL: out = v.i ? "true" : "false"; return OK;
    case INT: out = orc::fmt_i64(v.i); return OK;
    case UINT: out = orc::fmt_u64(v.u); return OK;
    case F64: out = orc::fmt_f64(v.f, orc::FMT_F); return OK;
    case F32: out = orc::fmt_f32((float)v.f, orc::FMT_F); return OK;
    case STRING: case JSONNUM: out = v.s; return OK;
    case BYTES: out = v.s; return OK;
    case DURATION: out = orc::fmt_duration(v.i); return OK;                       // fmt.Stringer
    case TIME: return UNPINNED;                                                  // time.Time.String() carries the location / monotonic reading
    default: return CAST_ERR;                                                    // maps: cast.ToStringE "unable to cast"
    }
}
inline int castx_to_json_number(const GoVal& v, std::string& out) {      // castx.ToJSONNumberE (caste.go:36-50)
    std::string t; const int rc = castx_to_string(v, t); if (rc) return rc;
    if (ff_parse_ok(t)) { out = t; return OK; }
    int64_t x; if (jsn::go_parse_int(t, 10, 64, x) == 0) { out = t; return OK; }
    return CAST_ERR;
}

// ---------------------------------------------------------------- strictify.go
// strictifyValue: out = the canonical Go value of column type `tf` (TF_* ids of include/tfgpu.h)
inline int strictify_value(const GoVal& v, int tf, GoVal& out) {
    out = GoVal();
    if (v.k == NIL) return OK;                                                    // :55-57
    auto sint = [&](int bits, int64_t lo, int64_t hi) {                           // toSignedInt :159-169
        int64_t x; if (cast_to_i64(v, x)) return (int)CAST_ERR;                   // castFn: ToIntNE = the int64 path + a Go conversion
        int64_t v64 = 0; cast_to_i64(v, v64);                                     // cast.ToInt64(v): errors give 0
        if (v64 < lo || v64 > hi) return (int)RANGE_ERR;
        out.k = INT; out.bits = bits; out.i = x; return (int)OK;
    };
    auto uint_ = [&](int bits, uint64_t hi) {                                     // toUnsignedInt :171-181
        uint64_t x; if (cast_to_un(v, bits, x)) return (int)CAST_ERR;
        uint64_t v64 = 0; cast_to_u64(v, v64);                                    // cast.ToUint64(v)
        if (v64 > hi) return (int)RANGE_ERR;
        out.k = UINT; out.bits = bits; out.u = x; return (int)OK;
    };
    switch (tf) {
    case TF_BOOLEAN: { bool b; if (cast_to_bool(v, b)) return CAST_ERR; out.k = BOOL; out.i = b; return OK; }
    case TF_INT8: return sint(8, INT8_MIN, INT8_MAX);
    case TF_INT16: return sint(16, INT16_MIN, INT16_MAX);
    case TF_INT32: return sint(32, INT32_MIN, INT32_MAX);
    case TF_INT64: return sint(64, INT64_MIN, INT64_MAX);
    case TF_UINT8: return uint_(8, UINT8_MAX);
    case TF_UINT16: return uint_(16, UINT16_MAX);
    case TF_UINT32: return uint_(32, UINT32_MAX);
    case TF_UINT64: return uint_(64, UINT64_MAX);
    case TF_FLOAT: {                                                              // cast.ToFloat32E: strings through ParseFloat(s, 32)
        if (v.k == INT) { out.k = F32; out.f = (double)(float)v.i; return OK; }      // float32(s): one conversion, not two
        if (v.k == UINT) { out.k = F32; out.f = (double)(float)v.u; return OK; }
        if (v.k == STRING) {                                                      // ParseFloat(s, 32): one rounding; a range error is cast's error
            double f; const int rc = jsn::go_parse_float(v.s, f); if (rc) return CAST_ERR;      // syntax, and overflow of float64 itself
            if (!std::isfinite(f)) { out.k = F32; out.f = f; return OK; }                       // inf / infinity / nan spellings
            std::string t = v.s; t.erase(std::remove(t.begin(), t.end(), '_'), t.end());
            const float g = std::strtof(t.c_str(), nullptr); if (std::isinf(g)) return CAST_ERR;
            out.k = F32; out.f = g; return OK;
        }
        double f; const int rc = cast_to_f64(v, f); if (rc) return rc;
        out.k = F32; out.f = (double)(float)f; return OK;
    }
    case TF_DOUBLE: { std::string t; const int rc = castx_to_json_number(v, t); if (rc) return rc; out.k = JSONNUM; out.s = t; return OK; }
    case TF_BYTES: if (v.k == BYTES || v.k == STRING) { out.k = BYTES; out.s = v.s; return OK; } return CAST_ERR;      // castx.ToByteSliceE
    case TF_UTF8: { std::string t; const int rc = castx_to_string(v, t); if (rc) return rc; out.k = STRING; out.s = t; return OK; }
    case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:                            // cast.ToTimeE
        if (v.k == TIME) { out = v; return OK; }
        if (v.k == INT || v.k == UINT) { out.k = TIME; out.i = v.k == INT ? v.i : (int64_t)v.u; return OK; }      // time.Unix(v, 0)
        if (v.k == JSONNUM) { int64_t x; if (cast_to_i64(v, x)) return CAST_ERR; out.k = TIME; out.i = x; return OK; }
        if (v.k == STRING) {
            int64_t sec; uint32_t ns; const int rc = orc::parse_time_iso((const uint8_t*)v.s.data(), v.s.size(), sec, ns);
            if (rc == 0) { out.k = TIME; out.i = sec; out.nsec = ns; return OK; }
            return rc == 2 ? UNPINNED : CAST_ERR;
        }
        return CAST_ERR;
    case TF_INTERVAL:                                                             // cast.ToDurationE
        if (v.k == DURATION) { out = v; return OK; }
        if (v.k == INT) { out.k = DURATION; out.i = v.i; return OK; }
        if (v.k == UINT) { out.k = DURATION; out.i = (int64_t)v.u; return OK; }
        if (v.k == F32 || v.k == F64) { out.k = DURATION; out.i = go_f2i64(v.f); return OK; }
        if (v.k == JSONNUM) { double f; if (cast_to_f64(v, f)) return CAST_ERR; out.k = DURATION; out.i = go_f2i64(f); return OK; }
        if (v.k == STRING) return UNPINNED;                                       // time.ParseDuration
        return CAST_ERR;
    case TF_ANY:                                                                  // castx.ToJSONMarshallableE: json.Marshal refuses NaN / Inf floats
        if ((v.k == F32 || v.k == F64) && !std::isfinite(v.f)) return CAST_ERR;
        out = v; return OK;
    }
    return PANIC;
}

// ---------------------------------------------------------------- restore.go
inline GoVal maybe_string_to_numeric(const GoVal& v) {      // :227-247
    GoVal r;
    auto from_string = [&](const std::string& s) {
        if (s.find('.') != std::string::npos) { double f = 0; jsn::go_parse_float(s, f); r.k = F64; r.f = f; return; }      // errors give 0
        if (!s.empty() && s[0] == '-') { int64_t x = 0; jsn::go_parse_int(s, 10, 64, x); r.k = INT; r.i = x; return; }
        uint64_t u = 0; jsn::go_parse_uint(s, 10, 64, u); r.k = UINT; r.u = u;
    };
    if (v.k == STRING) { from_string(v.s); return r; }
    if (v.k == DURATION) { r.k = INT; r.i = v.i; return r; }
    if (v.k == JSONNUM) { from_string(v.s); return r; }                            // fmt.Stringer
    return v;
}
// Restore for the column types whose result this restatement carries; rc PANIC where the reference panics, UNPINNED for dateparse
inline int restore_value(const GoVal& v, const std::string& data_type, GoVal& out) {
    out = v;
    if (v.k == NIL) return OK;
    if (v.k == TIME) {                                                             // :33-48
        if (data_type == "date" || data_type == "datetime" || data_type == "timestamp") return OK;
        const int64_t unano = v.i * 1000000000LL + v.nsec;
        if (data_type == "int64") { out = GoVal(); out.k = INT; out.i = -unano; return OK; }
        if (data_type == "uint64") { out = GoVal(); out.k = INT; out.i = unano; return OK; }
        if (data_type == "int32") { out = GoVal(); out.k = INT; out.i = -v.i; return OK; }
        if (data_type == "uint32") { out = GoVal(); out.k = INT; out.i = v.i; return OK; }
        if (data_type == "utf8" || data_type == "string" || data_type == "any") { out = GoVal(); out.k = STRING; out.s = orc::fmt_rfc3339nano_utc(v.i, v.nsec); return OK; }
    }
    auto to_int = [&](int bits) {
        const GoVal n = maybe_string_to_numeric(v); int64_t x = 0; cast_to_i64(n, x);      // cast.ToIntN: errors give 0
        out = GoVal(); out.k = INT; out.bits = bits;
        out.i = bits == 8 ? (int64_t)(int8_t)x : bits == 16 ? (int64_t)(int16_t)x : bits == 32 ? (int64_t)(int32_t)x : x; return OK;
    };
    auto to_uint = [&](int bits) {
        const GoVal n = maybe_string_to_numeric(v); uint64_t x = 0; if (cast_to_u64(n, x)) x = 0;
        out = GoVal(); out.k = UINT; out.bits = bits;
        out.u = bits == 8 ? (uint8_t)x : bits == 16 ? (uint16_t)x : bits == 32 ? (uint32_t)x : x; return OK;
    };
    if (data_type == "interval") {
        if (v.k == DURATION) return OK;
        if (v.k == F64) { out = GoVal(); out.k = DURATION; out.i = go_f2i64(v.f); return OK; }
        if (v.k == INT && v.bits == 64) { out = GoVal(); out.k = DURATION; out.i = v.i; return OK; }
        if (v.k == JSONNUM) { int64_t x; out = GoVal(); if (jsn::go_parse_int(v.s, 10, 64, x) == 0) { out.k = DURATION; out.i = x; } else { out.k = INT; out.i = 0; } return OK; }
        return PANIC;
    }
    if (data_type == "date" || data_type == "datetime" || data_type == "timestamp") {
        if (v.k == STRING) {
            int64_t sec; uint32_t ns; const int rc = orc::parse_time_iso((const uint8_t*)v.s.data(), v.s.size(), sec, ns);
            if (rc == 0) { out = GoVal(); out.k = TIME; out.i = sec; out.nsec = ns; return OK; }
            return UNPINNED;                                                       // araddon/dateparse
        }
        if (v.k == INT && v.bits == 64) {                                          // yt schema.Date / Datetime / Timestamp units: days, seconds, microseconds
            out = GoVal(); out.k = TIME;
            if (data_type == "date") out.i = v.i * 86400;
            else if (data_type == "datetime") out.i = v.i;
            else { out.i = orc::floor_div(v.i, 1000000); out.nsec = (uint32_t)((v.i - out.i * 1000000) * 1000); }
            return OK;
        }
        if (v.k == JSONNUM) { int64_t x; if (jsn::go_parse_int(v.s, 10, 64, x) == 0) { GoVal t; t.k = INT; t.bits = 64; t.i = x; return restore_value(t, data_type, out); } out = GoVal(); out.k = INT; out.i = 0; return OK; }
        return PANIC;
    }
    if (data_type == "int64") return to_int(64);
    if (data_type == "int32") return to_int(32);
    if (data_type == "int16") return to_int(16);
    if (data_type == "int8") return to_int(8);
    if (data_type == "uint64") return to_uint(64);
    if (data_type == "uint32") return to_uint(32);
    if (data_type == "uint16") return to_uint(16);
    if (data_type == "uint8") return to_uint(8);
    if (data_type == "double") {
        if (v.k == F32) { out = GoVal(); out.k = F64; out.f = v.f; return OK; }
        if (v.k == F64 || v.k == JSONNUM) return OK;
        if (v.k == STRING) { out = GoVal(); if (v.s.empty()) return OK; double f; const int rc = jsn::go_parse_float(v.s, f); if (rc == 2) return UNPINNED; if (rc == 0) { out.k = F64; out.f = f; } return OK; }
        out = GoVal(); return OK;                                                  // nil for everything else (an int32, a bool ...)
    }
    if (data_type == "boolean") return OK;
    if (data_type == "string" || data_type == "utf8") {                           // no OriginalType
        if (v.k == STRING) return OK;
        if (v.k == BYTES) { out = GoVal(); out.k = STRING; out.s = v.s; return OK; }
        return UNPINNED;                                                           // json.Marshal(value): handled where the value is a JSON tree (oracle.cpp)
    }
    if (data_type == "any") {
        if (v.k != STRING) return OK;
        // tryUnmarshalJSON: a decodable JSON document becomes the decoded value (numbers as json.Number), anything else stays the string
        const std::string& s = v.s; size_t a = 0, b = s.size();
        while (a < b && (s[a] == ' ' || s[a] == '\t' || s[a] == '\n' || s[a] == '\r')) a++;
        while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t' || s[b - 1] == '\n' || s[b - 1] == '\r')) b--;
        const std::string t = s.substr(a, b - a);
        if (!t.empty() && (t[0] == '{' || t[0] == '[')) { out = GoVal(); out.k = MAP; out.s = t; return OK; }
        if (jsn::valid_json_number(t)) { out = GoVal(); out.k = JSONNUM; out.s = t; return OK; }
        return OK;
    }
    return OK;
}

// ---------------------------------------------------------------- splitter.go
// ConsumeRow until EOF: the complete rows and what the last call (io.EOF) wrote
inline void csv_split_rows(const std::string& in, std::vector<std::string>& rows, std::string& eof_rest) {
    enum { OUTSIDE, OPEN, CLOSING } st = OUTSIDE;
    std::string cur;
    for (size_t i = 0; i < in.size(); i++) {
        const char c = in[i]; cur += c;
        switch (st) {
        case OUTSIDE: if (c == '"') st = OPEN; break;
        case OPEN: if (c == '"') st = CLOSING; break;
        case CLOSING: st = c == '"' ? OPEN : OUTSIDE; break;
        }
        if (c == '\n' && st == OUTSIDE) { rows.push_back(cur); cur.clear(); }
    }
    eof_rest = cur;
}

}  // namespace gocast
