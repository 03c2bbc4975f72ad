// ClickHouse JSONEachRow rows on the device.
//   reference: MarshalCItoJSON pkg/providers/clickhouse/httpuploader/marshal.go:88-253 (+ marshalTime :63-78,
//   questionableQuoter :264-266): `{"col":value,...}\n`, schema order, nil columns omitted, strings escape only
//   `\` and `"` (bytes otherwise untouched, non-UTF-8 included), ints/floats bare ('f', -1) unless the target column is
//   String, time by the target ClickHouse type, non-string `any` values as a JSON-quoted string of their JSON text.
// Row text has no fixed width: pass 1 sizes every kept row (CountSink), a tile scan places them, pass 2 writes them.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "kernels_fmt.cuh"
#include "kernels_mask.cuh"
#include "kernels_csv.cuh"

namespace tfk {

enum JsonChClass : int32_t { JC_OTHER = 0, JC_STRING = 1, JC_DATE = 2, JC_DATETIME = 3, JC_DT64 = 4 };
struct JsonCol { int32_t col; int32_t name_off, name_len; int32_t ch_class; int32_t prec; int32_t result_tf; int32_t pad0, pad1; };

template <typename Inner> struct EscSink {     // questionableQuoter: `\` -> `\\`, `"` -> `\"`
    Inner* in;
    __device__ __forceinline__ void put(uint8_t b) { if (b == '\\' || b == '"') in->put('\\'); in->put(b); }
};

template <typename Sink> __device__ __forceinline__ void json_time(Sink& s, int64_t sec, uint32_t nsec, const JsonCol& jc) {
    switch (jc.ch_class) {
    case JC_STRING: {      // v.Format("2006-01-02 15:04:05.999999999 -0700 MST") in UTC
        s.put('"');
        int64_t days = sec / 86400; int64_t sod = sec - days * 86400; if (sod < 0) { sod += 86400; days--; }
        int64_t y; unsigned m, d; civil_from_days_d(days, y, m, d);
        fmt_pad(s, y, 4); s.put('-'); fmt_pad(s, m, 2); s.put('-'); fmt_pad(s, d, 2); s.put(' ');
        fmt_pad(s, sod / 3600, 2); s.put(':'); fmt_pad(s, (sod / 60) % 60, 2); s.put(':'); fmt_pad(s, sod % 60, 2);
        if (nsec) { char b[9]; uint32_t v = nsec; for (int i = 8; i >= 0; i--) { b[i] = (char)('0' + v % 10); v /= 10; } int n = 9; while (n > 0 && b[n - 1] == '0') n--; s.put('.'); for (int i = 0; i < n; i++) s.put((uint8_t)b[i]); }
        fmt_lit(s, " +0000 UTC\""); break;
    }
    case JC_DT64: {        // UnixNano() / 10^(9-p) for 0 < p < 9 (Go integer division: toward zero)
        int64_t full = sec * 1000000000LL + (int64_t)nsec;
        if (jc.prec > 0 && jc.prec < 9) { int64_t div = 1; for (int i = 0; i < 9 - jc.prec; i++) div *= 10; full = full / div; }
        fmt_i64(s, full); break;
    }
    case JC_DATE: s.put('"'); fmt_time(s, sec, 0, true); s.put('"'); break;
    default: fmt_i64(s, sec);
    }
}

// one column's value; returns false when the column is omitted (nil, or a JSON `null`)
template <typename Sink> __device__ bool json_value(Sink& s, const DCol& c, uint64_t r, const JsonCol& jc, const MaskKey* keys, bool sizing) {
    const bool str = jc.ch_class == JC_STRING;
    if (c.out_kind == OK_MASK) {                 // hex digest, a Go string: never nil
        s.put('"');
        if (sizing) { for (int i = 0; i < 64; i++) s.put('0'); }
        else { uint8_t hx[64]; mask_digest_hex(c, r, keys[c.mask_slot], hx); for (int i = 0; i < 64; i++) s.put(hx[i]); }
        s.put('"'); return true;
    }
    if (c.out_kind == OK_TOSTR) { s.put('"'); EscSink<Sink> es{&s}; fmt_value(es, c, r); s.put('"'); return true; }
    if (c.out_kind == OK_TODT) {
        int64_t sec = 0; if (row_valid(c, r)) sec = c.type == TF_INT32 ? (int64_t)((const int32_t*)c.values)[r] : (int64_t)((const uint32_t*)c.values)[r];
        json_time(s, sec, 0, jc); return true;
    }
    if (!row_valid(c, r)) return false;
    switch (c.type) {
    case TF_INT8: if (str) s.put('"'); fmt_i64(s, ((const int8_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_INT16: if (str) s.put('"'); fmt_i64(s, ((const int16_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_INT32: if (str) s.put('"'); fmt_i64(s, ((const int32_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_INT64: if (str) s.put('"'); fmt_i64(s, ((const int64_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_UINT8: if (str) s.put('"'); fmt_u64(s, c.values[r]); if (str) s.put('"'); break;
    case TF_UINT16: if (str) s.put('"'); fmt_u64(s, ((const uint16_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_UINT32: if (str) s.put('"'); fmt_u64(s, ((const uint32_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_UINT64: if (str) s.put('"'); fmt_u64(s, ((const uint64_t*)c.values)[r]); if (str) s.put('"'); break;
    case TF_FLOAT: if (str) s.put('"'); fmt_float_bits(s, ((const uint32_t*)c.values)[r], true, FM_F); if (str) s.put('"'); break;
    case TF_DOUBLE: if (str) s.put('"'); fmt_float_bits(s, ((const uint64_t*)c.values)[r], false, FM_F); if (str) s.put('"'); break;
    case TF_BOOLEAN: fmt_lit(s, c.values[r] ? "true" : "false"); break;           // DataType == boolean (marshal.go:187-192)
    case TF_INTERVAL: {    // json.Marshal(time.Duration) is an integer; a non-`any` column re-marshals that text as a string
        s.put('"'); fmt_i64(s, ((const int64_t*)c.values)[r]); s.put('"'); break;
    }
    case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:
        json_time(s, ((const int64_t*)c.values)[r], c.aux ? ((const uint32_t*)c.aux)[r] : 0, jc); break;
    case TF_BYTES: case TF_UTF8: {
        const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
        s.put('"'); for (uint32_t k = 0; k < L; k++) { const uint8_t b = p[k]; if (b == '\\' || b == '"') s.put('\\'); s.put(b); } s.put('"'); break;
    }
    case TF_ANY: {
        const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
        if (c.aux && c.aux[r] == 1) { s.put('"'); for (uint32_t k = 0; k < L; k++) { const uint8_t b = p[k]; if (b == '\\' || b == '"') s.put('\\'); s.put(b); } s.put('"'); break; }
        if (L == 4 && p[0] == 'n' && p[1] == 'u' && p[2] == 'l' && p[3] == 'l') return false;      // :229-233
        fmt_json_string(s, p, L);      // any -> String column: json.Marshal(string(r)) (:234-239)
        break;
    }
    }
    return true;
}

template <typename Sink> __device__ void json_row(Sink& s, const DCol* cols, const JsonCol* jcols, int njc, const uint8_t* names, const MaskKey* keys, uint64_t r, bool sizing) {
    s.put('{');
    bool first = true;
    for (int k = 0; k < njc; k++) {
        const JsonCol jc = jcols[k]; const DCol& c = cols[jc.col];
        // is the column present? (decide before writing its name)
        bool present;
        if (c.out_kind == OK_MASK || c.out_kind == OK_TOSTR || c.out_kind == OK_TODT) present = true;
        else if (!row_valid(c, r)) present = false;
        else if (c.type == TF_ANY && !(c.aux && c.aux[r] == 1)) { const uint8_t* p = c.heap + c.offsets[r]; present = !((c.offsets[r + 1] - c.offsets[r]) == 4 && p[0] == 'n' && p[1] == 'u' && p[2] == 'l' && p[3] == 'l'); }
        else present = true;
        if (!present) continue;
        if (!first) s.put(',');
        first = false;
        s.put('"'); for (int i = 0; i < jc.name_len; i++) s.put(names[jc.name_off + i]); s.put('"'); s.put(':');
        json_value(s, c, r, jc, keys, sizing);
    }
    s.put('}'); s.put('\n');
}


// ------------------------------------------------------------------ batch serializers (pkg/serializer)
//   JSON: json.go:29-114 buildJsonKV + json.Encoder(SetEscapeHTML(false)) over a map (keys sorted: the host orders jcols and
//         pre-quotes `"name":`), values per json_format.go:32-82 on the canonical (strictified) Go type of the result schema
//   CSV:  csv.go:22-74 + csv_format.go:32-144 cells through encoding/csv (Comma ',', UseCRLF false)
// sink flags
#define TF_SER_NL 1u        /* AddClosingNewLine */
#define TF_SER_AAS 2u       /* AnyAsString */

template <typename Inner> struct B64Sink {       // base64.StdEncoding over a byte stream
    Inner* in; uint32_t acc; int n;
    __device__ __forceinline__ static uint8_t a(uint32_t v) { return (uint8_t)(v < 26 ? 'A' + v : v < 52 ? 'a' + v - 26 : v < 62 ? '0' + v - 52 : v == 62 ? '+' : '/'); }
    __device__ __forceinline__ void put(uint8_t b) { acc = (acc << 8) | b; if (++n == 3) { in->put(a(acc >> 18)); in->put(a((acc >> 12) & 63)); in->put(a((acc >> 6) & 63)); in->put(a(acc & 63)); acc = 0; n = 0; } }
    __device__ __forceinline__ void finish() {
        if (n == 1) { acc <<= 16; in->put(a(acc >> 18)); in->put(a((acc >> 12) & 63)); in->put('='); in->put('='); }
        else if (n == 2) { acc <<= 8; in->put(a(acc >> 18)); in->put(a((acc >> 12) & 63)); in->put(a((acc >> 6) & 63)); in->put('='); }
    }
};
template <typename Inner> struct CsvQuoteSink { Inner* in; __device__ __forceinline__ void put(uint8_t b) { if (b == '"') in->put('"'); in->put(b); } };

template <typename Sink> __device__ void ser_time_string(Sink& s, int64_t sec, uint32_t nsec) {     // Time.String() in UTC
    int64_t days = sec / 86400; int64_t sod = sec - days * 86400; if (sod < 0) { sod += 86400; days--; }
    int64_t y; unsigned m, d; civil_from_days_d(days, y, m, d);
    fmt_pad(s, y, 4); s.put('-'); fmt_pad(s, m, 2); s.put('-'); fmt_pad(s, d, 2); s.put(' ');
    fmt_pad(s, sod / 3600, 2); s.put(':'); fmt_pad(s, (sod / 60) % 60, 2); s.put(':'); fmt_pad(s, sod % 60, 2);
    if (nsec) { char b[9]; uint32_t v = nsec; for (int i = 8; i >= 0; i--) { b[i] = (char)('0' + v % 10); v /= 10; } int n = 9; while (n > 0 && b[n - 1] == '0') n--; s.put('.'); for (int i = 0; i < n; i++) s.put((uint8_t)b[i]); }
    fmt_lit(s, " +0000 UTC");
}
// JSON text written by json.Marshal (HTML escaping on) as a SetEscapeHTML(false) encoder writes the same value
template <typename Sink> __device__ void ser_unescape_html(Sink& s, const uint8_t* p, uint32_t n) {
    bool ins = false;
    for (uint32_t i = 0; i < n;) {
        const uint8_t c = p[i];
        if (!ins) { if (c == '"') ins = true; s.put(c); i++; continue; }
        if (c == '\\' && i + 1 < n) {
            if (p[i + 1] == 'u' && i + 5 < n && p[i + 2] == '0' && p[i + 3] == '0' && ((p[i + 4] == '3' && (p[i + 5] == 'c' || p[i + 5] == 'e')) || (p[i + 4] == '2' && p[i + 5] == '6'))) {
                s.put(p[i + 4] == '2' ? '&' : p[i + 5] == 'c' ? '<' : '>'); i += 6; continue;
            }
            s.put(c); s.put(p[i + 1]); i += 2; continue;
        }
        if (c == '"') ins = false;
        s.put(c); i++;
    }
}

// one JSON value; false = encoding/json would fail (NaN / Inf, year outside [0, 9999]) and `null` stands in
template <typename Sink> __device__ bool ser_json_value(Sink& s, const DCol& c, uint64_t r, const JsonCol& jc, const MaskKey* keys, bool sizing, uint32_t flags) {
    if (c.out_kind == OK_MASK) {
        s.put('"');
        if (sizing) { for (int i = 0; i < 64; i++) s.put('0'); }
        else { uint8_t hx[64]; mask_digest_hex(c, r, keys[c.mask_slot], hx); for (int i = 0; i < 64; i++) s.put(hx[i]); }
        s.put('"'); return true;
    }
    if (c.out_kind == OK_TOSTR) {                 // text of the value: a Go string (utf8) or []byte (string) cell
        s.put('"');
        if (jc.result_tf == TF_BYTES) { B64Sink<Sink> b{&s, 0, 0}; fmt_value(b, c, r); b.finish(); }
        else fmt_value(s, c, r);                  // numbers, times, "<nil>": ASCII (text cells are written by ser_json_row)
        s.put('"'); return true;
    }
    if (c.out_kind == OK_TODT) {
        int64_t sec = 0; if (row_valid(c, r)) sec = c.type == TF_INT32 ? (int64_t)((const int32_t*)c.values)[r] : (int64_t)((const uint32_t*)c.values)[r];
        s.put('"'); fmt_time(s, sec, 0, false); s.put('"'); return true;
    }
    if (!row_valid(c, r)) { fmt_lit(s, "null"); return true; }
    switch (c.type) {
    case TF_INT8: fmt_i64(s, ((const int8_t*)c.values)[r]); break;
    case TF_INT16: fmt_i64(s, ((const int16_t*)c.values)[r]); break;
    case TF_INT32: fmt_i64(s, ((const int32_t*)c.values)[r]); break;
    case TF_INT64: case TF_INTERVAL: fmt_i64(s, ((const int64_t*)c.values)[r]); break;
    case TF_UINT8: fmt_u64(s, c.values[r]); break;
    case TF_UINT16: fmt_u64(s, ((const uint16_t*)c.values)[r]); break;
    case TF_UINT32: fmt_u64(s, ((const uint32_t*)c.values)[r]); break;
    case TF_UINT64: fmt_u64(s, ((const uint64_t*)c.values)[r]); break;
    case TF_FLOAT: { const uint32_t b = ((const uint32_t*)c.values)[r]; if ((b & 0x7F800000u) == 0x7F800000u) { fmt_lit(s, "null"); return false; } fmt_float_bits(s, b, true, FM_JSON); break; }
    case TF_DOUBLE: { const uint64_t b = ((const uint64_t*)c.values)[r]; if ((b & 0x7FF0000000000000ull) == 0x7FF0000000000000ull) { fmt_lit(s, "null"); return false; } fmt_float_bits(s, b, false, FM_F); break; }
    case TF_BOOLEAN: fmt_lit(s, c.values[r] ? "true" : "false"); break;
    case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP: {
        const int64_t sec = ((const int64_t*)c.values)[r];
        if (sec < -62167219200LL || sec >= 253402300800LL) { fmt_lit(s, "null"); return false; }
        s.put('"'); fmt_time(s, sec, c.aux ? ((const uint32_t*)c.aux)[r] : 0, false); s.put('"'); break;
    }
    case TF_UTF8: fmt_json_string(s, c.heap + c.offsets[r], c.offsets[r + 1] - c.offsets[r], false); break;
    case TF_BYTES: { s.put('"'); B64Sink<Sink> b{&s, 0, 0}; const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r]; for (uint32_t k = 0; k < L; k++) b.put(p[k]); b.finish(); s.put('"'); break; }
    case TF_ANY: {
        const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
        const bool gostr = c.aux && c.aux[r] == 1, aas = flags & TF_SER_AAS;
        if (gostr && aas) { s.put('"'); EscSink<Sink> es{&s}; fmt_json_string(es, p, L, true); s.put('"'); }     // string(json.Marshal(v)) re-encoded
        else if (gostr || aas) fmt_json_string(s, p, L, false);
        else ser_unescape_html(s, p, L);
        break;
    }
    }
    return true;
}

template <typename Sink> __device__ int ser_json_row(Sink& s, const DCol* cols, const JsonCol* jcols, int njc, const uint8_t* names, const MaskKey* keys, uint64_t r, uint64_t j, bool sizing, uint32_t flags) {
    int bad = -1;
    if (!(flags & TF_SER_NL) && j) s.put('\n');               // items joined by "\n" (batch_factory.go:36-39)
    s.put('{');
    for (int k = 0; k < njc; k++) {
        const JsonCol jc = jcols[k]; const DCol& c = cols[jc.col];
        if (k) s.put(',');
        for (int i = 0; i < jc.name_len; i++) s.put(names[jc.name_off + i]);       // `"name":` quoted on the host
        if (c.out_kind == OK_TOSTR && jc.result_tf != TF_BYTES && (c.type == TF_UTF8 || c.type == TF_BYTES) && row_valid(c, r))
            fmt_json_string(s, c.heap + c.offsets[r], c.offsets[r + 1] - c.offsets[r], false);      // convert_to_string of a text cell: the same bytes
        else if (!ser_json_value(s, c, r, jc, keys, sizing, flags) && bad < 0) bad = jc.pad0;
    }
    s.put('}');
    if (flags & TF_SER_NL) s.put('\n');
    return bad;
}

// does the encoding/csv field need quotes? (fieldNeedsQuotes: empty no; `\.` yes; , " \r \n yes; leading unicode space yes)
static __device__ bool ser_csv_needs_quotes(const uint8_t* p, uint32_t n) {
    if (!n) return false;
    if (n == 2 && p[0] == '\\' && p[1] == '.') return true;
    for (uint32_t i = 0; i < n; i++) { const uint8_t c = p[i]; if (c == '\n' || c == '\r' || c == '"' || c == ',') return true; }
    uint32_t w; return d_space(p, n, w);
}

template <typename Sink> __device__ void ser_csv_row(Sink& s, const DCol* cols, const JsonCol* jcols, int njc, const MaskKey* keys, uint64_t r, bool sizing) {
    for (int k = 0; k < njc; k++) {
        const JsonCol jc = jcols[k]; const DCol& c = cols[jc.col];
        if (k) s.put(',');
        if (c.out_kind == OK_MASK) {
            if (sizing) { for (int i = 0; i < 64; i++) s.put('0'); }
            else { uint8_t hx[64]; mask_digest_hex(c, r, keys[c.mask_slot], hx); for (int i = 0; i < 64; i++) s.put(hx[i]); }
            continue;
        }
        if (c.out_kind == OK_TODT) { int64_t sec = 0; if (row_valid(c, r)) sec = c.type == TF_INT32 ? (int64_t)((const int32_t*)c.values)[r] : (int64_t)((const uint32_t*)c.values)[r]; ser_time_string(s, sec, 0); continue; }
        const bool tostr = c.out_kind == OK_TOSTR;
        if (tostr && jc.result_tf == TF_BYTES) { B64Sink<Sink> b{&s, 0, 0}; fmt_value(b, c, r); b.finish(); continue; }
        if (!row_valid(c, r)) { if (tostr) fmt_value(s, c, r); continue; }      // nil -> "" ; convert_to_string of nil is "<nil>" / "null"
        switch (c.type) {
        case TF_FLOAT: fmt_float_bits(s, ((const uint32_t*)c.values)[r], true, FM_F); break;
        case TF_DOUBLE: fmt_float_bits(s, ((const uint64_t*)c.values)[r], false, FM_F); break;
        case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:
            if (tostr) fmt_value(s, c, r); else ser_time_string(s, ((const int64_t*)c.values)[r], c.aux ? ((const uint32_t*)c.aux)[r] : 0);
            break;
        case TF_BYTES: if (!tostr) { B64Sink<Sink> b{&s, 0, 0}; const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r]; for (uint32_t i = 0; i < L; i++) b.put(p[i]); b.finish(); break; }
        // fall through: convert_to_string of bytes is the raw text
        case TF_UTF8: {
            const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
            if (ser_csv_needs_quotes(p, L)) { s.put('"'); for (uint32_t i = 0; i < L; i++) { if (p[i] == '"') s.put('"'); s.put(p[i]); } s.put('"'); }
            else for (uint32_t i = 0; i < L; i++) s.put(p[i]);
            break;
        }
        case TF_ANY: {
            const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
            if (c.aux && c.aux[r] == 1) { s.put('"'); CsvQuoteSink<Sink> q{&s}; fmt_json_string(q, p, L, true); s.put('"'); }     // json.Marshal(string) always holds a quote
            else if (ser_csv_needs_quotes(p, L)) { s.put('"'); for (uint32_t i = 0; i < L; i++) { if (p[i] == '"') s.put('"'); s.put(p[i]); } s.put('"'); }
            else for (uint32_t i = 0; i < L; i++) s.put(p[i]);
            break;
        }
        default: fmt_value(s, c, r);       // ints, bool, interval (Duration.String()): never quoted
        }
    }
    s.put('\n');
}

// ------------------------------------------------------------------ Debezium emitter (pkg/debezium), common path
//   Emitter.EmitKV emitter_value_converter.go:626-690 for INSERT rows: key message then value message. Everything that does not
//   change per row (envelope keys, `source` constants, schema wrapper / confluent prefix) is a host-built template of text
//   segments; a segment's code names the per-row piece that follows its text. Values: addCommon emitter_common.go:67-180.
__device__ __forceinline__ uint32_t sink_count(const CountSink& s) { return s.n; }
__device__ __forceinline__ uint32_t sink_count(const MemSink&) { return 0; }
__device__ __forceinline__ uint32_t sink_count(const WordSink&) { return 0; }
enum DbzCode : int32_t { DZ_NONE = 0, DZ_AFTER = 1, DZ_KEY = 2, DZ_LSN = 3, DZ_SRC_TS = 4, DZ_ID = 5, DZ_FILE = 6, DZ_POS = 7, DZ_GTID = 8, DZ_TS = 9, DZ_KEY_END = 10, DZ_BEFORE = 11, DZ_OP = 12 };
struct DbzSeg { int32_t text_off, text_len, code, pad; };
struct DbzEmitArgs {
    const DbzSeg* segs; int nseg; const uint8_t* text; const JsonCol* kcols; int nkc; const JsonCol* acols;     // acols: the sorted columns with their AddPg branch in pad1
    const uint32_t* id; const uint64_t* lsn; const uint64_t* ct; const uint32_t* gt_off; const uint8_t* gt_heap; uint32_t* key_size;
    // update / delete events (emitter_value_converter.go:626-674): ChangeItem.Kind per row and ChangeItem.OldKeys as a second set of columns
    const uint8_t* kinds;          // NULL = all insert
    const DCol* old_cols;          // OldKeys.KeyValues as typed cells, one DCol per input column (NULL: no row carries OldKeys)
    const uint8_t* old_present;    // per input column: the column is listed in OldKeys.KeyNames
    const uint8_t* old_has;        // per row: OldKeys.KeyNames is not empty (NULL: true for every update / delete row)
    int32_t n_old_present, n_pkeys, tombstones, mysql_src, snapshot;
    uint32_t* msg_size;            // [7 per output row]: message count, then (key bytes, value bytes | 0xFFFFFFFF for a tombstone) per message
};
template <typename Inner> struct JStrSink {      // the inside of a JSON string over text that is already valid JSON (ASCII escapes, UTF-8 intact)
    Inner* in;
    __device__ __forceinline__ void put(uint8_t b) {
        if (b >= 0x20 && b != '"' && b != '\\') { in->put(b); return; }
        in->put('\\');
        switch (b) {
        case '\\': case '"': in->put(b); break;
        case '\b': in->put('b'); break; case '\f': in->put('f'); break; case '\n': in->put('n'); break; case '\r': in->put('r'); break; case '\t': in->put('t'); break;
        default: { const char* hex = "0123456789abcdef"; in->put('u'); in->put('0'); in->put('0'); in->put((uint8_t)hex[b >> 4]); in->put((uint8_t)hex[b & 15]); }
        }
    }
};
// AddPg branches (pkg/debezium/pg/emitter.go:265-629) for columns that carry a pg: original type; jc.pad1 = branch, 0 = addCommon
enum DbzForm : int32_t { DF_COMMON = 0, DF_PG_REAL = 2, DF_PG_DOUBLE = 3, DF_PG_STRING = 4, DF_PG_JSON = 6, DF_PG_DATE = 7, DF_PG_TS_MICROS = 8, DF_PG_TS_MILLIS = 9, DF_PG_TSTZ = 10, DF_PG_INET = 11 };
template <typename Sink> __device__ bool dbz_pg_value(Sink& s, const DCol& c, uint64_t r, int form) {
    if (!row_valid(c, r)) { fmt_lit(s, "null"); return true; }                       // :266-269
    const uint8_t* p = nullptr; uint32_t L = 0; bool gostr = false;
    if (c.type == TF_UTF8 || c.type == TF_ANY || c.type == TF_BYTES) {
        p = c.heap + c.offsets[r]; L = c.offsets[r + 1] - c.offsets[r]; gostr = c.type != TF_ANY || (c.aux && c.aux[r] == 1);
        if (!gostr && L == 4 && p[0] == 'n' && p[1] == 'u' && p[2] == 'l' && p[3] == 'l') { fmt_lit(s, "null"); return true; }   // a nil interface inside `any`
    }
    switch (form) {
    case DF_PG_REAL: {                                                               // :342-356 float32(t)
        const float f = c.type == TF_FLOAT ? ((const float*)c.values)[r] : (float)((const double*)c.values)[r];
        const uint32_t b = __float_as_uint(f);
        if ((b & 0x7F800000u) == 0x7F800000u) { fmt_lit(s, "null"); return false; }
        fmt_float_bits(s, b, true, FM_JSON); return true;
    }
    case DF_PG_DOUBLE: {                                                             // :357-370 convertFloatNanInf
        const uint64_t b = ((const uint64_t*)c.values)[r];
        if ((b & 0x7FF0000000000000ull) == 0x7FF0000000000000ull) { fmt_lit(s, (b & 0x000FFFFFFFFFFFFFull) ? "\"NaN\"" : (b >> 63) ? "\"-Infinity\"" : "\"Infinity\""); return true; }
        fmt_float_bits(s, b, false, FM_JSON); return true;
    }
    case DF_PG_STRING:                                                               // colVal.(string)
        if (gostr) { fmt_json_string(s, p, L, false); return true; }
        if (L && p[0] == '"') { ser_unescape_html(s, p, L); return true; }
        fmt_lit(s, "null"); return false;
    case DF_PG_INET:                                                                 // :401-410 strings.TrimSuffix(t, "/32")
        if (!gostr) { fmt_lit(s, "null"); return false; }
        if (L >= 3 && p[L - 3] == '/' && p[L - 2] == '3' && p[L - 1] == '2') L -= 3;
        fmt_json_string(s, p, L, false); return true;
    case DF_PG_JSON:                                                                 // :377-382 string(JSONMarshalUnescape(colVal))
        s.put('"');
        { JStrSink<Sink> js{&s}; if (gostr) fmt_json_string(js, p, L, false); else ser_unescape_html(js, p, L); }
        s.put('"'); return true;
    case DF_PG_DATE: fmt_i64(s, ((const int64_t*)c.values)[r] / 86400); return true;                       // :476-478
    case DF_PG_TS_MICROS: case DF_PG_TS_MILLIS: {                                    // :558-580 UnixMicro() / divider
        const int64_t micro = ((const int64_t*)c.values)[r] * 1000000LL + (int64_t)((c.aux ? ((const uint32_t*)c.aux)[r] : 0u) / 1000u);
        fmt_i64(s, form == DF_PG_TS_MILLIS ? micro / 1000 : micro); return true;
    }
    case DF_PG_TSTZ:                                                                 // :581-594 SprintfDebeziumTime
        s.put('"'); fmt_time(s, ((const int64_t*)c.values)[r], c.aux ? ((const uint32_t*)c.aux)[r] : 0, false); s.put('"'); return true;
    }
    fmt_lit(s, "null"); return false;
}
template <typename Sink> __device__ bool dbz_json_value(Sink& s, const DCol& c, uint64_t r, const JsonCol& jc, const MaskKey* keys, bool sizing) {
    if (jc.pad1 != DF_COMMON) return dbz_pg_value(s, c, r, jc.pad1);              // (the plan refuses pg-typed columns a transformer rewrote)
    if (c.out_kind != OK_MASK && c.out_kind != OK_TOSTR && c.out_kind != OK_TODT) {      // the value keeps its input type (the sink cast kinds do not apply)
        if (!row_valid(c, r)) { fmt_lit(s, "null"); return true; }
        switch (c.type) {
        case TF_DATE: case TF_INTERVAL: fmt_lit(s, "null"); return false;            // emitter_common.go:161-163 unknown input data type
        case TF_DOUBLE: { const uint64_t b = ((const uint64_t*)c.values)[r]; if ((b & 0x7FF0000000000000ull) == 0x7FF0000000000000ull) { fmt_lit(s, "null"); return false; } fmt_float_bits(s, b, false, FM_JSON); return true; }
        case TF_ANY: {
            const uint8_t* p = c.heap + c.offsets[r]; const uint32_t L = c.offsets[r + 1] - c.offsets[r];
            if (c.aux && c.aux[r] == 1) { fmt_json_string(s, p, L, false); return true; }
            if (L == 4 && p[0] == 'n' && p[1] == 'u' && p[2] == 'l' && p[3] == 'l') { fmt_lit(s, "null"); return true; }
            if (L && p[0] == '"') { ser_unescape_html(s, p, L); return true; }
            if (L && p[0] == '{') { s.put('"'); JStrSink<Sink> js{&s}; ser_unescape_html(js, p, L); s.put('"'); return true; }
            fmt_lit(s, "null"); return false;                                        // :157-159 arrays / numbers / booleans
        }
        default: break;
        }
    }
    return ser_json_value(s, c, r, jc, keys, sizing, 0);
}
template <typename Sink> __device__ int dbz_object(Sink& s, const DCol* cols, const JsonCol* jcols, int njc, const uint8_t* names, const MaskKey* keys, uint64_t r, bool sizing) {
    int bad = -1;
    s.put('{');
    for (int k = 0; k < njc; k++) {
        const JsonCol jc = jcols[k]; const DCol& c = cols[jc.col];
        if (k) s.put(',');
        for (int i = 0; i < jc.name_len; i++) s.put(names[jc.name_off + i]);
        if (c.out_kind == OK_TOSTR && jc.result_tf != TF_BYTES && (c.type == TF_UTF8 || c.type == TF_BYTES) && row_valid(c, r))
            fmt_json_string(s, c.heap + c.offsets[r], c.offsets[r + 1] - c.offsets[r], false);
        else if (!dbz_json_value(s, c, r, jc, keys, sizing) && bad < 0) bad = jc.pad0;
    }
    s.put('}');
    return bad;
}
// before / key objects from OldKeys: mode 0 = only the listed columns (makeValues over OldKeys.KeyNames), mode 1 = every column, the
// listed ones from OldKeys and the others null (valPayload op "d": :461-483; a mysql source fills them from ColumnValues first)
template <typename Sink> __device__ int dbz_object_old(Sink& s, const DCol* cols, const DCol* old_cols, const uint8_t* present, const JsonCol* jcols, int njc,
                                                      const uint8_t* names, const MaskKey* keys, uint64_t r, bool sizing, int mode, bool mysql) {
    int bad = -1; bool first = true;
    s.put('{');
    for (int k = 0; k < njc; k++) {
        const JsonCol jc = jcols[k]; const bool pr = present && present[jc.col];
        if (mode == 0 && !pr) continue;
        if (!first) s.put(','); first = false;
        for (int i = 0; i < jc.name_len; i++) s.put(names[jc.name_off + i]);
        if (pr) { if (!dbz_json_value(s, old_cols[jc.col], r, jc, keys, sizing) && bad < 0) bad = jc.pad0; }
        else if (mysql) { if (!dbz_json_value(s, cols[jc.col], r, jc, keys, sizing) && bad < 0) bad = jc.pad0; }
        else fmt_lit(s, "null");
    }
    s.put('}');
    return bad;
}
// reflect.DeepEqual of a typed cell in two columns of the same type
__device__ __forceinline__ bool dbz_cell_equal(const DCol& a, const DCol& b, uint64_t r) {
    const bool va = row_valid(a, r), vb = row_valid(b, r);
    if (va != vb) return false;
    if (!va) return true;
    if (a.in_w) {
        const uint8_t* x = a.values + (size_t)a.in_w * r; const uint8_t* y = b.values + (size_t)b.in_w * r;
        for (int i = 0; i < a.in_w; i++) if (x[i] != y[i]) return false;
        if (a.aux && b.aux && (a.type == TF_TIMESTAMP || a.type == TF_DATETIME || a.type == TF_DATE) && ((const uint32_t*)a.aux)[r] != ((const uint32_t*)b.aux)[r]) return false;
        return true;
    }
    const uint32_t la = a.offsets[r + 1] - a.offsets[r], lb = b.offsets[r + 1] - b.offsets[r];
    if (la != lb) return false;
    const uint8_t* x = a.heap + a.offsets[r]; const uint8_t* y = b.heap + b.offsets[r];
    for (uint32_t i = 0; i < la; i++) if (x[i] != y[i]) return false;
    return true;
}
// One ChangeItem -> 1..3 Debezium messages (Emitter.emitKV :626-674): insert and plain update = one message; delete = the delete event and
// its tombstone (key, no value); an update that changes the primary key = delete event, tombstone, insert event.
template <typename Sink> __device__ int dbz_row(Sink& s, const DCol* cols, const JsonCol* jcols, int njc, const uint8_t* names, const MaskKey* keys,
                                               const DbzEmitArgs& z, uint64_t r, uint64_t j, bool sizing) {
    int bad = -1;
    const uint64_t lsn = z.lsn ? z.lsn[r] : 0, ct = z.ct ? z.ct[r] : 0;
    const int kind = z.kinds ? z.kinds[r] : TF_KIND_INSERT;
    const bool old_row = z.old_cols && kind != TF_KIND_INSERT && (z.old_has ? z.old_has[r] != 0 : true);      // len(OldKeys.KeyNames) > 0
    bool changed = false;
    if (kind == TF_KIND_UPDATE)                                                    // ChangeItem.KeysChanged change_item.go:235-284
        for (int k = 0; k < z.nkc && !changed; k++) {
            const int c = z.kcols[k].col;
            if (old_row && z.old_present[c]) changed = !dbz_cell_equal(z.old_cols[c], cols[c], r);
            else changed = row_valid(cols[c], r);                                  // a key OldKeys does not list compares as nil
        }
    // message plan: 0 regular, 1 delete event, 2 tombstone, 3 insert event
    int plan[3], np = 0;
    if (changed) { plan[np++] = 1; if (z.tombstones) plan[np++] = 2; plan[np++] = 3; }
    else if (kind == TF_KIND_DELETE) { plan[np++] = 1; if (z.tombstones) plan[np++] = 2; }
    else plan[np++] = 0;
    if (sizing && z.msg_size) z.msg_size[7 * j] = (uint32_t)np;
    const bool has_prev = old_row && z.n_old_present > z.n_pkeys;                  // hasPreviousValues :277-285
    for (int m = 0; m < np; m++) {
        const int mt = plan[m];
        const bool key_from_after = mt == 3 || !old_row;                            // makeKey :259-274
        const char op = mt == 1 ? 'd' : (mt == 3 ? 'c' : (kind == TF_KIND_UPDATE ? 'u' : (kind == TF_KIND_DELETE ? 'd' : (z.snapshot ? 'r' : 'c'))));      // kindToOp kind.go:8-31
        const uint32_t at0 = sink_count(s);
        uint32_t key_len = 0;
        for (int g = 0; g < z.nseg; g++) {
            const DbzSeg sg = z.segs[g];
            for (int i = 0; i < sg.text_len; i++) s.put(z.text[sg.text_off + i]);
            switch (sg.code) {
            case DZ_AFTER:
                if (op == 'd') fmt_lit(s, "null");
                else { const int b = dbz_object(s, cols, z.acols, njc, names, keys, r, sizing); if (bad < 0) bad = b; }
                break;
            case DZ_BEFORE:
                if (op == 'd') { const int b = dbz_object_old(s, cols, z.old_cols, old_row ? z.old_present : nullptr, z.acols, njc, names, keys, r, sizing, 1, z.mysql_src != 0); if (bad < 0) bad = b; }
                else if (op == 'u' && has_prev) { const int b = dbz_object_old(s, cols, z.old_cols, z.old_present, z.acols, njc, names, keys, r, sizing, 0, false); if (bad < 0) bad = b; }
                else fmt_lit(s, "null");
                break;
            case DZ_OP: s.put((uint8_t)op); break;
            case DZ_KEY:
                if (key_from_after) { const int b = dbz_object(s, cols, z.kcols, z.nkc, names, keys, r, sizing); if (bad < 0) bad = b; }
                else { const int b = dbz_object_old(s, cols, z.old_cols, z.old_present, z.kcols, z.nkc, names, keys, r, sizing, 0, false); if (bad < 0) bad = b; }
                break;
            case DZ_LSN: fmt_u64(s, lsn); break;
            case DZ_SRC_TS: fmt_u64(s, ct / 1000000ull); break;
            case DZ_ID: fmt_u64(s, z.id ? z.id[r] : 0); break;
            case DZ_FILE: { const uint64_t f = lsn / 1000000000000ull; fmt_pad(s, (int64_t)f, 6); break; }      // "mysql-log.%06d"
            case DZ_POS: fmt_u64(s, lsn % 1000000000000ull); break;
            case DZ_GTID: {
                const uint32_t a = z.gt_off ? z.gt_off[r] : 0, b = z.gt_off ? z.gt_off[r + 1] : 0;
                if (z.gt_heap && b > a) fmt_json_string(s, z.gt_heap + a, b - a, false); else fmt_lit(s, "null");
                break;
            }
            case DZ_TS: fmt_i64(s, (int64_t)ct / 1000000); break;
            case DZ_KEY_END:
                key_len = sink_count(s) - at0;
                if (sizing && m == 0) z.key_size[j] = key_len;
                break;
            default: break;
            }
            if (sg.code == DZ_KEY_END && mt == 2) break;                            // a tombstone is its key only
        }
        if (sizing && z.msg_size) { z.msg_size[7 * j + 1 + 2 * m] = key_len; z.msg_size[7 * j + 2 + 2 * m] = mt == 2 ? 0xffffffffu : sink_count(s) - at0 - key_len; }
    }
    return bad;
}

struct JsonArgs {
    const DCol* cols; const JsonCol* jcols; int njc; const uint8_t* names; const MaskKey* keys;
    const uint32_t* sel; DState* st; uint8_t* raw; uint32_t* row_size; uint32_t* tile_sum; const uint64_t* tile_base; const uint64_t* col_bytes;
    int mode; uint32_t flags; uint8_t* errcode; uint16_t* errstep;     // mode 0 ClickHouse JSONEachRow, 1 serializer JSON, 2 serializer CSV, 3 Debezium messages
    DbzEmitArgs dz;
};

template <typename Sink> __device__ __forceinline__ int json_any_row(Sink& s, const JsonArgs& a, uint64_t r, uint64_t j, bool sizing) {
    if (a.mode == 1) return ser_json_row(s, a.cols, a.jcols, a.njc, a.names, a.keys, r, j, sizing, a.flags);
    if (a.mode == 2) { ser_csv_row(s, a.cols, a.jcols, a.njc, a.keys, r, sizing); return -1; }
    if (a.mode == 3) return dbz_row(s, a.cols, a.jcols, a.njc, a.names, a.keys, a.dz, r, j, sizing);
    json_row(s, a.cols, a.jcols, a.njc, a.names, a.keys, r, sizing); return -1;
}

#define TF_JSON_TILE 256

__global__ void k_json_sizes(JsonArgs a);
#ifdef TF_KERNELS_JSON_OUT
__global__ void __launch_bounds__(TF_JSON_TILE) k_json_sizes(JsonArgs a) {
    __shared__ uint32_t sm[33];
    const uint64_t n = a.st->n_kept;
    const uint64_t j = (uint64_t)blockIdx.x * TF_JSON_TILE + threadIdx.x;
    if ((uint64_t)blockIdx.x * TF_JSON_TILE >= n) return;
    uint32_t sz = 0;
    if (j < n) {
        const uint64_t r = a.sel ? a.sel[j] : j; CountSink cs; cs.n = 0;
        const int bad = json_any_row(cs, a, r, j, true); sz = cs.n; a.row_size[j] = sz;
        if (bad >= 0) { a.errcode[r] = TF_ROWERR_SER_VALUE; a.errstep[r] = (uint16_t)bad; atomicAdd((unsigned long long*)&a.st->n_errors, 1ull); }
    }
    uint32_t tot; block_excl_scan(sz, &tot, sm);
    if (threadIdx.x == 0) a.tile_sum[blockIdx.x] = tot;
}
#endif  // TF_KERNELS_JSON_OUT

__global__ void k_json_write(JsonArgs a);
#ifdef TF_KERNELS_JSON_OUT
__global__ void __launch_bounds__(TF_JSON_TILE) k_json_write(JsonArgs a) {
    __shared__ uint32_t sm[33];
    const uint64_t n = a.st->n_kept;
    if (blockIdx.x == 0 && threadIdx.x == 0) { a.st->raw_total = n ? a.col_bytes[0] : 0; a.st->n_frames = 0; }
    const uint64_t j = (uint64_t)blockIdx.x * TF_JSON_TILE + threadIdx.x;
    if ((uint64_t)blockIdx.x * TF_JSON_TILE >= n) return;
    const uint32_t sz = j < n ? a.row_size[j] : 0;
    uint32_t tot; const uint32_t ex = block_excl_scan(sz, &tot, sm);
    if (j >= n) return;
    const uint64_t r = a.sel ? a.sel[j] : j;
    WordSink ms(a.raw + a.tile_base[blockIdx.x] + ex);
    json_any_row(ms, a, r, j, false);
    ms.flush();
}
#endif  // TF_KERNELS_JSON_OUT

}  // namespace tfk
