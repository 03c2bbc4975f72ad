// Host-side plan builder: the per-table, per-schema-hash "transformation plan" of the
// reference (pkg/transformer/transformation.go:46-85 AddTablePlan: Suitable() -> ResultSchema()
// chain), compiled into flat device programs.  Config-time only.
//
// Mirrors, for the transformers on the hot path:
//   filter_rows        pkg/transformer/registry/filter_rows/filter_rows.go:41-97,445-519
//     filter grammar   library/go/yandex/cloud/filter/grammar/grammar.go:256-313,
//                      library/go/yandex/cloud/filter/filters.go:237-313
//   mask_field         pkg/transformer/registry/mask/mask.go:20-67, hmac_hasher.go:35-47,76-89
//   table matching     pkg/transformer/registry/filter/filter.go:27-74, transformer_common.go:9-33,
//                      pkg/abstract/changeitem/table_id.go:14-30
//   ClickHouse types   pkg/providers/clickhouse/columntypes/types.go:210-248, sink_table.go:196-235
#pragma once
#include <cerrno>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <regex>
#include "host_regex.hpp"
#include <stdexcept>
#include <string>
#include <vector>
#include "json_min.hpp"
#include "../../include/tfgpu.h"

namespace tfplan {

struct FatalError : std::runtime_error { int code; FatalError(int c, const std::string& m) : std::runtime_error(m), code(c) {} };

// ------------------------------------------------------------------ schema
struct ColSchema {
    std::string table_schema, table_name, path, name, type, expression, original_type;
    bool key = false, fake_key = false, required = false;
    int tf = 0;
    int in_index = -1;      // position in the INPUT batch (filter_columns drops columns, it never reorders them)
};

inline int yt_to_tf(const std::string& t) {
    static const std::pair<const char*, int> m[] = {
        {"int8", TF_INT8}, {"int16", TF_INT16}, {"int32", TF_INT32}, {"int64", TF_INT64},
        {"uint8", TF_UINT8}, {"uint16", TF_UINT16}, {"uint32", TF_UINT32}, {"uint64", TF_UINT64},
        {"float", TF_FLOAT}, {"double", TF_DOUBLE}, {"boolean", TF_BOOLEAN}, {"string", TF_BYTES},
        {"utf8", TF_UTF8}, {"any", TF_ANY}, {"date", TF_DATE}, {"datetime", TF_DATETIME},
        {"timestamp", TF_TIMESTAMP}, {"interval", TF_INTERVAL}};
    for (auto& kv : m) if (t == kv.first) return kv.second;
    return 0;
}
inline const char* tf_to_yt(int tf) {
    static const char* n[] = {"", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float", "double",
                              "boolean", "string", "utf8", "any", "date", "datetime", "timestamp", "interval"};
    return (tf >= 1 && tf <= 18) ? n[tf] : "";
}

inline std::vector<ColSchema> parse_schema(const std::string& js) {
    auto root = tfj::parse(js);
    if (root->kind != tfj::Value::Arr) throw FatalError(TF_E_FATAL_CONFIG, "schema_json must be an array of ColSchema");
    std::vector<ColSchema> out;
    for (auto& e : root->arr) {
        ColSchema c;
        c.table_schema = e->get_str("table_schema"); c.table_name = e->get_str("table_name"); c.path = e->get_str("path");
        c.name = e->get_str("name"); c.type = e->get_str("type"); c.expression = e->get_str("expression");
        c.original_type = e->get_str("original_type");
        c.key = e->get_bool("key"); c.fake_key = e->get_bool("fake_key"); c.required = e->get_bool("required");
        c.tf = yt_to_tf(c.type);
        if (!c.tf) throw FatalError(TF_E_FATAL_UNSUPPORTED, "unsupported column type '" + c.type + "' for column " + c.name);
        out.push_back(c);
    }
    return out;
}

inline std::string schema_to_json(const std::vector<ColSchema>& s) {
    std::string o = "[";
    for (size_t i = 0; i < s.size(); i++) {
        const ColSchema& c = s[i];
        if (i) o += ",";
        o += "{\"table_schema\":" + tfj::quote(c.table_schema) + ",\"table_name\":" + tfj::quote(c.table_name) + ",\"path\":" + tfj::quote(c.path) +
             ",\"name\":" + tfj::quote(c.name) + ",\"type\":" + tfj::quote(c.type) + ",\"key\":" + (c.key ? "true" : "false") +
             ",\"fake_key\":" + (c.fake_key ? "true" : "false") + ",\"required\":" + (c.required ? "true" : "false") +
             ",\"expression\":" + tfj::quote(c.expression) + ",\"original_type\":" + tfj::quote(c.original_type) + "}";
    }
    return o + "]";
}

// ------------------------------------------------------------------ filter grammar
enum { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN, OP_NOTIN, OP_MATCH, OP_NOTMATCH };
enum { LV_INT = 1, LV_FLOAT = 2, LV_BOOL = 3, LV_STRING = 4, LV_TIME = 5, LV_NULL = 6, LV_LIST = 16 };

struct Literal { int kind = 0; int64_t i = 0; double f = 0; std::string s; };
struct Term { std::string attribute; int op = 0; int vtype = 0; Literal v; std::vector<Literal> list; };

struct Tok { int kind; std::string text; };   // kinds: 0 Operator 1 String 2 DateTime 3 Ident 4 Float 5 Int 6 Punct 7 WS 8 EOF
enum { T_OP, T_STR, T_DT, T_ID, T_FLOAT, T_INT, T_PUNCT, T_WS, T_EOF };

inline bool is_d(char c) { return c >= '0' && c <= '9'; }
inline bool is_a(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }

// grammar.go:256-266: one regexp, alternatives tried in order at each position
inline std::vector<Tok> lex(const std::string& s) {
    std::vector<Tok> out; size_t p = 0, n = s.size();
    auto digits = [&](size_t q, int cnt) { for (int i = 0; i < cnt; i++) if (q + i >= n || !is_d(s[q + i])) return false; return true; };
    while (p < n) {
        char c = s[p];
        // Operator
        if (p + 1 < n && ((c == '!' && (s[p + 1] == '=' || s[p + 1] == '~')) || ((c == '<' || c == '>') && s[p + 1] == '='))) { out.push_back({T_OP, s.substr(p, 2)}); p += 2; continue; }
        if (c == '=' || c == '<' || c == '>' || c == '~') { out.push_back({T_OP, std::string(1, c)}); p++; continue; }
        // String
        if (c == '\'' || c == '"') {
            size_t i = p + 1, last_esc = std::string::npos; bool closed = false;
            while (i < n) {
                if (s[i] == '\\' && i + 1 < n && s[i + 1] == c) { last_esc = i; i += 2; continue; }
                if (s[i] == c) { closed = true; break; }
                i++;
            }
            if (!closed && last_esc != std::string::npos) { i = last_esc + 1; closed = true; }   // regexp backtracking: "\'" re-read as '\' + closing quote
            if (closed) { out.push_back({T_STR, s.substr(p, i - p + 1)}); p = i + 1; continue; }
            throw FatalError(TF_E_FATAL_CONFIG, "filter: invalid token at " + std::to_string(p));
        }
        // DateTime
        if (digits(p, 4) && p + 4 < n && s[p + 4] == '-' && digits(p + 5, 2) && p + 7 < n && s[p + 7] == '-' && digits(p + 8, 2)) {
            size_t q = p + 10;
            if (q < n && s[q] == 'T' && digits(q + 1, 2) && q + 3 < n && s[q + 3] == ':' && digits(q + 4, 2)) {
                q += 6;
                if (q < n && s[q] == ':' && digits(q + 1, 2)) {
                    q += 3;
                    if (q + 1 < n && s[q] == '.' && is_d(s[q + 1])) { q++; while (q < n && is_d(s[q])) q++; }
                }
                if (q < n && s[q] == 'Z') q++;
                else if (q + 1 < n && (s[q] == '+' || s[q] == '-') && is_d(s[q + 1])) {
                    q++; while (q < n && is_d(s[q])) q++;
                    if (q + 1 < n && s[q] == ':' && is_d(s[q + 1])) { q++; while (q < n && is_d(s[q])) q++; }
                }
            }
            out.push_back({T_DT, s.substr(p, q - p)}); p = q; continue;
        }
        // Ident
        if (is_a(c)) { size_t q = p + 1; while (q < n && (is_a(s[q]) || is_d(s[q]) || s[q] == '_' || s[q] == '.')) q++; out.push_back({T_ID, s.substr(p, q - p)}); p = q; continue; }
        // Float / Int
        {
            size_t q = p; if (s[q] == '-' || s[q] == '+') q++;
            if (q < n && is_d(s[q])) {
                size_t r = q; while (r < n && is_d(s[r])) r++;
                if (r + 1 < n && s[r] == '.' && is_d(s[r + 1])) { size_t t = r + 1; while (t < n && is_d(s[t])) t++; out.push_back({T_FLOAT, s.substr(p, t - p)}); p = t; continue; }
                out.push_back({T_INT, s.substr(p, r - p)}); p = r; continue;
            }
        }
        if (c == '(' || c == ')' || c == ',') { out.push_back({T_PUNCT, std::string(1, c)}); p++; continue; }
        if (c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v') { size_t q = p; while (q < n && (s[q] == ' ' || s[q] == '\t' || s[q] == '\n' || s[q] == '\r' || s[q] == '\f' || s[q] == '\v')) q++; out.push_back({T_WS, s.substr(p, q - p)}); p = q; continue; }
        throw FatalError(TF_E_FATAL_CONFIG, "filter: invalid token at " + std::to_string(p));
    }
    out.push_back({T_EOF, ""});
    return out;
}

inline void put_utf8(std::string& o, uint32_t cp) {
    if (cp < 0x80) o += (char)cp;
    else if (cp < 0x800) { o += (char)(0xC0 | (cp >> 6)); o += (char)(0x80 | (cp & 0x3F)); }
    else if (cp < 0x10000) { o += (char)(0xE0 | (cp >> 12)); o += (char)(0x80 | ((cp >> 6) & 0x3F)); o += (char)(0x80 | (cp & 0x3F)); }
    else { o += (char)(0xF0 | (cp >> 18)); o += (char)(0x80 | ((cp >> 12) & 0x3F)); o += (char)(0x80 | ((cp >> 6) & 0x3F)); o += (char)(0x80 | (cp & 0x3F)); }
}
// participle.Unquote("String") == strconv.UnquoteChar over the body
inline std::string unquote(const std::string& tok) {
    char q = tok[0]; std::string b = tok.substr(1, tok.size() - 2), o; size_t i = 0;
    auto bad = [&]() -> FatalError { return FatalError(TF_E_FATAL_CONFIG, "filter: invalid quoted string " + tok); };
    while (i < b.size()) {
        char c = b[i];
        if (c != '\\') { o += c; i++; continue; }
        if (++i >= b.size()) throw bad();
        char e = b[i++];
        switch (e) {
        case 'a': o += '\a'; break; case 'b': o += '\b'; break; case 'f': o += '\f'; break; case 'n': o += '\n'; break;
        case 'r': o += '\r'; break; case 't': o += '\t'; break; case 'v': o += '\v'; break; case '\\': o += '\\'; break;
        case '\'': case '"': if (e != q) throw bad(); o += e; break;
        case 'x': { if (i + 2 > b.size()) throw bad(); o += (char)strtoul(b.substr(i, 2).c_str(), nullptr, 16); i += 2; break; }
        case 'u': case 'U': { size_t k = e == 'u' ? 4 : 8; if (i + k > b.size()) throw bad(); put_utf8(o, (uint32_t)strtoul(b.substr(i, k).c_str(), nullptr, 16)); i += k; break; }
        default:
            if (e >= '0' && e <= '7') { if (i + 2 > b.size()) throw bad(); o += (char)strtoul(b.substr(i - 1, 3).c_str(), nullptr, 8); i += 2; break; }
            throw bad();
        }
    }
    return o;
}

inline int64_t days_from_civil(int64_t y, unsigned m, unsigned d) {
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const unsigned yoe = (unsigned)(y - era * 400);
    const unsigned doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
    const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}
// DateTime.delayedParse grammar.go:176-188 (layout chosen by findTimeLayout :120-149); returns UnixMicro
inline int64_t parse_time_micro(const std::string& v) {
    auto bad = [&](const char* m) -> FatalError { return FatalError(TF_E_FATAL_CONFIG, std::string("filter: ") + m + " in '" + v + "'"); };
    auto num = [&](size_t p, size_t k) { return (int)strtol(v.substr(p, k).c_str(), nullptr, 10); };
    int y = num(0, 4), mo = num(5, 2), d = num(8, 2);
    static const int dm[] = {0, 31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    if (mo < 1 || mo > 12) throw bad("month out of range");
    if (d < 1 || d > dm[mo] + ((mo == 2 && leap) ? 1 : 0)) throw bad("day out of range");
    int hh = 0, mi = 0, ss = 0; int64_t nsec = 0, off = 0; size_t p = 10;
    if (p < v.size() && v[p] == 'T') {
        hh = num(p + 1, 2); mi = num(p + 4, 2); p += 6;
        if (p < v.size() && v[p] == ':') { ss = num(p + 1, 2); p += 3;
            if (p < v.size() && v[p] == '.') { size_t q = p + 1; std::string fr; while (q < v.size() && is_d(v[q])) fr += v[q++]; fr += "000000000"; nsec = strtoll(fr.substr(0, 9).c_str(), nullptr, 10); p = q; } }
        if (hh > 23) throw bad("hour out of range");
        if (mi > 59) throw bad("minute out of range");
        if (ss > 59) throw bad("second out of range");
        if (p < v.size() && v[p] != 'Z') {
            int sign = v[p] == '-' ? -1 : 1; std::string tz = v.substr(p + 1); size_t colon = tz.find(':');
            if (colon != std::string::npos) { if (colon != 2 || tz.size() != 5) throw bad("bad zone"); off = sign * (strtol(tz.substr(0, 2).c_str(), nullptr, 10) * 3600 + strtol(tz.substr(3, 2).c_str(), nullptr, 10) * 60); }
            else { if (tz.size() != 2) throw bad("bad zone"); off = sign * strtol(tz.c_str(), nullptr, 10) * 3600; }
        }
    }
    int64_t sec = days_from_civil(y, (unsigned)mo, (unsigned)d) * 86400 + hh * 3600 + mi * 60 + ss - off;
    return sec * 1000000 + nsec / 1000;
}

inline std::string upper(std::string s) { for (auto& c : s) if (c >= 'a' && c <= 'z') c -= 32; return s; }

class FilterParser {
public:
    explicit FilterParser(const std::string& src) : t_(lex(src)) {}
    std::vector<Term> parse() {
        std::vector<Term> out; ws();
        if (peek().kind == T_EOF) return out;
        out.push_back(term());
        for (;;) {
            ws(); if (peek().kind == T_EOF) break;
            if (!kw(peek(), "AND")) unexpected();
            p_++; ws(); out.push_back(term());
        }
        return out;
    }
private:
    std::vector<Tok> t_; size_t p_ = 0;
    const Tok& peek() const { return t_[p_ < t_.size() ? p_ : t_.size() - 1]; }
    void ws() { while (peek().kind == T_WS) p_++; }
    static bool kw(const Tok& t, const char* n) { return t.kind == T_ID && upper(t.text) == n; }
    [[noreturn]] void unexpected() { throw FatalError(TF_E_FATAL_CONFIG, "filter: unexpected token \"" + peek().text + "\""); }
    Literal scalar(int& kind) {
        Literal l; const Tok& t = peek();
        if (t.kind == T_STR) { kind = LV_STRING; l.s = unquote(t.text); p_++; }
        else if (t.kind == T_DT) { kind = LV_TIME; l.i = parse_time_micro(t.text); p_++; }
        else if (kw(t, "TRUE") || kw(t, "FALSE")) { kind = LV_BOOL; l.i = upper(t.text) == "TRUE"; p_++; }
        else if (t.kind == T_FLOAT) {
            kind = LV_FLOAT; l.f = strtod(t.text.c_str(), nullptr);
            if (l.f == HUGE_VAL || l.f == -HUGE_VAL) throw FatalError(TF_E_FATAL_CONFIG, "filter: value out of range");   // strconv.ParseFloat: ErrRange (an underflow to 0 is not one)
            p_++;
        }
        else if (t.kind == T_INT) {
            kind = LV_INT; errno = 0; l.i = strtoll(t.text.c_str(), nullptr, 10);
            if (errno == ERANGE) throw FatalError(TF_E_FATAL_CONFIG, "filter: value out of range");
            p_++;
        }
        else if (kw(t, "NULL") || kw(t, "NIL")) { kind = LV_NULL; p_++; }
        else unexpected();
        l.kind = kind; return l;
    }
    Term term() {
        Term tm; if (peek().kind != T_ID) unexpected();
        tm.attribute = peek().text; p_++; ws();
        const Tok& o = peek();
        if (o.kind == T_OP) {
            const std::string& x = o.text;
            tm.op = x == "=" ? OP_EQ : x == "!=" ? OP_NE : x == "<" ? OP_LT : x == "<=" ? OP_LE : x == ">" ? OP_GT : x == ">=" ? OP_GE : x == "~" ? OP_MATCH : OP_NOTMATCH;
            p_++;
        } else if (kw(o, "IN")) { tm.op = OP_IN; p_++; }
        else if (kw(o, "NOT")) { p_++; ws(); if (!kw(peek(), "IN")) unexpected(); tm.op = OP_NOTIN; p_++; }
        else unexpected();
        ws();
        bool is_list = false;
        if (peek().kind == T_PUNCT && peek().text == "(") {
            is_list = true; p_++; ws();
            int k0 = 0; tm.list.push_back(scalar(k0)); ws();
            while (peek().kind == T_PUNCT && peek().text == ",") {
                p_++; ws(); int k = 0; Literal l = scalar(k);
                if (k != k0) throw FatalError(TF_E_FATAL_CONFIG, "filter: list items should have same type");
                tm.list.push_back(l); ws();
            }
            if (!(peek().kind == T_PUNCT && peek().text == ")")) unexpected();
            p_++; tm.vtype = k0 | LV_LIST;
        } else { int k = 0; tm.v = scalar(k); tm.vtype = k; }
        ws();
        // validateTerm filters.go:255-287
        if (is_list && tm.op != OP_IN && tm.op != OP_NOTIN) throw FatalError(TF_E_FATAL_CONFIG, "filter: list values require [ NOT ] IN operator");
        if (!is_list && (tm.op == OP_IN || tm.op == OP_NOTIN)) throw FatalError(TF_E_FATAL_CONFIG, "filter: IN operator expect list value");
        if (tm.vtype == LV_NULL && tm.op != OP_EQ && tm.op != OP_NE) throw FatalError(TF_E_FATAL_CONFIG, "filter: NULL expects \"=\" or \"!=\" operator");
        return tm;
    }
};

// ------------------------------------------------------------------ table / column name filters
// The patterns are Go regular expressions (regexp.Compile in filter.NewFilter, filter.go:46-71): compiled by the Go-syntax engine of
// host_regex.hpp, so `\z`, POSIX classes, ASCII `\d` / `\w` and the errors are Go's, not ECMAScript's.
struct NameFilter {
    std::vector<std::string> inc_src, exc_src;
    std::vector<std::shared_ptr<tfre::Prog>> inc, exc;
    bool empty() const { return inc_src.empty() && exc_src.empty(); }
    bool match(const std::string& v) const {          // filter.go:27-44
        for (auto& r : exc) if (tfre::match_string(*r, v)) return false;
        if (inc_src.empty()) return true;
        for (auto& r : inc) if (tfre::match_string(*r, v)) return true;
        return false;
    }
};
inline NameFilter make_filter(const std::vector<std::string>& inc, const std::vector<std::string>& exc) {
    NameFilter f; f.inc_src = inc; f.exc_src = exc;
    try {
        for (auto& s : inc) f.inc.push_back(std::make_shared<tfre::Prog>(tfre::compile(s)));
        for (auto& s : exc) f.exc.push_back(std::make_shared<tfre::Prog>(tfre::compile(s)));
    } catch (const tfre::SyntaxError& e) { throw FatalError(TF_E_FATAL_CONFIG, std::string("unable to compile regexp: ") + e.what()); }
    catch (const tfre::Unsupported& e) { throw FatalError(TF_E_FATAL_UNSUPPORTED, std::string("a table / column filter expression this library does not carry: ") + e.what()); }
    return f;
}
inline NameFilter tables_filter(const tfj::Value* cfg) {
    if (!cfg) return NameFilter();
    auto inc = cfg->get_str_list("includeTables"); if (inc.empty()) inc = cfg->get_str_list("include_tables");
    auto exc = cfg->get_str_list("excludeTables"); if (exc.empty()) exc = cfg->get_str_list("exclude_tables");
    return make_filter(inc, exc);
}
inline std::string dq(const std::string& s) { std::string o = "\""; for (char c : s) { if (c == '"') o += "\"\""; else o += c; } return o + "\""; }
inline bool match_table(const NameFilter& f, const std::string& ns, const std::string& name) {   // transformer_common.go:9-33
    if (f.empty()) return true;
    std::string full = ns.empty() ? name : ns + "." + name;
    std::string fq = (ns.empty() ? "" : dq(ns) + ".") + (name == "*" ? name : dq(name));
    return f.match(full) || f.match(fq);
}

// ------------------------------------------------------------------ compiled plan
struct DTerm {            // device-visible predicate term (POD)
    int32_t col, op, vtype, nlist;
    int64_t i; double f;
    uint32_t s_off, s_len;      // string literal in the literal blob
    uint32_t list_off, pad;     // int64[] / double[] / (uint32 offs[nlist+1], bytes) in the blob, 8-byte aligned
};
struct FilterStep {
    std::vector<std::vector<DTerm>> exprs; std::vector<std::vector<Term>> src;
    bool is_skip = false; int kind_mask = 0;     // skip_events: bit TF_KIND_* set = drop rows of that kind
    bool pass_all = false;                       // filter_rows whose table filter does not match the (renamed) table
};
struct MaskStep { std::vector<int> cols; std::string salt; };

struct Plan {
    std::string ns, name, schema_json;
    std::vector<ColSchema> in_schema, out_schema;
    std::string out_ns, out_name;      // table identity after rename_tables
    std::vector<int> out_cols;         // input index of every output column, schema order
    std::vector<FilterStep> filters;   // in plan order
    std::vector<int> filter_step_index;
    std::vector<uint8_t> todt_col;     // [input column] 1 = convert_to_datetime applies (to_datetime.go:89-135)
    std::vector<int> todt_step_index; std::vector<std::vector<int>> todt_cols;
    std::vector<int> n2f_cols;         // input columns (still `any` at that step) number_to_float rewrites (number_to_float.go:75-85)
    std::vector<uint8_t> tostr_col;    // [input column] 1 = convert_to_string applies (to_string.go:58-97)
    std::vector<int> tostr_step_index; std::vector<std::vector<int>> tostr_cols;
    std::vector<MaskStep> masks;
    // sharder (registry/sharder/sharder.go:63-145): the LAST sharder of the chain sets ChangeItem.PartID. form: 0 = the text of the
    // input value (also after convert_to_string: the text of a text is itself), 1 = the mask digest, 3 = the converted datetime
    bool has_sharder = false; uint32_t shards = 0; std::vector<int> shard_cols, shard_form; int shard_step_index = -1;
    std::vector<int> mask_step_index;
    bool has_splitter = false; int splitter_step = -1;   // table_splitter@sink: the last step of the chain (checked at the end of build_plan)
    int n_regex_steps = 0;             // regex_replace_transformer@sink: rewrites the row image before the transposer, so these steps lead the chain
    std::vector<uint8_t> blob;         // literal pool referenced by DTerm
    std::string describe;
    // sink
    bool has_sink = false;
    std::vector<std::string> ch_types;
    std::vector<uint8_t> col_headers;        // per column: varint name, name, varint type, type, 0x00
    std::vector<uint32_t> col_header_off;    // ncols+1
};

inline uint32_t blob_put(std::vector<uint8_t>& b, const void* p, size_t n, size_t align = 8) {
    while (b.size() % align) b.push_back(0);
    uint32_t off = (uint32_t)b.size(); const uint8_t* q = (const uint8_t*)p; b.insert(b.end(), q, q + n); return off;
}

inline bool column_suitable(const Term& t, int tf) {   // checkColumnSuitable filter_rows.go:489-519
    int base = t.vtype & 15; bool list = t.vtype & LV_LIST;
    if (list) return base == LV_INT || base == LV_FLOAT || base == LV_STRING || base == LV_TIME;
    switch (base) {
    case LV_BOOL: return tf == TF_BOOLEAN;
    case LV_INT: case LV_FLOAT: return (tf >= TF_INT8 && tf <= TF_DOUBLE);
    case LV_STRING: return tf == TF_UTF8 || tf == TF_BYTES || tf == TF_ANY;
    case LV_TIME: return tf == TF_TIMESTAMP || tf == TF_DATE || tf == TF_DATETIME;
    case LV_NULL: return true;
    }
    return false;
}

inline std::string ch_type_of(const ColSchema& c) {    // columntypes.ToChType types.go:210-248 + sink_table.go:196-208
    if (c.original_type.rfind("ch:", 0) == 0) throw FatalError(TF_E_FATAL_UNSUPPORTED, "ch: original types are not supported by the device encoder (column " + c.name + ")");
    std::string b;
    switch (c.tf) {
    case TF_ANY: case TF_BYTES: case TF_UTF8: b = "String"; break;
    case TF_DOUBLE: b = "Float64"; break; case TF_FLOAT: b = "Float32"; break; case TF_BOOLEAN: b = "UInt8"; break;
    case TF_INT8: b = "Int8"; break; case TF_INT16: b = "Int16"; break; case TF_INT32: b = "Int32"; break; case TF_INT64: b = "Int64"; break;
    case TF_UINT8: b = "UInt8"; break; case TF_UINT16: b = "UInt16"; break; case TF_UINT32: b = "UInt32"; break; case TF_UINT64: b = "UInt64"; break;
    case TF_DATE: b = "Date"; break; case TF_DATETIME: b = "DateTime"; break; case TF_TIMESTAMP: b = "DateTime64(6)"; break;
    case TF_INTERVAL: b = "Int64"; break;
    default: b = "String";
    }
    return c.required ? b : "Nullable(" + b + ")";
}

inline void put_uvarint(std::vector<uint8_t>& o, uint64_t v) { while (v >= 0x80) { o.push_back((uint8_t)(v | 0x80)); v >>= 7; } o.push_back((uint8_t)v); }

inline std::string lit_json(int kind, const Literal& l) {
    switch (kind) {
    case LV_INT: case LV_TIME: return std::to_string(l.i);
    case LV_BOOL: return l.i ? "true" : "false";
    case LV_FLOAT: { char b[64]; snprintf(b, sizeof b, "%.17g", l.f); return b; }
    case LV_STRING: { std::string h; static const char* H = "0123456789abcdef"; for (unsigned char c : l.s) { h += H[c >> 4]; h += H[c & 15]; } return "\"" + h + "\""; }
    case LV_NULL: return "null";
    }
    return "null";
}

inline Plan build_plan(const std::string& ns, const std::string& name, const std::string& schema_json,
                       const std::string& transformers_json, const std::string& sink_json) {
    Plan pl; pl.ns = ns; pl.name = name; pl.schema_json = schema_json;
    pl.in_schema = parse_schema(schema_json);
    if (pl.in_schema.empty()) throw FatalError(TF_E_FATAL_CONFIG, "empty schema");
    for (size_t i = 0; i < pl.in_schema.size(); i++) pl.in_schema[i].in_index = (int)i;
    std::vector<ColSchema> cur = pl.in_schema;
    std::string cur_ns = ns, cur_name = name;
    std::string steps_desc;
    auto add_desc = [&](const std::string& d) { if (!steps_desc.empty()) steps_desc += ","; steps_desc += d; };
    auto trs = transformers_json.empty() ? tfj::parse("[]") : tfj::parse(transformers_json);
    if (trs->kind != tfj::Value::Arr) throw FatalError(TF_E_FATAL_CONFIG, "transformers_json must be a list");
    int step_no = 0;
    for (auto& tr : trs->arr) {
        if (tr->kind != tfj::Value::Obj) throw FatalError(TF_E_FATAL_CONFIG, "transformer entry must be an object");
        std::string ttype; const tfj::Value* cfg = nullptr;
        for (auto& kv : tr->obj) if (kv.first != "transformerId") { ttype = kv.first; cfg = kv.second.get(); }
        if (ttype.empty()) throw FatalError(TF_E_FATAL_CONFIG, "transformer entry without a type");
        static const tfj::Value empty_obj = [] { tfj::Value v; v.kind = tfj::Value::Obj; return v; }();
        if (!cfg || cfg->kind != tfj::Value::Obj) cfg = &empty_obj;
        auto col_pos = [&](const std::string& n) { for (size_t i = 0; i < cur.size(); i++) if (cur[i].name == n) return (int)i; return -1; };
        // NOTE transformation.AddTablePlan asks Suitable() with the ORIGINAL table id for every transformer
        // (transformation.go:54); only transformers that re-check the item's own id inside Apply see a rename.
        if (ttype == "filter_rows") {
            std::string one = cfg->get_str("filter"); auto many = cfg->get_str_list("filters");
            if (!one.empty() && !many.empty()) throw FatalError(TF_E_FATAL_CONFIG, "Settings 'filters' and 'filter' cannot be enabled at the same time");
            if (many.empty()) many.push_back(one);
            FilterStep fs;
            for (auto& f : many) fs.src.push_back(FilterParser(f).parse());
            NameFilter tf = tables_filter(cfg->get("tables"));
            if (!match_table(tf, ns, name)) continue;
            bool ok = true;                                         // Suitable filter_rows.go:445-476
            for (auto& terms : fs.src) for (auto& t : terms) { int ci = col_pos(t.attribute); if (ci < 0 || !column_suitable(t, cur[ci].tf)) ok = false; }
            if (!ok) continue;
            fs.pass_all = !match_table(tf, cur_ns, cur_name);       // Apply re-checks item.TableID() (filter_rows.go:109-113)
            std::string d = std::string("{\"type\":\"filter_rows\",\"pass_all\":") + (fs.pass_all ? "true" : "false") + ",\"exprs\":[";
            for (size_t e = 0; e < fs.src.size(); e++) {
                std::vector<DTerm> dt; if (e) d += ",";
                d += "[";
                for (size_t k = 0; k < fs.src[e].size(); k++) {
                    const Term& t = fs.src[e][k]; DTerm x; std::memset(&x, 0, sizeof x);
                    const int cp = col_pos(t.attribute);
                    x.col = cur[cp].in_index; x.op = t.op; x.vtype = t.vtype; x.nlist = (int)t.list.size();
                    int base = t.vtype & 15; int ctf = cur[cp].tf;
                    bool col_is_str = ctf == TF_UTF8 || ctf == TF_ANY;
                    if ((base == LV_INT || base == LV_FLOAT) && (col_is_str))
                        throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_rows: numeric literal against text column '" + t.attribute + "' (strconv.ParseFloat path) is not implemented on the device");
                    if (base == LV_TIME && (t.vtype & LV_LIST) && (col_is_str || ctf == TF_BYTES))
                        throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_rows: list of times against text column '" + t.attribute + "' (stringToTime path, filter_rows.go:340-352) is not implemented on the device");
                    if (k) d += ",";
                    d += "{\"col\":" + std::to_string(x.col) + ",\"op\":" + std::to_string(x.op) + ",\"vtype\":" + std::to_string(x.vtype) + ",\"value\":";
                    if (!(t.vtype & LV_LIST)) {
                        x.i = t.v.i; x.f = t.v.f;
                        if (base == LV_STRING) { x.s_off = blob_put(pl.blob, t.v.s.data(), t.v.s.size(), 1); x.s_len = (uint32_t)t.v.s.size(); }
                        d += lit_json(base, t.v);
                    } else {
                        d += "[";
                        for (size_t q = 0; q < t.list.size(); q++) { if (q) d += ","; d += lit_json(base, t.list[q]); }
                        d += "]";
                        if (base == LV_INT || base == LV_TIME) { std::vector<int64_t> v; for (auto& l : t.list) v.push_back(l.i); x.list_off = blob_put(pl.blob, v.data(), v.size() * 8); }
                        else if (base == LV_FLOAT) { std::vector<double> v; for (auto& l : t.list) v.push_back(l.f); x.list_off = blob_put(pl.blob, v.data(), v.size() * 8); }
                        else if (base == LV_STRING) {
                            std::vector<uint32_t> offs(1, 0); std::string bytes;
                            for (auto& l : t.list) { bytes += l.s; offs.push_back((uint32_t)bytes.size()); }
                            x.list_off = blob_put(pl.blob, offs.data(), offs.size() * 4); blob_put(pl.blob, bytes.data(), bytes.size(), 1);
                        }
                    }
                    d += "}";
                    dt.push_back(x);
                }
                d += "]";
                fs.exprs.push_back(dt);
            }
            d += "]}";
            add_desc(d);
            pl.filters.push_back(fs); pl.filter_step_index.push_back(step_no++);
        } else if (ttype == "skip_events") {                         // registry/filter/skip_events.go:52-66
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            FilterStep fs; fs.is_skip = true;
            for (auto& ev : cfg->get_str_list("events")) {
                if (ev == "insert") fs.kind_mask |= 1 << TF_KIND_INSERT;
                else if (ev == "update") fs.kind_mask |= 1 << TF_KIND_UPDATE;
                else if (ev == "delete") fs.kind_mask |= 1 << TF_KIND_DELETE;
            }
            add_desc("{\"type\":\"skip_events\",\"kind_mask\":" + std::to_string(fs.kind_mask) + "}");
            pl.filters.push_back(fs); pl.filter_step_index.push_back(step_no++);
        } else if (ttype == "filter_columns") {                      // registry/filter/filter_columns_transformer.go:215-236
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            const tfj::Value* cc = cfg->get("columns");
            std::vector<std::string> inc, exc;
            if (cc) { inc = cc->get_str_list("includeColumns"); if (inc.empty()) inc = cc->get_str_list("include_columns");
                      exc = cc->get_str_list("excludeColumns"); if (exc.empty()) exc = cc->get_str_list("exclude_columns"); }
            NameFilter cf = make_filter(inc, exc);
            bool valid = true;
            for (auto& c : cur) if (!cf.match(c.name) && c.key) valid = false;   // a primary key may not be dropped -> not Suitable
            if (!valid) continue;
            std::vector<ColSchema> nxt; std::string d = "{\"type\":\"filter_columns\",\"keep\":[";
            for (auto& c : cur) if (cf.match(c.name)) { if (!nxt.empty()) d += ","; d += std::to_string(c.in_index); nxt.push_back(c); }
            if (nxt.empty()) throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_columns leaves no columns");
            cur = nxt; add_desc(d + "]}"); step_no++;
        } else if (ttype == "replace_primary_key") {                 // registry/replace_primary_key/replace_primary_key.go:84-117
            const std::vector<std::string> keys = cfg->get_str_list("keys");
            for (size_t a = 0; a < keys.size(); a++) for (size_t b = a + 1; b < keys.size(); b++) if (keys[a] == keys[b])
                throw FatalError(TF_E_FATAL_CONFIG, "replace_primary_key: Can't use same keys column names twice");      // NewReplacePrimaryKeyTransformer :133-137
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            size_t have = 0; for (auto& c : cur) for (auto& k : keys) if (c.name == k) { have++; break; }
            if (have != keys.size()) continue;                       // Suitable: containsAllKeys :37-45
            auto is_key = [&](const std::string& n) { for (auto& k : keys) if (k == n) return true; return false; };
            if (keys.size() == 1) { for (auto& c : cur) c.key = is_key(c.name); }
            else {                                                   // composite key: the key columns lead the schema in the order given (:100-113)
                std::vector<ColSchema> nxt;
                for (auto& k : keys) for (auto& c : cur) if (c.name == k) { ColSchema x = c; x.key = true; nxt.push_back(x); break; }
                for (auto& c : cur) if (!is_key(c.name)) { ColSchema x = c; x.key = false; nxt.push_back(x); }
                cur = nxt;
            }
            std::string d = "{\"type\":\"replace_primary_key\",\"keys\":[";
            for (size_t i = 0; i < keys.size(); i++) d += (i ? "," : "") + tfj::quote(keys[i]);
            add_desc(d + "]}"); step_no++;
        } else if (ttype == "table_splitter@sink" || ttype == "table_splitter") {   // registry/table_splitter/table_splitter.go:36-101
            // The transformer changes ChangeItem.Table per ROW (original name + splitter + the text of the listed columns): nothing for the device to
            // compute on the values, but the rows of one batch then belong to several tables. tfgpu_sink_push groups the rows by the generated
            // name on the host and pushes every group on its own; it marks the step "@sink" when it forwards the list. Plain tfgpu_push_* callers
            // would get ONE block for all rows, so the unmarked form is refused.
            if (ttype == "table_splitter") throw FatalError(TF_E_FATAL_UNSUPPORTED, "table_splitter is applied by tfgpu_sink_push (rows are grouped by the generated table name on the host)");
            if (cfg->get_bool("useLegacyLf")) throw FatalError(TF_E_FATAL_UNSUPPORTED, "table_splitter: useLegacyLf is not implemented");
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            for (auto& cn : cfg->get_str_list("columns")) for (auto& c : cur) if (c.name == cn && (c.tf == TF_ANY || c.tf == TF_INTERVAL))
                throw FatalError(TF_E_FATAL_UNSUPPORTED, "table_splitter over an `any` / interval column is not implemented");
            pl.has_splitter = true; pl.splitter_step = step_no;
            add_desc("{\"type\":\"table_splitter\"}"); step_no++;
        } else if (ttype == "regex_replace_transformer@sink" || ttype == "regex_replace_transformer") {   // registry/regex_replace/transformer.go:64-142
            // Go's regexp over the string / []byte values of the matched columns; the schema does not change. tfgpu_sink_push applies it to the
            // row image before the transposer (csrc/host_regex.hpp) and marks the step "@sink": nothing on the device runs a regular expression,
            // so a plain tfgpu_push_* caller is refused, and so is a chain that would have to see the values before the replacement.
            if (ttype == "regex_replace_transformer") throw FatalError(TF_E_FATAL_UNSUPPORTED, "regex_replace_transformer is applied by tfgpu_sink_push (to the row image, before the device chain)");
            if (!tables_filter(cfg->get("tables")).match(name)) continue;       // Suitable :64-66: Tables.Match(table.Name), the bare name
            if (step_no != pl.n_regex_steps)
                throw FatalError(TF_E_FATAL_UNSUPPORTED, "regex_replace_transformer behind another transformer: tfgpu_sink_push rewrites the values before the chain runs (put it first)");
            pl.n_regex_steps++;
            add_desc("{\"type\":\"regex_replace_transformer\"}"); step_no++;
        } else if (ttype == "rename_tables") {                       // registry/rename/rename.go:46-67
            const tfj::Value* lst = cfg->get("renameTables");
            bool hit = false; std::string nns, nname;
            if (lst && lst->kind == tfj::Value::Arr) for (auto& r : lst->arr) {
                const tfj::Value* o = r->get("originalName"); const tfj::Value* nw = r->get("newName");
                if (!o || !nw) continue;
                if (o->get_str("nameSpace") == ns && o->get_str("name") == name) { hit = true; nns = nw->get_str("nameSpace"); nname = nw->get_str("name"); }
            }
            if (!hit) continue;                                      // Suitable: exact TableID in AltNames (ORIGINAL id)
            // Apply looks the item's CURRENT id up in AltNames (rename.go:50-54): after an earlier rename to B, a transformer that lists
            // both A -> B and B -> C takes the item on to C; the last entry for an id wins, like the map built from the list
            {
                bool found = false; std::string tns, tname;
                for (auto& r : lst->arr) {
                    const tfj::Value* o = r->get("originalName"); const tfj::Value* nw = r->get("newName");
                    if (!o || !nw) continue;
                    if (o->get_str("nameSpace") == cur_ns && o->get_str("name") == cur_name) { found = true; tns = nw->get_str("nameSpace"); tname = nw->get_str("name"); }
                }
                if (found) { cur_ns = tns; cur_name = tname; }
            }
            add_desc("{\"type\":\"rename_tables\",\"to\":" + tfj::quote(cur_ns.empty() ? cur_name : cur_ns + "." + cur_name) + "}"); step_no++;
        } else if (ttype == "mask_field") {
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            auto cols = cfg->get_str_list("columns");
            MaskStep ms; const tfj::Value* mf = cfg->get("maskFunctionHash");
            ms.salt = mf ? mf->get_str("userDefinedSalt") : "";
            std::vector<int> pos;
            for (size_t i = 0; i < cur.size(); i++) for (auto& c : cols) if (cur[i].name == c) { pos.push_back((int)i); break; }
            if (!cols.empty() && pos.empty()) continue;          // Suitable hmac_hasher.go:76-89
            std::string d = "{\"type\":\"mask_field\",\"cols\":[";
            for (size_t i = 0; i < pos.size(); i++) {
                ColSchema& c = cur[pos[i]];
                if (i) d += ","; d += std::to_string(c.in_index); ms.cols.push_back(c.in_index);
                c.type = "utf8"; c.tf = TF_UTF8; c.original_type = "";
            }
            add_desc(d + "]}");
            pl.masks.push_back(ms); pl.mask_step_index.push_back(step_no++);
        } else if (ttype == "convert_to_datetime") {                 // registry/to_datetime/to_datetime.go:56-151
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            const tfj::Value* cc = cfg->get("columns");
            std::vector<std::string> inc, exc;
            if (cc) { inc = cc->get_str_list("includeColumns"); exc = cc->get_str_list("excludeColumns"); }
            NameFilter cf = make_filter(inc, exc);
            if (cf.empty()) continue;                                // Suitable :64-66
            std::vector<int> pos;
            for (size_t i = 0; i < cur.size(); i++) if (cf.match(cur[i].name) && (cur[i].tf == TF_INT32 || cur[i].tf == TF_UINT32)) pos.push_back((int)i);
            if (pos.empty()) continue;
            if (pl.todt_col.empty()) pl.todt_col.assign(pl.in_schema.size(), 0);
            std::vector<int> cols; std::string d = "{\"type\":\"convert_to_datetime\",\"cols\":[";
            for (size_t i = 0; i < pos.size(); i++) {
                ColSchema& c = cur[pos[i]];
                if (c.tf != pl.in_schema[c.in_index].tf || (pl.tostr_col.size() && pl.tostr_col[c.in_index])) throw FatalError(TF_E_FATAL_UNSUPPORTED, "convert_to_datetime on a column an earlier transformer already rewrote");
                if (i) d += ","; d += std::to_string(c.in_index); cols.push_back(c.in_index); pl.todt_col[c.in_index] = 1;
                c.type = "datetime"; c.tf = TF_DATETIME;
            }
            add_desc(d + "]}");
            pl.todt_cols.push_back(cols); pl.todt_step_index.push_back(step_no++);
        } else if (ttype == "number_to_float_transformer") {         // registry/number_to_float/number_to_float.go:54-125
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;              // Suitable :123-125, original id
            if (!match_table(tables_filter(cfg->get("tables")), cur_ns, cur_name)) { add_desc("{\"type\":\"number_to_float_transformer\",\"cols\":[]}"); step_no++; continue; }   // Apply re-checks item.TableID() :62-66
            std::string d = "{\"type\":\"number_to_float_transformer\",\"cols\":["; bool first = true;
            for (size_t i = 0; i < cur.size(); i++) if (cur[i].tf == TF_ANY && cur[i].tf == pl.in_schema[cur[i].in_index].tf && !(pl.tostr_col.size() && pl.tostr_col[cur[i].in_index])) {
                bool dup = false; for (int c : pl.n2f_cols) if (c == cur[i].in_index) dup = true;
                if (!dup) pl.n2f_cols.push_back(cur[i].in_index);
                if (!first) d += ","; first = false; d += std::to_string(cur[i].in_index);
            }
            add_desc(d + "]}"); step_no++;
        } else if (ttype == "sharder_transformer") {                 // registry/sharder/sharder.go:20-145
            if (cfg->get_bool("is_random")) throw FatalError(TF_E_FATAL_UNSUPPORTED, "sharder_transformer is_random: PartID = uuid + rand.Intn, host only");
            const tfj::Value* cc = cfg->get("columns");
            std::vector<std::string> inc, exc;
            if (cc) { inc = cc->get_str_list("includeColumns"); exc = cc->get_str_list("excludeColumns"); }
            NameFilter cf = make_filter(inc, exc);
            const std::string sc = cfg->get_str("shardsCount");
            char* endp = nullptr; errno = 0; const long long sn = std::strtoll(sc.c_str(), &endp, 10);
            if (sc.empty() || *endp || errno) throw FatalError(TF_E_FATAL_CONFIG, "sharder_transformer: cannot parse shardsCount as int");        // :38-41
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            std::vector<int> pos;
            for (size_t i = 0; i < cur.size(); i++) if (cf.match(cur[i].name)) pos.push_back((int)i);
            if (!cf.empty() && pos.empty()) continue;                // Suitable :93-105
            if ((uint32_t)sn == 0) throw FatalError(TF_E_FATAL_CONFIG, "sharder_transformer: shardsCount is zero modulo 2^32 (the reference divides by zero)");
            pl.has_sharder = true; pl.shards = (uint32_t)sn; pl.shard_cols.clear(); pl.shard_form.clear(); pl.shard_step_index = step_no;
            std::string d = "{\"type\":\"sharder_transformer\",\"shards\":" + std::to_string(pl.shards) + ",\"cols\":[";
            for (size_t i = 0; i < pos.size(); i++) {
                const ColSchema& c = cur[pos[i]];
                int form = 0;
                for (auto& ms : pl.masks) for (int mc : ms.cols) if (mc == c.in_index) form = 1;
                if (pl.todt_col.size() && pl.todt_col[c.in_index]) form = 3;
                if (i) d += ","; d += std::to_string(c.in_index);
                pl.shard_cols.push_back(c.in_index); pl.shard_form.push_back(form);
            }
            add_desc(d + "]}"); step_no++;
        } else if (ttype == "convert_to_string") {                   // registry/to_string/to_string.go:24-113
            if (!match_table(tables_filter(cfg->get("tables")), ns, name)) continue;
            if (cfg->get_bool("skip_utc_conversion")) throw FatalError(TF_E_FATAL_UNSUPPORTED, "convert_to_string: skip_utc_conversion needs time zones, which the columnar layout does not carry");
            const tfj::Value* cc = cfg->get("columns");
            std::vector<std::string> inc, exc;
            if (cc) { inc = cc->get_str_list("includeColumns"); exc = cc->get_str_list("excludeColumns"); }
            NameFilter cf = make_filter(inc, exc);
            std::vector<int> pos;
            for (size_t i = 0; i < cur.size(); i++) if (cf.match(cur[i].name)) pos.push_back((int)i);
            if (!cf.empty() && pos.empty()) continue;                // Suitable :99-113
            const bool to_bytes = cfg->get_bool("convert_to_bytes");
            if (pl.tostr_col.empty()) pl.tostr_col.assign(pl.in_schema.size(), 0);
            std::vector<int> cols; std::string d = std::string("{\"type\":\"convert_to_string\",\"to_bytes\":") + (to_bytes ? "true" : "false") + ",\"cols\":[";
            for (size_t i = 0; i < pos.size(); i++) {
                ColSchema& c = cur[pos[i]];
                if (pl.tostr_col[c.in_index] || c.tf != pl.in_schema[c.in_index].tf || (pl.todt_col.size() && pl.todt_col[c.in_index]))
                    throw FatalError(TF_E_FATAL_UNSUPPORTED, "convert_to_string on column '" + c.name + "' that an earlier transformer already rewrote");
                if (i) d += ","; d += std::to_string(c.in_index); cols.push_back(c.in_index); pl.tostr_col[c.in_index] = 1;
                c.type = to_bytes ? "string" : "utf8"; c.tf = to_bytes ? TF_BYTES : TF_UTF8;
            }
            add_desc(d + "]}");
            pl.tostr_cols.push_back(cols); pl.tostr_step_index.push_back(step_no++);
        } else {
            throw FatalError(TF_E_FATAL_UNSUPPORTED, "transformer '" + ttype + "' is not implemented by the device engine");
        }
    }
    // a filter placed after a mask of the same column would see the digest, which the fused kernel does not model
    for (size_t m = 0; m < pl.masks.size(); m++) for (size_t f = 0; f < pl.filters.size(); f++)
        if (pl.filter_step_index[f] > pl.mask_step_index[m])
            for (auto& e : pl.filters[f].exprs) for (auto& t : e) for (int c : pl.masks[m].cols)
                if (t.col == c) throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_rows on a column masked earlier in the chain is not supported");
    for (size_t m = 0; m < pl.todt_cols.size(); m++) {
        for (size_t f = 0; f < pl.filters.size(); f++) if (pl.filter_step_index[f] > pl.todt_step_index[m])
            for (auto& e : pl.filters[f].exprs) for (auto& t : e) for (int c : pl.todt_cols[m])
                if (t.col == c) throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_rows on a column converted to datetime earlier in the chain is not supported");
        for (size_t k = 0; k < pl.masks.size(); k++) for (int c : pl.masks[k].cols) for (int c2 : pl.todt_cols[m])
            if (c == c2) throw FatalError(TF_E_FATAL_UNSUPPORTED, "mask_field and convert_to_datetime on the same column are not supported together");
    }
    for (size_t m = 0; m < pl.tostr_cols.size(); m++) {
        for (size_t f = 0; f < pl.filters.size(); f++) if (pl.filter_step_index[f] > pl.tostr_step_index[m])
            for (auto& e : pl.filters[f].exprs) for (auto& t : e) for (int c : pl.tostr_cols[m])
                if (t.col == c) throw FatalError(TF_E_FATAL_UNSUPPORTED, "filter_rows on a column converted to string earlier in the chain is not supported");
        for (size_t k = 0; k < pl.masks.size(); k++) for (int c : pl.masks[k].cols) for (int c2 : pl.tostr_cols[m])
            if (c == c2) throw FatalError(TF_E_FATAL_UNSUPPORTED, "mask_field and convert_to_string on the same column are not supported together");
    }
    if (pl.has_sharder) {     // transformers placed AFTER the sharder must not change what it read (the device evaluates it on the final column forms)
        for (size_t k = 0; k < pl.shard_cols.size(); k++) {
            const int c = pl.shard_cols[k];
            for (size_t m = 0; m < pl.masks.size(); m++) if (pl.mask_step_index[m] > pl.shard_step_index) for (int mc : pl.masks[m].cols) if (mc == c)
                pl.shard_form[k] = 0;                                 // masked later: the sharder saw the value itself
            for (size_t m = 0; m < pl.todt_cols.size(); m++) if (pl.todt_step_index[m] > pl.shard_step_index) for (int tc : pl.todt_cols[m]) if (tc == c) pl.shard_form[k] = 0;
            if (pl.in_schema[c].tf == TF_ANY) for (int nc : pl.n2f_cols) if (nc == c)
                throw FatalError(TF_E_FATAL_UNSUPPORTED, "sharder_transformer over an `any` column that number_to_float rewrites is not supported");
        }
    }
    if (pl.has_splitter && pl.splitter_step != step_no - 1)
        throw FatalError(TF_E_FATAL_UNSUPPORTED, "a transformer behind table_splitter would see per-row table names: not implemented (put table_splitter last)");
    pl.out_schema = cur; pl.out_ns = cur_ns; pl.out_name = cur_name;
    for (auto& c : cur) pl.out_cols.push_back(c.in_index);
    std::string sink_desc = "null";
    if (!sink_json.empty()) {
        auto sk = tfj::parse(sink_json);
        std::string st = sk->get_str("type", "clickhouse");
        if (st != "clickhouse") throw FatalError(TF_E_FATAL_UNSUPPORTED, "sink type '" + st + "' is not implemented");
        pl.has_sink = true; pl.col_header_off.push_back(0);
        sink_desc = "{\"type\":\"clickhouse\",\"revision\":54460,\"columns\":[";
        for (size_t i = 0; i < cur.size(); i++) {
            std::string t = ch_type_of(cur[i]); pl.ch_types.push_back(t);
            put_uvarint(pl.col_headers, cur[i].name.size()); pl.col_headers.insert(pl.col_headers.end(), cur[i].name.begin(), cur[i].name.end());
            put_uvarint(pl.col_headers, t.size()); pl.col_headers.insert(pl.col_headers.end(), t.begin(), t.end());
            pl.col_headers.push_back(0);   // has-custom-serialization = false (revision >= 54454)
            pl.col_header_off.push_back((uint32_t)pl.col_headers.size());
            if (i) sink_desc += ","; sink_desc += tfj::quote(t);
        }
        sink_desc += "]}";
    }
    std::string oc = "[";
    for (size_t i = 0; i < pl.out_cols.size(); i++) { if (i) oc += ","; oc += std::to_string(pl.out_cols[i]); }
    pl.describe = "{\"table\":" + tfj::quote(ns.empty() ? name : ns + "." + name) + ",\"result_table\":" + tfj::quote(cur_ns.empty() ? cur_name : cur_ns + "." + cur_name) +
                  ",\"steps\":[" + steps_desc + "],\"out_cols\":" + oc + "],\"result_schema\":" + schema_to_json(cur) + ",\"sink\":" + sink_desc + "}";
    return pl;
}

}  // namespace tfplan
