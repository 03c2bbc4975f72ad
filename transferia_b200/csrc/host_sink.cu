// Sinker.Push as one call: the reference's sink pipeline below the user's transformers (pkg/sink_factory/sink_factory.go:79-108) over items in
// row form — transformation.Push (pkg/transformer/transformation.go:122-158,236-282) with the device running each table's chain, then
// NonRowSeparator (pkg/middlewares/nonrow_separator.go:29-55), Filter(ExcludeSystemTables) (pkg/middlewares/filter.go:60-77), the Statistician's
// counters (pkg/middlewares/statistician.go:55-68, pkg/stats/sink_wrapper.go:63-78, sink_wrapper_util.go:10-50) and the destination.
// Host-only C++ above the C-ABI of tfgpu.h: it calls tfgpu_plan / tfgpu_push_encode / tfgpu_push_columns like any other client of the library.
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/tfgpu_sink.h"
#include "plan.hpp"
#include "row_image.hpp"
#include "host_regex.hpp"
#include "host_internal.hpp"
#include <charconv>
#include <chrono>
#include <cstdio>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <thread>

namespace {

struct SinkFail { int rc; std::string msg; };

const char* kind_name(uint8_t k) {            // abstract.Kind strings (kind.go:5-43)
    switch (k) {
    case TF_KIND_INSERT: return "insert"; case TF_KIND_UPDATE: return "update"; case TF_KIND_DELETE: return "delete";
    case TF_KIND_INIT_SHARDED_TABLE_LOAD: return "init_sharded_table_load"; case TF_KIND_INIT_TABLE_LOAD: return "init_load_table";
    case TF_KIND_DONE_TABLE_LOAD: return "done_load_table"; case TF_KIND_DONE_SHARDED_TABLE_LOAD: return "done_sharded_table_load";
    case TF_KIND_DROP_TABLE: return "drop_table"; case TF_KIND_TRUNCATE: return "truncate"; case TF_KIND_DDL: return "DDL";
    case TF_KIND_PG_DDL: return "pg:DDL"; case TF_KIND_SYNCHRONIZE: return ""; default: return "\x01other";
    }
}

// what a transformer does to an item that is not a row event: skip_events may drop it, rename_tables renames it, the rest pass it through
// (filter_rows.go:110, number_to_float.go:59, mask / to_string / to_datetime touch ColumnValues of row events only)
struct HostStep {
    int type = 0;                              // 1 skip_events, 2 rename_tables, 3 table_splitter, 4 regex_replace_transformer
    std::vector<std::string> split_cols; std::string splitter;
    tfplan::NameFilter columns; std::shared_ptr<tfre::Prog> prog; tfre::Template tpl; std::shared_ptr<tfre::Machine> vm;    // type 4
    tfplan::NameFilter tables; std::set<std::string> events;
    std::vector<std::pair<std::pair<std::string, std::string>, std::pair<std::string, std::string>>> renames;
};

struct TablePlan {
    int plan_id = -1;
    std::string out_ns, out_name, insert_query;
    std::vector<std::string> col_names; std::vector<int> col_tf;      // the table's input schema (table_splitter reads values by column name)
    std::map<std::string, std::string> insert_by_table;               // INSERT statement per generated table name
    std::string aug_schema;                                           // updatable ClickHouse tables: the schema with the two system columns behind it
};

// fmt "%v" of a float = strconv 'g' with the shortest digits: exponent form when exp < -4 || exp >= 6 (ftoa.go: eprec = 6 for the shortest form)
std::string go_v_float(double v, bool is32) {
    if (v != v) return "NaN";
    if (v == 1.0 / 0.0) return "+Inf";
    if (v == -1.0 / 0.0) return "-Inf";
    char buf[64];
    auto r = is32 ? std::to_chars(buf, buf + sizeof buf, (float)v, std::chars_format::scientific) : std::to_chars(buf, buf + sizeof buf, v, std::chars_format::scientific);
    std::string sci(buf, r.ptr);                                     // d[.ddd]e[+-]XX, shortest digits that round-trip
    const size_t epos = sci.find('e');
    std::string mant = sci.substr(0, epos); const int exp = std::atoi(sci.c_str() + epos + 1);
    bool neg = false; if (!mant.empty() && mant[0] == '-') { neg = true; mant.erase(0, 1); }
    std::string digits; for (char c : mant) if (c != '.') digits += c;
    std::string out;
    if (exp < -4 || exp >= 6) {                                      // %e form: d.ddde+XX (at least two exponent digits)
        out = digits.substr(0, 1); if (digits.size() > 1) out += "." + digits.substr(1);
        char e[16]; std::snprintf(e, sizeof e, "e%c%02d", exp < 0 ? '-' : '+', exp < 0 ? -exp : exp); out += e;
    } else if (exp < 0) { out = "0." + std::string((size_t)(-exp - 1), '0') + digits; }
    else {
        if ((int)digits.size() <= exp + 1) out = digits + std::string((size_t)(exp + 1 - (int)digits.size()), '0');
        else out = digits.substr(0, (size_t)exp + 1) + "." + digits.substr((size_t)exp + 1);
    }
    return (neg ? "-" : "") + out;
}
// time.Time.UTC().Format(time.DateOnly / time.RFC3339Nano)
std::string go_time_text(int64_t sec, uint32_t nsec, bool date_only) {
    int64_t days = sec / 86400, rem = sec % 86400; if (rem < 0) { rem += 86400; days--; }
    int64_t z = days + 719468; const int64_t era = (z >= 0 ? z : z - 146096) / 146097; const unsigned doe = (unsigned)(z - era * 146097);
    const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365; int64_t y = (int64_t)yoe + era * 400;
    const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100), mp = (5 * doy + 2) / 153, d = doy - (153 * mp + 2) / 5 + 1, m = mp < 10 ? mp + 3 : mp - 9;
    if (m <= 2) y++;
    char b[64];
    if (date_only) { std::snprintf(b, sizeof b, "%04lld-%02u-%02u", (long long)y, m, d); return b; }
    std::snprintf(b, sizeof b, "%04lld-%02u-%02uT%02d:%02d:%02d", (long long)y, m, d, (int)(rem / 3600), (int)(rem / 60 % 60), (int)(rem % 60));
    std::string out = b;
    if (nsec) { char f[16]; std::snprintf(f, sizeof f, ".%09u", nsec); std::string fs = f; while (fs.back() == '0') fs.pop_back(); out += fs; }
    return out + "Z";
}
// to_string.SerializeToString (registry/to_string/to_string.go:145-172) of one boxed value for a column of YT type tf; false = a form the
// host side does not print (maps, a time.Time outside a time column, ...): the batch stays on the Go path
bool serialize_to_string(int tf, const Val& v, std::string& out) {
    switch (v.tag) {
    case TF_V_NIL: out = "<nil>"; return true;
    case TF_V_BOOL: out = v.p[0] ? "true" : "false"; return true;
    case TF_V_UINT64: { uint64_t x; std::memcpy(&x, v.p, 8); out = std::to_string(x); return true; }
    case TF_V_INT8: case TF_V_INT16: case TF_V_INT32: case TF_V_INT64: case TF_V_UINT8: case TF_V_UINT16: case TF_V_UINT32: out = std::to_string(val_i64(v)); return true;
    case TF_V_FLOAT32: { float f; std::memcpy(&f, v.p, 4); out = go_v_float(f, true); return true; }
    case TF_V_FLOAT64: { double f; std::memcpy(&f, v.p, 8); out = go_v_float(f, false); return true; }
    case TF_V_STRING: case TF_V_JSONNUM: out.assign((const char*)v.p, v.n); return true;
    case TF_V_BYTES: if (tf == TF_BYTES) { out.assign((const char*)v.p, v.n); return true; } return false;          // %v of a []byte elsewhere prints the byte list
    case TF_V_TIME: {
        int64_t sec; uint32_t ns; std::memcpy(&sec, v.p, 8); std::memcpy(&ns, v.p + 8, 4);
        if (tf == TF_DATE) { out = go_time_text(sec, ns, true); return true; }
        if (tf == TF_DATETIME || tf == TF_TIMESTAMP) { out = go_time_text(sec, ns, false); return true; }
        return false;
    }
    default: return false;
    }
}

}  // namespace

struct tfgpu_sink {
    tfgpu_engine* e = nullptr;
    std::string err, transformers_json, sink_json, database, debezium_opts;
    bool has_transformers = false, needs_device = false, errors_to_sink = true, exclude_sys = true, updateable = false;
    int wire_fmt = 0;
    std::set<std::string> system_tables;
    std::vector<HostStep> host_steps;
    bool regex_on_columns = false;             // this push: the replace steps run on the transposed text columns (push_rows) instead of the row image
    tf_sink_fn fn = nullptr; void* ctx = nullptr; tfgpu_ch_conn* ch = nullptr;
    tfgpu_columnar* pool = nullptr;
    std::map<std::string, TablePlan> plans;
    tf_sink_stats st{};
    // delivery gate (tfgpu_dispatcher): entered before the first downstream delivery of a push, left when the push is over
    void (*gate_enter)(void*) = nullptr; void (*gate_leave)(void*) = nullptr; void* gate_ctx = nullptr; bool in_gate = false;

    TablePlan& plan_for(const tf_table& t) {
        std::string key = std::string(t.schema ? t.schema : "") + '\0' + (t.table ? t.table : "") + '\0' + (t.schema_json ? t.schema_json : "");
        auto it = plans.find(key);
        if (it != plans.end()) return it->second;
        TablePlan tp;
        const std::string ns = t.schema ? t.schema : "", name = t.table ? t.table : "";
        const bool want_sink = wire_fmt == TF_WIRE_CH_NATIVE || wire_fmt == TF_WIRE_CH_NATIVE_LZ4 || wire_fmt == TF_WIRE_CH_JSONEACHROW ||
                               wire_fmt == (TF_WIRE_CH_JSONEACHROW | TF_WIRE_F_ZSTD);
        tfplan::Plan pl;
        std::string schema_text = t.schema_json ? t.schema_json : "[]";
        if (updateable) {
            // sink_table.go:633-650: an updatable table takes `__data_transfer_commit_time` and `__data_transfer_delete_time` (UInt64) behind its columns
            const size_t close = schema_text.rfind(']');
            if (close == std::string::npos) throw SinkFail{TF_E_FATAL_CONFIG, "schema_json is not an array"};
            const bool empty = schema_text.find('{') == std::string::npos;
            schema_text = schema_text.substr(0, close) + (empty ? "" : ",") +
                "{\"name\":\"__data_transfer_commit_time\",\"type\":\"uint64\",\"required\":true},{\"name\":\"__data_transfer_delete_time\",\"type\":\"uint64\",\"required\":true}]";
            tp.aug_schema = schema_text;
        }
        try { pl = tfplan::build_plan(ns, name, schema_text, transformers_json, want_sink ? sink_json : ""); }
        catch (const tfplan::FatalError& f) { throw SinkFail{f.code, std::string("unable to add table plan: ") + f.what()}; }
        catch (const std::exception& x) { throw SinkFail{TF_E_FATAL_CONFIG, std::string("unable to add table plan: ") + x.what()}; }
        tp.out_ns = pl.out_ns.empty() && pl.out_name.empty() ? ns : pl.out_ns; tp.out_name = pl.out_name.empty() ? name : pl.out_name;
        for (auto& c : pl.in_schema) { tp.col_names.push_back(c.name); tp.col_tf.push_back(c.tf); }
        if (e && (needs_device || wire_fmt)) {
            const int rc = tfgpu_plan(e, ns.c_str(), name.c_str(), schema_text.c_str(), transformers_json.c_str(), want_sink ? sink_json.c_str() : nullptr, &tp.plan_id);
            if (rc) throw SinkFail{rc, std::string("unable to add table plan: ") + tfgpu_last_error(e)};
        }
        {
            std::string cols = "[";
            for (size_t i = 0; i < pl.out_schema.size(); i++) cols += (i ? "," : "") + tfj::quote(pl.out_schema[i].name);
            tp.insert_query = cols + "]";                      // the column list; the statement is built per destination table name (insert_for)
        }
        return plans.emplace(std::move(key), std::move(tp)).first->second;
    }

    const std::string& insert_for(TablePlan& tp, const std::string& table_name) {
        auto it = tp.insert_by_table.find(table_name);
        if (it != tp.insert_by_table.end()) return it->second;
        std::vector<char> q(tp.insert_query.size() + table_name.size() + database.size() + 256);
        const int64_t n = tfgpu_ch_insert_query(database.c_str(), table_name.c_str(), tp.insert_query.c_str(), 0 /* the plan's schema already lists the system columns */, q.data(), q.size());
        if (n < 0) throw SinkFail{(int)n, "cannot build the INSERT statement"};
        return tp.insert_by_table.emplace(table_name, std::string(q.data(), (size_t)n)).first->second;
    }

    // a non-row item through the transformer list: false = dropped by skip_events; the table id it leaves with in (ns, name)
    bool host_chain(const std::string& orig_ns, const std::string& orig_name, uint8_t kind, std::string& ns, std::string& name, const TablePlan* tp) const {
        ns = orig_ns; name = orig_name;
        for (const HostStep& h : host_steps) {
            if (h.type == 1) { if (tfplan::match_table(h.tables, orig_ns, orig_name) && h.events.count(kind_name(kind))) return false; }
            else if (h.type == 3) {
                // GenerateTableName over an item without values (table_splitter.go:36-58): AsMap() is empty, every listed column the schema knows
                // contributes SerializeToString(nil) = "<nil>"
                if (!tfplan::match_table(h.tables, orig_ns, orig_name) || !tp) continue;
                std::vector<std::string> parts; if (!name.empty()) parts.push_back(name);
                for (auto& cn : h.split_cols) for (auto& have : tp->col_names) if (have == cn) { parts.push_back("<nil>"); break; }
                std::string j; for (size_t i = 0; i < parts.size(); i++) j += (i ? h.splitter : "") + parts[i];
                name = j;
            }
            else {
                bool suitable = false; for (auto& r : h.renames) if (r.first.first == orig_ns && r.first.second == orig_name) suitable = true;   // Suitable on the original id
                if (!suitable) continue;
                for (auto& r : h.renames) if (r.first.first == ns && r.first.second == name) { const auto to = r.second; ns = to.first; name = to.second; }   // last entry wins (map built from the list)
            }
        }
        return true;
    }

    int deliver(const tf_sink_event& ev, const tf_rows* rows, TablePlan* tp) {
        int rc = 0;
        if (gate_enter && !in_gate) { gate_enter(gate_ctx); in_gate = true; }
        if (ev.type == TF_SINK_EV_ROWS && ch && ev.wire) {
            rc = tfgpu_ch_insert_begin(ch, insert_for(*tp, ev.out_table).c_str(), "", nullptr);
            if (!rc) rc = tfgpu_ch_insert_data(ch, ev.wire, ev.wire_len);
            if (!rc) rc = tfgpu_ch_insert_end(ch, nullptr, nullptr);
            if (rc) throw SinkFail{rc, std::string("clickhouse: ") + tfgpu_ch_last_error(ch)};
        } else if (fn) {
            rc = fn(ctx, &ev);
            if (rc) throw SinkFail{rc, "the downstream Push failed"};
        }
        // Statistician: counted after the downstream Push succeeded (statistician.go:60-66)
        st.downstream_pushes++; st.change_items_pushed += ev.n_items; st.wire_bytes += ev.wire_len; st.metering_output_rows += ev.n_items;
        if (ev.type != TF_SINK_EV_ITEM) st.row_events_pushed += ev.n_items;
        if (ev.item_idx) for (uint64_t k = 0; k < ev.n_items; k++) {
            const tf_item& it = rows->items[ev.item_idx[k]];
            if (!(TF_KIND_IS_ROW(it.kind) || it.kind == TF_KIND_SYNCHRONIZE)) continue;              // batchStats :16-18
            st.inflight_bytes += it.size_values;
            if (!it.commit_time) { st.without_commit_time++; continue; }
            if (!st.max_commit_time || it.commit_time > st.max_commit_time) st.max_commit_time = it.commit_time;
            if (!st.min_commit_time || it.commit_time < st.min_commit_time) st.min_commit_time = it.commit_time;
        }
        return 0;
    }

    // one maximal run of row events of one (table, schema): what the host-level steps do to it (skip_events without a device plan,
    // table_splitter's per-row table names), then every group of rows that shares a destination table goes down on its own
    void push_run(const tf_rows* rows, uint32_t table, const std::vector<uint64_t>& idx_in, TablePlan& tp) {
        if (idx_in.empty()) return;
        const tf_table& t = rows->tables[table];
        const std::string ons = t.schema ? t.schema : "", oname = t.table ? t.table : "";
        std::vector<uint64_t> kept; const std::vector<uint64_t>* idx = &idx_in;
        if (tp.plan_id < 0) {                                   // no device plan: skip_events drops row kinds here (skip_events.go:52-62)
            for (const HostStep& h : host_steps) if (h.type == 1 && tfplan::match_table(h.tables, ons, oname)) {
                std::vector<uint64_t> nxt;
                for (uint64_t i : *idx) { if (h.events.count(kind_name(rows->items[i].kind))) st.transform_dropped++; else nxt.push_back(i); }
                kept.swap(nxt); idx = &kept;
            }
            if (idx->empty()) return;
        }
        const HostStep* sp = nullptr;
        for (const HostStep& h : host_steps) if (h.type == 3 && tfplan::match_table(h.tables, ons, oname)) sp = &h;       // the plan keeps table_splitter last: at most one applies
        if (!sp) { push_rows(rows, table, *idx, tp, tp.out_name); return; }
        // GenerateTableName (table_splitter.go:36-58): current table name, then SerializeToString of every listed column the schema knows
        std::vector<int> cols;                                  // schema index of every split column (in the configured order)
        for (auto& cn : sp->split_cols) for (size_t c = 0; c < tp.col_names.size(); c++) if (tp.col_names[c] == cn) { cols.push_back((int)c); break; }
        int max_col = -1; for (int c : cols) max_col = std::max(max_col, c);
        std::vector<std::pair<std::string, std::vector<uint64_t>>> groups; std::map<std::string, size_t> where;
        const uint8_t* vend = rows->values + rows->values_len;
        std::vector<Val> vals(tp.col_names.size()); std::vector<uint8_t> have(tp.col_names.size());
        for (uint64_t i : *idx) {
            const tf_item& it = rows->items[i];
            std::fill(have.begin(), have.end(), 0);
            const uint8_t* at = rows->values + it.values_off; const bool sparse = it.flags & TF_ITEM_SPARSE;
            for (uint32_t k = 0; k < it.n_values && max_col >= 0; k++) {
                uint32_t c = k;
                if (sparse) { if (vend - at < 2) throw SinkFail{TF_E_FATAL_ARG, "truncated value image"}; uint16_t ci; std::memcpy(&ci, at, 2); at += 2; c = ci; }
                Val v; if (!read_val(at, vend, v)) throw SinkFail{TF_E_FATAL_ARG, "malformed value image"};
                if (c < vals.size()) { vals[c] = v; have[c] = 1; }
                if (!sparse && (int)c >= max_col) break;
            }
            std::string name = tp.out_name.empty() ? "" : tp.out_name; bool first = tp.out_name.empty();
            for (int c : cols) {
                std::string text; Val nil{TF_V_NIL, nullptr, 0};
                if (!serialize_to_string(tp.col_tf[c], have[c] ? vals[c] : nil, text))
                    throw SinkFail{TF_E_FATAL_UNSUPPORTED, "table_splitter: a value of column '" + tp.col_names[c] + "' has a form the host side does not print"};
                if (!first) name += sp->splitter; name += text; first = false;
            }
            auto w = where.find(name);
            if (w == where.end()) { w = where.emplace(name, groups.size()).first; groups.emplace_back(name, std::vector<uint64_t>()); }
            groups[w->second].second.push_back(i);
        }
        for (auto& g : groups) push_rows(rows, table, g.second, tp, g.first);
    }

    // rows of one destination table: transformers + encode on the device, then downstream
    void push_rows(const tf_rows* rows, uint32_t table, const std::vector<uint64_t>& idx, TablePlan& tp, const std::string& out_name) {
        const uint64_t n = idx.size();
        if (!n) return;
        tf_sink_event ev{}; ev.table = table; ev.out_schema = tp.out_ns.c_str(); ev.out_table = out_name.c_str(); ev.plan_id = tp.plan_id;
        if (exclude_sys && system_tables.count(out_name)) { st.filter_dropped += n; return; }           // ChangeItem.IsSystemTable looks at Table only
        const tf_batch* batch = nullptr; const tf_row_meta* meta = nullptr; const tf_old_keys* old = nullptr;
        int rc;
        if (updateable) {
            // buildChangeItemArgs (sink_table.go:411-432) on the row image: an insert keeps its values and gets (CommitTime, 0) behind them; a delete
            // is rebuilt from OldKeys (buildDeleteKindArgs :397-409: the key columns' old values, nil for the rest — insert_null_as_default fills them
            // on the server) with (CommitTime, CommitTime). Updates need Collapse and the toast lookup of doOperation (:618-626): Go sink.
            const uint32_t ncols = (uint32_t)tp.col_names.size() - 2;
            std::vector<tf_item> aitems(n); std::vector<uint8_t> avals; avals.reserve((size_t)n * 64);
            const uint8_t* vend = rows->values + rows->values_len;
            auto put_u64 = [&](uint64_t v) { avals.push_back(TF_V_UINT64); const uint8_t* b = (const uint8_t*)&v; avals.insert(avals.end(), b, b + 8); };
            auto put_idx = [&](uint16_t c) { const uint8_t* b = (const uint8_t*)&c; avals.insert(avals.end(), b, b + 2); };
            for (uint64_t j = 0; j < n; j++) {
                const tf_item& it = rows->items[idx[j]]; tf_item& a = aitems[j]; a = it;
                a.table = 0; a.kind = TF_KIND_INSERT; a.old_keys_off = UINT64_MAX; a.values_off = avals.size();
                if (it.kind == TF_KIND_INSERT) {
                    if ((it.flags & TF_ITEM_SPARSE) || it.n_values != ncols) throw SinkFail{TF_E_FATAL_UNSUPPORTED, "updatable table: an insert with a column subset needs the Go sink"};
                    const uint8_t* at = rows->values + it.values_off; const uint8_t* p = at;
                    for (uint32_t k = 0; k < ncols; k++) { Val v; if (!read_val(p, vend, v)) throw SinkFail{TF_E_FATAL_ARG, "malformed value image"}; }
                    avals.insert(avals.end(), at, p); put_u64(it.commit_time); put_u64(0);
                    a.n_values = ncols + 2; a.flags = 0;
                } else if (it.kind == TF_KIND_DELETE) {
                    if (it.old_keys_off == UINT64_MAX || it.old_keys_off + 2 > rows->values_len) throw SinkFail{TF_E_FATAL_UNSUPPORTED, "updatable table: a delete without OldKeys"};
                    const uint8_t* p = rows->values + it.old_keys_off; uint16_t cnt; std::memcpy(&cnt, p, 2); p += 2; const uint8_t* at = p;
                    for (uint16_t k = 0; k < cnt; k++) { if (vend - p < 2) throw SinkFail{TF_E_FATAL_ARG, "truncated OldKeys image"}; uint16_t c; std::memcpy(&c, p, 2); p += 2; Val v; if (c >= ncols || !read_val(p, vend, v)) throw SinkFail{TF_E_FATAL_ARG, "malformed OldKeys image"}; }
                    avals.insert(avals.end(), at, p);                                        // {u16 column, value}*: already the sparse row form
                    put_idx((uint16_t)ncols); put_u64(it.commit_time); put_idx((uint16_t)(ncols + 1)); put_u64(it.commit_time);
                    a.n_values = (uint32_t)cnt + 2; a.flags = TF_ITEM_SPARSE;
                } else throw SinkFail{TF_E_FATAL_UNSUPPORTED, "updatable table: update items go through abstract.Collapse and the toast lookup of the Go sink (sink_table.go:618-626)"};
            }
            avals.push_back(0);
            tf_table at_{rows->tables[table].schema, rows->tables[table].table, tp.aug_schema.c_str()};
            tf_rows ar{}; ar.n_items = n; ar.items = aitems.data(); ar.n_tables = 1; ar.tables = &at_; ar.values = avals.data(); ar.values_len = avals.size() - 1;
            ar.strings = rows->strings; ar.strings_len = rows->strings_len;
            rc = tfgpu_rows_to_batch(pool, &ar, 0, nullptr, 0, 0, &batch, &meta, &old);
        } else rc = tfgpu_rows_to_batch(pool, rows, table, idx.data(), n, 0, &batch, &meta, &old);
        if (rc) throw SinkFail{rc, std::string("transpose: ") + tfgpu_columnar_last_error(pool)};
        Rewritten rw_run;
        if (regex_on_columns) {
            const std::string name = rows->tables[table].table ? rows->tables[table].table : "";
            std::vector<std::vector<const HostStep*>> by_col(tp.col_names.size()); bool mixed = false;
            for (const HostStep& h : host_steps) if (h.type == 4 && h.tables.match(name))
                for (size_t c = 0; c < tp.col_names.size(); c++) if ((tp.col_tf[c] == TF_UTF8 || tp.col_tf[c] == TF_BYTES) && h.columns.match(tp.col_names[c])) {
                    by_col[c].push_back(&h); mixed |= tfgpu_columnar_text_was_mixed(pool, (uint32_t)c);
                }
            if (mixed) {
                // a []byte inside a utf8 column (or a string inside a `string` column) fails the transformer's type assertion and stays as it is:
                // only the row image knows which cells those are
                if (regex_rewrite(rows, rw_run)) rc = tfgpu_rows_to_batch(pool, &rw_run.rows, table, idx.data(), n, 0, &batch, &meta, &old);
                if (rc) throw SinkFail{rc, std::string("transpose: ") + tfgpu_columnar_last_error(pool)};
            } else for (size_t c = 0; c < by_col.size(); c++) {
                if (by_col[c].empty()) continue;
                const std::vector<const HostStep*>& steps = by_col[c];
                rc = tfgpu_columnar_rewrite_text(pool, (uint32_t)c, [&steps]() -> tf_text_fn {
                    auto vms = std::make_shared<std::vector<tfre::Machine>>(); for (const HostStep* h : steps) vms->emplace_back(*h->prog);
                    auto tmp = std::make_shared<std::string>();
                    return [vms, tmp, &steps](const uint8_t* p, uint32_t len, std::string& out) {
                        const uint8_t* src = p; size_t n = len;
                        for (size_t k = 0; k < steps.size(); k++) {
                            std::string& dst = (k & 1) ? *tmp : out;
                            tfre::replace_all((*vms)[k], steps[k]->tpl, src, n, dst); src = (const uint8_t*)dst.data(); n = dst.size();
                        }
                        if (!(steps.size() & 1)) out.swap(*tmp);                  // an even number of steps left the result in tmp
                    };
                }, 0);
                if (rc) throw SinkFail{rc, std::string("regex_replace: ") + tfgpu_columnar_last_error(pool)};
            }
        }
        if (tp.plan_id < 0) {                                                                           // no transformers, columnar hand-over
            ev.type = TF_SINK_EV_ROWS; ev.n_items = n; ev.item_idx = idx.data(); ev.batch = batch;
            deliver(ev, rows, &tp); return;
        }
        tfgpu_result* res = nullptr;
        if (wire_fmt == TF_WIRE_DEBEZIUM)       // queue Debezium serializer: every row kind, OldKeys and the source block's fields from the transposer
            rc = tfgpu_emit_debezium_crud(e, tp.plan_id, debezium_opts.c_str(), batch, old, meta, &res);
        else
            rc = wire_fmt ? tfgpu_push_encode(e, tp.plan_id, wire_fmt, batch, &res) : tfgpu_push_columns(e, tp.plan_id, batch, &res);
        if (rc) throw SinkFail{rc, std::string("device: ") + tfgpu_last_error(e)};
        struct Release { tfgpu_result* r; ~Release() { tfgpu_result_release(r); } } guard{res};
        const uint64_t n_out = tfgpu_result_rows_out(res), n_err = tfgpu_result_n_errors(res);
        st.transform_dropped += n - n_out; st.transform_errors += n_err;
        if (n_err) {
            if (wire_fmt && n_err) {                                                                      // a sink format refuses some rows outright (UPDATE / DELETE kinds): the Go sink must take the run
                const tf_rowerr* er = tfgpu_result_errors(res);
                for (uint64_t k = 0; k < n_err; k++) if (er[k].code == TF_ROWERR_SINK_KIND_HOST || er[k].code == TF_ROWERR_SER_VALUE)
                    throw SinkFail{TF_E_FATAL_UNSUPPORTED, "a row of this run needs the Go sink (update / delete kind or a value the wire format refuses)"};
            }
            if (errors_to_sink) {                                                                         // pushErrors before the transformed items (transformation.go:152-157)
                std::vector<uint64_t> eidx(n_err); std::vector<tf_rowerr> errs(tfgpu_result_errors(res), tfgpu_result_errors(res) + n_err);
                for (uint64_t k = 0; k < n_err; k++) { eidx[k] = idx[errs[k].row]; errs[k].row = (uint32_t)k; }
                tf_sink_event ee = ev; ee.type = TF_SINK_EV_ERRORS; ee.n_items = n_err; ee.item_idx = eidx.data(); ee.errors = errs.data();
                deliver(ee, rows, &tp);
            }
        }
        if (!n_out) return;                                                                              // filter.go:73-75 / an empty Push is not forwarded
        ev.type = TF_SINK_EV_ROWS; ev.n_items = n_out; ev.item_idx = n_out == n ? idx.data() : nullptr;
        if (wire_fmt) { ev.wire = tfgpu_result_bytes(res); ev.wire_len = tfgpu_result_bytes_len(res); ev.raw_len = tfgpu_result_raw_len(res); ev.n_frames = tfgpu_result_n_frames(res); ev.msg_sizes = wire_fmt == TF_WIRE_DEBEZIUM ? tfgpu_result_dbz_msg_sizes(res) : nullptr; }
        else ev.batch = tfgpu_result_batch(res);
        deliver(ev, rows, &tp);
    }

    // regex_replace_transformer (registry/regex_replace/transformer.go:87-142) over the row image, before anything else looks at the values
    // (the plan keeps these steps at the head of the chain): every row event of a table the step's table filter takes gets its string values
    // (schema type utf8 holding a Go string) and []byte values (schema type string) of the matched columns replaced. The type is read at the
    // value's POSITION in the item (`item.TableSchema.Columns()[i]`, :108), the name from ColumnNames — they differ for an item that carries
    // a column subset. The image is copied once with the rewritten value lists appended; OldKeys are not touched by Apply.
    struct Rewritten { tf_rows rows; std::vector<tf_item> items; std::vector<uint8_t> values; };
    bool regex_rewrite(const tf_rows* in, Rewritten& out) {
        bool any = false; for (const HostStep& h : host_steps) if (h.type == 4) any = true;
        if (!any) return false;
        struct PerTable { bool looked = false; std::vector<std::vector<const HostStep*>> by_col; const TablePlan* tp = nullptr; bool hit = false; };
        std::vector<PerTable> per(in->n_tables);
        out.values.reserve((size_t)in->values_len * 2 + 4096);
        out.values.assign(in->values, in->values + in->values_len);
        out.items.assign(in->items, in->items + in->n_items);
        const uint8_t* vend = in->values + in->values_len;
        std::string a, b; const auto t_begin = std::chrono::steady_clock::now(); double rx_ns = 0; const bool trace = std::getenv("TFGPU_SINK_TRACE") != nullptr;
        for (uint64_t i = 0; i < in->n_items; i++) {
            const tf_item& it = in->items[i];
            if (!TF_KIND_IS_ROW(it.kind)) continue;
            if (it.table >= in->n_tables) throw SinkFail{TF_E_FATAL_ARG, "item names a table outside tf_rows.tables"};
            PerTable& pt = per[it.table];
            if (!pt.looked) {
                pt.looked = true;
                const tf_table& t = in->tables[it.table]; const std::string name = t.table ? t.table : "";
                pt.tp = &plan_for(t); pt.by_col.resize(pt.tp->col_names.size());
                for (const HostStep& h : host_steps) if (h.type == 4 && h.tables.match(name))
                    for (size_t c = 0; c < pt.tp->col_names.size(); c++) if (h.columns.match(pt.tp->col_names[c])) { pt.by_col[c].push_back(&h); pt.hit = true; }
            }
            if (!pt.hit || !it.n_values) continue;
            if (it.values_off > in->values_len) throw SinkFail{TF_E_FATAL_ARG, "values offset outside the image"};
            const uint8_t* at = in->values + it.values_off; const bool sparse = it.flags & TF_ITEM_SPARSE;
            const uint64_t new_off = out.values.size();
            const uint8_t* run = at;                             // bytes of the list not yet copied: untouched values go over in one piece
            for (uint32_t k = 0; k < it.n_values; k++) {
                uint32_t c = k;
                if (sparse) { if (vend - at < 2) throw SinkFail{TF_E_FATAL_ARG, "truncated value image"}; uint16_t ci; std::memcpy(&ci, at, 2); at += 2; c = ci; }
                const uint8_t* v0 = at; Val v; if (!read_val(at, vend, v)) throw SinkFail{TF_E_FATAL_ARG, "malformed value image"};
                const int typ = k < pt.tp->col_tf.size() ? pt.tp->col_tf[k] : -1;
                const bool takes = c < pt.by_col.size() && !pt.by_col[c].empty() && ((typ == TF_UTF8 && v.tag == TF_V_STRING) || (typ == TF_BYTES && v.tag == TF_V_BYTES));
                if (!takes) continue;
                out.values.insert(out.values.end(), run, v0); run = at;        // (the column index of a sparse value lies before v0: copied with the run)
                a.assign((const char*)v.p, v.n);
                const auto t0 = trace ? std::chrono::steady_clock::now() : std::chrono::steady_clock::time_point();
                for (const HostStep* h : pt.by_col[c]) { tfre::replace_all(*h->vm, h->tpl, (const uint8_t*)a.data(), a.size(), b); a.swap(b); }
                if (trace) rx_ns += std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t0).count();
                if (a.size() > 0xffffffffull) throw SinkFail{TF_E_FATAL_UNSUPPORTED, "regex_replace_transformer: a value grew past 4 GiB"};
                const uint32_t len = (uint32_t)a.size();
                out.values.push_back((uint8_t)v.tag); out.values.insert(out.values.end(), (const uint8_t*)&len, (const uint8_t*)&len + 4);
                out.values.insert(out.values.end(), a.begin(), a.end());
            }
            out.values.insert(out.values.end(), run, at);
            out.items[i].values_off = new_off;
        }
        if (std::getenv("TFGPU_SINK_TRACE")) fprintf(stderr, "[sink] regex step: %.2f ms over %llu items (%.2f ms inside ReplaceAll)\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count(), (unsigned long long)in->n_items, rx_ns / 1e6);
        out.values.push_back(0);
        out.rows = *in; out.rows.items = out.items.data(); out.rows.values = out.values.data(); out.rows.values_len = out.values.size() - 1;
        return true;
    }

    void push(const tf_rows* rows) {
        st.pushes++; st.max_commit_time = st.min_commit_time = 0;
        // regex_replace steps: on the transposed text columns when that is the same thing (every row event lists all its columns, so the
        // type-by-position rule of transformer.go:108 is the column's type, and nothing reads the values before the transposer does);
        // else on the row image up front
        Rewritten rw; regex_on_columns = false;
        bool has_regex = false, has_splitter = false;
        for (const HostStep& h : host_steps) { has_regex |= h.type == 4; has_splitter |= h.type == 3; }
        if (has_regex) {
            bool dense = !has_splitter && !std::getenv("TFGPU_REGEX_ON_ROWS");
            for (uint64_t i = 0; dense && i < rows->n_items; i++) if (TF_KIND_IS_ROW(rows->items[i].kind) && (rows->items[i].flags & TF_ITEM_SPARSE)) dense = false;
            if (dense) regex_on_columns = true;
            else if (regex_rewrite(rows, rw)) rows = &rw.rows;
        }
        // SplitByTableID (utils.go:130-136): groups in order of first appearance, items in input order
        std::vector<std::pair<std::string, std::vector<uint64_t>>> groups; std::map<std::string, size_t> where;
        for (uint64_t i = 0; i < rows->n_items; i++) {
            const tf_item& it = rows->items[i];
            if (it.table >= rows->n_tables) throw SinkFail{TF_E_FATAL_ARG, "item names a table outside tf_rows.tables"};
            const tf_table& t = rows->tables[it.table];
            std::string id = std::string(t.schema ? t.schema : "") + '\0' + (t.table ? t.table : "");
            auto w = where.find(id);
            if (w == where.end()) { w = where.emplace(id, groups.size()).first; groups.emplace_back(id, std::vector<uint64_t>()); }
            groups[w->second].second.push_back(i);
        }
        std::vector<uint64_t> run;
        for (auto& g : groups) {
            uint32_t run_table = 0; TablePlan* run_plan = nullptr;
            auto flush = [&] { if (!run.empty()) { push_run(rows, run_table, run, *run_plan); run.clear(); } };
            for (uint64_t i : g.second) {
                const tf_item& it = rows->items[i];
                const tf_table& t = rows->tables[it.table];
                if (TF_KIND_IS_ROW(it.kind)) {
                    if (!run.empty() && it.table != run_table) flush();                                   // another TableSchema of the same table: its own plan (transformation.go:243-277)
                    if (run.empty()) { run_table = it.table; run_plan = &plan_for(t); }
                    run.push_back(i); continue;
                }
                std::string ns, name;
                // DDL / drop / truncate items may come without a TableSchema: only table_splitter looks at it (which columns it knows)
                const TablePlan* tpp = nullptr;
                if (t.schema_json && t.schema_json[0] && std::strcmp(t.schema_json, "[]") != 0) for (const HostStep& h : host_steps) if (h.type == 3) { tpp = &plan_for(t); break; }
                if (!host_chain(t.schema ? t.schema : "", t.table ? t.table : "", it.kind, ns, name, tpp)) { st.transform_dropped++; continue; }   // the run is NOT cut: the item is gone before NonRowSeparator sees it
                flush();                                                                                  // nonrow_separator.go:38-47
                if (exclude_sys && system_tables.count(name)) { st.filter_dropped++; continue; }
                tf_sink_event ev{}; ev.type = TF_SINK_EV_ITEM; ev.table = it.table; ev.out_schema = ns.c_str(); ev.out_table = name.c_str();
                ev.n_items = 1; ev.item_idx = &i; ev.plan_id = -1;
                deliver(ev, rows, nullptr);
            }
            flush();
        }
    }
};

extern "C" {

int tfgpu_sink_create(tfgpu_engine* e, const char* cfg_json, tfgpu_sink** out) {
    if (!out) return TF_E_FATAL_ARG;
    *out = nullptr;
    auto s = std::make_unique<tfgpu_sink>();
    try {
        tfj::ValuePtr cfg = tfj::parse(cfg_json && *cfg_json ? cfg_json : "{}");
        s->e = e; s->wire_fmt = (int)cfg->get_num("wire_fmt", 0);
        const tfj::Value* trs = cfg->get("transformers");
        s->has_transformers = trs && trs->kind == tfj::Value::Arr && !trs->arr.empty();
        if (s->has_transformers) for (auto& tr : trs->arr) if (tr->kind == tfj::Value::Obj) for (auto& kv : tr->obj)
            if (kv.first != "transformerId" && kv.first != "skip_events" && kv.first != "rename_tables" && kv.first != "table_splitter" && kv.first != "regex_replace_transformer") s->needs_device = true;
        // skip_events / rename_tables / table_splitter act on kinds and table names only: with wire_fmt 0 they run on the host alone; every
        // other transformer and every wire format computes on the device — nothing here computes on the CPU in its place
        if ((s->needs_device || s->wire_fmt) && !e) return TF_E_FATAL_NODEVICE;
        // the transformer list, re-serialised for tfgpu_plan, and its effect on non-row items
        std::string tj = "[";
        if (s->has_transformers) {
            // the caller's text is passed on verbatim: find the array in cfg_json by re-reading it with the same parser the plans use
            const std::string src = cfg_json; const size_t k = src.find("\"transformers\"");
            size_t a = src.find('[', k), depth = 0, b = a; bool in_str = false;
            for (; b < src.size(); b++) {
                const char c = src[b];
                if (in_str) { if (c == '\\') b++; else if (c == '"') in_str = false; continue; }
                if (c == '"') in_str = true; else if (c == '[') depth++; else if (c == ']' && --depth == 0) break;
            }
            tj = src.substr(a, b - a + 1);
            for (auto& tr : trs->arr) {
                if (tr->kind != tfj::Value::Obj) continue;
                for (auto& kv : tr->obj) {
                    const tfj::Value* c = kv.second.get();
                    if (kv.first == "skip_events") { HostStep h; h.type = 1; h.tables = tfplan::tables_filter(c->get("tables")); for (auto& ev : c->get_str_list("events")) h.events.insert(ev); s->host_steps.push_back(std::move(h)); }
                    else if (kv.first == "table_splitter") {
                        HostStep h; h.type = 3; h.tables = tfplan::tables_filter(c->get("tables")); h.split_cols = c->get_str_list("columns");
                        h.splitter = c->get_str("splitter", ""); if (h.splitter.empty()) h.splitter = "/";      // defaultSplitter table_splitter.go:17,48-50
                        if (c->get_bool("useLegacyLf")) return TF_E_FATAL_UNSUPPORTED;
                        s->host_steps.push_back(std::move(h));
                    }
                    else if (kv.first == "regex_replace_transformer") {
                        // regexp.Compile(cfg.RegexMatch) + the two filters, transformer.go:18-41: a bad expression fails the construction
                        HostStep h; h.type = 4; h.tables = tfplan::tables_filter(c->get("tables"));
                        const tfj::Value* cc = c->get("columns");
                        h.columns = tfplan::make_filter(cc ? cc->get_str_list("includeColumns") : std::vector<std::string>(), cc ? cc->get_str_list("excludeColumns") : std::vector<std::string>());
                        try {
                            h.prog = std::make_shared<tfre::Prog>(tfre::compile(c->get_str("regexMatch", "")));
                            h.tpl = tfre::parse_template(c->get_str("replaceRule", ""), *h.prog);
                        } catch (const tfre::Unsupported&) { return TF_E_FATAL_UNSUPPORTED; }
                        h.vm = std::make_shared<tfre::Machine>(*h.prog);
                        s->host_steps.push_back(std::move(h));
                    }
                    else if (kv.first == "rename_tables") {
                        HostStep h; h.type = 2; const tfj::Value* lst = c->get("renameTables");
                        if (lst && lst->kind == tfj::Value::Arr) for (auto& r : lst->arr) {
                            const tfj::Value* o = r->get("originalName"); const tfj::Value* nw = r->get("newName");
                            if (o && nw) h.renames.push_back({{o->get_str("nameSpace"), o->get_str("name")}, {nw->get_str("nameSpace"), nw->get_str("name")}});
                        }
                        s->host_steps.push_back(std::move(h));
                    }
                }
            }
        } else tj = "[]";
        for (size_t at = 0; (at = tj.find("\"table_splitter\"", at)) != std::string::npos; at += 22) tj.replace(at, 16, "\"table_splitter@sink\"");   // see plan.hpp: the unmarked form is refused
        for (size_t at = 0; (at = tj.find("\"regex_replace_transformer\"", at)) != std::string::npos; at += 32) tj.replace(at, 27, "\"regex_replace_transformer@sink\"");
        s->transformers_json = tj;
        if (s->wire_fmt == TF_WIRE_DEBEZIUM) {               // the emitter's options are passed on verbatim (tfgpu_emit_debezium's opts_json)
            const std::string src = cfg_json ? cfg_json : ""; const size_t k = src.find("\"debezium\"");
            if (k == std::string::npos) return TF_E_FATAL_CONFIG;
            size_t a = src.find('{', k), depth = 0, b = a; bool in_str = false;
            for (; a != std::string::npos && b < src.size(); b++) {
                const char c = src[b];
                if (in_str) { if (c == '\\') b++; else if (c == '"') in_str = false; continue; }
                if (c == '"') in_str = true; else if (c == '{') depth++; else if (c == '}' && --depth == 0) break;
            }
            if (a == std::string::npos || b >= src.size()) return TF_E_FATAL_CONFIG;
            s->debezium_opts = src.substr(a, b - a + 1);
        }
        s->sink_json = "{\"type\":\"clickhouse\"}";
        s->database = cfg->get_str("database", "default"); s->updateable = cfg->get_bool("updateable", false);
        if (s->updateable && s->has_transformers) return TF_E_FATAL_UNSUPPORTED;      // the system columns are the SINK's: a chain over the augmented schema would see them
        s->errors_to_sink = cfg->get_str("errors_output", "sink") != "devnull";
        s->exclude_sys = cfg->get_bool("exclude_system_tables", true);
        for (auto& t : cfg->get_str_list("system_tables")) s->system_tables.insert(t);
        const int rc = tfgpu_columnar_create(&s->pool); if (rc) return rc;
    } catch (const std::exception& x) { return TF_E_FATAL_CONFIG; }
    *out = s.release();
    return TF_OK;
}

int64_t tfgpu_regex_replace_all(const char* pattern, const char* rule, const uint8_t* src, uint64_t src_len, uint8_t* dst, uint64_t cap) {
    if (!pattern || !rule || (!src && src_len) || (!dst && cap)) return TF_E_FATAL_ARG;
    try {
        const tfre::Prog prog = tfre::compile(pattern);
        const tfre::Template tpl = tfre::parse_template(rule, prog);
        tfre::Machine vm(prog); std::string out;
        static const uint8_t none = 0;
        tfre::replace_all(vm, tpl, src ? src : &none, src_len, out);
        if (out.size() <= cap && !out.empty()) std::memcpy(dst, out.data(), out.size());
        return (int64_t)out.size();
    } catch (const tfre::Unsupported&) { return TF_E_FATAL_UNSUPPORTED; }
    catch (const tfre::SyntaxError&) { return TF_E_FATAL_CONFIG; }
    catch (const std::exception&) { return TF_E_FATAL_CONFIG; }
}

int tfgpu_sink_destroy(tfgpu_sink* s) { if (!s) return TF_E_FATAL_ARG; if (s->pool) tfgpu_columnar_destroy(s->pool); delete s; return TF_OK; }
const char* tfgpu_sink_last_error(const tfgpu_sink* s) { return s ? s->err.c_str() : "null sink"; }
int tfgpu_sink_set_callback(tfgpu_sink* s, tf_sink_fn fn, void* ctx) { if (!s) return TF_E_FATAL_ARG; s->fn = fn; s->ctx = ctx; return TF_OK; }
int tfgpu_sink_set_clickhouse(tfgpu_sink* s, tfgpu_ch_conn* conn) {
    if (!s) return TF_E_FATAL_ARG;
    if (conn && s->wire_fmt != TF_WIRE_CH_NATIVE_LZ4 && s->wire_fmt != TF_WIRE_CH_NATIVE) { s->err = "the ClickHouse writer takes wire_fmt TF_WIRE_CH_NATIVE_LZ4 (compression on) or TF_WIRE_CH_NATIVE"; return TF_E_FATAL_CONFIG; }
    s->ch = conn; s->plans.clear(); return TF_OK;
}

int tfgpu_sink_push(tfgpu_sink* s, const tf_rows* items) {
    if (!s || !items) return TF_E_FATAL_ARG;
    struct Leave { tfgpu_sink* s; ~Leave() { if (s->gate_enter && !s->in_gate) s->gate_enter(s->gate_ctx); if (s->gate_leave) s->gate_leave(s->gate_ctx); s->in_gate = false; } } leave{s};   // a push without deliveries still takes its turn
    try { s->push(items); s->st.metering_input_rows += items->n_items; return TF_OK; }
    catch (const SinkFail& f) { s->err = f.msg; return f.rc; }
    catch (const std::bad_alloc&) { s->err = "host allocation failed"; return TF_E_RETRY_OOM; }
    catch (const std::exception& x) { s->err = x.what(); return TF_E_FATAL_CONFIG; }
}

int tfgpu_sink_stats(const tfgpu_sink* s, tf_sink_stats* out) { if (!s || !out) return TF_E_FATAL_ARG; *out = s->st; return TF_OK; }

}  // extern "C"


// ------------------------------------------------------------------ round-robin dispatcher over N sinks (SURVEY §8e)
struct tfgpu_dispatcher {
    struct Job { uint64_t seq; const tf_rows* items; };
    struct Lane { tfgpu_sink* sink; std::deque<Job> q; std::thread th; uint64_t cur_seq = 0; tfgpu_dispatcher* d = nullptr; };
    std::vector<std::unique_ptr<Lane>> lanes;
    std::mutex m; std::condition_variable cv;
    uint64_t submitted = 0, deliver_turn = 0;               // deliver_turn: the batch whose deliveries may run
    std::map<uint64_t, int> done;                            // seq -> rc of finished batches not yet waited for
    bool stop = false; int first_error = 0;

    static void enter(void* ctx) { Lane* l = (Lane*)ctx; std::unique_lock<std::mutex> lk(l->d->m); l->d->cv.wait(lk, [&] { return l->d->deliver_turn == l->cur_seq; }); }
    static void leave(void* ctx) { Lane* l = (Lane*)ctx; { std::lock_guard<std::mutex> g(l->d->m); l->d->deliver_turn = l->cur_seq + 1; } l->d->cv.notify_all(); }

    void loop(Lane* l) {
        for (;;) {
            Job j;
            {
                std::unique_lock<std::mutex> lk(m);
                cv.wait(lk, [&] { return stop || !l->q.empty(); });
                if (l->q.empty()) return;
                j = l->q.front(); l->cur_seq = j.seq;
            }
            const int rc = tfgpu_sink_push(l->sink, j.items);      // its deliveries wait for their turn inside (gate), and pass it on when the push is over
            {
                std::lock_guard<std::mutex> g(m);
                l->q.pop_front(); done[j.seq] = rc; if (rc && !first_error) first_error = rc;
            }
            cv.notify_all();
        }
    }
    std::set<uint64_t> waited;
};

extern "C" {

int tfgpu_dispatcher_create(tfgpu_sink* const* sinks, int n, tfgpu_dispatcher** out) {
    if (!sinks || n <= 0 || !out) return TF_E_FATAL_ARG;
    auto d = std::make_unique<tfgpu_dispatcher>();
    for (int i = 0; i < n; i++) {
        if (!sinks[i] || sinks[i]->gate_enter) return TF_E_FATAL_ARG;
        auto l = std::make_unique<tfgpu_dispatcher::Lane>(); l->sink = sinks[i]; l->d = d.get();
        d->lanes.push_back(std::move(l));
    }
    for (auto& l : d->lanes) { l->sink->gate_enter = &tfgpu_dispatcher::enter; l->sink->gate_leave = &tfgpu_dispatcher::leave; l->sink->gate_ctx = l.get(); tfgpu_dispatcher* dp = d.get(); tfgpu_dispatcher::Lane* lp = l.get(); l->th = std::thread([dp, lp] { dp->loop(lp); }); }
    *out = d.release();
    return TF_OK;
}

int tfgpu_dispatcher_submit(tfgpu_dispatcher* d, const tf_rows* items, uint64_t* seq) {
    if (!d || !items) return TF_E_FATAL_ARG;
    std::unique_lock<std::mutex> lk(d->m);
    const uint64_t s = d->submitted; tfgpu_dispatcher::Lane* l = d->lanes[s % d->lanes.size()].get();
    d->cv.wait(lk, [&] { return l->q.size() < 2; });                  // one batch in work + one waiting per sink
    l->q.push_back({s, items}); d->submitted++;
    if (seq) *seq = s;
    lk.unlock(); d->cv.notify_all();
    return TF_OK;
}

int tfgpu_dispatcher_wait(tfgpu_dispatcher* d, uint64_t seq) {
    if (!d) return TF_E_FATAL_ARG;
    std::unique_lock<std::mutex> lk(d->m);
    if (seq >= d->submitted) return TF_E_FATAL_ARG;
    d->cv.wait(lk, [&] { return d->done.count(seq) || d->waited.count(seq); });
    if (d->waited.count(seq)) return TF_E_FATAL_ARG;                  // waited for twice
    const int rc = d->done[seq]; d->done.erase(seq); d->waited.insert(seq);
    while (!d->waited.empty() && *d->waited.begin() + 1024 < seq) d->waited.erase(d->waited.begin());      // bounded memory on long runs
    return rc;
}

int tfgpu_dispatcher_drain(tfgpu_dispatcher* d) {
    if (!d) return TF_E_FATAL_ARG;
    std::unique_lock<std::mutex> lk(d->m);
    d->cv.wait(lk, [&] { for (auto& l : d->lanes) if (!l->q.empty()) return false; return true; });
    const int rc = d->first_error; d->first_error = 0;
    return rc;
}

int tfgpu_dispatcher_destroy(tfgpu_dispatcher* d) {
    if (!d) return TF_E_FATAL_ARG;
    tfgpu_dispatcher_drain(d);
    { std::lock_guard<std::mutex> g(d->m); d->stop = true; }
    d->cv.notify_all();
    for (auto& l : d->lanes) { if (l->th.joinable()) l->th.join(); l->sink->gate_enter = nullptr; l->sink->gate_leave = nullptr; l->sink->gate_ctx = nullptr; }
    delete d;
    return TF_OK;
}

}  // extern "C"
