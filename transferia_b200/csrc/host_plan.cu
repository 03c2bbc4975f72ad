// Host-only entry points of include/tfgpu.h (no device needed) and the host helpers tfgpu.cu shares with them: plan validation,
// the queue serializer batchers, the describe / error-buffer convention of the *_validate calls and column-name quoting.
#include <cstring>
#include <string>

#include "../../include/tfgpu.h"
#include "plan.hpp"
#include "host_internal.hpp"

namespace {
void put_text(char* dst, uint64_t cap, const std::string& s) {
    if (!dst || !cap) return;
    const size_t n = s.size() < cap - 1 ? s.size() : cap - 1;
    std::memcpy(dst, s.data(), n); dst[n] = 0;
}
}  // namespace

int host_validate(char* describe_out, uint64_t cap, char* err_out, uint64_t err_cap, const std::function<std::string()>& describe) {
    try {
        const std::string d = describe();
        if (describe_out && d.size() + 1 > cap) { put_text(err_out, err_cap, "describe buffer too small"); return TF_E_FATAL_ARG; }
        put_text(describe_out, cap, d);
        return TF_OK;
    } catch (const tfplan::FatalError& f) { put_text(err_out, err_cap, f.what()); return f.code; }
    catch (const std::exception& x) { put_text(err_out, err_cap, x.what()); return TF_E_FATAL_CONFIG; }
}

// encoding/json appendString with escapeHTML off, for column names (json.go:56-58)
std::string host_json_quote_nohtml(const std::string& in) {
    static const char* hex = "0123456789abcdef";
    std::string d = "\""; const uint8_t* s = (const uint8_t*)in.data(); const size_t n = in.size();
    for (size_t i = 0; i < n;) {
        const uint8_t b = s[i];
        if (b < 0x80) {
            if (b >= 0x20 && b != '"' && b != '\\') d += (char)b;
            else { d += '\\'; switch (b) { case '"': case '\\': d += (char)b; break; case '\b': d += 'b'; break; case '\f': d += 'f'; break; case '\n': d += 'n'; break; case '\r': d += 'r'; break; case '\t': d += 't'; break;
                                            default: d += "u00"; d += hex[b >> 4]; d += hex[b & 15]; } }
            i++; continue;
        }
        uint32_t r = 0xFFFD; size_t w = 1;
        if (b >= 0xC2 && b <= 0xDF && i + 1 < n && (s[i + 1] & 0xC0) == 0x80) { r = ((b & 0x1Fu) << 6) | (s[i + 1] & 0x3Fu); w = 2; }
        else if (b >= 0xE0 && b <= 0xEF && i + 2 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80) { const uint32_t t = ((b & 0x0Fu) << 12) | ((s[i + 1] & 0x3Fu) << 6) | (s[i + 2] & 0x3Fu); if (t >= 0x800 && !(t >= 0xD800 && t <= 0xDFFF)) { r = t; w = 3; } }
        else if (b >= 0xF0 && b <= 0xF4 && i + 3 < n && (s[i + 1] & 0xC0) == 0x80 && (s[i + 2] & 0xC0) == 0x80 && (s[i + 3] & 0xC0) == 0x80) { const uint32_t t = ((b & 0x07u) << 18) | ((s[i + 1] & 0x3Fu) << 12) | ((s[i + 2] & 0x3Fu) << 6) | (s[i + 3] & 0x3Fu); if (t >= 0x10000 && t <= 0x10FFFF) { r = t; w = 4; } }
        if (r == 0xFFFD && w == 1) d += "\\ufffd";
        else if (r == 0x2028 || r == 0x2029) { d += "\\u202"; d += hex[r & 0xF]; }
        else d.append((const char*)s + i, w);
        i += w;
    }
    return d + "\"";
}

extern "C" {

// Host-only: build the plan (Suitable / ResultSchema chain, filter grammar, ClickHouse types) without touching a
// device, so a transfer's YAML can be validated where no GPU is present (cmd/trcli validate does the same for the
// reference's transformers: cmd/trcli/config/model.go:57-72).
int tfgpu_plan_validate(const char* ns, const char* name, const char* schema_json, const char* transformers_json,
                        const char* sink_json, char* describe_out, uint64_t cap, char* err_out, uint64_t err_cap) {
    if (!schema_json || !name) return TF_E_FATAL_ARG;
    return host_validate(describe_out, cap, err_out, err_cap, [&] {
        return tfplan::build_plan(ns ? ns : "", name, schema_json, transformers_json ? transformers_json : "", sink_json ? sink_json : "").describe;
    });
}

// queue JSON serializer batching (pkg/serializer/queue/json_batcher.go:13-66): host only, no device needed
int tfgpu_queue_debezium_batches(const uint32_t* value_sizes, uint64_t n, uint64_t max_message_size, uint64_t* starts, uint64_t cap, uint64_t* n_msgs) {
    if ((!value_sizes && n) || !starts || !n_msgs) return TF_E_FATAL_ARG;
    uint64_t k = 0, cur = 0;
    for (uint64_t i = 0; i < n; i++) {
        // expandArrIfNeeded :76-86: a new message for the first value and whenever len(last) + 1 + len(new) > maxMessageSize;
        // without a limit every value stays its own message (MergeBack :53-65)
        if (i == 0 || !max_message_size || cur + 1 + value_sizes[i] > max_message_size) { if (k >= cap) return TF_E_FATAL_ARG; starts[k++] = i; cur = 0; }
        cur += value_sizes[i];
    }
    if (k >= cap) return TF_E_FATAL_ARG;
    starts[k] = n; *n_msgs = k;
    return TF_OK;
}
int tfgpu_queue_json_batches(const uint32_t* row_sizes, uint64_t n, uint64_t max_message_size, uint64_t max_change_items, uint64_t* starts, uint64_t cap, uint64_t* n_msgs) {
    if ((!row_sizes && n) || !starts || !n_msgs) return TF_E_FATAL_ARG;
    uint64_t k = 0, start = 0, sum = 0;
    auto emit = [&](uint64_t s) -> bool { if (k >= cap) return false; starts[k++] = s; return true; };
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t count = i - start + 1;
        const bool viol = (max_message_size && sum + (count - 1) + row_sizes[i] > max_message_size) || (max_change_items && count > max_change_items);
        if (!viol) { sum += row_sizes[i]; continue; }
        if (!emit(start)) return TF_E_FATAL_ARG;
        if (i == start) { start = i + 1; sum = 0; }        // a single item over the size limit goes out alone
        else { start = i; sum = row_sizes[i]; }
    }
    if (start != n && !emit(start)) return TF_E_FATAL_ARG;
    if (k >= cap) return TF_E_FATAL_ARG;
    starts[k] = n; *n_msgs = k;
    return TF_OK;
}

}  // extern "C"
