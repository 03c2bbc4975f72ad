// Calls between the host translation units of libtfgpu.so that are not part of the C-ABI.
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include "../../include/tfgpu_sink.h"

// One text cell through a replacement: (cell bytes, length, result). A worker asks `make` for its own replacer (a regexp machine is not shared).
using tf_text_fn = std::function<void(const uint8_t*, uint32_t, std::string&)>;

// Rewrites var-width column `col` of the batch the pool handed out last (tfgpu_rows_to_batch) cell by cell — null cells stay null — into
// pooled buffers, with the narrowest length array the new cells allow; patches the batch's column in place. TF_OK or a TF_E_* code
// (tfgpu_columnar_last_error has the text).
int tfgpu_columnar_rewrite_text(tfgpu_columnar* pool, uint32_t col, const std::function<tf_text_fn()>& make, int threads);

// Did a cell of text column `col` of the last transposed batch carry the OTHER text type of Go (a []byte in a utf8 column, a string in a
// `string` column)? The regex_replace transformer's type assertion leaves such cells alone (transformer.go:127-142).
bool tfgpu_columnar_text_was_mixed(const tfgpu_columnar* pool, uint32_t col);

// The host-only *_validate calls of tfgpu.h: `describe` checks the input and returns its description, which goes to describe_out
// (TF_E_FATAL_ARG if it does not fit in cap bytes with its NUL); a refusal puts its text in err_out and returns its code
// (TF_E_FATAL_CONFIG for an error that carries none). Both buffers may be NULL.
int host_validate(char* describe_out, uint64_t cap, char* err_out, uint64_t err_cap, const std::function<std::string()>& describe);

// encoding/json's string quoting with HTML escaping off (json.go:56-58): column names and template text
std::string host_json_quote_nohtml(const std::string& in);
