/* ORACLE — test infrastructure only (tests/, __graft_entry__.smoke(), bench.py cpu_baseline /
 * --impl reference).  Never linked into or called from the product path.
 *
 * C API of the CPU restatement of transferia's per-batch hot path.  Every function cites the
 * reference file:line it follows in oracle.cpp.  The batch layout is the product's tf_batch
 * (include/tfgpu.h) with HOST pointers; processing is row-at-a-time over boxed values, like
 * the Go reference (`[]interface{}` per ChangeItem).
 *
 * Parity status (also in DESIGN.md):
 *   pinned by reference goldens: mask_field digests, %v / RFC3339 text forms, filter_rows
 *     matrices, filter grammar;  pinned by independent implementations here: shortest float
 *     digits (CPython repr / numpy), SHA-256/HMAC (hashlib), LZ4 decode (liblz4, pyarrow);
 *   PARITY UNPINNED: ClickHouse native block bytes, LZ4 compressed bytes, CityHash128 — third
 *     party in the reference (clickhouse-go/v2 v2.46.0, ch-go v0.71.0, pierrec/lz4/v4 v4.1.25,
 *     go-faster/city v1.0.1), not vendored, and no reference test pins them.
 */
#ifndef ORACLE_H_
#define ORACLE_H_
#include <stdint.h>
#include "../include/tfgpu.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Go dynamic type of a boxed value */
enum { OG_NIL = 0, OG_INT8, OG_INT16, OG_INT32, OG_INT64, OG_UINT8, OG_UINT16, OG_UINT32, OG_UINT64,
       OG_FLOAT32, OG_FLOAT64, OG_BOOL, OG_STRING, OG_BYTES, OG_TIME, OG_DURATION, OG_JSON /* any: non-string value, JSON text */,
       OG_INT /* Go int */, OG_UINT };

typedef struct orc_val {
    int32_t kind; uint32_t nsec;
    int64_t i;          /* signed ints, bool, duration ns, time seconds */
    uint64_t u;         /* unsigned ints */
    double f;           /* float32 (exactly representable) / float64 */
    const uint8_t* s; uint64_t slen;
} orc_val;

/* filter.OperatorType order: library/go/yandex/cloud/filter/filters.go:12-23 */
enum { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN, OP_NOTIN, OP_MATCH, OP_NOTMATCH };
/* literal kinds */
enum { LV_INT = 1, LV_FLOAT = 2, LV_BOOL = 3, LV_STRING = 4, LV_TIME = 5, LV_NULL = 6, LV_LIST = 16 };

typedef struct orc_term {
    int32_t col;        /* column index in the batch */
    int32_t op;
    int32_t vtype;      /* LV_* (| LV_LIST) */
    int32_t nlist;
    int64_t i;          /* int / bool / time as UnixMicro */
    double f;
    const uint8_t* s; uint64_t slen;
    const int64_t* ilist;       /* int list, time list (UnixMicro) */
    const double* flist;
    const uint32_t* soffs; const uint8_t* sheap;  /* string list: nlist+1 offsets */
} orc_term;

typedef struct orc_colschema {
    const char* name;
    int32_t type;       /* tf_type */
    int32_t required;
    const char* original_type;  /* may be NULL */
} orc_colschema;

enum { STEP_FILTER_ROWS = 1, STEP_MASK = 2, STEP_TO_STRING = 3, STEP_SKIP_EVENTS = 4, STEP_SELECT_COLS = 5, STEP_TO_DATETIME = 6, STEP_NUMBER_TO_FLOAT = 7, STEP_SHARDER = 8 };
typedef struct orc_step {
    int32_t kind;
    /* filter_rows */
    const orc_term* terms; const uint32_t* expr_off; int32_t nexpr;
    /* mask_field / convert_to_string: column indexes */
    const int32_t* cols; int32_t ncols;
    const uint8_t* salt; uint64_t salt_len;
    int32_t convert_to_bytes;
    int32_t pass_all;      /* filter_rows: table filter misses the renamed table -> rows pass, kinds still checked */
    int32_t kind_mask;     /* skip_events: bit TF_KIND_* set = drop; sharder: ShardsNum */
} orc_step;

typedef struct orc_buf { uint8_t* data; uint64_t len; } orc_buf;
void orc_free(orc_buf* b);

/* ---- scalar entry points (golden-vector tests) ---- */
int  orc_fmt_float64(double v, int fmt /*0 %v,1 'f',2 json*/, char* dst, int cap);
int  orc_fmt_float32(float v, int fmt, char* dst, int cap);
int  orc_fmt_duration(int64_t ns, char* dst, int cap);
int  orc_fmt_rfc3339nano(int64_t sec, uint32_t nsec, char* dst, int cap);
int  orc_serialize_to_string(const orc_val* v, int32_t yt_type, char* dst, int cap);  /* to_string.go:149-171 */
void orc_hmac_sha256_hex(const uint8_t* key, uint64_t klen, const uint8_t* msg, uint64_t mlen, char out[65]);
void orc_sha256(const uint8_t* msg, uint64_t mlen, uint8_t out[32]);
void orc_cityhash128(const uint8_t* p, uint64_t n, uint64_t* lo, uint64_t* hi);
uint64_t orc_lz4_bound(uint64_t n);
uint64_t orc_lz4_compress(const uint8_t* src, uint64_t n, uint8_t* dst);
/* Strict: decodes a block of exactly rs raw bytes that obeys the LZ4 end-of-block rules (lz4_block.hpp), else -1. */
int64_t  orc_lz4_decompress(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t rs);
/* matchValue: returns 0 ok (*matched set), else TF_ROWERR_* */
int  orc_match_value(const orc_val* v, const orc_term* t, int* matched);

/* typesystem casts over one boxed Go value, values as (Go type name, text) pairs — see tests/golden/cast_goldens.json.
 * rc: 0 ok, 1 cast error, 2 StrictifyRangeError, 3 the reference panics, 4 outside this restatement (dateparse / StringToDate tail), -1 bad call */
int  orc_strictify_value(const char* go, const char* v, uint64_t vlen, int32_t tf, char* out_go, int go_cap, char* out_v, uint64_t v_cap, uint64_t* out_vlen);   /* strictify.go:46-157 */
int  orc_restore_value(const char* go, const char* v, uint64_t vlen, const char* data_type, char* out_go, int go_cap, char* out_v, uint64_t v_cap, uint64_t* out_vlen);   /* restore.go:20-223 */
uint64_t orc_csv_split_rows(const uint8_t* p, uint64_t n, uint64_t* row_ends, uint64_t cap);   /* splitter.go:38-85 */

/* ---- batch entry points ---- */
/* ClickHouse column type the sink DDL gives this column: sink_table.go:196-208 + columntypes/types.go:210-248 */
int  orc_ch_type(const orc_colschema* c, char* dst, int cap);

/* Whole hot path, row by row: transformer steps -> columntypes.Restore -> native block (-> LZ4 frames).
 * out_raw: uncompressed native block; out_wire: what goes on the socket for wire_fmt.
 * errs must hold nrows entries. Returns 0 or a negative fatal code. */
int orc_push_encode(const tf_batch* in, const orc_colschema* schema,
                    const orc_step* steps, int nsteps,
                    int wire_fmt, uint64_t frame_bytes,
                    orc_buf* out_raw, orc_buf* out_wire,
                    uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs);

/* Transformer chain only (TransformerResult.Transformed, pkg/abstract/transformer.go:40-48): the kept rows, columnar,
 * in one buffer; regions[k] = {values, validity, aux, offsets, heap, heap_len} offsets into it (~0 = absent). */
/* Debezium emitter (pkg/debezium/emitter_value_converter.go:626-690 + emitter_common.go:67-180), INSERT rows, columns without
 * a database-specific original_type. Messages back to back: key then value per output row. */
typedef struct orc_dbz_emit_opts {
    const char* version; const char* name; const char* database; const char* schema; const char* table;
    int32_t source_type;                   /* 0 none, 1 pg, 2 mysql */
    uint8_t snapshot, drop_keys, pad[2];
    const char* key_schema; const char* val_schema;      /* NULL: schemas disabled */
    int64_t key_schema_id, val_schema_id;                /* >= 0: confluent schema registry framing */
} orc_dbz_emit_opts;
/* forms[input column]: 0 = addCommon, else the AddPg branch (pkg/debezium/pg/emitter.go:265-629): 2 real, 3 double precision, 4 string
 * types, 6 json / jsonb, 7 date, 8 / 9 timestamp without time zone (micros / millis), 10 timestamp with time zone, 11 inet */
int orc_debezium_emit(const tf_batch* in, const orc_colschema* schema, const uint8_t* is_key, const uint8_t* forms, const orc_step* steps, int nsteps,
                      const tf_row_meta* meta, const orc_dbz_emit_opts* opts, orc_buf* out, uint32_t* key_sizes, uint32_t* row_sizes,
                      uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs);
/* every row kind: ChangeItem.OldKeys as a second batch (tf_old_keys of include/tfgpu.h); msg_sizes: 7 per output row */
int  orc_debezium_emit_crud(const tf_batch* in, const tf_old_keys* old, int tombstones, const orc_colschema* schema, const uint8_t* is_key, const uint8_t* forms, const orc_step* steps, int nsteps,
                            const tf_row_meta* meta, const orc_dbz_emit_opts* o, orc_buf* out, uint32_t* key_sizes, uint32_t* row_sizes, uint32_t* msg_sizes,
                            uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs);

/* sharder transformer (pkg/transformer/registry/sharder/sharder.go:130-145): ChangeItem.PartID of every row the chain keeps =
 * decimal(CRC32-IEEE(join(".", SerializeToString(value) of the matched columns)) % uint32(ShardsNum)). part_ids: nrows entries. */
int orc_shard_ids(const tf_batch* in, const orc_colschema* schema, const orc_step* steps, int nsteps, uint32_t* part_ids, uint64_t* rows_out);
uint32_t orc_crc32_ieee(const uint8_t* p, uint64_t n);

typedef struct orc_regions { uint64_t values, validity, aux, offsets, heap, heap_len; } orc_regions;
int orc_push_columns(const tf_batch* in, const orc_colschema* schema, const orc_step* steps, int nsteps,
                     orc_buf* out, orc_regions* regions /* one per output column */, int32_t* out_types,
                     uint64_t* rows_out, tf_rowerr* errs, uint64_t* nerrs);

/* CSV: raw bytes -> typed columns (pkg/csv/reader.go + s3 reader_csv.go + strictify), see csv_oracle.hpp.
 * list arguments are '\n'-separated. Output layout as orc_push_columns. errs[].row = data line index (after skip_lines). */
typedef struct orc_csv_opts {
    uint8_t delimiter, quote, escape, double_quote, strings_can_be_null, quoted_strings_can_be_null, include_missing, pad;
    const char* null_values; const char* true_values; const char* false_values;
    uint64_t skip_lines;
} orc_csv_opts;
int orc_csv_parse(const uint8_t* buf, uint64_t len, const int32_t* types, const int32_t* paths, int ncols, const orc_csv_opts* opts,
                  orc_buf* out, orc_regions* regions, uint64_t* rows, uint64_t* lines, uint64_t* consumed,
                  tf_rowerr* errs, uint64_t errs_cap, uint64_t* nerrs);

/* Generic JSON parser (pkg/parsers/generic/generic_parser.go, format "json"), see json_oracle.hpp. `cols` is the parser's
 * RESULT schema: the declared fields, then `_rest` (add_rest), then _timestamp,_partition,_offset,_idx (add_dedupe_keys).
 * names/keys/required are parallel arrays; msgs[k].end = one past message k in buf. errs[].row = non-empty line index. */
typedef struct orc_json_opts { uint8_t add_rest, add_dedupe_keys, null_keys_allowed, use_numbers_in_any, unpack_bytes_base64, pad[3]; const char* partition; } orc_json_opts;
typedef struct orc_json_msg { uint64_t end, offset; int64_t write_sec; uint32_t write_nsec, pad; } orc_json_msg;
int orc_json_parse(const uint8_t* buf, uint64_t len, const orc_json_msg* msgs, uint64_t nmsgs,
                   const char* const* names, const int32_t* types, const uint8_t* keys, const uint8_t* required, int ncols,
                   const orc_json_opts* opts, orc_buf* out, orc_regions* regions, uint64_t* rows, uint64_t* lines,
                   tf_rowerr* errs, uint64_t errs_cap, uint64_t* nerrs);

/* Debezium parser (pkg/parsers/registry/debezium/engine/parser.go + pkg/debezium/receiver*.go), see debezium_oracle.hpp.
 * One row per message (a schema-registry message holding several events is reported DBZ_HOST). errs[].row = message index.
 * Outputs: columns of `fields` (validity always present) + per-row kind / txId / lsn / commit time / message index. */
typedef struct orc_dbz_field { const char* name; int32_t recv; int32_t scale; int32_t key; } orc_dbz_field;
typedef struct orc_dbz_opts { const uint8_t* schema_text; uint64_t schema_len; uint8_t use_sr, check_table, pad[2]; uint32_t schema_id; const char* table_schema; const char* table_name; } orc_dbz_opts;
int orc_debezium_parse(const uint8_t* buf, uint64_t len, const uint64_t* msg_ends, uint64_t nmsgs, const orc_dbz_field* fields, int nfields, const orc_dbz_opts* o,
                       orc_buf* out, orc_regions* regions, int32_t* out_types, uint8_t* kinds, uint32_t* tx_ids, uint64_t* lsns, uint64_t* commit_times, uint32_t* row_msg,
                       uint64_t* rows, tf_rowerr* errs, uint64_t* nerrs);
int orc_base64_to_numeric(const char* b64, int scale, char* dst, int cap);

/* BatchJSON (pkg/serializer/queue/json_batcher.go:29-66): starts needs n + 1 entries. */
int orc_queue_json_batches(const uint64_t* len_elements, uint64_t n, uint64_t max_message_size, uint64_t max_change_items, uint64_t* starts, uint64_t* n_msgs);

/* Measurer middleware: Size.Values = util.DeepSizeof(ColumnValues) per row (pkg/util/sizeof.go:7-110). */
int orc_measure(const tf_batch* in, uint64_t* per_row, uint64_t* total);

/* Verify + decode a frame stream with the oracle's own (strict) LZ4 decoder and CityHash. */
int orc_ch_decode_frames(const uint8_t* wire, uint64_t n, orc_buf* raw, uint64_t* n_frames);

#ifdef __cplusplus
}
#endif
#endif
