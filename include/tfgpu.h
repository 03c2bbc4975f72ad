/*
 * tfgpu.h — C-ABI of the H100 columnar transform engine.
 *
 * This is the drop-in boundary for ONE hot path of transferia/transferia:
 *
 *   Sinker.Push([]abstract.ChangeItem) -> pkg/middlewares -> pkg/transformer chain
 *     -> sink typesystem cast -> sink wire format
 *
 * The Go side (cgo shim, see INTEGRATION.md) transposes a []ChangeItem batch of
 * one table into the columnar `tf_batch` below (pinned host memory it owns),
 * calls one of the tfgpu_* entry points, and rebuilds ChangeItems / writes the
 * wire bytes from the result.  No torch / C++ types cross this boundary: plain
 * pointers, sizes and NUL-terminated JSON strings only.
 *
 * Reference interfaces each entry point stands in for (paths relative to the
 * reference repository root):
 *
 *   tfgpu_engine_create / _destroy
 *       middleware construction: func(Sinker) Sinker
 *       pkg/abstract/middleware.go:3, pkg/middlewares/pluggable_transformer.go:19-30,
 *       pkg/abstract/sink.go:14-19 (Close)
 *   tfgpu_plan
 *       transformation.AddTablePlan (Suitable + ResultSchema per transformer,
 *       cached by TableSchema.Hash())  pkg/transformer/transformation.go:46-85,93-121
 *       pkg/abstract/transformer.go:32-48, pkg/abstract/changeitem/table_schema.go:54-67
 *   tfgpu_push_columns
 *       transformation.Push / do -> Transformer.Apply chain
 *       pkg/transformer/transformation.go:122-158,236-282
 *   tfgpu_push_encode
 *       the same chain followed by the destination's per-row cast + wire encode:
 *       pkg/providers/clickhouse/sink_table.go:605-684 (doOperation),
 *       :698-704 (restoreVals) -> columntypes.Restore columntypes/types.go:74-115
 *       -> clickhouse-go/v2 native block + LZ4 frames (conn/connection.go:46)
 *   tfgpu_result_* accessors
 *       abstract.TransformerResult{Transformed, Errors}  pkg/abstract/transformer.go:40-48
 *
 * Threading (pkg/abstract/sink.go:12): calls on ONE engine handle are never
 * concurrent; distinct handles are independent (one per pipeline / per GPU).
 *
 * Error classes (pkg/abstract/sink.go:16-17, pkg/abstract/errors.go:14):
 *   rc == 0  ok
 *   rc  > 0  retriable (device OOM, launch failure) — Push may be retried
 *   rc  < 0  fatal (unsupported schema/type, malformed config) — NewFatalError
 * Per-row transformer failures are DATA, not errors: they come back as an
 * error-row list (row index + message id), mirroring TransformerResult.Errors.
 */
#ifndef TFGPU_H_
#define TFGPU_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- return codes ------------------------------------------------------- */
#define TF_OK                 0
#define TF_E_RETRY_OOM        1   /* retriable: device / pinned allocation failed  */
#define TF_E_RETRY_LAUNCH     2   /* retriable: kernel launch / stream error       */
#define TF_E_FATAL_CONFIG    -1   /* fatal: malformed cfg / schema / transformers   */
#define TF_E_FATAL_UNSUPPORTED -2 /* fatal: type or transformer not supported       */
#define TF_E_FATAL_ARG       -3   /* fatal: bad handle / NULL argument              */
#define TF_E_FATAL_NODEVICE  -4   /* fatal: no CUDA device — there is no CPU fallback */

/* ---- logical column types: the YT type strings of pkg/abstract/typesystem/schema.go:48-68.
 * NOTE the naming trap (SURVEY §2.4): YT "string" is BYTES, YT "utf8" is text. */
typedef enum tf_type {
    TF_INT8 = 1, TF_INT16 = 2, TF_INT32 = 3, TF_INT64 = 4,
    TF_UINT8 = 5, TF_UINT16 = 6, TF_UINT32 = 7, TF_UINT64 = 8,
    TF_FLOAT = 9,        /* "float"    -> Go float32            */
    TF_DOUBLE = 10,      /* "double"   -> Go float64            */
    TF_BOOLEAN = 11,     /* "boolean"  -> Go bool, 1 byte       */
    TF_BYTES = 12,       /* "string"   -> Go []byte             */
    TF_UTF8 = 13,        /* "utf8"     -> Go string             */
    TF_ANY = 14,         /* "any"      -> JSON text (or raw Go string, see aux tags) */
    TF_DATE = 15,        /* "date"     -> Go time.Time          */
    TF_DATETIME = 16,    /* "datetime" -> Go time.Time          */
    TF_TIMESTAMP = 17,   /* "timestamp"-> Go time.Time          */
    TF_INTERVAL = 18     /* "interval" -> Go time.Duration (int64 ns) */
} tf_type;

/* ---- physical layout of one column ---------------------------------------
 * fixed-width (ints, float, double, boolean, interval):
 *     values = nrows little-endian elements of the natural width (boolean: u8 0/1).
 * time types (date / datetime / timestamp), i.e. Go time.Time:
 *     values = nrows int64 Unix seconds (UTC instant),
 *     aux    = optional nrows uint32 nanoseconds [0, 1e9); NULL = all zero.
 * var-width (string / utf8 / any):
 *     offsets = nrows+1 uint32, heap = offsets[nrows] bytes.
 *     any: heap holds the value's JSON text (what json.Marshal gives); aux is an
 *     optional nrows uint8 tag array, tag 1 = the Go value was a `string` and the
 *     heap holds its raw bytes (columntypes.Restore passes such values through
 *     unquoted, columntypes/types.go:77-79).
 * validity: optional bitmap, bit r (LSB-first in byte r/8) = 1 means non-nil.
 */
typedef struct tf_col {
    int32_t         type;       /* tf_type */
    int32_t         flags;      /* 0, or TF_COL_LENS8 / TF_COL_LENS16 (var-width columns) */
    const void*     values;
    const uint8_t*  validity;
    const uint32_t* offsets;
    const uint8_t*  heap;
    const void*     aux;
    uint64_t        heap_len;
} tf_col;

/* A var-width column may carry per-row LENGTHS instead of offsets: `offsets` then points at nrows uint8 (TF_COL_LENS8) or uint16
 * (TF_COL_LENS16) values and the engine builds the uint32 offsets on the device — a quarter / half of the offset bytes over PCIe for
 * columns whose cells are shorter than 256 / 65536 bytes. heap_len must still be the heap's byte count. */
#define TF_COL_LENS8  1
#define TF_COL_LENS16 2

#define TF_MEM_HOST   0   /* pointers are host memory (pinned preferred): copies are inside the call */
#define TF_MEM_DEVICE 1   /* pointers are device memory on the engine's GPU: batch is HBM-resident   */

/* abstract.Kind of each row (pkg/abstract/changeitem/kind.go:5-43); only row kinds travel */
#define TF_KIND_INSERT 0
#define TF_KIND_UPDATE 1
#define TF_KIND_DELETE 2

typedef struct tf_batch {
    uint64_t        nrows;
    uint32_t        ncols;
    uint32_t        mem;        /* TF_MEM_HOST | TF_MEM_DEVICE */
    const tf_col*   cols;       /* ncols entries, host memory, schema order */
    const uint8_t*  kinds;      /* optional nrows TF_KIND_*; NULL = all insert */
} tf_batch;

/* ---- per-row transformer errors (TransformerResult.Errors) ----------------- */
#define TF_ROWERR_FILTER_KIND      1  /* filter_rows.go:103-107 "Found non-supported kind '%s'"  */
#define TF_ROWERR_FILTER_OVERFLOW  2  /* filter_rows util.go:66-68 errIntOverflow                  */
#define TF_ROWERR_FILTER_TYPEPAIR  3  /* filter_rows.go:364 "Unsupported type pair"                */
#define TF_ROWERR_CSV_MISSING_CELL 16 /* reader_csv.go:299-312 missing row element                        */
#define TF_ROWERR_CSV_SINGLE_QUOTE 17 /* reader.go:293-295 element is a lone quote (file-level in the reference) */
#define TF_ROWERR_CSV_BAD_INT      18 /* strictify: cannot cast to int / negative into unsigned              */
#define TF_ROWERR_CSV_RANGE        19 /* strictify.go:159-181 StrictifyRangeError                            */
#define TF_ROWERR_CSV_BAD_BOOL     20
#define TF_ROWERR_CSV_BAD_TIME     21
#define TF_ROWERR_CSV_BAD_FLOAT    22
#define TF_ROWERR_CSV_UNSUPPORTED  23 /* valid for Go's parsers, but a syntax the device does not implement   */
#define TF_ROWERR_CSV_DQ_DISABLED  24 /* reader.go:305-311 errDoubleQuotesDisabled                           */
#define TF_ROWERR_CSV_QUOTING_DISABLED 25 /* reader.go:185-187 errQuotingDisabled: a '"' on a line read with "quote":"" */

/* generic JSON parser (tfgpu_parse_json) */
#define TF_ROWERR_JSON_PARSE        32 /* fastjson rejects the line -> unparsed row (generic_parser.go:548-553)            */
#define TF_ROWERR_JSON_SKIP         33 /* valid JSON but not an object with keys: the line yields nothing (:536)           */
#define TF_ROWERR_JSON_NIL_REQUIRED 34 /* "ParseVal nil": key / required column without a value (:369-371); term = column  */
#define TF_ROWERR_JSON_PARSEVAL     35 /* "ParseVal error" on a key / required column (:361-366); term = column             */
#define TF_ROWERR_JSON_HOST         36 /* the line needs the Go parser (see tfgpu_parse_json); term = column                */

/* number_to_float: a number literal inside an `any` value whose float64 rounding the device cannot decide (hex / underscored /
 * > 19 digit literals with an open Eisel-Lemire result); the shim applies the Go transformer to that row */
#define TF_ROWERR_N2F_HOST 52
#define TF_ROWERR_STRICT_CAST  57 /* strictify.go:46-157: the value cannot be cast to the column type (a negative into an unsigned column); term = column */
#define TF_ROWERR_STRICT_RANGE 58 /* strictify.go:159-181 StrictifyRangeError; term = column */
#define TF_ROWERR_SINK_KIND_HOST 54 /* tfgpu_push_encode*: an UPDATE / DELETE row reached a sink or serializer wire format; the device encodes INSERT rows only
                                     (sink_table.go:296-305, marshal.go:92-95, json_serializer.go:17-20) — the shim routes the row through the Go sink */
#define TF_ROWERR_DBZ_EMIT_HOST 53 /* (round 1; no longer raised: tfgpu_emit_debezium_crud emits update / delete events) */

/* serializers: a value encoding/json refuses (NaN / Inf float, time.Time with a year outside [0,9999]); the reference
 * fails the whole Serialize call on it, so a result carrying this code must not be written; term = output column */
#define TF_ROWERR_SER_VALUE 40

typedef struct tf_rowerr {
    uint32_t row;      /* index into the INPUT batch */
    uint16_t code;     /* TF_ROWERR_* */
    uint16_t term;     /* index of the transformer in the plan that raised it, or the column (any index below 65536) for the codes documented
                          "term = column"; 0xff = raised before the chain (parser, host hand-off) */
} tf_rowerr;

/* ---- wire formats for tfgpu_push_encode ----------------------------------- */
#define TF_WIRE_CH_NATIVE      1  /* ClickHouse native block, uncompressed                       */
#define TF_WIRE_CH_NATIVE_LZ4  2  /* same, cut into [CityHash128][0x82][sizes][LZ4 block] frames */
#define TF_WIRE_CH_JSONEACHROW 3  /* httpuploader/marshal.go:88-253                              */
/* batch serializers (pkg/serializer/batch.go:73-231 over json.go:29-114 + json_format.go:32-82 / csv.go:22-74 +
 * csv_format.go:32-144): the object-storage / queue sinks' row text. OR the flags into the format id. */
#define TF_WIRE_SER_JSON       4  /* one JSON object per row, keys sorted, rows joined by '\n'    */
#define TF_WIRE_SER_CSV        5  /* encoding/csv records, each ending in '\n'                    */
#define TF_WIRE_DEBEZIUM       6  /* tfgpu_emit_debezium only: key message + value message per row  */
#define TF_WIRE_F_CLOSING_NEWLINE 0x100  /* JSONSerializerConfig.AddClosingNewLine (json.go:15)   */
#define TF_WIRE_F_ANY_AS_STRING   0x200  /* JSONSerializerConfig.AnyAsString (json_format.go:69-76) */
/* The S3 sink's OutputEncoding (pkg/providers/s3/sink/writer/writer.go:45-55, uploader.go:29-47): the row text of TF_WIRE_SER_JSON /
 * TF_WIRE_SER_CSV compressed on the device, as one gzip member (RFC 1952) or one zlib stream (RFC 1950). At most one of the two, and
 * only on the serializer formats (any other combination is TF_E_FATAL_UNSUPPORTED). tfgpu_result_bytes / _bytes_len give the
 * container, tfgpu_result_raw_len the length of the text inside it; row sizes, rows, selection, errors and part ids are those of the
 * same call without the flag. Layout of the container (tfgpu_deflate_stream_* relies on it):
 *   header      gzip 1f 8b 08 00 00000000 00 ff (no name, MTIME 0, XFL 0, OS 255) | zlib 78 9c: what Go's default writers emit
 *   chunks      the text cut into 16 KiB chunks, compressed independently (no back-reference crosses a chunk start); every chunk
 *               starts byte-aligned and ends with a sync-flush marker (an empty non-final stored block: ... 00 00 ff ff)
 *   final block 03 00 (an empty final fixed-Huffman block)
 *   trailer     gzip CRC-32 + ISIZE (little-endian) | zlib Adler-32 (big-endian)
 * The compressed bytes are not those of Go's compress/flate: the text they decode to and the framing above are what is pinned. */
#define TF_WIRE_F_GZIP            0x400
#define TF_WIRE_F_ZLIB            0x800
/* The ClickHouse HTTP uploader's Content-Encoding: zstd (httpclient/http_client_impl.go:54-86): the TF_WIRE_CH_JSONEACHROW text compressed
 * on the device into one zstd frame (RFC 8878). Only on TF_WIRE_CH_JSONEACHROW, and not with TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB (any other
 * combination is TF_E_FATAL_UNSUPPORTED). tfgpu_result_bytes / _bytes_len give the frame, tfgpu_result_raw_len the length of the text
 * inside it; row sizes, rows, errors and part ids are those of the same call without the flag. Layout of the frame (tfgpu_zstd_prefix
 * relies on it):
 *   header      28 b5 2f fd | c0 (8-byte Frame_Content_Size, no single segment, no checksum, no dictionary) | 28 (Window_Size 32 KiB,
 *               so Block_Maximum_Size 32 KiB) | Frame_Content_Size = the text length, 8 bytes little-endian: 14 bytes
 *   blocks      the text cut into 16 KiB chunks, one block per chunk in text order (Raw_Block, RLE_Block or Compressed_Block, whichever
 *               is smallest); Last_Block on the last one only. An empty text is one empty last Raw_Block (01 00 00). A block's matches
 *               reach at most 16 KiB before its chunk, never before the text's start, and a block uses no state of the blocks before it
 *               (no repeat offsets, treeless literals or Repeat_Mode tables)
 *   no content checksum: XXH64 is one serial chain over the whole content and cannot be combined from per-chunk pieces; decoders,
 *               ClickHouse's included, accept frames without it
 * The compressed bytes are not those of the reference's encoder: the text they decode to and the framing above are what is pinned. */
#define TF_WIRE_F_ZSTD            0x1000

typedef struct tfgpu_engine tfgpu_engine;
typedef struct tfgpu_result tfgpu_result;

/* cfg_json: {"frame_bytes":15360,...} or NULL for defaults; frame_bytes = uncompressed bytes per ClickHouse
 * compressed frame: a multiple of 16 in [1024, 15360] (one CTA of 256 threads compresses one frame in shared memory, four CTAs per SM).
 * One engine drives one device (device_ids[0]); n_devices must be 1 — multi-GPU
 * is one engine per GPU with batches dealt round-robin by the host (SURVEY §8e). */
int tfgpu_engine_create(const char* cfg_json, const int* device_ids, int n_devices,
                        tfgpu_engine** out);
int tfgpu_engine_destroy(tfgpu_engine* e);
const char* tfgpu_last_error(const tfgpu_engine* e);

/* Launch all work on this CUstream/cudaStream_t (NULL = the engine's own stream). */
int tfgpu_engine_set_stream(tfgpu_engine* e, void* cuda_stream);

/* Build (or fetch from the schema-hash cache) the plan for one table.
 *   table_namespace/table_name : abstract.TableID
 *   schema_json       : JSON array of ColSchema objects with the reference's tags
 *                       (pkg/abstract/changeitem/col_schema.go:14-29)
 *   transformers_json : the transfer YAML's `transformation.transformers` list as JSON
 *                       (pkg/transformer/abstract.go:20-48)
 *   sink_json         : {"type":"clickhouse", ...} or NULL when only push_columns is used
 * Returns plan id >= 0 in *plan_id. */
int tfgpu_plan(tfgpu_engine* e, const char* table_namespace, const char* table_name,
               const char* schema_json, const char* transformers_json, const char* sink_json,
               int* plan_id);
/* Same plan construction, host-only (no device, no engine): validates a transfer's transformer list against a
 * table schema and returns the describe JSON. rc < 0 with a message in err_out for configs the engine rejects. */
int tfgpu_plan_validate(const char* table_namespace, const char* table_name, const char* schema_json,
                        const char* transformers_json, const char* sink_json,
                        char* describe_out, uint64_t describe_cap, char* err_out, uint64_t err_cap);
/* JSON of the plan: result schema (ResultSchema chain), transformers kept by Suitable(),
 * the compiled predicate terms — owned by the engine, valid until the engine is destroyed. */
const char* tfgpu_plan_describe(tfgpu_engine* e, int plan_id);

/* Transformer chain only: Transformed rows come back columnar (host memory owned by the
 * result), Errors as a row-error list. */
int tfgpu_push_columns(tfgpu_engine* e, int plan_id, const tf_batch* in, tfgpu_result** out);

/* Transformer chain + sink cast + wire encode, fused on the device. */
int tfgpu_push_encode(tfgpu_engine* e, int plan_id, int wire_fmt, const tf_batch* in,
                      tfgpu_result** out);

/* tfgpu_push_encode in two phases, for host batches whose plan filters rows (the headline workload keeps 28 %): only the columns the
 * predicates read cross PCIe first and the device answers with one keep flag per row; host threads gather the kept rows (`threads` <= 0:
 * up to 32) and only those go through the chain and the encoder. The result is the one tfgpu_push_encode gives (all transformers are
 * row-local, filter_rows keeps what it kept; rows dropped with an error in phase one are reported with their input index). Plans without
 * filter steps, device batches, loosely typed predicate columns and batches under 8192 rows take the one-phase path. */
int tfgpu_push_encode_selective(tfgpu_engine* e, int plan_id, int wire_fmt, const tf_batch* in, int threads, tfgpu_result** out);
/* Bytes the engine has copied host -> device for batch columns since it was created (bench accounting of the e2e legs). */
uint64_t tfgpu_engine_h2d_bytes(const tfgpu_engine* e);

/* Queue Debezium serializer (pkg/serializer/queue/debezium_serializer.go:25-92 -> debezium.Emitter.EmitKV
 * pkg/debezium/emitter_value_converter.go:566-690). Runs the plan's chain on the device and writes, for every surviving INSERT row,
 * the Kafka key message immediately followed by the value message:
 *   key   = pack({"<pk col>":v,...})                                   (keys sorted: encoding/json map order)
 *   value = pack({"after":{...},"before":null,"op":"c"|"r","source":{...},"transaction":null,"ts_ms":CommitTime/1e6})
 *   pack(p) = p                                        schemas disabled (packer_skip_schema.go)
 *           | {"payload":p,"schema":<schema text>}      packer_include_schema.go:24-44
 *           | 0x00 | u32be schema id | p                packer_schema_registry.go:66-76
 * tfgpu_result_bytes holds the messages back to back; tfgpu_result_row_sizes[j] = key + value bytes of output row j,
 * tfgpu_result_key_sizes[j] = the key part (0 with drop_keys).
 * Values, by the column's original_type (emitter_value_converter.go:139-193):
 *   none              addCommon emitter_common.go:67-180: ints / uints bare, float / double as encoding/json writes float32 / float64,
 *                     boolean, `string` (bytes) base64, `utf8` JSON string (SetEscapeHTML(false)), datetime / timestamp RFC3339Nano,
 *                     `any`: Go string as is, object -> its JSON text as a string, JSON null -> null. Needs "ignore_unknown_sources"
 *                     (without it the reference answers errUnknownSource for such columns, :183-191).
 *   pg:...            AddPg pkg/debezium/pg/emitter.go:265-629 for boolean, smallint, integer, bigint, real (float32), double
 *                     precision ("NaN" / "Infinity" strings), text, character[ varying][(n)], uuid, cidr, macaddr, citext, inet, int4range,
 *                     int8range, bytea (base64), json / jsonb (JSON text as a string), date (days), timestamp[(p)] without time zone
 *                     (micro- or milliseconds by p), timestamp[(p)] with time zone (ZonedTimestamp string), on the column type the
 *                     pg source gives them. Other pg types, mysql: / ydb: types, and pg-typed columns a transformer rewrote are
 *                     refused by the call (TF_E_FATAL_UNSUPPORTED): the table stays on the Go emitter.
 * A value EmitKV fails on (date / interval without a pg type, `any` arrays / scalars, NaN, years outside [0,9999], a non-string in a
 * pg string type) is reported as TF_ROWERR_SER_VALUE (term = output column) and the shim fails the batch like Serialize does.
 * UPDATE / DELETE rows need ChangeItem.OldKeys: tfgpu_emit_debezium_crud (below) takes them as a second typed batch and emits every row kind;
 * this INSERT-only entry point is the same call with old == NULL.
 * opts_json: {"ignore_unknown_sources":bool, "snapshot":bool, "drop_keys":bool, "source_type":""|"pg"|"mysql", "version":"..",
 *   "topic_prefix":"..", "database":"..", "key_schema":"<json>"|null, "val_schema":"<json>"|null (what
 *   Emitter.ToKafkaSchemaKey/Val return for the plan's result schema; the lightning cache computes them once per table,
 *   packer/lightning_cache), "key_schema_id":N, "val_schema_id":N (confluent framing instead)}.
 * meta: the ChangeItem fields the envelope's `source` block carries (buildSource :329-372), in the memory space of `in`. */
typedef struct tf_row_meta {
    const uint32_t* id;            /* ChangeItem.ID  -> source.txId (pg); NULL = 0              */
    const uint64_t* lsn;           /* ChangeItem.LSN -> source.lsn (pg) / file + pos (mysql)    */
    const uint64_t* commit_time;   /* ChangeItem.CommitTime ns -> source.ts_ms and payload ts_ms */
    const uint32_t* txid_offsets;  /* ChangeItem.TxID -> source.gtid (mysql): nrows+1 offsets    */
    const uint8_t*  txid_heap;     /*   into this heap; NULL = "" (gtid null)                    */
} tf_row_meta;
int tfgpu_emit_debezium(tfgpu_engine* e, int plan_id, const char* opts_json, const tf_batch* in, const tf_row_meta* meta,
                        tfgpu_result** out);
/* ChangeItem.OldKeys (pkg/abstract/changeitem/old_keys.go:3-7) for a batch: KeyValues as typed cells in a second tf_batch with the
 * plan's input schema and the batch's row count (only the listed columns are read), present_cols[c] != 0 = column c is listed in
 * OldKeys.KeyNames, row_has[r] != 0 = row r carries OldKeys at all (NULL: every update / delete row does). */
typedef struct tf_old_keys {
    const tf_batch* values;
    const uint8_t*  present_cols;   /* ncols flags (host memory) */
    const uint8_t*  row_has;        /* nrows flags in the memory space of the batch, or NULL */
} tf_old_keys;
/* Emitter.emitKV for every row kind (pkg/debezium/emitter_value_converter.go:626-674): in->kinds says insert / update / delete;
 *   insert, update that keeps its primary key  -> one message (op c|r / u; `before` = OldKeys when they list more than the keys,
 *                                                  hasPreviousValues :277-285, else null; key from OldKeys, else from the row)
 *   delete                                      -> the delete event (op d, after null, before = every column null + OldKeys) and its
 *                                                  tombstone (key only) unless opts "tombstones_on_delete":false
 *   update that changes its primary key (ChangeItem.KeysChanged) -> delete event, tombstone, insert event (op c, key from the row)
 * The messages of a row are contiguous in the result bytes; tfgpu_result_dbz_msg_sizes gives, per output row, the message count and
 * (key bytes, value bytes | 0xFFFFFFFF for a tombstone) per message. `old` may be NULL (no row carries OldKeys: keys come from the row
 * and every update counts as key-changing, as in the reference). Plans whose transformers rewrite values are refused here. */
int tfgpu_emit_debezium_crud(tfgpu_engine* e, int plan_id, const char* opts_json, const tf_batch* in, const tf_old_keys* old,
                             const tf_row_meta* meta, tfgpu_result** out);
const uint32_t* tfgpu_result_dbz_msg_sizes(const tfgpu_result* r);   /* 7 * rows_out entries */
/* Host-only (no GPU): the set-up tfgpu_emit_debezium derives from a table and opts_json — the value branch of every result column
 * (0 addCommon, else the AddPg branch), the key columns in message order and the message template (text pieces + the per-row field
 * that follows each) — or the error the call would return. Same arguments as tfgpu_plan_validate plus opts_json. */
int tfgpu_emit_debezium_validate(const char* ns, const char* name, const char* schema_json, const char* transformers_json, const char* opts_json,
                                 char* describe_out, uint64_t cap, char* err_out, uint64_t err_cap);

/* Measurer middleware (pkg/middlewares/synchronizer/measurer.go:38-42): ChangeItem.Size.Values = util.DeepSizeof(ColumnValues)
 * (pkg/util/sizeof.go:7-110) for every row of `in`, computed in closed form from the column types and lengths instead of a
 * reflection walk. per_row (host, nrows entries) may be NULL; *total receives the sum. `any` cells that are not Go strings
 * are counted as their JSON text (the reference walks the map / slice). */
int tfgpu_measure(tfgpu_engine* e, const tf_batch* in, uint64_t* per_row, uint64_t* total);

/* parsers.Parser for CSV (pkg/parsers/abstract.go:35-38 shape; algorithm of the S3 CSV reader:
 * pkg/csv/reader.go:89-324 + pkg/providers/s3/reader/registry/csv/reader_csv.go:186-452 + strictify.go:18-181).
 * One chunk of raw bytes (host, or device memory at any alignment, < 4 GiB) is split into lines and typed columns ON THE DEVICE and fed straight
 * into the plan's transformer chain; wire_fmt 0 returns the Transformed rows columnar (tfgpu_result_batch), otherwise the
 * sink wire bytes. The schema's `path` of each column is the field index (reader_csv.go:286); opts_json:
 * {"delimiter":",","quote":"\"","escape":"\\","double_quote":true,"null_values":[..],"strings_can_be_null":false,
 *  "quoted_strings_can_be_null":false,"true_values":[..],"false_values":[..],"include_missing_columns":false,"skip_lines":0}.
 * Inside an element, the quote character written twice stands for one '"' (the S3 reader's DoubleQuoteStr = quote + quote,
 * swapToSingleQuotes reader.go:309-324), whatever the quote character is; with "double_quote":false such a pair is
 * TF_ROWERR_CSV_DQ_DISABLED. With "quote":"" a data line that contains '"' is TF_ROWERR_CSV_QUOTING_DISABLED, which outranks
 * every other error of the line; lines dropped by skip_lines are not checked (in the reference such a line fails the whole read).
 * Row-level failures come back as row errors with TF_ROWERR_CSV_* codes (row = data line index); an unterminated last
 * line is left unconsumed (tfgpu_result_consumed) exactly as the reference drops it (reader.go:162-165). */
int tfgpu_parse_csv(tfgpu_engine* e, int plan_id, const char* opts_json, const uint8_t* bytes, uint64_t len, int mem,
                    int wire_fmt, tfgpu_result** out);
uint64_t tfgpu_result_consumed(const tfgpu_result* r);

/* Same as tfgpu_push_encode but asynchronous and HBM-resident: `in` must be
 * TF_MEM_DEVICE, nothing is copied back and no host sync happens; the wire
 * bytes stay in the engine's device arena (tfgpu_result_device_*) until the
 * next call on this engine. Used to time kernels without PCIe in the way. */
int tfgpu_push_encode_resident(tfgpu_engine* e, int plan_id, int wire_fmt, const tf_batch* in);
/* After a stream sync: counters of the last resident call. */
int tfgpu_resident_stats(tfgpu_engine* e, uint64_t* rows_out, uint64_t* raw_bytes,
                         uint64_t* wire_bytes, uint64_t* n_errors);
/* Copy the last resident call's uncompressed block / wire bytes to host (tests). */
int tfgpu_resident_fetch(tfgpu_engine* e, int what /*0=raw block,1=wire*/, uint8_t* dst, uint64_t cap);

/* Result accessors. Row errors and the columnar batch are owned by the result until
 * tfgpu_result_release; the wire bytes live in the engine's pinned landing buffer and stay valid
 * until the NEXT push on the same engine (the Go shim writes them to the socket before that). */
uint64_t          tfgpu_result_rows_in(const tfgpu_result* r);
/* parsers.Parser.DoBatch for the generic JSON parser (pkg/parsers/abstract.go:35-38; algorithm
 * pkg/parsers/generic/generic_parser.go:406-430 DoBatch, :519-555 doGenericParser, :672-730 Unmarshal, :888-1123 ParseVal,
 * :297-404 makeChangeItem; config pkg/parsers/registry/json/parser_json.go:51-87).
 * `bytes` holds n_msgs message payloads back to back (host or device, < 4 GiB); msgs[k] gives message k's end offset and
 * the queue metadata the aux columns need. The plan's schema is the parser's RESULT schema (addAuxFields :115-164): the
 * declared fields (int8..uint64, double, boolean, utf8, string, any, datetime; flat keys), then `_rest` when add_rest,
 * then _timestamp,_partition,_offset,_idx when add_dedupe_keys. Lines are split, parsed and typed ON THE DEVICE and fed
 * straight into the plan's transformer chain; wire_fmt 0 returns the rows columnar, otherwise the sink wire bytes.
 * opts_json: {"add_rest":false,"add_dedupe_keys":false,"null_keys_allowed":false,"use_numbers_in_any":false,
 *             "unpack_bytes_base64":false,"partition":"<abstract.Partition.String()>"}; any other AuxParserOpts switch
 * (time_field, table_splitter, unescape_string_values, add_system_columns, ...) is refused with TF_E_FATAL_UNSUPPORTED.
 * Row errors: row = index of the line among the non-empty lines of the call, code TF_ROWERR_JSON_*, term = column.
 * PARSE / NIL_REQUIRED / PARSEVAL lines are the reference's `_unparsed` rows (the shim builds them, reason text from Go);
 * SKIP lines produce nothing; HOST lines carry a value whose reference result needs a Go library the device does not
 * restate (dateparse, goccy re-parse of JSON inside a string, > 19 digit floats with undecided rounding, NaN/Inf or an
 * invalid number inside `any`, nesting deeper than 24, a key named like an aux column) and must be re-parsed by the
 * host parser. */
typedef struct tf_msg { uint64_t end; uint64_t offset; int64_t write_sec; uint32_t write_nsec; uint32_t pad; } tf_msg;
int tfgpu_parse_json(tfgpu_engine* e, int plan_id, const char* opts_json, const uint8_t* bytes, uint64_t len, int mem,
                     const tf_msg* msgs, uint32_t n_msgs, int wire_fmt, tfgpu_result** out);

/* parsers.Parser.DoBatch for the Debezium parser (pkg/parsers/registry/debezium/engine/parser.go:34-137; receive path
 * pkg/debezium/receiver.go:142-220, receiver_engine.go:143-330, common/field_receiver_default.go:15-330).
 * `bytes` holds n_msgs queue messages back to back (msg_ends[k] = end offset of message k), each either
 * {"schema":<Kafka Connect schema>,"payload":{before,after,source,op,ts_ms}} or, with "schema_registry":true, a confluent
 * frame 0x00 | u32be schema id | payload JSON. opts_json: {"schema_text":"<the exact schema JSON text the plan was built
 * for>","schema_registry":false,"schema_id":0,"check_table":false}. The plan's schema must be the table schema the
 * reference derives from the schema's `after` struct with the DEFAULT receivers: int8/16/32/64, boolean, string -> utf8,
 * float/double -> double, bytes -> string (base64) or utf8 for org.apache.kafka.connect.data.Decimal, struct -> utf8 for
 * io.debezium.data.geometry.Point / double for io.debezium.data.VariableScaleDecimal; key = !optional. Messages are validated
 * with encoding/json's grammar, typed and fed into the plan's chain ON THE DEVICE; one row per message.
 * Row errors (row = message index): TF_ROWERR_DBZ_UNPARSED = the reference's `_unparsed` row; TF_ROWERR_DBZ_HOST = the
 * message needs the Go parser (several events in one frame, keys matching only case-insensitively or with escapes,
 * __debezium_unavailable_value, magnitudes over 256 bits, nesting over 256); TF_ROWERR_DBZ_OTHER_SCHEMA / _OTHER_TABLE = the
 * message belongs to another plan. Per message metadata (ChangeItem.Kind / ID / LSN / CommitTime, receiver.go:182-190) comes
 * back through tfgpu_result_meta_*; tfgpu_result_selection maps output rows to messages. */
#define TF_ROWERR_DBZ_UNPARSED     48
#define TF_ROWERR_DBZ_HOST         49
#define TF_ROWERR_DBZ_OTHER_SCHEMA 50
#define TF_ROWERR_DBZ_OTHER_TABLE  51
int tfgpu_parse_debezium(tfgpu_engine* e, int plan_id, const char* opts_json, const uint8_t* bytes, uint64_t len, int mem,
                         const uint64_t* msg_ends, uint32_t n_msgs, int wire_fmt, tfgpu_result** out);
/* Host-only (no GPU): the table schema tfgpu_parse_debezium expects the plan to be built for — name, YT type, key = !optional — and the
 * receiver of every field, derived from the envelope schema as the reference does (receiver.go:46-62, receiver_engine.go:104-141), or
 * the error the call would return (database specific original types, struct kinds without a default receiver, before != after). */
int tfgpu_debezium_schema_validate(const char* schema_text, char* describe_out, uint64_t cap, char* err_out, uint64_t err_cap);
/* Profiling aid: cycles thread 0 of every k_lz4_frames CTA spent in {stage, match finding, parse, scan, emit} since the last read. */
int tfgpu_debug_lz4_phases(tfgpu_engine* e, int enable, uint64_t out[8]);
const uint32_t*   tfgpu_result_selection(const tfgpu_result* r);          /* rows_out entries: input row of each output row */
const uint8_t*    tfgpu_result_meta_kinds(const tfgpu_result* r);         /* per message (rows_in entries) */
const uint32_t*   tfgpu_result_meta_tx_id(const tfgpu_result* r);
const uint64_t*   tfgpu_result_meta_lsn(const tfgpu_result* r);
const uint64_t*   tfgpu_result_meta_commit_time(const tfgpu_result* r);

uint64_t          tfgpu_result_rows_out(const tfgpu_result* r);
uint64_t          tfgpu_result_n_errors(const tfgpu_result* r);
const tf_rowerr*  tfgpu_result_errors(const tfgpu_result* r);
const tf_batch*   tfgpu_result_batch(const tfgpu_result* r);      /* push_columns only   */
const uint8_t*    tfgpu_result_bytes(const tfgpu_result* r);      /* push_encode: wire    */
uint64_t          tfgpu_result_bytes_len(const tfgpu_result* r);
uint64_t          tfgpu_result_raw_len(const tfgpu_result* r);    /* uncompressed block   */
uint64_t          tfgpu_result_n_frames(const tfgpu_result* r);
/* Row-text formats (TF_WIRE_SER_JSON/CSV, TF_WIRE_CH_JSONEACHROW): bytes of every output row in the order written,
 * separator included (SER_JSON without CLOSING_NEWLINE: rows after the first start with '\n'). rows_out entries or NULL. */
const uint32_t*   tfgpu_result_row_sizes(const tfgpu_result* r);
/* sharder_transformer in the plan (pkg/transformer/registry/sharder/sharder.go:130-145): ChangeItem.PartID of every output row
 * as the integer the reference prints with %d (CRC32-IEEE of the joined text forms of the matched columns, modulo ShardsNum);
 * rows_out entries, NULL when the plan has no sharder. is_random sharders are refused by tfgpu_plan (uuid + rand.Intn: host). */
const uint32_t*   tfgpu_result_part_ids(const tfgpu_result* r);
const uint32_t*   tfgpu_result_key_sizes(const tfgpu_result* r);  /* tfgpu_emit_debezium: key bytes of every output row */

/* Queue JSON serializer (pkg/serializer/queue/json_serializer.go:22-83 + json_batcher.go:13-66): the message VALUES are the
 * TF_WIRE_SER_JSON rows (key = ChangeItem.Fqtn(), built by the shim); with batching enabled BatchJSON packs consecutive rows
 * joined by '\n' greedily under MaxMessageSize / MaxChangeItems. Given the JSON length of every row (row_sizes minus the
 * separator byte) this returns the first row of every message: message k = rows [starts[k], starts[k+1]); starts needs
 * n + 1 entries. Host only. Update / delete items are refused by the reference (json_serializer.go:17-20): check kinds first. */
int tfgpu_queue_json_batches(const uint32_t* json_row_sizes, uint64_t n, uint64_t max_message_size, uint64_t max_change_items,
                             uint64_t* starts, uint64_t cap, uint64_t* n_msgs);
/* Queue Debezium serializer with batching.max.size (pkg/serializer/queue/debezium_multithreading.go:67-106 MergeWithMaxMessageSize):
 * the VALUES of consecutive messages are appended to one another (no separator, Key nil) while
 * len(current) + 1 + len(next) <= max_message_size; the first value always opens a message. Given the value length of every row
 * (tfgpu_result_row_sizes - tfgpu_result_key_sizes; emit with "drop_keys" so that the values lie back to back) this returns the first
 * row of every merged message as tfgpu_queue_json_batches does. max_message_size == 0: the reference does not merge (MergeBack). Host only. */
int tfgpu_queue_debezium_batches(const uint32_t* value_sizes, uint64_t n, uint64_t max_message_size, uint64_t* starts, uint64_t cap, uint64_t* n_msgs);
void              tfgpu_result_release(tfgpu_result* r);

/* One object out of many pushes (host only): the snapshot writer streams every batch of a file through one gzip / zlib writer, and a
 * zlib object cannot be a concatenation of streams. A stream joins the results of TF_WIRE_F_GZIP (or TF_WIRE_F_ZLIB) pushes, in
 * order, into one gzip member (one zlib stream) that decodes to the concatenation of their texts: the header once, every result's
 * chunks, then the final block and a trailer with the checksums combined (ISIZE = total text length mod 2^32).
 *   open    container = TF_WIRE_F_GZIP | TF_WIRE_F_ZLIB
 *   append  one result: its bytes / bytes_len / raw_len (tfgpu_result_bytes, _bytes_len, _raw_len). The first append also writes
 *           the header. *written = bytes put at out. A result whose header, final block or trailer does not match the container
 *           (or whose gzip ISIZE is not raw_len mod 2^32) is refused with TF_E_FATAL_ARG, as is out too small (cap); the stream
 *           is unchanged then.
 *   close   the final block and the trailer (after the header when nothing was appended): *written bytes at out.
 * Returns TF_OK or TF_E_FATAL_ARG. */
typedef struct tfgpu_deflate_stream tfgpu_deflate_stream;
int  tfgpu_deflate_stream_open(int container, tfgpu_deflate_stream** out);
int  tfgpu_deflate_stream_append(tfgpu_deflate_stream* s, const uint8_t* bytes, uint64_t len, uint64_t raw_len, uint8_t* out, uint64_t cap,
                                 uint64_t* written);
int  tfgpu_deflate_stream_close(tfgpu_deflate_stream* s, uint8_t* out, uint64_t cap, uint64_t* written);
void tfgpu_deflate_stream_free(tfgpu_deflate_stream* s);

/* The INSERT line in front of a TF_WIRE_F_ZSTD result, inside the same frame (host only): the reference compresses
 * `INSERT INTO ... FORMAT JSONEachRow\n` and the rows as one zstd frame. Writes to out a frame header whose content size is text_len plus
 * the frame's, then `text` as Raw_Blocks of at most 32 KiB; the body to send is out[0, *written) followed by frame[14, frame_len) (the
 * engine's frame after its fixed header, never copied). A frame whose header is not the engine's layout, or whose block headers do not
 * walk exactly to frame_len, is refused with TF_E_FATAL_ARG, as is out too small (cap). Returns TF_OK or TF_E_FATAL_ARG. */
int tfgpu_zstd_prefix(const uint8_t* text, uint64_t text_len, const uint8_t* frame, uint64_t frame_len, uint8_t* out, uint64_t cap,
                      uint64_t* written);

/* Number of kernel launches issued by this engine since creation (bench `gpu_launches`). */
uint64_t tfgpu_engine_launch_count(const tfgpu_engine* e);

/* Optional per-kernel timing with CUDA events on the streams the kernels run on (bench.py roofline): the profile holds every launch,
 * in launch order, of the last call that launched a kernel after tfgpu_profile_enable; calls that launch none (tfgpu_resident_stats,
 * tfgpu_profile_read itself) leave it as it is. tfgpu_profile_read synchronises the stream and returns JSON
 * [{"name":"k_lz4_frames","ms":..},..] owned by the engine. */
int tfgpu_profile_enable(tfgpu_engine* e, int on);
const char* tfgpu_profile_read(tfgpu_engine* e);

/* Library identity: "tfgpu <version> sm_90a". */
const char* tfgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TFGPU_H_ */
