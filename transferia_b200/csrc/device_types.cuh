// Device-visible descriptors shared by all kernels (sm_90a).
#pragma once
#include <cstdint>
#include "../../include/tfgpu.h"

namespace tfk {

// how one output column is produced in the ClickHouse native block
enum OutKind : int32_t {
    OK_COPY = 0,      // fixed width, bytes copied as is (ints, floats, interval)
    OK_BOOL = 1,      // boolean -> UInt8 0/1
    OK_DATE = 2,      // time seconds -> clamp [1970-01-01, 2106-01-01] -> u16 days       (columntypes/types.go:15-29,93-104)
    OK_DATETIME = 3,  // time seconds -> same clamp -> u32 seconds
    OK_TS64 = 4,      // time (sec, nsec) -> DateTime64(6) = UnixMicro, no clamp          (columntypes/types.go:242)
    OK_STR = 5,       // LEB128 length + bytes
    OK_MASK = 6,      // mask_field digest: 0x40 + 64 lowercase hex chars                  (hmac_hasher.go:29-33)
    OK_TODT = 8,      // convert_to_datetime: int32/uint32 seconds -> time.Unix(s, 0), never nil     (to_datetime.go:137-151)
    OK_TOSTR = 7      // convert_to_string: LEB128 length + text form of the value         (to_string.go:145-171)
};

struct DCol {
    int32_t type;       // input tf_type
    int32_t out_kind;   // OutKind
    int32_t in_w;       // bytes per input element (fixed types), 0 for var-width
    int32_t out_w;      // bytes per output element (fixed kinds, 65 for OK_MASK), 0 for OK_STR
    int32_t nullable;   // Nullable(T): a null map precedes the data
    int32_t str_slot;   // index among OK_STR columns, else -1
    int32_t mask_slot;  // index of the mask step touching this column, else -1
    int32_t pad;
    const uint8_t* values;
    const uint8_t* validity;
    const uint32_t* offsets;
    const uint8_t* heap;
    const uint8_t* aux;
    uint64_t hdr_off;   // where this column's name/type header starts in the block  (k_layout)
    uint64_t null_off;  // null map start                                               (k_layout)
    uint64_t out_off;   // data start                                                   (k_layout)
    uint64_t aux_off;   // columnar output only: nanos / any-tags region
    uint64_t offs_off;  // columnar output only: uint32 offsets region (nrows+1)
};

struct DTerm {          // must match tfplan::DTerm
    int32_t col, op, vtype, nlist;
    int64_t i; double f;
    uint32_t s_off, s_len;
    uint32_t list_off, pad;
};

// flags: bit0 = skip_events step (expr_begin holds the kind mask), bit1 = filter_rows that lets every row pass
// (its table filter does not match the renamed table) but still rejects update/delete kinds
struct DFilterStep { int32_t expr_begin, nexpr, step_index, flags; };

// counters / layout results living in device memory, read back only by the host API that needs them
struct DState {
    uint64_t n_kept;
    uint64_t n_errors;
    uint64_t raw_total;     // bytes of the uncompressed native block
    uint64_t n_frames;
    uint64_t wire_total;    // bytes of the framed, compressed stream
    uint32_t frame_ticket;  // persistent-kernel work counter
    uint32_t pad;
};

__host__ __device__ inline int varint_len(uint64_t v) { int n = 1; while (v >= 0x80) { v >>= 7; n++; } return n; }

}  // namespace tfk
