// filter_rows predicate, row compaction, typesystem cast + ClickHouse native block encode.
// All kernels are HBM-streaming: coalesced element loads along rows, one launch covers every
// column (blockIdx.y = column slot), no tensor cores (there is no contraction on this path).
#pragma once
#include "device_types.cuh"

namespace tfk {

// ------------------------------------------------------------------ small block-scan helpers
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
    const unsigned lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, v, d); if (lane >= (unsigned)d) v += t; }
    return v;
}
// exclusive scan over blockDim.x (<= 1024) threads; returns exclusive prefix, *total = block sum
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total, uint32_t* smem33) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    uint32_t inc = warp_incl_scan(v);
    if (lane == 31) smem33[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nw ? smem33[lane] : 0;
        uint32_t wi = warp_incl_scan(w);
        smem33[lane] = wi - w;
        if (lane == 31) smem33[32] = wi;
    }
    __syncthreads();
    uint32_t res = inc - v + smem33[warp];
    *total = smem33[32];
    __syncthreads();
    return res;
}

// ------------------------------------------------------------------ Strictify over typed columns
// strictify.Strictify / strictifyValue / toSignedInt / toUnsignedInt (pkg/abstract/changeitem/strictify/strictify.go:18-181) for values
// that arrive in another fixed-width type than the column's schema type (a Go int64 in an int32 column, a float64 in an int8 column ...):
// the spf13/cast conversion (Go conversion semantics, negatives refused by the unsigned targets), then the range check on
// cast.ToInt64 / cast.ToUint64 of the value. One thread per row walks the loose columns in schema order, so the row's error is the first
// failing column's, like Strictify's.
struct StrictCol { const uint8_t* src; uint8_t* dst; const uint8_t* validity; int32_t src_tf, dst_tf, col, pad; };
struct StrictArgs { const StrictCol* cols; int ncols; uint64_t nrows; uint8_t* err; uint16_t* term; };
__device__ __forceinline__ int64_t go_f2i64(double f) { return (f >= -9223372036854775808.0 && f < 9223372036854775808.0) ? (int64_t)f : INT64_MIN; }   // CVTTSD2SQ
__device__ __forceinline__ uint64_t go_f2u64(double f) { return f < 9223372036854775808.0 ? (uint64_t)go_f2i64(f) : ((uint64_t)go_f2i64(f - 9223372036854775808.0) ^ 0x8000000000000000ull); }
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_strictify(StrictArgs a) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.nrows) return;
    int err = 0, term = 0xff;
    for (int k = 0; k < a.ncols; k++) {
        const StrictCol c = a.cols[k];
        if (c.validity && !((c.validity[r >> 3] >> (r & 7)) & 1)) continue;            // nil stays nil (:55-57); the slot keeps whatever it held
        // the value as the three views spf13/cast takes of it
        int cls; int64_t si = 0; uint64_t ui = 0; double f = 0;                          // cls: 0 signed, 1 unsigned, 2 float, 3 bool
        switch (c.src_tf) {
        case TF_INT8: cls = 0; si = ((const int8_t*)c.src)[r]; break;
        case TF_INT16: cls = 0; si = ((const int16_t*)c.src)[r]; break;
        case TF_INT32: cls = 0; si = ((const int32_t*)c.src)[r]; break;
        case TF_INT64: cls = 0; si = ((const int64_t*)c.src)[r]; break;
        case TF_UINT8: cls = 1; ui = c.src[r]; break;
        case TF_UINT16: cls = 1; ui = ((const uint16_t*)c.src)[r]; break;
        case TF_UINT32: cls = 1; ui = ((const uint32_t*)c.src)[r]; break;
        case TF_UINT64: cls = 1; ui = ((const uint64_t*)c.src)[r]; break;
        case TF_FLOAT: cls = 2; f = ((const float*)c.src)[r]; break;
        case TF_DOUBLE: cls = 2; f = ((const double*)c.src)[r]; break;
        default: cls = 3; si = c.src[r] ? 1 : 0; break;                                   // TF_BOOLEAN
        }
        int e = 0;
        const int64_t as_i = cls == 0 || cls == 3 ? si : (cls == 1 ? (int64_t)ui : go_f2i64(f));                 // ToInt64E
        const bool neg = cls == 0 ? si < 0 : (cls == 2 ? f < 0 : false);
        const uint64_t as_u = cls == 0 || cls == 3 ? (uint64_t)si : (cls == 1 ? ui : go_f2u64(f));               // ToUint64E (negatives refused below)
        auto sint = [&](int64_t lo, int64_t hi) { if (as_i < lo || as_i > hi) e = TF_ROWERR_STRICT_RANGE; };
        auto uint_ = [&](uint64_t hi) { if (neg) e = TF_ROWERR_STRICT_CAST; else if (as_u > hi) e = TF_ROWERR_STRICT_RANGE; };
        switch (c.dst_tf) {
        case TF_INT8: sint(INT8_MIN, INT8_MAX); ((int8_t*)c.dst)[r] = (int8_t)as_i; break;
        case TF_INT16: sint(INT16_MIN, INT16_MAX); ((int16_t*)c.dst)[r] = (int16_t)as_i; break;
        case TF_INT32: sint(INT32_MIN, INT32_MAX); ((int32_t*)c.dst)[r] = (int32_t)as_i; break;
        case TF_INT64: case TF_INTERVAL: case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:       // int64 targets: ToInt64E / Duration(v) / time.Unix(v, 0)
            ((int64_t*)c.dst)[r] = as_i; break;
        case TF_UINT8: uint_(UINT8_MAX); c.dst[r] = (uint8_t)as_u; break;
        case TF_UINT16: uint_(UINT16_MAX); ((uint16_t*)c.dst)[r] = (uint16_t)as_u; break;
        case TF_UINT32: uint_(UINT32_MAX); ((uint32_t*)c.dst)[r] = (uint32_t)as_u; break;
        case TF_UINT64: uint_(UINT64_MAX); ((uint64_t*)c.dst)[r] = as_u; break;
        case TF_FLOAT: ((float*)c.dst)[r] = cls == 0 || cls == 3 ? (float)si : (cls == 1 ? (float)ui : (float)f); break;     // ToFloat32E: one Go conversion
        case TF_DOUBLE: ((double*)c.dst)[r] = cls == 0 ? (double)si : (cls == 1 ? (double)ui : f); break;                    // json.Number of the decimal text: the nearest float64
        default: c.dst[r] = cls == 2 ? (f != 0) : (cls == 1 ? ui != 0 : si != 0); break;                                     // TF_BOOLEAN: ToBoolE
        }
        if (e && !err) { err = e; term = c.col; }
    }
    const bool mine = err && !a.err[r];                    // an error raised upstream (parser) keeps its code and term 0xff
    if (mine) a.err[r] = (uint8_t)err;
    a.term[r] = (uint16_t)(mine ? term : 0xff);
}
#endif  // TF_KERNELS_ENCODE

// ------------------------------------------------------------------ filter_rows
// matchValue (pkg/transformer/registry/filter_rows/filter_rows.go:180-365) for typed columns.
struct RowVal {
    int cls;            // 0 nil, 1 int, 2 float, 3 bool, 4 string(Go string), 5 bytes, 6 time, 7 opaque (Duration / JSON tree), 8 uint64 overflow
    int64_t i; double f; const uint8_t* s; uint32_t slen; uint32_t nsec;
};

__device__ __forceinline__ bool row_valid(const DCol& c, uint64_t r) { return !c.validity || ((c.validity[r >> 3] >> (r & 7)) & 1); }

__device__ __forceinline__ RowVal load_val(const DCol& c, uint64_t r) {
    RowVal v; v.cls = 0; v.i = 0; v.f = 0; v.s = nullptr; v.slen = 0; v.nsec = 0;
    if (!row_valid(c, r)) return v;
    switch (c.type) {
    case TF_INT8:  v.cls = 1; v.i = ((const int8_t*)c.values)[r]; break;
    case TF_INT16: v.cls = 1; v.i = ((const int16_t*)c.values)[r]; break;
    case TF_INT32: v.cls = 1; v.i = ((const int32_t*)c.values)[r]; break;
    case TF_INT64: v.cls = 1; v.i = ((const int64_t*)c.values)[r]; break;
    case TF_UINT8:  v.cls = 1; v.i = ((const uint8_t*)c.values)[r]; break;
    case TF_UINT16: v.cls = 1; v.i = ((const uint16_t*)c.values)[r]; break;
    case TF_UINT32: v.cls = 1; v.i = ((const uint32_t*)c.values)[r]; break;
    case TF_UINT64: { uint64_t u = ((const uint64_t*)c.values)[r]; if (u > 0x7fffffffffffffffULL) v.cls = 8; else { v.cls = 1; v.i = (int64_t)u; } break; }   // util.go:66-68
    case TF_FLOAT:  v.cls = 2; v.f = ((const float*)c.values)[r]; break;
    case TF_DOUBLE: v.cls = 2; v.f = ((const double*)c.values)[r]; break;
    case TF_BOOLEAN: v.cls = 3; v.i = c.values[r] != 0; v.f = v.i ? 1.0 : 0.0; break;
    case TF_INTERVAL: v.cls = 7; break;
    case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP:
        v.cls = 6; v.i = ((const int64_t*)c.values)[r]; v.nsec = c.aux ? ((const uint32_t*)c.aux)[r] : 0; break;
    case TF_BYTES: v.cls = 5; v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; break;
    case TF_UTF8:  v.cls = 4; v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; break;
    case TF_ANY:
        if (c.aux && c.aux[r] == 1) { v.cls = 4; v.s = c.heap + c.offsets[r]; v.slen = c.offsets[r + 1] - c.offsets[r]; }
        else v.cls = 7;
        break;
    }
    return v;
}

template <typename T> __device__ __forceinline__ bool ordered(T a, T b, int op) {
    switch (op) { case 0: return a == b; case 1: return a != b; case 2: return a < b; case 3: return a <= b; case 4: return a > b; default: return a >= b; }
}
__device__ __forceinline__ int cmp_bytes(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {
    uint32_t m = an < bn ? an : bn;
    for (uint32_t k = 0; k < m; k++) { int d = (int)a[k] - (int)b[k]; if (d) return d < 0 ? -1 : 1; }
    return an < bn ? -1 : (an > bn ? 1 : 0);
}
__device__ __forceinline__ bool contains_bytes(const uint8_t* h, uint32_t hn, const uint8_t* n, uint32_t nn) {
    if (nn == 0) return true;
    if (nn > hn) return false;
    const uint8_t n0 = n[0];
    for (uint32_t i = 0; i + nn <= hn; i++) {
        if (h[i] != n0) continue;
        uint32_t k = 1; while (k < nn && h[i + k] == n[k]) k++;
        if (k == nn) return true;
    }
    return false;
}

// returns 0 and sets matched, or a TF_ROWERR_* code
static __device__ int eval_term(const RowVal& v, const DTerm& t, const uint8_t* blob, bool& matched) {
    const int op = t.op; const bool is_set = (op == 6 || op == 7);
    const int base = t.vtype & 15; const bool is_list = (t.vtype & 16) != 0;
    if (v.cls == 8) return TF_ROWERR_FILTER_OVERFLOW;                       // filter_rows.go:193-197
    if (op >= 8 && base != 4) return TF_ROWERR_FILTER_TYPEPAIR;             // ~ / !~ on a non-string literal: matchOrderedValue has no such operation (:367-383)
    const bool is_int1 = v.cls == 1;
    const bool is_float1 = v.cls == 2 || v.cls == 3 || v.cls == 0;          // cast.ToFloat64E: floats, bool, nil (-> 0)
    const double float1 = v.cls == 2 ? v.f : (v.cls == 3 ? v.f : 0.0);
    const int64_t* il = (const int64_t*)(blob + t.list_off);
    const double* fl = (const double*)(blob + t.list_off);
    switch (base) {
    case 1:   // int literal(s)
        if (is_int1) {
            if (is_set) { bool c = false; for (int k = 0; k < t.nlist; k++) c |= (il[k] == v.i); matched = (op == 6) ? c : !c; return 0; }
            matched = ordered<int64_t>(v.i, t.i, op); return 0;
        }
        if (is_float1) {
            if (is_set) {                                                   // int64(float1) of amd64, not cvt.rzi's saturation
                if (trunc(float1) == float1) { int64_t x = go_f2i64(float1); bool c = false; for (int k = 0; k < t.nlist; k++) c |= (il[k] == x); matched = (op == 6) ? c : !c; }
                else matched = false;
                return 0;
            }
            matched = ordered<double>(float1, (double)t.i, op); return 0;
        }
        break;
    case 2:   // float literal(s)
        if (is_int1 || is_float1) {
            const double x = is_int1 ? (double)v.i : float1;
            if (is_set) { bool c = false; for (int k = 0; k < t.nlist; k++) c |= (fl[k] == x); matched = (op == 6) ? c : !c; return 0; }
            matched = ordered<double>(x, t.f, op); return 0;
        }
        break;
    case 3:   // bool
        if (!is_list && v.cls == 3) { matched = ordered<int>(v.i ? 1 : 0, t.i ? 1 : 0, op); return 0; }
        break;
    case 4:   // string
        if (v.cls == 4 || v.cls == 5) {
            const uint8_t* lit = blob + t.s_off;
            if (!is_list) {
                if (op == 8) { matched = contains_bytes(v.s, v.slen, lit, t.s_len); return 0; }
                if (op == 9) { matched = !contains_bytes(v.s, v.slen, lit, t.s_len); return 0; }
                if (is_set) return TF_ROWERR_FILTER_TYPEPAIR;
                const int c = cmp_bytes(v.s, v.slen, lit, t.s_len);
                matched = ordered<int>(c, 0, op); return 0;
            }
            if (!is_set) return TF_ROWERR_FILTER_TYPEPAIR;
            const uint32_t* so = (const uint32_t*)(blob + t.list_off);
            const uint8_t* sh = (const uint8_t*)(so + t.nlist + 1);
            bool c = false;
            for (int k = 0; k < t.nlist && !c; k++) { uint32_t a = so[k], b = so[k + 1]; c = (b - a == v.slen) && cmp_bytes(sh + a, b - a, v.s, v.slen) == 0; }
            matched = (op == 6) ? c : !c; return 0;
        }
        break;
    case 5:   // time: compared as UnixMicro (filter_rows.go:330-339)
        if (v.cls == 6) {
            const int64_t um = v.i * 1000000LL + (int64_t)(v.nsec / 1000u);
            if (is_set) { bool c = false; for (int k = 0; k < t.nlist; k++) c |= (il[k] == um); matched = (op == 6) ? c : !c; return 0; }
            matched = ordered<int64_t>(um, t.i, op); return 0;
        }
        break;
    case 6:   // NULL
        if (op == 0) { matched = v.cls == 0; return 0; }
        if (op == 1) { matched = v.cls != 0; return 0; }
        break;
    }
    return TF_ROWERR_FILTER_TYPEPAIR;
}

struct FilterArgs {
    const DCol* cols; const uint8_t* kinds; uint64_t nrows;
    const DFilterStep* steps; int nsteps;
    const uint32_t* expr_off;      // term ranges per expression (global expr index)
    const DTerm* terms; const uint8_t* blob;
    uint8_t* keep; uint8_t* errcode; uint16_t* errstep; uint32_t* blockcnt; DState* st;
    const uint8_t* pre_err;        // optional per-row error already raised upstream (parser): the row is dropped and reported
    const uint16_t* pre_term;      // optional: the column an upstream error belongs to (Strictify), else the term is 0xff
    int sink_guard;                // the rows go to a sink / serializer wire format that only takes INSERT rows here: update / delete rows that survive the chain are reported
};

// FilterRowsTransformer.Apply (filter_rows.go:99-130): one thread per row.
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_filter(FilterArgs a) {
    __shared__ uint32_t s_cnt, s_err;
    if (threadIdx.x == 0) { s_cnt = 0; s_err = 0; }
    __syncthreads();
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false, is_err = false;
    if (r < a.nrows) {
        keep = true; int err = 0, estep = 0;
        const int kind = a.kinds ? a.kinds[r] : TF_KIND_INSERT;
        if (a.pre_err && a.pre_err[r]) { err = a.pre_err[r]; estep = a.pre_term ? a.pre_term[r] : 0xff; keep = false; }
        for (int s = 0; s < a.nsteps && keep; s++) {
            const DFilterStep st = a.steps[s];
            if (st.flags & 1) { if ((st.expr_begin >> kind) & 1) keep = false; continue; }            // skip_events.go:52-62
            if (kind == TF_KIND_UPDATE || kind == TF_KIND_DELETE) { err = TF_ROWERR_FILTER_KIND; estep = st.step_index; keep = false; break; }
            if (st.flags & 2) continue;
            bool any = false;
            for (int e = 0; e < st.nexpr && !any && !err; e++) {            // matchItem: OR over filters
                bool all = true;
                const uint32_t kb = a.expr_off[st.expr_begin + e], ke = a.expr_off[st.expr_begin + e + 1];
                for (uint32_t k = kb; k < ke; k++) {                         // matchExpression: AND over terms
                    const DTerm t = a.terms[k];
                    const RowVal v = load_val(a.cols[t.col], r);
                    bool m = false; const int rc = eval_term(v, t, a.blob, m);
                    if (rc) { err = rc; break; }
                    if (!m) { all = false; break; }
                }
                if (!err && all) any = true;
            }
            if (err) { estep = st.step_index; keep = false; break; }
            if (!any) keep = false;
        }
        if (keep && a.sink_guard && (kind == TF_KIND_UPDATE || kind == TF_KIND_DELETE)) { err = TF_ROWERR_SINK_KIND_HOST; estep = 0xff; keep = false; }
        a.keep[r] = keep ? 1 : 0;
        a.errcode[r] = (uint8_t)err; a.errstep[r] = (uint16_t)estep; is_err = err != 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    const unsigned be = __ballot_sync(0xffffffffu, is_err);
    if ((threadIdx.x & 31) == 0) { if (b) atomicAdd(&s_cnt, __popc(b)); if (be) atomicAdd(&s_err, __popc(be)); }
    __syncthreads();
    if (threadIdx.x == 0) { a.blockcnt[blockIdx.x] = s_cnt; if (s_err) atomicAdd((unsigned long long*)&a.st->n_errors, (unsigned long long)s_err); }
}
#endif  // TF_KERNELS_ENCODE

// The rows that raised an error as (row, code, term) triples: appended through a counter (the host sorts the few it gets by row), so a
// batch with a handful of failing rows does not ship its whole error-code arrays back.
struct DevRowErr { uint32_t row; uint16_t code, term; };
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_collect_errors(const uint8_t* errcode, const uint16_t* errstep, uint64_t nrows, DevRowErr* out, unsigned long long* counter, unsigned long long cap) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint8_t c = r < nrows ? errcode[r] : 0;
    if (!c) return;
    const unsigned long long at = atomicAdd(counter, 1ull);
    if (at < cap) out[at] = DevRowErr{(uint32_t)r, c, errstep[r]};
}
#endif  // TF_KERNELS_ENCODE

// exclusive scan of per-block kept counts (single block), total -> state.n_kept
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(1024) k_scan_blockcnt(const uint32_t* blockcnt, uint32_t* blockoff, uint32_t nblocks, DState* st) {
    __shared__ uint32_t sm[33];
    uint32_t carry = 0;
    for (uint32_t base = 0; base < nblocks; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < nblocks ? blockcnt[i] : 0;
        uint32_t tot; const uint32_t ex = block_excl_scan(v, &tot, sm);
        if (i < nblocks) blockoff[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) st->n_kept = carry;
}
#endif  // TF_KERNELS_ENCODE

// sel[j] = index of the j-th kept row (order preserved)
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_compact_sel(const uint8_t* keep, const uint32_t* blockoff, uint64_t nrows, uint32_t* sel) {
    __shared__ uint32_t sm[33];
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = (r < nrows && keep[r]) ? 1u : 0u;
    uint32_t tot; const uint32_t ex = block_excl_scan(k, &tot, sm);
    if (k) sel[blockoff[blockIdx.x] + ex] = (uint32_t)r;
}
#endif  // TF_KERNELS_ENCODE

// ------------------------------------------------------------------ layout of the native block
struct LayoutArgs {
    DCol* cols; int ncols;                     // ncols = OUTPUT columns; out_cols[k] = index into cols
    const int32_t* out_cols;
    const int32_t* str_cols; int nstr;         // column index of each OK_STR slot
    const uint32_t* tile_sum;                  // [nstr][ntiles_cap] encoded bytes per tile of STR_TILE kept rows
    uint64_t* tile_base;                       // [nstr][ntiles_cap] exclusive prefix within the column
    uint32_t ntiles_cap;
    const uint8_t* col_headers; const uint32_t* col_header_off;   // pre-serialized "name,type,0" per column
    uint8_t* raw; DState* st;
    uint64_t nrows_in; int has_sel; uint32_t frame_bytes;
    uint64_t* col_bytes;                       // [nstr] encoded bytes of each String column
};

#define TF_STR_TILE 256
#define TF_STR_THREADS 256
#define TF_STR_STAGE 16384   // bytes of shared memory staging per tile in k_encode_str

// k_layout_scan: one CTA per String column: exclusive prefix of the column's tile sizes, column total.
// k_layout_finish: column offsets, then the block / column headers.
// Block layout (clickhouse-go/v2 v2.46.0 lib/proto/block.go, revision 54460):
//   uvarint 1, u8 is_overflows=0, uvarint 2, i32 bucket_num=-1, uvarint 0, uvarint ncols, uvarint nrows,
//   per column: string name, string type, u8 custom_serialization=0, [null map], data
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(1024) k_layout_scan(LayoutArgs a) {
    __shared__ uint32_t sm[33];
    const int s = blockIdx.x;
    const uint64_t n = a.st->n_kept;
    const uint32_t ntiles = (uint32_t)((n + TF_STR_TILE - 1) / TF_STR_TILE);
    uint64_t carry = 0;
    for (uint32_t base = 0; base < ntiles; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < ntiles ? a.tile_sum[(size_t)s * a.ntiles_cap + i] : 0;
        uint32_t tot; const uint32_t ex = block_excl_scan(v, &tot, sm);
        if (i < ntiles) a.tile_base[(size_t)s * a.ntiles_cap + i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) a.col_bytes[s] = carry;
}
#endif  // TF_KERNELS_ENCODE

#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_layout_finish(LayoutArgs a) {
    __shared__ uint64_t s_size[3][256];     // header, null map, data bytes per column (ncols <= 256 per pass)
    __shared__ uint64_t s_pos[256];
    __shared__ uint64_t s_run;
    const uint64_t n = a.st->n_kept;
    if (threadIdx.x == 0) {
        uint8_t* o = a.raw; uint64_t p = 0;
        o[p++] = 1; o[p++] = 0; o[p++] = 2; o[p++] = 0xff; o[p++] = 0xff; o[p++] = 0xff; o[p++] = 0xff; o[p++] = 0;
        uint64_t v = (uint64_t)a.ncols; while (v >= 0x80) { o[p++] = (uint8_t)(v | 0x80); v >>= 7; } o[p++] = (uint8_t)v;
        v = n; while (v >= 0x80) { o[p++] = (uint8_t)(v | 0x80); v >>= 7; } o[p++] = (uint8_t)v;
        s_run = p;
    }
    for (int base = 0; base < a.ncols; base += 256) {
        const int c = base + threadIdx.x;
        __syncthreads();
        if (c < a.ncols) {       // every thread fetches its own column's sizes (global latency paid once, in parallel)
            const DCol& d = a.cols[a.out_cols[c]];
            s_size[0][threadIdx.x] = a.col_header_off[c + 1] - a.col_header_off[c];
            s_size[1][threadIdx.x] = (d.nullable && n) ? n : 0;
            s_size[2][threadIdx.x] = n ? ((d.out_kind == OK_STR || d.out_kind == OK_TOSTR) ? a.col_bytes[d.str_slot] : (uint64_t)d.out_w * n) : 0;
        }
        __syncthreads();
        if (threadIdx.x == 0) {  // serial prefix over shared memory only
            uint64_t p = s_run; const int m = a.ncols - base < 256 ? a.ncols - base : 256;
            for (int k = 0; k < m; k++) { s_pos[k] = p; p += s_size[0][k] + s_size[1][k] + s_size[2][k]; }
            s_run = p;
        }
        __syncthreads();
        if (c < a.ncols) {
            DCol& d = a.cols[a.out_cols[c]];
            const uint64_t p = s_pos[threadIdx.x];
            d.hdr_off = p; d.null_off = p + s_size[0][threadIdx.x]; d.out_off = d.null_off + s_size[1][threadIdx.x];
            const uint32_t hb = a.col_header_off[c], hn = (uint32_t)s_size[0][threadIdx.x];
            for (uint32_t k = 0; k < hn; k++) a.raw[p + k] = a.col_headers[hb + k];       // this column's "name,type,0"
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint64_t p = s_run;
        a.st->raw_total = p;
        a.st->n_frames = p ? (p + a.frame_bytes - 1) / a.frame_bytes : 1;
        a.st->frame_ticket = 0;
    }
}
#endif  // TF_KERNELS_ENCODE

// Columnar (tf_batch-shaped) output for tfgpu_push_columns: per output column 16-byte aligned regions
// [values | validity bitmap | aux | offsets | heap]; the region table goes back to the host with the data.
struct ColRegions { uint64_t values, validity, aux, offsets, heap, heap_len; };   // offsets into the buffer; ~0 = absent

#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_layout_columnar(LayoutArgs a, ColRegions* regions) {
    __shared__ uint64_t s_sz[5][256];
    __shared__ uint64_t s_pos[256];
    __shared__ uint64_t s_run;
    const uint64_t n = a.st->n_kept;
    if (threadIdx.x == 0) s_run = 0;
    for (int base = 0; base < a.ncols; base += 256) {
        const int k = base + threadIdx.x;
        __syncthreads();
        if (k < a.ncols) {
            const DCol& d = a.cols[a.out_cols[k]];
            const bool var = d.out_kind == OK_STR || d.out_kind == OK_MASK || d.out_kind == OK_TOSTR;
            const bool fresh = d.out_kind == OK_MASK || d.out_kind == OK_TOSTR || d.out_kind == OK_TODT;      // a new value: never nil, no aux
            const uint64_t heap = (d.out_kind == OK_STR || d.out_kind == OK_TOSTR) ? a.col_bytes[d.str_slot] : (d.out_kind == OK_MASK ? 64 * n : 0);
            s_sz[0][threadIdx.x] = var ? 0 : (uint64_t)d.out_w * n;                                   // values
            s_sz[1][threadIdx.x] = (d.validity && !fresh) ? (n + 7) / 8 : 0;          // validity bitmap
            s_sz[2][threadIdx.x] = (d.aux && !fresh) ? (d.type == TF_ANY ? n : 4 * n) : 0;   // aux
            s_sz[3][threadIdx.x] = var ? 4 * (n + 1) : 0;                                             // offsets
            s_sz[4][threadIdx.x] = heap;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t p = s_run; const int m = a.ncols - base < 256 ? a.ncols - base : 256;
            for (int q = 0; q < m; q++) { s_pos[q] = p; for (int z = 0; z < 5; z++) p += (s_sz[z][q] + 15) & ~15ull; }
            s_run = p;
        }
        __syncthreads();
        if (k < a.ncols) {
            DCol& d = a.cols[a.out_cols[k]];
            uint64_t p = s_pos[threadIdx.x]; ColRegions r;
            auto take = [&](int z) { const uint64_t at = p; p += (s_sz[z][threadIdx.x] + 15) & ~15ull; return at; };
            const uint64_t v = take(0), val = take(1), ax = take(2), of = take(3), hp = take(4);
            const bool var = d.out_kind == OK_STR || d.out_kind == OK_MASK || d.out_kind == OK_TOSTR;
            d.out_off = var ? hp : v; d.null_off = val; d.aux_off = ax; d.offs_off = of;
            r.values = var ? ~0ull : v; r.validity = s_sz[1][threadIdx.x] ? val : ~0ull; r.aux = s_sz[2][threadIdx.x] ? ax : ~0ull;
            r.offsets = var ? of : ~0ull; r.heap = var ? hp : ~0ull; r.heap_len = s_sz[4][threadIdx.x];
            regions[k] = r;
            if (var) ((uint32_t*)(a.raw + of))[n] = (uint32_t)s_sz[4][threadIdx.x];      // offsets[nrows] = heap length
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) { a.st->raw_total = s_run; a.st->n_frames = 0; a.st->frame_ticket = 0; }
}
#endif  // TF_KERNELS_ENCODE

// ------------------------------------------------------------------ fixed-width columns
struct EncodeArgs {
    const DCol* cols;
    const int32_t* slots;          // per blockIdx.y: column index, bit 30 set = this slot is the column's null map
    const uint32_t* sel; const DState* st; uint8_t* raw;
    uint32_t* tile_sum; const uint64_t* tile_base; uint32_t ntiles_cap;
    int columnar;                  // 1: Transformed batch back in tf_batch layout (no LEB128, offsets arrays, no cast)
};

#define TF_SLOT_NULLMAP (1 << 30)
#define TF_SLOT_AUX (1 << 29)
#define TF_SLOT_ZEROMAP (1 << 28)   // null map of a column whose transformer made every value non-nil: all zeros       // columnar output: the column's aux array (time nanos u32 / any tags u8)
#define TF_FIX_TILE_WORDS 2048
#define CH_MAX_DATE_SEC 4291747200LL   // 2106-01-01T00:00:00Z (columntypes/types.go:15-18)

// Stream kinds of k_encode_fixed, resolved ONCE per CTA (every thread of a CTA works on the same column), so the
// per-element code below is straight-line for its kind.
enum StreamKind { SK_COPY = 0, SK_BOOL, SK_DATE, SK_DATETIME, SK_TS64, SK_NULLMAP, SK_AUX32, SK_AUX8, SK_ZERO, SK_TODT_CH, SK_TODT_SEC };

// One output element after the typesystem cast (columntypes.Restore -> abstract.Restore are the identity for values
// whose Go type already matches the column type; what remains is the ClickHouse clamp / unit rule).
template <int K, int INW> __device__ __forceinline__ uint64_t elem_t(const DCol& c, const uint32_t* sel, uint64_t j, uint64_t n) {
    if (j >= n) return 0;
    const uint64_t r = sel ? sel[j] : j;
    if (K == SK_ZERO) return 0;
    if (K == SK_TODT_CH || K == SK_TODT_SEC) {     // SerializeToDateTime to_datetime.go:137-151: nil -> time.Unix(0, 0)
        int64_t s = 0;
        if (row_valid(c, r)) s = c.type == TF_INT32 ? (int64_t)((const int32_t*)c.values)[r] : (int64_t)((const uint32_t*)c.values)[r];
        if (K == SK_TODT_SEC) return (uint64_t)s;
        if (s > CH_MAX_DATE_SEC) s = CH_MAX_DATE_SEC;          // applyClickhouseDateBoundaries columntypes/types.go:20-29
        if (s < 0) s = 0;
        return (uint64_t)s;
    }
    if (K == SK_AUX8) return (uint64_t)c.aux[r];
    if (K == SK_AUX32) return (uint64_t)((const uint32_t*)c.aux)[r];
    const bool valid = row_valid(c, r);
    if (K == SK_NULLMAP) return valid ? 0 : 1;
    if (!valid) return 0;
    if (K == SK_COPY) {
        if (INW == 1) return c.values[r];
        if (INW == 2) return ((const uint16_t*)c.values)[r];
        if (INW == 4) return ((const uint32_t*)c.values)[r];
        return ((const uint64_t*)c.values)[r];
    }
    if (K == SK_BOOL) return c.values[r] != 0;
    if (K == SK_DATE || K == SK_DATETIME) {
        int64_t s = ((const int64_t*)c.values)[r];
        const uint32_t ns = c.aux ? ((const uint32_t*)c.aux)[r] : 0;
        if (s > CH_MAX_DATE_SEC || (s == CH_MAX_DATE_SEC && ns > 0)) s = CH_MAX_DATE_SEC;
        if (s < 0) s = 0;
        return K == SK_DATE ? (uint64_t)(s / 86400) : (uint64_t)s;
    }
    // SK_TS64
    const int64_t s = ((const int64_t*)c.values)[r];
    const uint32_t ns = c.aux ? ((const uint32_t*)c.aux)[r] : 0;
    return (uint64_t)(s * 1000000LL + (int64_t)(ns / 1000u));
}

// 4 consecutive bytes [4q, 4q+4) of the column's little-endian element stream (W = output element width)
template <int K, int INW, int W> __device__ __forceinline__ uint32_t stream_word_t(const DCol& c, const uint32_t* sel, uint64_t q, uint64_t n) {
    if (W == 1) return (uint32_t)elem_t<K, INW>(c, sel, 4 * q, n) | ((uint32_t)elem_t<K, INW>(c, sel, 4 * q + 1, n) << 8) |
                       ((uint32_t)elem_t<K, INW>(c, sel, 4 * q + 2, n) << 16) | ((uint32_t)elem_t<K, INW>(c, sel, 4 * q + 3, n) << 24);
    if (W == 2) return (uint32_t)(elem_t<K, INW>(c, sel, 2 * q, n) & 0xffff) | ((uint32_t)(elem_t<K, INW>(c, sel, 2 * q + 1, n) & 0xffff) << 16);
    if (W == 4) return (uint32_t)elem_t<K, INW>(c, sel, q, n);
    const uint64_t v = elem_t<K, INW>(c, sel, q >> 1, n); return (uint32_t)(v >> ((q & 1) * 32));
}

// The column's data starts at an arbitrary byte of the block (ClickHouse's format has no padding), so each lane builds
// one 4-byte word of the element stream, takes its left neighbour's word by shuffle and funnel-shifts the pair onto
// the 4-byte grid of the OUTPUT address: every store is an aligned, fully coalesced 128 B per warp.
template <int K, int INW, int W> __device__ __forceinline__ void encode_stream(const DCol& c, const EncodeArgs& a, uint64_t base, uint64_t n) {
    const uint32_t m = (uint32_t)(base & 3);
    const uint64_t total = n * (uint64_t)W;
    const uint64_t T = (m + total + 3) >> 2;
    uint8_t* dst0 = a.raw + (base - m);
    const unsigned lane = threadIdx.x & 31;
    // the grid is sized on the host for at most n INPUT rows of the widest type; the CTAs stride over the tiles the kept
    // rows actually fill, so a selective filter does not leave tens of thousands of CTAs that only start and exit
    for (uint64_t t0 = (uint64_t)blockIdx.x * TF_FIX_TILE_WORDS; t0 < T; t0 += (uint64_t)gridDim.x * TF_FIX_TILE_WORDS)
#pragma unroll 2
    for (uint32_t it = 0; it < TF_FIX_TILE_WORDS / 256; it++) {
        const uint64_t t = t0 + it * 256 + threadIdx.x;      // uniform trip count: the shuffle below needs the whole warp
        const uint32_t wcur = (t < T) ? stream_word_t<K, INW, W>(c, a.sel, t, n) : 0;
        uint32_t wprev = __shfl_up_sync(0xffffffffu, wcur, 1);
        if (lane == 0) wprev = (m && t > 0 && t <= T) ? stream_word_t<K, INW, W>(c, a.sel, t - 1, n) : 0;
        if (t >= T) continue;
        const uint32_t val = m ? __funnelshift_r(wprev, wcur, 8 * (4 - m)) : wcur;
        const int64_t sb = (int64_t)(4 * t) - (int64_t)m;          // stream offset of this word's first byte
        uint8_t* dst = dst0 + 4 * t;
        if (sb >= 0 && (uint64_t)sb + 4 <= total) *(uint32_t*)dst = val;
        else {
#pragma unroll
            for (int b = 0; b < 4; b++) { const int64_t x = sb + b; if (x >= 0 && (uint64_t)x < total) dst[b] = (uint8_t)(val >> (8 * b)); }
        }
    }
}

// Fixed-width columns, null maps and (columnar output) aux arrays: blockIdx.y = stream slot.
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_encode_fixed(EncodeArgs a) {
    const int32_t slot = a.slots[blockIdx.y];
    const DCol c = a.cols[slot & ~(TF_SLOT_NULLMAP | TF_SLOT_AUX | TF_SLOT_ZEROMAP)];
    const uint64_t n = a.st->n_kept;
    if (n == 0) return;
    const DCol& cc = c;
    if (slot & TF_SLOT_ZEROMAP) { encode_stream<SK_ZERO, 1, 1>(cc, a, c.null_off, n); return; }
    if (slot & TF_SLOT_NULLMAP) { encode_stream<SK_NULLMAP, 1, 1>(c, a, c.null_off, n); return; }
    if (slot & TF_SLOT_AUX) { if (c.type == TF_ANY) encode_stream<SK_AUX8, 1, 1>(c, a, c.aux_off, n); else encode_stream<SK_AUX32, 4, 4>(c, a, c.aux_off, n); return; }
    switch (c.out_kind) {
    case OK_COPY:
        switch (c.in_w) {
        case 1: encode_stream<SK_COPY, 1, 1>(c, a, c.out_off, n); break;
        case 2: encode_stream<SK_COPY, 2, 2>(c, a, c.out_off, n); break;
        case 4: encode_stream<SK_COPY, 4, 4>(c, a, c.out_off, n); break;
        default: encode_stream<SK_COPY, 8, 8>(c, a, c.out_off, n); break;
        }
        break;
    case OK_BOOL: encode_stream<SK_BOOL, 1, 1>(c, a, c.out_off, n); break;
    case OK_DATE: encode_stream<SK_DATE, 8, 2>(c, a, c.out_off, n); break;
    case OK_DATETIME: encode_stream<SK_DATETIME, 8, 4>(c, a, c.out_off, n); break;
    case OK_TS64: encode_stream<SK_TS64, 8, 8>(c, a, c.out_off, n); break;
    case OK_TODT: if (a.columnar) encode_stream<SK_TODT_SEC, 4, 8>(c, a, c.out_off, n); else encode_stream<SK_TODT_CH, 4, 4>(c, a, c.out_off, n); break;
    }
}
#endif  // TF_KERNELS_ENCODE

// validity bitmap of the kept rows: one thread per output byte (8 rows)
#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_pack_validity(EncodeArgs a) {
    const DCol c = a.cols[a.slots[blockIdx.y]];
    const uint64_t n = a.st->n_kept;
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b * 8 >= n) return;
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint64_t j = b * 8 + k;
        if (j < n) { const uint64_t r = a.sel ? a.sel[j] : j; v |= (row_valid(c, r) ? 1u : 0u) << k; }
    }
    a.raw[c.null_off + b] = (uint8_t)v;
}
#endif  // TF_KERNELS_ENCODE


// ------------------------------------------------------------------ Measurer
// middlewares/synchronizer/measurer.go:38-42: item.Size.Values = util.DeepSizeof(item.ColumnValues) (pkg/util/sizeof.go:7-110),
// a reflection walk over every value in the reference. For the canonical Go types the walk is a closed form:
//   []interface{} header 24, then per value 16 (interface) + its payload: nil 0; bool/int8/uint8 1; int16/uint16 2;
//   int32/uint32/float32 4; int64/uint64/float64/Duration 8; string 16 + len; []byte 24 + len; time.Time 24 (three words).
// `any` holding a Go string counts as a string; other `any` values (maps / slices in the reference) are counted as their
// JSON text in a string -- an estimate, flagged in DESIGN.md.
struct MeasureArgs { const DCol* cols; int ncols; uint64_t nrows; uint64_t* per_row; unsigned long long* total; };

#ifdef TF_KERNELS_ENCODE
__global__ void __launch_bounds__(256) k_measure(MeasureArgs a) {
    __shared__ uint32_t sm[33];
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t sz = 0;
    if (r < a.nrows) {
        sz = 24;
        for (int c = 0; c < a.ncols; c++) {
            const DCol& d = a.cols[c];
            sz += 16;
            if (!row_valid(d, r)) continue;
            switch (d.type) {
            case TF_UTF8: sz += 16 + (d.offsets[r + 1] - d.offsets[r]); break;
            case TF_ANY: sz += 16 + (d.offsets[r + 1] - d.offsets[r]); break;
            case TF_BYTES: sz += 24 + (d.offsets[r + 1] - d.offsets[r]); break;
            case TF_DATE: case TF_DATETIME: case TF_TIMESTAMP: sz += 24; break;
            default: sz += (uint64_t)d.in_w;
            }
        }
        if (a.per_row) a.per_row[r] = sz;
    }
    // block sum (sizes of one block fit 32 bits: 256 rows x < 16 MiB would not, so reduce in two halves)
    const uint32_t lo = (uint32_t)(sz & 0xffffffu), hi = (uint32_t)(sz >> 24);
    uint32_t tl, th; block_excl_scan(lo, &tl, sm); __syncthreads(); block_excl_scan(hi, &th, sm);
    if (threadIdx.x == 0) atomicAdd(a.total, (unsigned long long)tl + ((unsigned long long)th << 24));
}
#endif  // TF_KERNELS_ENCODE

}  // namespace tfk
