// number_to_float on the device (pkg/transformer/registry/number_to_float/number_to_float.go:75-123): inside every `any` value
// each json.Number becomes a float64. On the columnar layout an `any` cell is the JSON text json.Marshal gives the value, so
// the transformer is a text rewrite: every number literal outside strings is parsed like json.Number.Float64 does
// (strconv.ParseFloat: exact path + Eisel-Lemire, kernels_json_in.cuh) and printed the way encoding/json prints a float64; a
// literal that overflows float64 keeps its text (the reference keeps the json.Number when Float64 fails). Cells holding a Go
// string (tag 1) or nil and rows that are not insert / update (supportedKinds :21) are left alone. A literal whose rounding
// the device cannot decide marks the row TF_ROWERR_N2F_HOST.
// Runs as a pre-pass of the chain: the rewritten text replaces the column's heap / offsets, so later steps (mask_field,
// convert_to_string, the sinks) see what they would see after the reference's transformer.
#pragma once
#include "kernels_json_in.cuh"

namespace tfk {

#define N2F_HOST 52

struct N2fArgs {
    const DCol* cols; const int32_t* which; const uint8_t* kinds; uint64_t nrows;
    uint32_t* out_len;              // [ncols][nrows]
    const uint32_t* offsets; uint8_t* heap; const uint64_t* col_base;     // pass 2
    uint8_t* err;
};

template <typename Sink> __device__ bool n2f_rewrite(Sink& sk, const uint8_t* s, uint32_t n) {      // false: undecided literal
    bool ins = false;
    for (uint32_t i = 0; i < n;) {
        const uint8_t c = s[i];
        if (ins) { sk.put(c); if (c == '\\' && i + 1 < n) { sk.put(s[i + 1]); i += 2; continue; } if (c == '"') ins = false; i++; continue; }
        if (c == '"') { ins = true; sk.put(c); i++; continue; }
        if (c == '-' || (c >= '0' && c <= '9')) {
            uint32_t q = i; while (q < n && jsn_numch(s[q])) q++;
            double f; const int rc = d_go_parse_float(s + i, q - i, f);
            if (rc == 3) return false;
            if (rc == 0 && !isnan(f) && !isinf(f)) fmt_float_bits(sk, (uint64_t)__double_as_longlong(f), false, FM_JSON);
            else for (uint32_t k = i; k < q; k++) sk.put(s[k]);
            i = q; continue;
        }
        sk.put(c); i++;
    }
    return true;
}
__device__ __forceinline__ bool n2f_applies(const N2fArgs& a, const DCol& c, uint64_t r) {
    if (a.kinds && a.kinds[r] != TF_KIND_INSERT && a.kinds[r] != TF_KIND_UPDATE) return false;
    if (!row_valid(c, r)) return false;
    return !(c.aux && c.aux[r] == 1);
}

__global__ void k_n2f_sizes(N2fArgs a);
#ifdef TF_KERNELS_N2F
__global__ void __launch_bounds__(128) k_n2f_sizes(N2fArgs a) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.nrows) return;
    const DCol c = a.cols[a.which[blockIdx.y]];
    const uint32_t off = c.offsets[r], L = c.offsets[r + 1] - off;
    uint32_t out = L;
    if (n2f_applies(a, c, r)) { CountSink cs{0}; if (n2f_rewrite(cs, c.heap + off, L)) out = cs.n; else { a.err[r] = N2F_HOST; out = 0; } }
    a.out_len[(size_t)blockIdx.y * a.nrows + r] = out;
}
#endif  // TF_KERNELS_N2F
__global__ void k_n2f_write(N2fArgs a);
#ifdef TF_KERNELS_N2F
__global__ void __launch_bounds__(128) k_n2f_write(N2fArgs a) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.nrows) return;
    const DCol c = a.cols[a.which[blockIdx.y]];
    const uint32_t off = c.offsets[r], L = c.offsets[r + 1] - off;
    uint8_t* o = a.heap + a.col_base[blockIdx.y] + a.offsets[(size_t)blockIdx.y * (a.nrows + 1) + r];
    if (a.out_len[(size_t)blockIdx.y * a.nrows + r] == 0) return;
    if (n2f_applies(a, c, r)) { MemSink ms{o}; n2f_rewrite(ms, c.heap + off, L); }
    else for (uint32_t k = 0; k < L; k++) o[k] = c.heap[off + k];
}
#endif  // TF_KERNELS_N2F

}  // namespace tfk
