// String columns of the ClickHouse block / the columnar output: sizes, offsets, payload.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "kernels_fmt.cuh"

namespace tfk {

// ------------------------------------------------------------------ String columns
__device__ __forceinline__ uint32_t str_len(const DCol& c, const uint32_t* sel, uint64_t j, uint64_t n, uint64_t& r) {
    if (j >= n) { r = 0; return 0xffffffffu; }
    r = sel ? sel[j] : j;
    if (c.out_kind == OK_TOSTR) { CountSink cs; cs.n = 0; fmt_value(cs, c, r); return cs.n; }    // convert_to_string: length of the text form
    if (!row_valid(c, r)) return 0;
    return c.offsets[r + 1] - c.offsets[r];
}

// encoded size (LEB128 length + payload) of every tile of TF_STR_TILE kept rows, for every String column
#define TF_STR_GROUP 4      /* tiles per CTA: their loads are issued together, which hides the gather latency */
__global__ void k_str_sizes(EncodeArgs a);
#ifdef TF_KERNELS_STR
__global__ void __launch_bounds__(TF_STR_THREADS) k_str_sizes(EncodeArgs a) {
    __shared__ uint32_t sm[33];
    const DCol c = a.cols[a.slots[blockIdx.y]];
    const uint64_t n = a.st->n_kept;
    const uint64_t jg = (uint64_t)blockIdx.x * TF_STR_TILE * TF_STR_GROUP;
    if (jg >= n) return;
    uint32_t Ls[TF_STR_GROUP];
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) { uint64_t r; Ls[g] = str_len(c, a.sel, jg + (uint64_t)g * TF_STR_TILE + threadIdx.x, n, r); }
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) {
        uint32_t tot; block_excl_scan(Ls[g] != 0xffffffffu ? Ls[g] + (a.columnar ? 0 : varint_len(Ls[g])) : 0u, &tot, sm);
        if (threadIdx.x == 0 && jg + (uint64_t)g * TF_STR_TILE < n) a.tile_sum[(size_t)c.str_slot * a.ntiles_cap + blockIdx.x * TF_STR_GROUP + g] = tot;
        __syncthreads();
    }
}
#endif  // TF_KERNELS_STR

// LEB128 length + bytes. Plain String columns (the hot case): every thread first publishes its row's piece (offset in the
// tile, heap offset, length) in shared memory; then the tile's OUTPUT is cut into aligned 4-byte words and every thread
// produces whole words: a binary search over the piece offsets finds the row that owns the word, payload bytes come from
// two aligned source words re-aligned with a funnel shift. Work is proportional to output bytes (no skew between short
// and long strings, no staging limit) and every store is an aligned, coalesced word.
// convert_to_string columns produce their text with fmt_value: those tiles keep the row-per-thread path below.
__device__ __forceinline__ uint32_t str_find_row(const uint32_t* ex, uint32_t x) {      // largest r with ex[r] <= x, ex[0] = 0
    uint32_t lo = 0, hi = TF_STR_TILE;
#pragma unroll
    for (int it = 0; it < 8; it++) { const uint32_t mid = (lo + hi) >> 1; if (ex[mid] <= x) lo = mid; else hi = mid; }
    return lo;
}
__global__ void k_encode_str_plain(EncodeArgs a);
#ifdef TF_KERNELS_STR
__global__ void __launch_bounds__(TF_STR_THREADS) k_encode_str_plain(EncodeArgs a) {
    __shared__ uint32_t sm[33];
    __shared__ uint32_t s_ex[TF_STR_GROUP][TF_STR_TILE + 1];
    __shared__ uint32_t s_src[TF_STR_GROUP][TF_STR_TILE];
    __shared__ uint64_t s_tb[TF_STR_GROUP];
    const DCol c = a.cols[a.slots[blockIdx.y]];
    if (c.out_kind == OK_TOSTR) return;                       // handled by k_encode_str
    const uint64_t n = a.st->n_kept;
    const uint64_t jg = (uint64_t)blockIdx.x * TF_STR_TILE * TF_STR_GROUP;
    if (jg >= n) return;
    const uint32_t vlb = a.columnar ? 0u : 1u;                // a length prefix exists
    uint32_t Ls[TF_STR_GROUP]; uint64_t Rs[TF_STR_GROUP]; uint32_t src[TF_STR_GROUP];
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) Ls[g] = str_len(c, a.sel, jg + (uint64_t)g * TF_STR_TILE + threadIdx.x, n, Rs[g]);
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) src[g] = (Ls[g] != 0xffffffffu && Ls[g]) ? c.offsets[Rs[g]] : 0u;
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) {
        const bool have = Ls[g] != 0xffffffffu;
        uint32_t tot; const uint32_t ex = block_excl_scan(have ? Ls[g] + (vlb ? varint_len(Ls[g]) : 0) : 0u, &tot, sm);
        const uint64_t j0 = jg + (uint64_t)g * TF_STR_TILE;
        const uint64_t tb = j0 < n ? a.tile_base[(size_t)c.str_slot * a.ntiles_cap + blockIdx.x * TF_STR_GROUP + g] : 0;
        if (a.columnar && have) ((uint32_t*)(a.raw + c.offs_off))[j0 + threadIdx.x] = (uint32_t)(tb + ex);
        s_ex[g][threadIdx.x] = ex; s_src[g][threadIdx.x] = src[g];
        if (threadIdx.x == 0) { s_ex[g][TF_STR_TILE] = tot; s_tb[g] = tb; }
        __syncthreads();                                       // also separates the scans' use of `sm`
    }
    const uint32_t hsh = ((uint32_t)(uintptr_t)c.heap & 3);   // alignment of the heap base
    const uint32_t* hw = (const uint32_t*)(c.heap - hsh);
#pragma unroll 1
    for (int g = 0; g < TF_STR_GROUP; g++) {
        const uint32_t* ex_ = s_ex[g]; const uint32_t* src_ = s_src[g];
        const uint32_t tot = ex_[TF_STR_TILE];
        if (!tot) continue;
        uint8_t* gdst = a.raw + c.out_off + s_tb[g];
        const uint32_t m = (uint32_t)((uintptr_t)gdst & 3);
        const uint32_t T = (m + tot + 3) >> 2;
        uint8_t* dst0 = gdst - m;
        for (uint32_t t = threadIdx.x; t < T; t += TF_STR_THREADS) {
            const int32_t sb = (int32_t)(4 * t) - (int32_t)m;      // stream offset of this word's first byte
            const uint32_t x0 = sb < 0 ? 0u : (uint32_t)sb;
            uint32_t r = str_find_row(ex_, x0);
            // piece r = [ex[r], ex[r+1]): LEB128 of its payload length, then the payload
            uint32_t pe = ex_[r + 1], pl = pe - ex_[r];
            uint32_t plen = pl, vl = 0;
            if (vlb) { vl = pl < 129 ? 1 : (pl < 16386 ? 2 : (pl < 2097155 ? 3 : (pl < 268435460 ? 4 : 5))); plen = pl - vl; }
            const uint32_t k0 = x0 - ex_[r];
            if (sb >= 0 && (uint32_t)sb + 4 <= pe && k0 >= vl) {   // the whole word is payload of one row
                const uint32_t so = src_[r] + (k0 - vl) + hsh; const uint32_t sh = (so & 3) * 8;
                const uint32_t w0 = __ldg(hw + (so >> 2)); uint32_t val = w0;
                if (sh) val = __funnelshift_r(w0, __ldg(hw + (so >> 2) + 1), sh);
                *(uint32_t*)(dst0 + 4 * (size_t)t) = val;
                continue;
            }
            uint32_t val = 0, mask = 0;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int32_t xs = sb + b;
                if (xs < 0 || (uint32_t)xs >= tot) continue;
                const uint32_t x = (uint32_t)xs;
                while (x >= pe) { r++; pe = ex_[r + 1]; pl = pe - ex_[r]; if (vlb) { vl = pl < 129 ? 1 : (pl < 16386 ? 2 : (pl < 2097155 ? 3 : (pl < 268435460 ? 4 : 5))); plen = pl - vl; } else plen = pl; }
                const uint32_t k = x - ex_[r];
                uint32_t byte;
                if (k < vl) { const uint32_t v = plen >> (7 * k); byte = (v & 0x7f) | ((v >> 7) ? 0x80u : 0u); }
                else byte = c.heap[src_[r] + (k - vl)];
                val |= byte << (8 * b); mask |= 1u << b;
            }
            uint8_t* dst = dst0 + 4 * (size_t)t;
            if (mask == 15) *(uint32_t*)dst = val;
            else { for (int b = 0; b < 4; b++) if ((mask >> b) & 1) dst[b] = (uint8_t)(val >> (8 * b)); }
        }
    }
}
#endif  // TF_KERNELS_STR

// LEB128 length + text of convert_to_string columns, one kept row per thread, staged in shared memory.
__global__ void k_encode_str(EncodeArgs a);
#ifdef TF_KERNELS_STR
__global__ void __launch_bounds__(TF_STR_THREADS) k_encode_str(EncodeArgs a) {
    __shared__ uint32_t sm[33];
    __shared__ __align__(16) uint8_t stage[TF_STR_STAGE + 8];
    const DCol c = a.cols[a.slots[blockIdx.y]];
    if (c.out_kind != OK_TOSTR) return;                       // plain String columns: k_encode_str_plain
    const uint64_t n = a.st->n_kept;
    const uint64_t j0 = (uint64_t)blockIdx.x * TF_STR_TILE;
    if (j0 >= n) return;
    uint64_t R; const uint32_t L = str_len(c, a.sel, j0 + threadIdx.x, n, R);
    if (c.nullable && !a.columnar && L != 0xffffffffu) a.raw[c.null_off + j0 + threadIdx.x] = 0;   // "<nil>" is a value
    uint32_t tot; const uint32_t ex = block_excl_scan(L != 0xffffffffu ? L + (a.columnar ? 0 : varint_len(L)) : 0u, &tot, sm);
    const uint64_t tb = a.tile_base[(size_t)c.str_slot * a.ntiles_cap + blockIdx.x];
    uint8_t* gdst = a.raw + c.out_off + tb;
    if (a.columnar && L != 0xffffffffu) ((uint32_t*)(a.raw + c.offs_off))[j0 + threadIdx.x] = (uint32_t)(tb + ex);
    const bool staged = tot <= TF_STR_STAGE;
    uint8_t* o = staged ? stage + ex : gdst + ex;
    if (L != 0xffffffffu) {
        if (!a.columnar) {
            uint32_t v = L;
            while (v >= 0x80) { *o++ = (uint8_t)(v | 0x80); v >>= 7; }
            *o++ = (uint8_t)v;
        }
        MemSink ms; ms.p = o; fmt_value(ms, c, R);
    }
    if (!staged) return;
    __syncthreads();
    const uint32_t m = (uint32_t)((uintptr_t)gdst & 3);
    const uint32_t T = (m + tot + 3) >> 2;
    uint8_t* dst0 = gdst - m;
    const uint32_t* sw = (const uint32_t*)stage;
    for (uint32_t t = threadIdx.x; t < T; t += TF_STR_THREADS) {
        const uint32_t wcur = sw[t], wprev = t ? sw[t - 1] : 0;
        const uint32_t val = m ? __funnelshift_r(wprev, wcur, 8 * (4 - m)) : wcur;
        const int32_t sb = (int32_t)(4 * t) - (int32_t)m;
        uint8_t* dst = dst0 + 4 * (size_t)t;
        if (sb >= 0 && (uint32_t)sb + 4 <= tot) *(uint32_t*)dst = val;
        else {
#pragma unroll
            for (int b = 0; b < 4; b++) { const int32_t x = sb + b; if (x >= 0 && (uint32_t)x < tot) dst[b] = (uint8_t)(val >> (8 * b)); }
        }
    }
}
#endif  // TF_KERNELS_STR


}  // namespace tfk
