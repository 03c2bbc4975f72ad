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

#define TF_STR_GROUP 4      /* tiles per CTA: their loads are issued together, which hides the gather latency */
#define TF_STR_WARPS (TF_STR_THREADS / 32)
static_assert(TF_STR_GROUP <= TF_STR_WARPS, "one warp scans each tile's warp sums");

// Exclusive scans of the CTA's TF_STR_GROUP tiles at once (v[g] = this thread's piece size in tile g): one pair of barriers
// for all of them, not one set per tile. On return v[g] is the exclusive prefix and ws[g][TF_STR_WARPS] tile g's total.
__device__ __forceinline__ void str_group_scan(uint32_t (&v)[TF_STR_GROUP], uint32_t (*ws)[TF_STR_WARPS + 1]) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc[TF_STR_GROUP];
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) inc[g] = warp_incl_scan(v[g]);
    if (lane == 31) {
#pragma unroll
        for (int g = 0; g < TF_STR_GROUP; g++) ws[g][warp] = inc[g];
    }
    __syncthreads();
    if (warp < TF_STR_GROUP) {                                 // warp g scans tile g's warp sums
        const uint32_t w = lane < TF_STR_WARPS ? ws[warp][lane] : 0u, wi = warp_incl_scan(w);
        if (lane < TF_STR_WARPS) ws[warp][lane] = wi - w;
        if (lane == TF_STR_WARPS - 1) ws[warp][TF_STR_WARPS] = wi;
    }
    __syncthreads();
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) v[g] = inc[g] - v[g] + ws[g][warp];
}

// encoded size (LEB128 length + payload) of every tile of TF_STR_TILE kept rows, for every String column
__global__ void k_str_sizes(EncodeArgs a);
#ifdef TF_KERNELS_STR
__global__ void __launch_bounds__(TF_STR_THREADS) k_str_sizes(EncodeArgs a) {
    __shared__ uint32_t s_ws[TF_STR_GROUP][TF_STR_WARPS + 1];
    const uint64_t n = a.st->n_kept;                          // (both loads issued before the first exit)
    const int32_t slot = a.slots[blockIdx.y];
    const uint64_t jg = (uint64_t)blockIdx.x * TF_STR_TILE * TF_STR_GROUP;
    if (jg >= n) return;
    const DCol c = a.cols[slot];
    uint32_t Ls[TF_STR_GROUP];
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) { uint64_t r; Ls[g] = str_len(c, a.sel, jg + (uint64_t)g * TF_STR_TILE + threadIdx.x, n, r); }
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) Ls[g] = Ls[g] != 0xffffffffu ? Ls[g] + (a.columnar ? 0 : varint_len(Ls[g])) : 0u;
    str_group_scan(Ls, s_ws);
    if (threadIdx.x < TF_STR_GROUP && jg + (uint64_t)threadIdx.x * TF_STR_TILE < n)
        a.tile_sum[(size_t)c.str_slot * a.ntiles_cap + blockIdx.x * TF_STR_GROUP + threadIdx.x] = s_ws[threadIdx.x][TF_STR_WARPS];
}
#endif  // TF_KERNELS_STR

// LEB128 length + bytes. Plain String columns (the hot case): every thread first publishes its row's piece (offset in the
// tile, heap offset, length) in shared memory; then the OUTPUT of the CTA's tiles is cut into aligned chunks of
// TF_STR_CHUNK_WORDS 4-byte words, numbered across the tiles as one index space (a sparse column's four tiles then share one
// pass of the CTA instead of four mostly idle ones), and every thread produces whole chunks: a binary search over the piece
// offsets finds the row that owns the chunk's first byte and the later words walk forward from it. A word that is payload of
// one row comes from two aligned source words re-aligned with a funnel shift; those loads are all issued before the first
// word is assembled, so a thread keeps the chunk's loads in flight together. Work is proportional to output bytes (no skew
// between short and long strings, no staging limit) and a chunk inside its tile is one aligned, coalesced 16-byte store.
// convert_to_string columns produce their text with fmt_value: those tiles keep the row-per-thread path below.
#define TF_STR_CHUNK_WORDS 4   /* a 16-byte chunk: stored as one uint4 */
__device__ __forceinline__ uint32_t str_find_row(const uint32_t* ex, uint32_t x) {      // largest r with ex[r] <= x, ex[0] = 0
    uint32_t lo = 0, hi = TF_STR_TILE;
#pragma unroll
    for (int it = 0; it < 8; it++) { const uint32_t mid = (lo + hi) >> 1; if (ex[mid] <= x) lo = mid; else hi = mid; }
    return lo;
}
// bytes of the LEB128 length in a piece of pl bytes (length prefix + payload)
__device__ __forceinline__ uint32_t str_piece_vl(uint32_t pl) {
    return pl < 129 ? 1 : (pl < 16386 ? 2 : (pl < 2097155 ? 3 : (pl < 268435460 ? 4 : 5)));
}
// One output word of a tile that is not payload of a single row, byte by byte: LEB128 bytes computed, payload bytes loaded.
// sb = stream offset of its first byte in the tile (bytes outside [0, tile total) are left alone), r = piece holding max(sb, 0).
__device__ __forceinline__ void str_word_bytes(const uint32_t* ex_, const uint32_t* src_, const uint8_t* heap, uint32_t vlb, int32_t sb,
                                               uint32_t r, uint8_t* dst) {
    const uint32_t tot = ex_[TF_STR_TILE];
    uint32_t ps = ex_[r], pe = ex_[r + 1], val = 0, mask = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) {
        const int32_t xs = sb + b;
        if (xs < 0 || (uint32_t)xs >= tot) continue;
        const uint32_t x = (uint32_t)xs;
        while (x >= pe) { r++; ps = pe; pe = ex_[r + 1]; }
        const uint32_t pl = pe - ps, vl = vlb ? str_piece_vl(pl) : 0, k = x - ps;
        uint32_t byte;
        if (k < vl) { const uint32_t v = (pl - vl) >> (7 * k); byte = (v & 0x7f) | ((v >> 7) ? 0x80u : 0u); }
        else byte = heap[src_[r] + (k - vl)];
        val |= byte << (8 * b); mask |= 1u << b;
    }
    if (mask == 15) *(uint32_t*)dst = val;
    else { for (int b = 0; b < 4; b++) if ((mask >> b) & 1) dst[b] = (uint8_t)(val >> (8 * b)); }
}
__global__ void k_encode_str_plain(EncodeArgs a);
#ifdef TF_KERNELS_STR
__global__ void __launch_bounds__(TF_STR_THREADS, 2048 / TF_STR_THREADS) k_encode_str_plain(EncodeArgs a) {
    constexpr uint32_t CB = 4 * TF_STR_CHUNK_WORDS;           // bytes per chunk
    static_assert(TF_STR_CHUNK_WORDS == 4, "a whole chunk is one uint4 store");
    __shared__ uint32_t s_ws[TF_STR_GROUP][TF_STR_WARPS + 1];
    __shared__ uint32_t s_ex[TF_STR_GROUP][TF_STR_TILE + 1];
    __shared__ uint32_t s_src[TF_STR_GROUP][TF_STR_TILE];
    __shared__ uint64_t s_tb[TF_STR_GROUP];
    __shared__ uint32_t s_cp[TF_STR_GROUP + 1];               // first chunk of every tile in the CTA's index space
    __shared__ uint2 s_q[TF_STR_WARPS][32 * TF_STR_CHUNK_WORDS];   // per warp: queued words (word index in the tile, tile | piece << 8)
    const uint64_t n = a.st->n_kept;                          // (both loads issued before the first exit)
    const int32_t slot = a.slots[blockIdx.y];
    const uint64_t jg = (uint64_t)blockIdx.x * TF_STR_TILE * TF_STR_GROUP;
    if (jg >= n) return;
    const DCol c = a.cols[slot];
    if (c.out_kind == OK_TOSTR) return;                       // handled by k_encode_str
    const uint32_t vlb = a.columnar ? 0u : 1u;                // a length prefix exists
    if (threadIdx.x < TF_STR_GROUP) {                         // the tiles' block offsets load beside the row gather below
        const uint64_t j0 = jg + (uint64_t)threadIdx.x * TF_STR_TILE;
        s_tb[threadIdx.x] = j0 < n ? a.tile_base[(size_t)c.str_slot * a.ntiles_cap + blockIdx.x * TF_STR_GROUP + threadIdx.x] : 0;
    }
    uint32_t Ls[TF_STR_GROUP]; uint64_t Rs[TF_STR_GROUP]; uint32_t src[TF_STR_GROUP];
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) Ls[g] = str_len(c, a.sel, jg + (uint64_t)g * TF_STR_TILE + threadIdx.x, n, Rs[g]);
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) src[g] = (Ls[g] != 0xffffffffu && Ls[g]) ? c.offsets[Rs[g]] : 0u;
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) Ls[g] = Ls[g] != 0xffffffffu ? Ls[g] + (vlb ? varint_len(Ls[g]) : 0) : 0u;
    str_group_scan(Ls, s_ws);                                  // Ls[g]: the piece's offset in tile g; its barriers publish s_tb
    uint32_t cp = 0;                                           // chunks of the tiles before g
#pragma unroll
    for (int g = 0; g < TF_STR_GROUP; g++) {
        const uint32_t ex = Ls[g], tot = s_ws[g][TF_STR_WARPS];
        const uint64_t tb = s_tb[g];
        const uint64_t j = jg + (uint64_t)g * TF_STR_TILE + threadIdx.x;
        if (a.columnar && j < n) ((uint32_t*)(a.raw + c.offs_off))[j] = (uint32_t)(tb + ex);
        s_ex[g][threadIdx.x] = ex; s_src[g][threadIdx.x] = src[g];
        // a tile's chunks are aligned to CB bytes of the block: the first and last may be shared with the neighbouring tiles
        if (tot) cp += ((uint32_t)((uintptr_t)(a.raw + c.out_off + tb) & (CB - 1)) + tot + CB - 1) / CB;
        if (threadIdx.x == 0) { s_ex[g][TF_STR_TILE] = tot; s_cp[g + 1] = cp; }
    }
    if (threadIdx.x == 0) s_cp[0] = 0;
    __syncthreads();
    const uint32_t hsh = ((uint32_t)(uintptr_t)c.heap & 3);   // alignment of the heap base
    const uint32_t* hw = (const uint32_t*)(c.heap - hsh);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // A warp runs the loop while any of its lanes has a chunk. Words that are not payload of one row are queued, and the warp
    // then produces its queue together, so that the byte-wise path runs once per 32 such words, not once per word position.
    for (uint32_t f0 = threadIdx.x & ~31u; f0 < cp; f0 += TF_STR_THREADS) {
        const uint32_t f = f0 + lane;
        uint32_t slow = 0, rs = 0, g = 0, ci = 0;             // word w is queued with piece (rs >> 8w) & 255
        if (f < cp) {
            while (f >= s_cp[g + 1]) g++;                     // the tile of chunk f (tiles without output have no chunks)
            const uint32_t* ex_ = s_ex[g]; const uint32_t* src_ = s_src[g];
            const uint32_t tot = ex_[TF_STR_TILE];
            uint8_t* gdst = a.raw + c.out_off + s_tb[g];
            const uint32_t m = (uint32_t)((uintptr_t)gdst & (CB - 1));
            ci = f - s_cp[g];
            uint8_t* dst = gdst - m + (size_t)CB * ci;
            const int32_t sb0 = (int32_t)(CB * ci) - (int32_t)m;   // stream offset of the chunk's first byte
            uint32_t r = str_find_row(ex_, sb0 < 0 ? 0u : (uint32_t)sb0);
            // piece r = [ps, pe): LEB128 of its payload length, then the payload
            uint32_t ps = ex_[r], pe = ex_[r + 1];
            uint32_t lo[TF_STR_CHUNK_WORDS], hi[TF_STR_CHUNK_WORDS], sh = 0, full = 0;
#pragma unroll
            for (int w = 0; w < TF_STR_CHUNK_WORDS; w++) {
                lo[w] = 0; hi[w] = 0;
                const int32_t sb = sb0 + 4 * w;                // stream offset of this word's first byte
                const uint32_t x0 = sb < 0 ? 0u : (uint32_t)sb;
                if (sb <= -4 || x0 >= tot) continue;           // wholly before or after the tile
                while (x0 >= pe) { r++; ps = pe; pe = ex_[r + 1]; }
                const uint32_t vl = vlb ? str_piece_vl(pe - ps) : 0, k0 = x0 - ps;
                if (sb >= 0 && (uint32_t)sb + 4 <= pe && k0 >= vl) {   // the whole word is payload of one row: load now, assemble below
                    const uint32_t so = src_[r] + (k0 - vl) + hsh;
                    lo[w] = __ldg(hw + (so >> 2));
                    if (so & 3) hi[w] = __ldg(hw + (so >> 2) + 1);
                    sh |= (so & 3) << (8 * w); full |= 1u << w;
                } else { slow |= 1u << w; rs |= r << (8 * w); }
            }
#pragma unroll
            for (int w = 0; w < TF_STR_CHUNK_WORDS; w++) lo[w] = __funnelshift_r(lo[w], hi[w], 8 * ((sh >> (8 * w)) & 3));
            if (full == (1u << TF_STR_CHUNK_WORDS) - 1) *(uint4*)dst = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            else {
#pragma unroll
                for (int w = 0; w < TF_STR_CHUNK_WORDS; w++) if ((full >> w) & 1) ((uint32_t*)dst)[w] = lo[w];
            }
        }
        const uint32_t cnt = __popc(slow), qe = warp_incl_scan(cnt), qn = __shfl_sync(0xffffffffu, qe, 31);
        uint2* q = s_q[warp];
        for (uint32_t i = qe - cnt; slow; slow &= slow - 1, i++) {
            const uint32_t w = __ffs(slow) - 1;
            q[i] = make_uint2(TF_STR_CHUNK_WORDS * ci + w, g | (((rs >> (8 * w)) & 255) << 8));
        }
        __syncwarp();
        for (uint32_t e = lane; e < qn; e += 32) {
            const uint2 it = q[e];
            const uint32_t qg = it.y & 255;
            uint8_t* gdst = a.raw + c.out_off + s_tb[qg];
            const uint32_t m = (uint32_t)((uintptr_t)gdst & (CB - 1));
            str_word_bytes(s_ex[qg], s_src[qg], c.heap, vlb, (int32_t)(4 * it.x) - (int32_t)m, it.y >> 8, gdst - m + 4 * (size_t)it.x);
        }
        __syncwarp();                                          // the queue is refilled by the next pass
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
