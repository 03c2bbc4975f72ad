// LZ4 block compression of the native block, cut into ClickHouse compressed frames and written straight to their
// final place in the wire buffer, plus the CityHash128 (v1.0.2) frame checksum.
//
// GPU-native LZ4 (not a port of any CPU compressor): one CTA per frame, the frame lives in shared memory and
// every phase is data-parallel:
//   P1  stage the frame in shared memory (16-byte coalesced loads, all of a thread's loads in flight at once)
//   P2  match finding in rounds of 4 x LZ_THREADS positions (4 consecutive per thread: two shared-memory words give the four
//       4-byte sequences). Every position is inserted into a 2^LZ_HASH_BITS-entry hash table (tag16 | position); every EVEN
//       position gets a candidate: the same sequence 4 or 8 bytes back (runs of fixed-width values: the nearest
//       candidate gives the longest match), else the table entry of an earlier round, else (after this round's
//       inserts) an entry of this round. Result: one u16 candidate per even position + two warp ballots per round.
//       This phase is bound by instruction issue: rounds that lie wholly inside the frame run without bounds tests.
//   P3  greedy parse, one thread per 60-byte segment (15 words: an odd stride keeps the segment walkers on
//       different banks). A match found at an even position is extended backwards; matches are cut at the
//       segment end. Descriptors (offset | length | start) overwrite the segment's candidate slots. The walkers
//       wait on shared memory, so comparisons go 8 bytes forward / 4 bytes backward per round trip.
//   P3b continuation: a match that was cut at a segment end is carried on by the next segments: each tests how
//       far the cut match's offset still holds from its first byte (the offset travels over fully matched
//       segments by a segmented scan); what holds is merged into the running match, so a long match costs one
//       sequence however many segments it crosses.
//   P4  segmented scan carries pending literals across segments; a block scan gives every segment its output
//       offset; the frame's size is published for the frames behind it (decoupled look-back)
//   P5  every thread emits its segment's tokens / lengths / offsets / literals into a shared-memory image of the
//       compressed frame, which is then copied to the wire buffer with aligned 16-byte stores at the frame's
//       final offset (prefix of the earlier frames' sizes, looked back through global memory)
// The emitted stream is a standard LZ4 block (last 5 bytes literals, last match starts >= 12 bytes before the
// end) and decodes with stock liblz4; the bytes are NOT those of pierrec/lz4 (parity for compressed bytes is
// unpinned in the reference, see DESIGN.md). scripts/lz4_model.cpp is the CPU model these rules were chosen with.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"

namespace tfk {

#ifndef LZ_THREADS
#define LZ_THREADS 256     /* 4 CTAs x 256 threads on 15 KiB frames measured faster than 2 x 512 on 30 KiB frames, for 3 % of ratio (1.694 / 1.751) */
#endif
#define LZ_CTAS_PER_SM (LZ_THREADS <= 256 ? 4 : 2)   /* register file: 64 registers x LZ_THREADS x CTAs = 64 K */
#define LZ_ROUND (4 * LZ_THREADS)                   /* positions per match-finding round */
#define LZ_SEG 60
#ifndef LZ_HASH_BITS
#define LZ_HASH_BITS 11      /* 2048 entries of u32: tag16 << 16 | position (8 KiB: with a 15 KiB frame four CTAs fit the 227 KiB of an SM) */
#endif
#define LZ_MAX_FRAME (LZ_THREADS * LZ_SEG)   /* 15360 */
#define LZ_HDR 25            /* 16 checksum + 1 method + 4 compressed size + 4 raw size */
#define LZ_NONE 0xffffffffu
#define LZ_FLAG_AGG (1ull << 62)
#define LZ_FLAG_INCL (2ull << 62)
#define LZ_VAL_MASK ((1ull << 62) - 1)

__host__ __device__ inline uint32_t lz4_bound(uint32_t n) { return n + n / 255 + 16; }

// shared-memory carve-up (byte offsets)
struct LzSmem { uint32_t data, cand, bitmap, table, stg, total; };
__host__ __device__ inline LzSmem lz_smem(uint32_t F) {
    LzSmem s; uint32_t o = 0;
    const uint32_t F16 = (F + 15) & ~15u;
    s.data = o + 16; o += 16 + F16 + 16;                          // guard words in front of and behind the frame
    s.cand = o; o += F16;                                         // u16 per even position
    s.bitmap = o; o += ((F + LZ_ROUND - 1) / LZ_ROUND) * (LZ_THREADS / 4) + 16;            // 1 bit per even position, whole rounds (+ spare words)
    s.table = o; o += 4u << LZ_HASH_BITS;                         // later: the per-segment arrays
    s.stg = o + 16; o += 16 + ((9 + lz4_bound(F) + 15) & ~15u) + 32;   // image of [method][sizes][LZ4 block]
    s.total = o; return s;
}

struct Lz4Args {
    const uint8_t* raw; DState* st; uint8_t* wire; uint32_t* comp_size; uint64_t* wire_off;
    unsigned long long* pfx;        // [n_frames] decoupled look-back cells, zeroed before the launch
    uint64_t* tail;                 // tail[0] = frame count for the checksum kernel (it may still run when the next batch resets DState)
    uint32_t frame_bytes;
    unsigned long long* phases;     // optional [8]: cycles thread 0 of every CTA spent per phase (tfgpu_debug_lz4_phases), NULL = off
};
__global__ void k_lz4_frames(Lz4Args a);
#define LZ_PHASE(k) do { if (a.phases && tid == 0) { const long long t_ = clock64(); atomicAdd(&a.phases[k], (unsigned long long)(t_ - t_ph)); t_ph = t_; } } while (0)

__device__ __forceinline__ uint32_t ld32u(const uint32_t* w, uint32_t p) {   // 4 bytes at byte offset p of the frame in shared memory
    const uint32_t i = p >> 2, s = (p & 3) * 8;
    return __funnelshift_r(w[i], w[i + 1], s);
}
__device__ __forceinline__ uint32_t ext_bytes(uint32_t x) { return x < 15 ? 0u : 1u + (x - 15u) / 255u; }
__device__ __forceinline__ uint8_t* put_ext(uint8_t* o, uint32_t x) {   // x >= 15
    x -= 15; while (x >= 255) { *o++ = 255; x -= 255; } *o++ = (uint8_t)x; return o;
}
__device__ __forceinline__ void put_bytes3(uint8_t* dst, uint32_t x, uint32_t n) {     // the low n (< 4) bytes of x
#pragma unroll
    for (uint32_t k = 0; k < 3; k++) if (k < n) dst[k] = (uint8_t)(x >> (8 * k));
}
// literal copy inside shared memory: frame bytes [src, src + n) -> image bytes at dst (aligned words once dst is aligned). Every
// shared-memory load is a word, and the loads of a step come ahead of its stores: one round trip per 8 bytes and one per ragged end.
__device__ __forceinline__ void copy_lit(uint8_t* dst, const uint32_t* dw, uint32_t src, uint32_t n) {
    const uint32_t h = min(n, (0u - (uint32_t)(uintptr_t)dst) & 3u);
    if (h) { put_bytes3(dst, ld32u(dw, src), h); dst += h; src += h; n -= h; }
    for (; n >= 8; n -= 8, dst += 8, src += 8) {
        const uint32_t x = ld32u(dw, src), y = ld32u(dw, src + 4);
        *(uint32_t*)dst = x; *(uint32_t*)(dst + 4) = y;
    }
    if (n >= 4) { *(uint32_t*)dst = ld32u(dw, src); n -= 4; dst += 4; src += 4; }
    if (n) put_bytes3(dst, ld32u(dw, src), n);
}
// common prefix of frame bytes at c and p, at most maxl (> 0). 8 bytes per step: the loads of a step are independent, so a long
// match waits on half as many shared-memory round trips (the reads run at most 12 bytes past p + maxl, into the guard words)
__device__ __forceinline__ uint32_t lz_match_len(const uint32_t* dw, uint32_t c, uint32_t p, uint32_t maxl) {
    uint32_t ic = c >> 2, ip = p >> 2; const uint32_t sc = (c & 3) * 8, sp = (p & 3) * 8;
    uint32_t wc0 = dw[ic], wp0 = dw[ip], ml = 0;
    for (;;) {
        const uint32_t wc1 = dw[ic + 1], wp1 = dw[ip + 1], wc2 = dw[ic + 2], wp2 = dw[ip + 2];
        const uint32_t x0 = __funnelshift_r(wc0, wc1, sc) ^ __funnelshift_r(wp0, wp1, sp);
        const uint32_t x1 = __funnelshift_r(wc1, wc2, sc) ^ __funnelshift_r(wp1, wp2, sp);
        if (x0 | x1) { ml += x0 ? (uint32_t)(__ffs((int)x0) - 1) >> 3 : 4u + ((uint32_t)(__ffs((int)x1) - 1) >> 3); break; }
        ml += 8; if (ml >= maxl) break;
        ic += 2; ip += 2; wc0 = wc2; wp0 = wp2;
    }
    return ml < maxl ? ml : maxl;
}
// common suffix of the frame bytes in front of c and p, at most maxb: how far a match found at p extends backwards
__device__ __forceinline__ uint32_t lz_back_len(const uint32_t* dw, uint32_t c, uint32_t p, uint32_t maxb) {
    uint32_t n = 0;
    while (n < maxb) {      // 4 bytes per step, the last one highest; maxb <= c, so a read starts at most 3 bytes in front of the frame (zero guards)
        const int32_t qc = (int32_t)(c - n) - 4, qp = (int32_t)(p - n) - 4;
        const uint32_t x = __funnelshift_r(dw[qc >> 2], dw[(qc >> 2) + 1], (qc & 3) * 8) ^ __funnelshift_r(dw[qp >> 2], dw[(qp >> 2) + 1], (qp & 3) * 8);
        if (x) { n += (uint32_t)__clz((int)x) >> 3; break; }
        n += 4;
    }
    return n < maxb ? n : maxb;
}

// Decoupled look-back (warp 0 only): the exclusive prefix of the sizes of frames [0, f). Cells hold AGG | own size or INCL | inclusive prefix.
__device__ __forceinline__ unsigned long long lz_lookback(const Lz4Args& a, uint32_t f, uint32_t lane) {
    unsigned long long excl = 0;
    if (!f) return 0;
    int64_t base = (int64_t)f;           // cells [0, base) are still to be summed
    for (uint32_t spins = 0;;) {
        // four windows of 32 cells per round trip
        unsigned long long v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) { const int64_t j = base - 1 - 32 * k - (int64_t)lane; v[k] = j >= 0 ? *(volatile unsigned long long*)&a.pfx[j] : LZ_FLAG_INCL; }
        bool done = false, stale = false;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (done || stale) continue;
            const uint32_t fl = (uint32_t)(v[k] >> 62);
            const uint32_t incl = __ballot_sync(0xffffffffu, fl == 2), none = __ballot_sync(0xffffffffu, fl == 0);
            const uint32_t upto = incl ? (uint32_t)__ffs((int)incl) - 1 : 31u;       // lanes 0..upto are needed
            const uint32_t need = upto == 31 ? 0xffffffffu : ((2u << upto) - 1);
            if (none & need) { stale = true; continue; }      // an earlier frame has not got that far yet (its CTA holds a lower ticket and is running)
            unsigned long long part = lane <= upto ? (v[k] & LZ_VAL_MASK) : 0ull;
#pragma unroll
            for (int d = 16; d; d >>= 1) part += __shfl_xor_sync(0xffffffffu, part, d);
            excl += part; base -= 32;
            if (incl) done = true;
        }
        if (done) break;
        if (stale) { if (++spins > (1u << 20)) { if (lane == 0) a.st->pad = 1; break; } __nanosleep(100); }      // a bounded wait keeps a bug from hanging the device
    }
    return excl;
}

#ifdef TF_KERNELS_LZ4
// One match-finding round (P2): thread wi takes positions 4 wi .. 4 wi + 3. FULL: every position of the round is inside the frame
// (all rounds but a short last one), so the round runs without the per-thread bounds test and the branches around it.
template <bool FULL>
__device__ __forceinline__ void lz_match_round(const uint32_t* dw, uint32_t* table, uint32_t* cand_w, uint32_t* bm, uint32_t wi, uint32_t lane, uint32_t len) {
    const uint32_t p0 = wi * 4;
    const bool active = FULL || p0 < len;
    uint32_t i0 = 0, i1 = 0, i2 = 0, i3 = 0, e0 = 0, e1 = 0, e2 = 0, e3 = 0, c0 = LZ_NONE, c2 = LZ_NONE, t0 = 0, t2 = 0;
    if (active) {
        const uint32_t wm2 = dw[(int)wi - 2], wm1 = dw[(int)wi - 1], w0 = dw[wi], w1 = dw[wi + 1];
        const uint32_t s1 = __funnelshift_r(w0, w1, 8), s2 = __funnelshift_r(w0, w1, 16), s3 = __funnelshift_r(w0, w1, 24);
        const uint32_t h0 = w0 * 2654435761u, h1 = s1 * 2654435761u, h2 = s2 * 2654435761u, h3 = s3 * 2654435761u;
        i0 = h0 >> (32 - LZ_HASH_BITS); i1 = h1 >> (32 - LZ_HASH_BITS); i2 = h2 >> (32 - LZ_HASH_BITS); i3 = h3 >> (32 - LZ_HASH_BITS);
        e0 = ((h0 << LZ_HASH_BITS) & 0xffff0000u) | p0; e1 = ((h1 << LZ_HASH_BITS) & 0xffff0000u) | (p0 + 1);
        e2 = ((h2 << LZ_HASH_BITS) & 0xffff0000u) | (p0 + 2); e3 = ((h3 << LZ_HASH_BITS) & 0xffff0000u) | (p0 + 3);
        // the same 4 bytes 4 or 8 back: a run of a fixed-width value (from the third word on; the first two read the zero guards)
        const uint32_t a2 = __funnelshift_r(wm1, w0, 16), b2 = __funnelshift_r(wm2, wm1, 16);
        c0 = w0 == wm1 ? p0 - 4 : (w0 == wm2 ? p0 - 8 : LZ_NONE);
        c2 = s2 == a2 ? p0 - 2 : (s2 == b2 ? p0 - 6 : LZ_NONE);
        if (p0 < 8) c0 = c2 = LZ_NONE;
        t0 = table[i0]; t2 = table[i2];
    }
    __syncthreads();
    if (active) {
        table[i3] = e3; table[i2] = e2; table[i1] = e1; table[i0] = e0;
        if (c0 == LZ_NONE && ((t0 ^ e0) >> 16) == 0) c0 = t0 & 0xffffu;      // an entry of an earlier round: position < p0
        if (c2 == LZ_NONE && ((t2 ^ e2) >> 16) == 0) c2 = t2 & 0xffffu;
    }
    __syncthreads();
    if (active) {   // second probe: sees this round's inserts, recovers repeats whose first occurrence is in this round
        if (c0 == LZ_NONE) { const uint32_t t = table[i0]; if (((t ^ e0) >> 16) == 0 && (t & 0xffffu) < p0) c0 = t & 0xffffu; }
        if (c2 == LZ_NONE) { const uint32_t t = table[i2]; if (((t ^ e2) >> 16) == 0 && (t & 0xffffu) < p0 + 2) c2 = t & 0xffffu; }
        cand_w[wi] = (c0 & 0xffffu) | (c2 << 16);
    }
    const uint32_t b0 = __ballot_sync(0xffffffffu, c0 != LZ_NONE), b2 = __ballot_sync(0xffffffffu, c2 != LZ_NONE);
    if (lane == 0) { bm[2 * (wi >> 5)] = b0; bm[2 * (wi >> 5) + 1] = b2; }
}
// bit j of x (< 2^16) -> bit 2 j
__device__ __forceinline__ uint32_t lz_spread(uint32_t x) {
    x = (x | (x << 8)) & 0x00ff00ffu; x = (x | (x << 4)) & 0x0f0f0f0fu; x = (x | (x << 2)) & 0x33333333u; return (x | (x << 1)) & 0x55555555u;
}

__global__ void __launch_bounds__(LZ_THREADS, LZ_CTAS_PER_SM) k_lz4_frames(Lz4Args a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t F = a.frame_bytes;
    const LzSmem L = lz_smem(F);
    uint32_t* dw = (uint32_t*)(smem + L.data);                   // the frame; dw[-2], dw[-1] and 4 words behind it are zero guards
    uint16_t* cand = (uint16_t*)(smem + L.cand);                // candidate of even position p at cand[p >> 1]; later: sequence descriptors
    uint32_t* cand_w = (uint32_t*)(smem + L.cand);
    uint32_t* bm = (uint32_t*)(smem + L.bitmap);                // per warp and round the ballots [p0 has a candidate][p0 + 2 has one]: bit i of word 2 j (+ 1) is P2 thread 32 j + i
    uint32_t* table = (uint32_t*)(smem + L.table);
    uint8_t* stg = smem + L.stg;                                // [0x82][u32 size + 9][u32 raw size][LZ4 block]
    __shared__ uint32_t s_frame;
    __shared__ uint32_t scratch[80];
    __shared__ unsigned long long s_woff;
    // per-segment arrays, aliased onto the hash table once match finding is over
    int32_t* delta0 = (int32_t*)table;                           // [512]
    uint32_t* scanv = (uint32_t*)(delta0 + LZ_THREADS);          // [512]
    uint16_t* carry_incl = (uint16_t*)(scanv + LZ_THREADS);      // [512]
    uint16_t* ext16 = carry_incl + LZ_THREADS;                   // [514]
    uint8_t* clt8 = (uint8_t*)(ext16 + LZ_THREADS + 4);          // [512]
    uint8_t* flg8 = clt8 + LZ_THREADS;                           // [512]
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t raw_total = a.st->raw_total, n_frames = a.st->n_frames;

    // The image of a finished frame stays in shared memory while the NEXT frame is staged, matched and parsed (none of that touches the
    // image): its place in the wire buffer is looked up only then, when the frames before it have long published their sizes, so a slow
    // predecessor costs nothing.
    uint32_t pend_f = 0xffffffffu, pend_cs = 0;
    auto resolve_flush = [&](uint32_t pf, uint32_t pcs) {
        if (warp == 0) {
            const unsigned long long excl = lz_lookback(a, pf, lane);
            if (lane == 0) {
                *(volatile unsigned long long*)&a.pfx[pf] = LZ_FLAG_INCL | (excl + pcs + LZ_HDR);
                s_woff = excl;
                a.comp_size[pf] = pcs; a.wire_off[pf] = excl;
                if (pf + 1 == n_frames) { a.st->wire_total = excl + pcs + LZ_HDR; a.tail[0] = n_frames; }
            }
        }
        __syncthreads();
        // the image goes to wire + offset + 16 (behind the checksum field) in aligned 16-byte stores; the bytes a first / last store
        // carries beyond the image land in checksum fields, which k_frame_seal writes afterwards
        uint8_t* G = a.wire + s_woff + 16;
        const uint32_t m = (uint32_t)((uintptr_t)G & 15), total = 9 + pcs;
        const uint32_t nchunks = (m + total + 15) >> 4;
        int4* g4 = (int4*)(G - m);
        const uint32_t* sw = (const uint32_t*)(stg - 16);                 // image byte x is at sw byte x + 16
        const uint32_t o0 = 16 - m, sh = (o0 & 3) * 8;
        for (uint32_t j = tid; j < nchunks; j += LZ_THREADS) {
            const uint32_t wi0 = (o0 + 16 * j) >> 2;
            const uint32_t q0 = sw[wi0], q1 = sw[wi0 + 1], q2 = sw[wi0 + 2], q3 = sw[wi0 + 3], q4 = sw[wi0 + 4];
            int4 v;
            v.x = (int)__funnelshift_r(q0, q1, sh); v.y = (int)__funnelshift_r(q1, q2, sh);
            v.z = (int)__funnelshift_r(q2, q3, sh); v.w = (int)__funnelshift_r(q3, q4, sh);
            g4[j] = v;
        }
        __syncthreads();
    };
    for (;;) {
        __syncthreads();
        if (tid == 0) s_frame = atomicAdd(&a.st->frame_ticket, 1u);
        __syncthreads();
        const uint32_t f = s_frame;
        if (f >= n_frames) break;
        long long t_ph = a.phases ? clock64() : 0;
        const uint64_t pos0 = (uint64_t)f * F;
        const uint32_t len = (uint32_t)((raw_total - pos0 < F) ? raw_total - pos0 : F);

        // ---- P1: stage
        {
            const int4* g = (const int4*)(a.raw + pos0);
            const uint32_t nv = (len + 15) >> 4;
            int4* d4 = (int4*)(smem + L.data);
            constexpr uint32_t NLD = (LZ_MAX_FRAME / 16 + LZ_THREADS) / LZ_THREADS;     // the frame and a zero guard: all loads in flight at once
            int4 v[NLD];
#pragma unroll
            for (uint32_t k = 0; k < NLD; k++) { const uint32_t i = tid + k * LZ_THREADS; v[k] = i < nv ? __ldg(g + i) : make_int4(0, 0, 0, 0); }
#pragma unroll
            for (uint32_t k = 0; k < NLD; k++) { const uint32_t i = tid + k * LZ_THREADS; if (i < nv + 1) d4[i] = v[k]; }
            int4* t4 = (int4*)table;
            for (uint32_t i = tid; i < (1u << LZ_HASH_BITS) / 4; i += LZ_THREADS) t4[i] = make_int4(0, 0, 0, 0);
            if (tid < 4) ((uint32_t*)smem)[tid] = 0;
        }
        __syncthreads();

        LZ_PHASE(0);
        // ---- P2: match finding
        const uint32_t nrounds = (len + LZ_ROUND - 1) / LZ_ROUND;
        const uint32_t nfull = len / LZ_ROUND;
        for (uint32_t rd = 0; rd < nfull; rd++) lz_match_round<true>(dw, table, cand_w, bm, rd * LZ_THREADS + tid, lane, len);
        if (nfull < nrounds) lz_match_round<false>(dw, table, cand_w, bm, nfull * LZ_THREADS + tid, lane, len);
        if (tid == 0) { bm[((nrounds * LZ_THREADS) >> 4)] = 0; bm[((nrounds * LZ_THREADS) >> 4) + 1] = 0; }
        __syncthreads();
        if (tid == 0) bm[0] &= ~1u;        // position 0 has nothing before it

        LZ_PHASE(1);
        // ---- P3: greedy parse, one thread per 60-byte segment
        const uint32_t nseg = (len + LZ_SEG - 1) / LZ_SEG;
        const uint32_t lim5 = len >= 5 ? len - 5 : 0;
        const int32_t pmax = (int32_t)len - 12;                               // MFLIMIT: no match starts behind it
        const uint32_t sa = tid * LZ_SEG;
        uint32_t sb = 0, slimit = 0, nseq = 0, d_last = 0;
        bool reach = false, pure = false;
        uint32_t* desc = cand_w + tid * (LZ_SEG / 4);
        if (tid < nseg) {
            sb = sa + LZ_SEG < len ? sa + LZ_SEG : len;
            slimit = sb < lim5 ? sb : lim5;
            const uint32_t k = tid * (LZ_SEG / 4), bw = 2 * (k >> 5);      // the segment's first P2 thread, its ballot pair
            const uint32_t m0 = __funnelshift_r(bm[bw], bm[bw + 2], k & 31) & 0x7fffu, m2 = __funnelshift_r(bm[bw + 1], bm[bw + 3], k & 31) & 0x7fffu;
            const uint32_t m = lz_spread(m0) | (lz_spread(m2) << 1);       // bit j: position sa + 2 j has a candidate
            uint32_t cur = 0, anchor = sa;
            for (;;) {
                const uint32_t cb = (cur + 1) >> 1;
                if (cb >= LZ_SEG / 2) break;
                const uint32_t mm = m >> cb;
                if (!mm) break;
                const uint32_t r = cb + (uint32_t)__ffs((int)mm) - 1;
                uint32_t p = sa + 2 * r;
                if (p + 4 > slimit || (int32_t)p > pmax) break;
                uint32_t c = cand[p >> 1];
                uint32_t ml = lz_match_len(dw, c, p, slimit - p);
                if (ml < 4) { cur = 2 * r + 1; continue; }              // the tag agreed but the bytes do not: not a match
                const uint32_t nb = lz_back_len(dw, c, p, min(p - anchor, c));
                p -= nb; c -= nb; ml += nb;
                desc[nseq++] = ((p - c) << 16) | (ml << 8) | (p - sa);
                d_last = p - c;
                anchor = p + ml; cur = anchor - sa;
            }
            reach = nseq && anchor == sa + LZ_SEG;
            pure = nseq == 1 && reach && (desc[0] & 0xffu) == 0;
        }
        __syncthreads();     // the hash table is dead from here on: its memory holds the per-segment arrays

        // ---- P3b: continuation of matches that were cut at a segment end
        // scan value: 0 = fully matched segment (the running offset passes through), 1 = no running match behind it, else (offset << 2) | 2
        uint32_t k0 = 0, cl = 0, D = 0; bool merged = false, head = false;
        {
            uint32_t sv = tid < nseg ? (pure ? 0u : (reach ? (d_last << 2) | 2u : 1u)) : 1u;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, sv, d); if (lane >= (uint32_t)d && sv == 0) sv = o; }
            if (lane == 31) scratch[warp] = sv;
            __syncthreads();
            if (sv == 0) { for (int w = (int)warp - 1; w >= 0; w--) { const uint32_t o = scratch[w]; if (o) { sv = o; break; } } if (sv == 0) sv = 1; }
            scanv[tid] = sv;
            __syncthreads();
            const uint32_t prev = tid ? scanv[tid - 1] : 1u;
            const bool dvalid = tid < nseg && prev >= 2;
            D = prev >> 2;
            uint32_t n = 0;
            if (dvalid && slimit > sa) {        // how far does the running match's offset still hold from the first byte of this segment
                const uint32_t maxn = slimit - sa;
                const uint32_t q = sa - D; uint32_t iq = q >> 2; const uint32_t sq = (q & 3) * 8;
                uint32_t wq0 = dw[iq]; const uint32_t* pw = dw + tid * (LZ_SEG / 4);
                for (;;) {      // 8 bytes per step, as lz_match_len
                    const uint32_t wq1 = dw[iq + 1], wq2 = dw[iq + 2];
                    const uint32_t x0 = __funnelshift_r(wq0, wq1, sq) ^ pw[n >> 2], x1 = __funnelshift_r(wq1, wq2, sq) ^ pw[(n >> 2) + 1];
                    if (x0 | x1) { n += x0 ? (uint32_t)(__ffs((int)x0) - 1) >> 3 : 4u + ((uint32_t)(__ffs((int)x1) - 1) >> 3); break; }
                    n += 8; if (n >= maxn) break;
                    iq += 2; wq0 = wq2;
                }
                if (n > maxn) n = maxn;
            }
            clt8[tid] = (uint8_t)n; flg8[tid] = (uint8_t)((pure ? 1 : 0) | (reach ? 2 : 0) | (dvalid ? 4 : 0));
            __syncthreads();
            if (dvalid) {
                const uint32_t pf = flg8[tid - 1];
                const bool alive = (pf & 1) ? (clt8[tid - 1] == LZ_SEG && (pf & 4)) : (pf & 2) != 0;
                if (pure) {
                    if (!(alive && n > 0) && n != LZ_SEG) n = 0;
                    if (n && n < LZ_SEG && LZ_SEG - n < 4) n = LZ_SEG - 4;
                } else {
                    if (!alive) n = 0;
                    if (reach && n > LZ_SEG - 4) n = LZ_SEG - 4;
                }
                if (n && !alive && (int32_t)sa > pmax) n = 0;         // a head piece starts a match
                cl = n;
                if (n) {
                    merged = alive; head = !alive;
                    while (k0 < nseq) {      // own sequences against the piece [sa, sa + n)
                        const uint32_t dsc = desc[k0], pr = dsc & 0xffu, ml = (dsc >> 8) & 0xffu;
                        if (pr + ml <= n) { k0++; continue; }
                        if (pr >= n) break;
                        const uint32_t nml = pr + ml - n;      // what is left of it behind the piece is still a match with the same offset ...
                        if (nml >= 4 && (int32_t)(sa + n) <= pmax) desc[k0] = (dsc & 0xffff0000u) | (nml << 8) | n; else k0++;      // ... unless it would start in the last 12 bytes
                        break;
                    }
                }
            }
            // ext(t) = bytes the running match gains from segment t on: reverse segmented sum over merged pieces
            uint32_t es = merged ? cl : 0u, ec = (merged && cl == LZ_SEG) ? 1u : 0u;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t os = __shfl_down_sync(0xffffffffu, es, d), oc = __shfl_down_sync(0xffffffffu, ec, d);
                if (lane + d < 32 && ec) { es += os; ec = oc; }
            }
            if (lane == 0) { scratch[32 + warp] = es; scratch[48 + warp] = ec; }
            __syncthreads();
            if (ec) for (uint32_t w = warp + 1; w < LZ_THREADS / 32; w++) { es += scratch[32 + w]; if (!scratch[48 + w]) break; }
            ext16[tid] = (uint16_t)es;
            if (tid == 0) ext16[LZ_THREADS] = 0;
        }
        __syncthreads();
        const uint32_t ext_next = ext16[tid + 1];

        LZ_PHASE(2);
        // ---- P4a: segmented scan of pending literals: combine(a, b) = b.has ? b : (a.has, a.tr + b.tr)
        const bool emits = tid < nseg && (head || k0 < nseq);
        uint32_t my_trail = 0;
        if (tid < nseg) {
            uint32_t last_end = sa + cl;
            if (k0 < nseq) { const uint32_t dsc = desc[nseq - 1]; last_end = sa + (dsc & 0xffu) + ((dsc >> 8) & 0xffu); }
            my_trail = sb - last_end;
        }
        {
            uint32_t has = emits ? 1u : 0u, tr = my_trail;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t h2 = __shfl_up_sync(0xffffffffu, has, d), t2 = __shfl_up_sync(0xffffffffu, tr, d);
                if (lane >= (uint32_t)d && !has) { tr += t2; has = h2; }
            }
            if (lane == 31) { scratch[warp] = has; scratch[16 + warp] = tr; }
            __syncthreads();
            if (warp == 0) {
                uint32_t wh = lane < LZ_THREADS / 32 ? scratch[lane] : 0, wt = lane < LZ_THREADS / 32 ? scratch[16 + lane] : 0;
#pragma unroll
                for (int d = 1; d < 16; d <<= 1) {
                    const uint32_t h2 = __shfl_up_sync(0xffffffffu, wh, d), t2 = __shfl_up_sync(0xffffffffu, wt, d);
                    if (lane >= (uint32_t)d && !wh) { wt += t2; wh = h2; }
                }
                const uint32_t eh = __shfl_up_sync(0xffffffffu, wh, 1), et = __shfl_up_sync(0xffffffffu, wt, 1);
                if (lane < LZ_THREADS / 32) { scratch[lane] = lane ? eh : 0; scratch[16 + lane] = lane ? et : 0; }
            }
            __syncthreads();
            if (!has) { tr += scratch[16 + warp]; }
            carry_incl[tid] = (uint16_t)tr;
        }
        __syncthreads();
        const uint32_t carry_in = (tid > 0 && tid < nseg) ? carry_incl[tid - 1] : 0;

        // ---- P4b: encoded bytes per segment, block scan -> output offsets
        uint32_t my_bytes = 0, p_first = 0, ll_first = 0;
        if (emits) {
            uint32_t prev_end = sa + (merged ? cl : 0u); bool first = true;
            if (head) {
                const uint32_t ml = LZ_SEG + ext_next;
                my_bytes += 1 + ext_bytes(carry_in) + carry_in + 2 + ext_bytes(ml - 4);
                p_first = sa; ll_first = carry_in; prev_end = sa + LZ_SEG; first = false;
            }
            for (uint32_t k = k0; k < nseq; k++) {
                const uint32_t dsc = desc[k], pr = dsc & 0xffu; uint32_t ml = (dsc >> 8) & 0xffu;
                const uint32_t p = sa + pr, ll = (first ? carry_in : 0u) + (p - prev_end);
                prev_end = p + ml;
                if (k + 1 == nseq && pr + ml == LZ_SEG) ml += ext_next;
                my_bytes += 1 + ext_bytes(ll) + ll + 2 + ext_bytes(ml - 4);
                if (first) { p_first = p; ll_first = ll; first = false; }
            }
        }
        uint32_t total_seq_bytes;
        const uint32_t my_off = block_excl_scan(my_bytes, &total_seq_bytes, scratch);
        if (emits) delta0[tid] = (int32_t)(my_off + 1 + ext_bytes(ll_first)) - (int32_t)(p_first - ll_first);
        // first later segment that emits a sequence (it owns this segment's trailing literals): warp ballots + one barrier
        uint32_t my_next_has = 0xffff;
        {
            const uint32_t hm = __ballot_sync(0xffffffffu, emits);
            if (lane == 0) scratch[40 + warp] = hm;
            __syncthreads();
            const uint32_t above = lane == 31 ? 0u : (hm >> (lane + 1));
            if (above) my_next_has = tid + (uint32_t)__ffs((int)above);
            else for (uint32_t w = warp + 1; w < LZ_THREADS / 32; w++) { const uint32_t m = scratch[40 + w]; if (m) { my_next_has = w * 32 + (uint32_t)__ffs((int)m) - 1; break; } }
        }
        const uint32_t ll_final = nseg ? carry_incl[nseg - 1] : 0;
        const int32_t delta_final = (int32_t)(total_seq_bytes + 1 + ext_bytes(ll_final)) - (int32_t)(len - ll_final);
        const uint32_t cs = total_seq_bytes + 1 + ext_bytes(ll_final) + ll_final;
        if (tid == 0) { *(volatile unsigned long long*)&a.pfx[f] = LZ_FLAG_AGG | (unsigned long long)(cs + LZ_HDR); }   // the frames behind can start summing
        LZ_PHASE(3);
        if (pend_f != 0xffffffffu) resolve_flush(pend_f, pend_cs);      // the previous frame leaves the image
        LZ_PHASE(5);
        // ---- P5: emit into the shared-memory image
        uint8_t* out = stg + 9;
        if (tid < nseg) {
            uint32_t prev_end = sa + (merged ? cl : 0u);
            if (emits) {
                uint8_t* o = out + my_off; bool first = true;
                if (head) {
                    const uint32_t mt = LZ_SEG + ext_next - 4, ll = carry_in;
                    *o++ = (uint8_t)(((ll < 15 ? ll : 15) << 4) | 15);
                    if (ll >= 15) o = put_ext(o, ll);
                    o += ll;
                    *o++ = (uint8_t)D; *o++ = (uint8_t)(D >> 8);
                    o = put_ext(o, mt);
                    prev_end = sa + LZ_SEG; first = false;
                }
                for (uint32_t k = k0; k < nseq; k++) {
                    const uint32_t dsc = desc[k], pr = dsc & 0xffu, off = dsc >> 16; uint32_t ml = (dsc >> 8) & 0xffu;
                    const uint32_t p = sa + pr, cin = first ? carry_in : 0u, ll = cin + (p - prev_end);
                    const uint32_t lit0 = prev_end, nlit = p - prev_end;
                    prev_end = p + ml;
                    if (k + 1 == nseq && pr + ml == LZ_SEG) ml += ext_next;
                    const uint32_t mt = ml - 4;
                    *o++ = (uint8_t)(((ll < 15 ? ll : 15) << 4) | (mt < 15 ? mt : 15));
                    if (ll >= 15) o = put_ext(o, ll);
                    copy_lit(o + cin, dw, lit0, nlit);
                    o += ll;
                    *o++ = (uint8_t)off; *o++ = (uint8_t)(off >> 8);
                    if (mt >= 15) o = put_ext(o, mt);
                    first = false;
                }
            }
            if (sb > prev_end) {   // trailing literals belong to the next sequence downstream
                const uint32_t nh = my_next_has;
                const int32_t dl = (nh != 0xffff && nh < nseg) ? delta0[nh] : delta_final;
                copy_lit(out + ((int32_t)prev_end + dl), dw, prev_end, sb - prev_end);
            }
        }
        if (tid == 0) {
            uint8_t* o = out + total_seq_bytes;
            *o++ = (uint8_t)((ll_final < 15 ? ll_final : 15) << 4);
            if (ll_final >= 15) o = put_ext(o, ll_final);
            const uint32_t c9 = cs + 9;
            stg[0] = 0x82; stg[1] = (uint8_t)c9; stg[2] = (uint8_t)(c9 >> 8); stg[3] = (uint8_t)(c9 >> 16); stg[4] = (uint8_t)(c9 >> 24);
            stg[5] = (uint8_t)len; stg[6] = (uint8_t)(len >> 8); stg[7] = (uint8_t)(len >> 16); stg[8] = (uint8_t)(len >> 24);
        }
        LZ_PHASE(4);
        pend_f = f; pend_cs = cs;      // written to the wire buffer while the next frame is being parsed (resolve_flush above), or after the loop
    }
    if (pend_f != 0xffffffffu) { __syncthreads(); resolve_flush(pend_f, pend_cs); }
}
#endif  // TF_KERNELS_LZ4

// ------------------------------------------------------------------ CityHash128 v1.0.2 over [method byte .. end of block]
namespace cityd {
#define CK0 0xc3a5c85c97cb3127ULL
#define CK1 0xb492b66fbe98f273ULL
#define CK2 0x9ae16a3b2f90404fULL
#define CK3 0xc949d7c7509e6557ULL
__device__ __forceinline__ uint64_t f64(const uint8_t* p) {
    const uintptr_t a = (uintptr_t)p; const uint64_t* q = (const uint64_t*)(a & ~(uintptr_t)7); const uint32_t s = (uint32_t)(a & 7) * 8;
    if (s == 0) return q[0];
    return (q[0] >> s) | (q[1] << (64 - s));
}
__device__ __forceinline__ uint32_t f32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint64_t rot(uint64_t v, int s) { return s == 0 ? v : ((v >> s) | (v << (64 - s))); }
__device__ __forceinline__ uint64_t smix(uint64_t v) { return v ^ (v >> 47); }
__device__ __forceinline__ uint64_t hl16(uint64_t u, uint64_t v) {
    const uint64_t kMul = 0x9ddfea08eb382d69ULL;
    uint64_t a = (u ^ v) * kMul; a ^= (a >> 47);
    uint64_t b = (v ^ a) * kMul; b ^= (b >> 47); b *= kMul; return b;
}
static __device__ uint64_t hl0to16(const uint8_t* s, size_t len) {
    if (len > 8) { uint64_t a = f64(s), b = f64(s + len - 8); return hl16(a, rot(b + len, (int)len)) ^ b; }
    if (len >= 4) { uint64_t a = f32(s); return hl16(len + (a << 3), f32(s + len - 4)); }
    if (len > 0) { uint8_t a = s[0], b = s[len >> 1], c = s[len - 1]; uint32_t y = (uint32_t)a + ((uint32_t)b << 8); uint32_t z = (uint32_t)len + ((uint32_t)c << 2); return smix(y * CK2 ^ z * CK3) * CK2; }
    return CK2;
}
struct P { uint64_t first, second; };
__device__ __forceinline__ P weak32(uint64_t w, uint64_t x, uint64_t y, uint64_t z, uint64_t a, uint64_t b) {
    a += w; b = rot(b + a + z, 21); const uint64_t c = a; a += x; a += y; b += rot(a, 44); P r; r.first = a + z; r.second = b + c; return r;
}
__device__ __forceinline__ P weak32p(const uint8_t* s, uint64_t a, uint64_t b) { return weak32(f64(s), f64(s + 8), f64(s + 16), f64(s + 24), a, b); }
static __device__ P murmur(const uint8_t* s, size_t len, P seed) {
    uint64_t a = seed.first, b = seed.second, c = 0, d = 0; long l = (long)len - 16;
    if (l <= 0) { a = smix(a * CK1) * CK1; c = b * CK1 + hl0to16(s, len); d = smix(a + (len >= 8 ? f64(s) : c)); }
    else {
        c = hl16(f64(s + len - 8) + CK1, a); d = hl16(b + len, c + f64(s + len - 16)); a += d;
        do { a ^= smix(f64(s) * CK1) * CK1; a *= CK1; b ^= a; c ^= smix(f64(s + 8) * CK1) * CK1; c *= CK1; d ^= c; s += 16; l -= 16; } while (l > 0);
    }
    a = hl16(a, c); b = hl16(d, b);
    P r; r.first = a ^ b; r.second = hl16(b, a); return r;
}
static __device__ P hash128_seed(const uint8_t* s, size_t len, P seed) {
    if (len < 128) return murmur(s, len, seed);
    P v, w; uint64_t x = seed.first, y = seed.second, z = len * CK1;
    v.first = rot(y ^ CK1, 49) * CK1 + f64(s);
    v.second = rot(v.first, 42) * CK1 + f64(s + 8);
    w.first = rot(y + z, 35) * CK1 + x;
    w.second = rot(x + f64(s + 88), 53) * CK1;
    do {
#pragma unroll
        for (int rep = 0; rep < 2; rep++) {
            x = rot(x + y + v.first + f64(s + 16), 37) * CK1;
            y = rot(y + v.second + f64(s + 48), 42) * CK1;
            x ^= w.second; y ^= v.first; z = rot(z ^ w.first, 33);
            v = weak32p(s, v.second * CK1, x + w.first);
            w = weak32p(s + 32, z + w.second, y);
            const uint64_t t = z; z = x; x = t; s += 64;
        }
        len -= 128;
    } while (len >= 128);
    y += rot(w.first, 37) * CK0 + z;
    x += rot(v.first + z, 49) * CK0;
    for (size_t tail = 0; tail < len;) {
        tail += 32;
        y = rot(y - x, 42) * CK0 + v.second;
        w.first += f64(s + len - tail + 16);
        x = rot(x, 49) * CK0 + w.first;
        w.first += v.first;
        v = weak32p(s + len - tail, v.first, v.second);
    }
    x = hl16(x, v.first); y = hl16(y, w.first);
    P r; r.first = hl16(x + v.second, w.second) + y; r.second = hl16(x + w.second, y + v.second); return r;
}
static __device__ P hash128(const uint8_t* s, size_t len) {
    P seed;
    if (len >= 16) { seed.first = f64(s) ^ CK3; seed.second = f64(s + 8); return hash128_seed(s + 16, len - 16, seed); }
    if (len >= 8) { seed.first = f64(s) ^ (len * CK0); seed.second = f64(s + len - 8) ^ CK1; return hash128_seed(nullptr, 0, seed); }
    seed.first = CK0; seed.second = CK1; return hash128_seed(s, len, seed);
}
}  // namespace cityd

struct FrameArgs { const uint32_t* comp_size; const uint64_t* wire_off; uint8_t* wire; const uint64_t* tail; };   // tail[0] = frame count, written by k_lz4_frames

// CityHash128 is a serial chain per frame, so the parallelism is ACROSS frames: one thread per frame. What a
// thread-per-frame loop would ruin is the memory access (every lane striding through its own frame), so each
// warp stages the next 512 bytes of all its 32 frames with coalesced 16-byte cp.async copies into shared
// memory (double buffered) while the lanes hash the previous 512 bytes out of it. The frames sit at byte
// offsets in the wire buffer, so the copies start at the 16-byte boundary below the frame and every lane
// reads its 8-byte words at its own shift.
#define SEAL_STEP 512
#define SEAL_STRIDE 544
#define SEAL_TAIL 320
#define SEAL_STAGES 2      /* deeper pipelines do not help: the per-frame hash is a serial dependency chain (~43 k instructions) */
#define SEAL_SMEM ((size_t)SEAL_STAGES * 32 * SEAL_STRIDE + 32 * SEAL_TAIL)
__device__ __forceinline__ uint64_t sm64u(const uint8_t* base, uint32_t off) {      // 8 bytes at any byte offset of a shared-memory row
    const uint32_t al = off & ~7u, s = (off & 7u) * 8;
    const uint64_t lo = *(const uint64_t*)(base + al), hi = *(const uint64_t*)(base + al + 8);
    return (lo >> s) | ((hi << 1) << (63 - s));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

__global__ void k_frame_seal(FrameArgs a);
#ifdef TF_KERNELS_LZ4
__global__ void __launch_bounds__(32) k_frame_seal(FrameArgs a) {
    extern __shared__ __align__(16) uint8_t seal_smem[];
    uint8_t (*s_buf)[32][SEAL_STRIDE] = (uint8_t (*)[32][SEAL_STRIDE])seal_smem;                                  // [SEAL_STAGES][32][SEAL_STRIDE]
    uint8_t (*s_tail)[SEAL_TAIL] = (uint8_t (*)[SEAL_TAIL])(seal_smem + (size_t)SEAL_STAGES * 32 * SEAL_STRIDE);  // [32][SEAL_TAIL]
    const uint32_t lane = threadIdx.x;
    const uint64_t nf = a.tail[0];
    const uint64_t f = (uint64_t)blockIdx.x * 32 + lane;
    const bool have = f < nf;
    // the frame: [16 checksum][0x82][u32 compressed size + 9][u32 raw size][LZ4 block]; the hash covers everything behind the checksum
    const uint8_t* H = a.wire + (have ? a.wire_off[f] : 0) + 16;
    const uint32_t cs = have ? a.comp_size[f] + 9 : 0;
    uint8_t* wck = (uint8_t*)H - 16;
    auto put_checksum = [&](uint64_t lo, uint64_t hi) {
#pragma unroll
        for (int b = 0; b < 8; b++) { wck[b] = (uint8_t)(lo >> (8 * b)); wck[8 + b] = (uint8_t)(hi >> (8 * b)); }
    };
    const bool big = have && cs >= 16 + 128 + 16;
    if (have && !big) { const cityd::P h = cityd::hash128(H, cs); put_checksum(h.first, h.second); }
    const uint8_t* body = H + 16; const uint32_t len = big ? cs - 16 : 0;
    const uint32_t bsh = (uint32_t)((uintptr_t)body & 15);
    const uint8_t* body_al = body - bsh;
    const uint32_t nblk = len / 128, used = nblk * 128;
    const uint32_t nsteps = (used + SEAL_STEP - 1) / SEAL_STEP;
    uint32_t max_steps = nsteps;
#pragma unroll
    for (int d = 16; d; d >>= 1) { const uint32_t o = __shfl_xor_sync(0xffffffffu, max_steps, d); max_steps = o > max_steps ? o : max_steps; }
    if (max_steps == 0) return;
    const uint32_t tail_rel = (bsh + (len > 272 ? (len - 272) : 0)) & ~15u;      // relative to body_al
    // cooperative staging: lane l copies bytes [16 l, 16 l + 16) of every frame's current step (+ 2 more chunks for the shifted reads)
    auto stage_step = [&](uint32_t st, uint32_t bi) {
#pragma unroll 4
        for (int j = 0; j < 32; j++) {
            const uint8_t* bj = (const uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)body_al, j);
            const uint32_t uj = __shfl_sync(0xffffffffu, used ? used + 32 : 0, j);
            const uint32_t off = st * SEAL_STEP + lane * 16;
            if (off < uj) cp_async16(&s_buf[bi][j][lane * 16], bj + off);
            if (lane < 2 && off + 512 < uj) cp_async16(&s_buf[bi][j][512 + lane * 16], bj + off + 512);
        }
        cp_async_commit();
    };
    for (int j = 0; j < 32; j++) {      // tail windows
        const uint8_t* bj = (const uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)body_al, j);
        const uint32_t lj = __shfl_sync(0xffffffffu, len, j), tj = __shfl_sync(0xffffffffu, tail_rel, j);
        if (lane < SEAL_TAIL / 16 && lj) cp_async16(&s_tail[j][16 * lane], bj + tj + 16 * lane);
    }
#pragma unroll
    for (int k = 0; k < SEAL_STAGES - 1; k++) { if ((uint32_t)k < max_steps) stage_step(k, k); else cp_async_commit(); }      // the tail windows ride in the first group
    cityd::P v, w; uint64_t x = 0, y = 0, z = 0;
    if (big) {
        x = cityd::f64(H) ^ CK3; y = cityd::f64(H + 8); z = (uint64_t)len * CK1;
        v.first = cityd::rot(y ^ CK1, 49) * CK1 + cityd::f64(body);
        v.second = cityd::rot(v.first, 42) * CK1 + cityd::f64(body + 8);
        w.first = cityd::rot(y + z, 35) * CK1 + x;
        w.second = cityd::rot(x + cityd::f64(body + 88), 53) * CK1;
    }
    for (uint32_t st = 0; st < max_steps; st++) {
        if (st + SEAL_STAGES - 1 < max_steps) stage_step(st + SEAL_STAGES - 1, (st + SEAL_STAGES - 1) % SEAL_STAGES); else cp_async_commit();
        cp_async_wait<SEAL_STAGES - 1>();      // every group but the newest SEAL_STAGES - 1 has landed: step st is in shared memory
        __syncwarp();
        if (st < nsteps) {
            const uint8_t* b = s_buf[st % SEAL_STAGES][lane];
            const uint32_t nb = (nblk - st * 4 < 4) ? nblk - st * 4 : 4;
            for (uint32_t i = 0; i < 2 * nb; i++) {
                const uint32_t o = i * 64 + bsh;
                const uint64_t q0 = sm64u(b, o), q1 = sm64u(b, o + 8), q2 = sm64u(b, o + 16), q3 = sm64u(b, o + 24);
                const uint64_t q4 = sm64u(b, o + 32), q5 = sm64u(b, o + 40), q6 = sm64u(b, o + 48), q7 = sm64u(b, o + 56);
                x = cityd::rot(x + y + v.first + q2, 37) * CK1;
                y = cityd::rot(y + v.second + q6, 42) * CK1;
                x ^= w.second; y ^= v.first; z = cityd::rot(z ^ w.first, 33);
                v = cityd::weak32(q0, q1, q2, q3, v.second * CK1, x + w.first);
                w = cityd::weak32(q4, q5, q6, q7, z + w.second, y);
                const uint64_t t = z; z = x; x = t;
            }
        }
        __syncwarp();
    }
    if (big) {
        const uint32_t rem = len - used;                 // 0..127 bytes; the tail reads reach back into hashed data
        const uint8_t* tb = s_tail[lane];
        auto t64 = [&](uint32_t off) -> uint64_t { return sm64u(tb, off + bsh - tail_rel); };      // 8 bytes at body + off
        y += cityd::rot(w.first, 37) * CK0 + z;
        x += cityd::rot(v.first + z, 49) * CK0;
        for (uint32_t td = 0; td < rem;) {
            td += 32;
            const uint32_t base = len - td;
            y = cityd::rot(y - x, 42) * CK0 + v.second;
            w.first += t64(base + 16);
            x = cityd::rot(x, 49) * CK0 + w.first;
            w.first += v.first;
            v = cityd::weak32(t64(base), t64(base + 8), t64(base + 16), t64(base + 24), v.first, v.second);
        }
        x = cityd::hl16(x, v.first); y = cityd::hl16(y, w.first);
        put_checksum(cityd::hl16(x + v.second, w.second) + y, cityd::hl16(x + w.second, y + v.second));
    }
}
#endif  // TF_KERNELS_LZ4

}  // namespace tfk
