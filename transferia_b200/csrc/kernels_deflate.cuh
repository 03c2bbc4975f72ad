// DEFLATE (RFC 1951) of the batch serializers' row text inside a gzip member (RFC 1952) or a zlib stream (RFC 1950), the S3
// sink's OutputEncoding GZIP / ZLIB (TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB).
//
// The text is cut into DF_CHUNK-byte chunks that do not depend on each other: no back-reference crosses a chunk start, every
// chunk starts byte-aligned and ends with a sync-flush marker (an empty non-final stored block). One CTA compresses one chunk
// in shared memory at a time (persistent CTAs take chunks by ticket), every phase data-parallel:
//   P1  stage the chunk; CRC-32 or the Adler-32 sums of every thread's 32 bytes, combined into the chunk's value
//   P2  match finding in rounds of DF_THREADS positions: the same 4 bytes 1, 2 or 4 back (runs), else a hash-table entry of an
//       earlier round, else one of this round; the match length (4..258, inside the chunk) is measured for each position
//   P3  greedy parse by pointer doubling: next(p) = p + match length, or p + 1 for a literal; the positions of the path
//       from 0 are marked in log2(tokens) rounds of "mark next(marked)" and "next = next(next)"
//   P4  histograms of the literal/length and distance symbols of the marked tokens
//   P5  block choice by exact bit count: stored, fixed Huffman, or dynamic Huffman (length-limited codes: 15 bits, 7 for the
//       code-length code, built by the in-place Moffat-Katajainen algorithm and a Kraft-sum repair)
//   P6  every thread bit-packs its tokens at the bit offset a block scan gives it into a shared-memory image of the chunk
//   P7  the chunk's size is published for the chunks behind it and the image is written at its final offset (decoupled
//       look-back over the earlier chunks' sizes)
// k_deflate_finish then combines the chunk checksums and writes the container header, the final empty fixed block and the
// trailer, so the bytes are complete when they land on the host. The compressed bytes are not those of Go's compress/flate
// (the decoded text and the container framing are what is pinned, DESIGN.md §3).
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "deflate_sum.hpp"

namespace tfk {

#define DF_CHUNK 16384       /* bytes per chunk: positions and successors fit u16; ~105 KiB of shared memory, two CTAs per SM */
#define DF_THREADS 512
#define DF_PPT (DF_CHUNK / DF_THREADS)     /* 32 positions per thread: one word of the path bitmap */
#define DF_HASH_BITS 12
#define DF_CHUNK_OVERHEAD 10               /* a stored block's header (5) + the sync-flush marker (5) */
#define DF_FLAG_AGG (1ull << 62)
#define DF_FLAG_INCL (2ull << 62)
#define DF_VAL_MASK ((1ull << 62) - 1)

// shared-memory carve-up (byte offsets)
struct DfSmem { uint32_t data, dist, lenb, work, path, hist, lens, codes, sort, crct, total; };
__host__ __device__ inline DfSmem df_smem() {
    DfSmem s; uint32_t o = 0;
    s.data = o; o += 16 + DF_CHUNK + 32;                  // zero guard words in front of and behind the chunk
    s.dist = o; o += 2 * DF_CHUNK;                        // u16 match distance per position
    s.lenb = o; o += DF_CHUNK;                            // u8 match length - 3 per position (0 = literal)
    s.work = o; o += 2 * DF_CHUNK + 64;                   // P2 hash table; P3 successors (DF_CHUNK + 1 u16); P6 the image
    s.path = o; o += (DF_CHUNK / 32 + 4) * 4;             // bitmap of the parse's token starts
    s.hist = o; o += (288 + 32 + 20) * 4;                 // literal/length, distance, code-length histograms
    s.lens = o; o += 288 + 32 + 32;                       // code lengths
    s.codes = o; o += (288 + 32 + 32) * 2;                // bit-reversed codes
    s.sort = o; o += 320 * 4 * 2 + 320 * 2 + 320 * 2;     // build weights, sorted weights, sorted symbols, code-length RLE
    s.crct = o; o += 256 * 4;                             // CRC-32 byte table
    s.total = o; return s;
}

struct DeflateArgs {
    const uint8_t* text; uint64_t total;     // the row text and its byte count (the host read it before sizing the arena)
    uint8_t* out;                            // header | chunk bodies | 03 00 | trailer
    unsigned long long* pfx;                 // [nchunks] decoupled look-back cells, zeroed before the launch
    uint32_t* sums;                          // [2 nchunks]: CRC-32 of the chunk, or its Adler sums (s1, s2)
    uint32_t* ticket;                        // work counter, zeroed before the launch
    uint32_t nchunks;
    int zlib;                                // 0 gzip, 1 zlib
    DState* st;                              // wire_total
};
__global__ void k_deflate_chunks(DeflateArgs a);
__global__ void k_deflate_finish(DeflateArgs a);

__device__ __forceinline__ uint32_t df_ld32(const uint32_t* w, uint32_t p) {   // 4 bytes at byte offset p of the chunk
    const uint32_t i = p >> 2, s = (p & 3) * 8;
    return __funnelshift_r(w[i], w[i + 1], s);
}
// common prefix of the chunk bytes at c < p, at most maxl
__device__ __forceinline__ uint32_t df_match_len(const uint32_t* dw, uint32_t c, uint32_t p, uint32_t maxl) {
    uint32_t n = 0;
    while (n < maxl) {
        const uint32_t x = df_ld32(dw, c + n) ^ df_ld32(dw, p + n);
        if (x) { n += (uint32_t)(__ffs((int)x) - 1) >> 3; break; }
        n += 4;
    }
    return n < maxl ? n : maxl;
}
// RFC 1951 §3.2.5: length 3..258 -> symbol 257..285 + extra bits; distance 1..32768 -> symbol 0..29 + extra bits
__device__ __forceinline__ void df_len_sym(uint32_t len, uint32_t& sym, uint32_t& eb, uint32_t& ev) {
    const uint32_t l = len - 3;
    if (l < 8) { sym = 257 + l; eb = 0; ev = 0; }
    else if (l == 255) { sym = 285; eb = 0; ev = 0; }
    else { const uint32_t nb = 31 - __clz(l); eb = nb - 2; sym = 257 + 4 * (nb - 1) + ((l >> eb) & 3); ev = l & ((1u << eb) - 1); }
}
__device__ __forceinline__ void df_dist_sym(uint32_t d, uint32_t& sym, uint32_t& eb, uint32_t& ev) {
    const uint32_t v = d - 1;
    if (v < 4) { sym = v; eb = 0; ev = 0; }
    else { const uint32_t nb = 31 - __clz(v); eb = nb - 1; sym = 2 * nb + ((v >> eb) & 1); ev = v & ((1u << eb) - 1); }
}
__device__ __forceinline__ uint32_t df_fixed_len(uint32_t s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
// OR n (<= 32) bits of v into the image at bit offset at (LSB first)
__device__ __forceinline__ void df_put(uint32_t* img, uint32_t at, uint32_t v, uint32_t n) {
    if (!n) return;
    const uint32_t w = at >> 5, s = at & 31;
    atomicOr(&img[w], v << s);
    if (s + n > 32) atomicOr(&img[w + 1], v >> (32 - s));
}

#if defined(TF_KERNELS_DEFLATE) || defined(TF_KERNELS_ZSTD)
// Code lengths of a minimum-redundancy code limited to maxbits (one thread). w[0..n) holds the weights in ascending order
// (n >= 2) and sym[] their symbols; lens[sym] receives the lengths (the caller zeroed the others). w is overwritten.
static __device__ void df_huff_lengths(uint32_t* w, const uint16_t* sym, int n, uint32_t maxbits, uint8_t* lens) {
    // Moffat & Katajainen, in place: tree (parent pointers), internal node depths, leaf depths
    w[0] += w[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < n - 1; next++) {
        if (leaf >= n || w[root] < w[leaf]) { w[next] = w[root]; w[root++] = (uint32_t)next; }
        else w[next] = w[leaf++];
        if (leaf >= n || (root < next && w[root] < w[leaf])) { w[next] += w[root]; w[root++] = (uint32_t)next; }
        else w[next] += w[leaf++];
    }
    w[n - 2] = 0;
    for (int next = n - 3; next >= 0; next--) w[next] = w[w[next]] + 1;
    {
        int avail = 1, used = 0, depth = 0, r = n - 2, next = n - 1;
        while (avail > 0) {
            while (r >= 0 && (int)w[r] == depth) { used++; r--; }
            while (avail > used) { w[next--] = (uint32_t)depth; avail--; }
            avail = 2 * used; depth++; used = 0;
        }
    }
    // length limit: clamp, then repair the Kraft sum (each step moves one code one level down and removes one at maxbits)
    uint32_t cnt[16];
    for (uint32_t l = 0; l <= 15; l++) cnt[l] = 0;
    for (int i = 0; i < n; i++) cnt[w[i] < maxbits ? w[i] : maxbits]++;
    uint32_t kraft = 0;
    for (uint32_t l = 1; l <= maxbits; l++) kraft += cnt[l] << (maxbits - l);
    while (kraft > (1u << maxbits)) {
        cnt[maxbits]--;
        for (uint32_t l = maxbits - 1; l > 0; l--) if (cnt[l]) { cnt[l]--; cnt[l + 1] += 2; break; }
        kraft--;
    }
    // the heaviest symbols take the shortest codes
    int i = n - 1;
    for (uint32_t l = 1; l <= maxbits; l++) for (uint32_t k = 0; k < cnt[l]; k++) lens[sym[i--]] = (uint8_t)l;
}
#endif

// Exclusive prefix of the sizes of chunks [0, f) (warp 0). Cells hold AGG | own size or INCL | inclusive prefix; a wait past the
// bound sets st->pad.
__device__ __forceinline__ unsigned long long df_lookback(unsigned long long* pfx, DState* st, uint32_t f, uint32_t lane) {
    unsigned long long excl = 0;
    int64_t base = (int64_t)f;
    for (uint32_t spins = 0; base > 0;) {
        const int64_t j = base - 1 - (int64_t)lane;
        const unsigned long long v = j >= 0 ? *(volatile unsigned long long*)&pfx[j] : DF_FLAG_INCL;
        const uint32_t fl = (uint32_t)(v >> 62);
        const uint32_t incl = __ballot_sync(0xffffffffu, fl == 2), none = __ballot_sync(0xffffffffu, fl == 0);
        const uint32_t upto = incl ? (uint32_t)__ffs((int)incl) - 1 : 31u;
        const uint32_t need = upto == 31 ? 0xffffffffu : ((2u << upto) - 1);
        if (none & need) {       // an earlier chunk has not published yet (its CTA holds a lower ticket and is running)
            if (++spins > (1u << 20)) { if (lane == 0) st->pad = 1; break; }      // a bounded wait keeps a bug from hanging the device
            __nanosleep(100); continue;
        }
        unsigned long long part = lane <= upto ? (v & DF_VAL_MASK) : 0ull;
#pragma unroll
        for (int d = 16; d; d >>= 1) part += __shfl_xor_sync(0xffffffffu, part, d);
        excl += part; base -= 32;
        if (incl) break;
    }
    return excl;
}

#ifdef TF_KERNELS_DEFLATE
// canonical codes (RFC 1951 §3.2.2), stored bit-reversed for the LSB-first bit stream (one thread)
__device__ void df_codes(const uint8_t* lens, int n, uint16_t* codes) {
    uint32_t cnt[16], next[16];
    for (int l = 0; l < 16; l++) cnt[l] = 0;
    for (int s = 0; s < n; s++) cnt[lens[s]]++;
    cnt[0] = 0; uint32_t c = 0;
    for (int l = 1; l < 16; l++) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
    for (int s = 0; s < n; s++) { const uint32_t l = lens[s]; codes[s] = l ? (uint16_t)(__brev(next[l]++) >> (32 - l)) : 0; }
}

__device__ __forceinline__ uint32_t df_block_xor(uint32_t v, uint32_t* red) {
#pragma unroll
    for (int d = 16; d; d >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t r = 0;
    for (uint32_t w = 0; w < (blockDim.x + 31) / 32; w++) r ^= red[w];
    __syncthreads();
    return r;
}
__device__ __forceinline__ uint64_t df_block_sum64(uint64_t v, unsigned long long* red) {
#pragma unroll
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint64_t r = 0;
    for (uint32_t w = 0; w < (blockDim.x + 31) / 32; w++) r += red[w];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(DF_THREADS, 2) k_deflate_chunks(DeflateArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const DfSmem S = df_smem();
    uint8_t* db = smem + S.data + 16;                       // the chunk; 16 zero bytes in front, 32 behind
    const uint32_t* dw = (const uint32_t*)db;
    uint16_t* dist = (uint16_t*)(smem + S.dist);
    uint8_t* lenb = smem + S.lenb;
    uint16_t* J = (uint16_t*)(smem + S.work);               // P2: hash table (position + 1); P3: successor of every position
    uint32_t* img = (uint32_t*)(smem + S.work);              // P6: the compressed chunk
    uint32_t* path = (uint32_t*)(smem + S.path);
    uint32_t* hl = (uint32_t*)(smem + S.hist); uint32_t* hd = hl + 288; uint32_t* hc = hd + 32;
    uint8_t* ll_len = smem + S.lens; uint8_t* d_len = ll_len + 288; uint8_t* c_len = d_len + 32;
    uint16_t* ll_code = (uint16_t*)(smem + S.codes); uint16_t* d_code = ll_code + 288; uint16_t* c_code = d_code + 32;
    uint32_t* bw = (uint32_t*)(smem + S.sort);               // [320] build weights (literal/length at 0, distance at 288)
    uint32_t* sw = bw + 320;                                 // [320] sorted weights
    uint16_t* ssym = (uint16_t*)(sw + 320);                  // [320] sorted symbols
    uint16_t* rle = ssym + 320;                              // [320] code-length RLE: symbol | extra value << 8
    uint32_t* crct = (uint32_t*)(smem + S.crct);
    __shared__ uint32_t s_f, s_btype, s_hdr_bits, s_nbytes, s_nrle, s_hlit, s_hdist, s_hclen;
    __shared__ uint32_t red[33];
    __shared__ unsigned long long red64[32], s_off;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (uint32_t i = tid; i < 256; i += DF_THREADS) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ tfdf::CRC_POLY : c >> 1;
        crct[i] = c;
    }
    for (;;) {
        __syncthreads();
        if (tid == 0) s_f = atomicAdd(a.ticket, 1u);
        __syncthreads();
        const uint32_t f = s_f;
        if (f >= a.nchunks) break;
        const uint64_t pos0 = (uint64_t)f * DF_CHUNK;
        const uint32_t L = (uint32_t)((a.total - pos0 < DF_CHUNK) ? a.total - pos0 : DF_CHUNK);

        // ---- P1: stage, clear, checksum
        {
            const int4* g = (const int4*)(a.text + pos0);
            const uint32_t nv = (L + 15) >> 4;
            int4* d4 = (int4*)db;
            for (uint32_t i = tid; i < DF_CHUNK / 16 + 2; i += DF_THREADS) d4[i] = i < nv ? __ldg(g + i) : make_int4(0, 0, 0, 0);
            if (tid < 4) ((uint32_t*)(smem + S.data))[tid] = 0;
            int4* t4 = (int4*)J;
            for (uint32_t i = tid; i < (2u << DF_HASH_BITS) / 16; i += DF_THREADS) t4[i] = make_int4(0, 0, 0, 0);
            for (uint32_t i = tid; i < DF_CHUNK / 32 + 4; i += DF_THREADS) path[i] = 0;
            for (uint32_t i = tid; i < 288 + 32 + 20; i += DF_THREADS) hl[i] = 0;
        }
        __syncthreads();
        if (tid < 16 && L + tid < ((L + 15) & ~15u)) db[L + tid] = 0;     // the bytes the last 16-byte load brought in past the chunk
        {
            const uint32_t b0 = tid * DF_PPT, b1 = b0 + DF_PPT < L ? b0 + DF_PPT : L, nb = b1 > b0 ? b1 - b0 : 0;
            if (a.zlib) {       // s1 = sum of bytes, s2 = sum of (bytes from here to the chunk end) * byte
                uint64_t s1 = 0, s2 = 0;
                for (uint32_t i = 0; i < nb; i++) { const uint32_t v = db[b0 + i]; s1 += v; s2 += (uint64_t)(L - b0 - i) * v; }
                s1 = df_block_sum64(s1, red64) % tfdf::ADLER_MOD; s2 = df_block_sum64(s2, red64) % tfdf::ADLER_MOD;
                if (tid == 0) { a.sums[2 * f] = (uint32_t)s1; a.sums[2 * f + 1] = (uint32_t)s2; }
            } else {            // CRC-32 of the thread's bytes, shifted past the rest of the chunk: the chunk's CRC is their xor
                uint32_t c = 0;
                if (nb) {
                    c = 0xffffffffu;
                    for (uint32_t i = 0; i < nb; i++) c = crct[(c ^ db[b0 + i]) & 0xff] ^ (c >> 8);
                    c = tfdf::crc_mulmod(tfdf::crc_xpow8(L - b1), ~c);
                }
                c = df_block_xor(c, red);
                if (tid == 0) a.sums[2 * f] = c;
            }
        }

        // ---- P2: match finding
        const uint32_t nrounds = (L + DF_THREADS - 1) / DF_THREADS;
        for (uint32_t r = 0; r < nrounds; r++) {
            const uint32_t p = r * DF_THREADS + tid;
            const bool valid = p + 4 <= L;
            const uint32_t w = valid ? df_ld32(dw, p) : 0, h = (w * 2654435761u) >> (32 - DF_HASH_BITS);
            const uint32_t t1 = valid ? J[h] : 0;          // an entry of an earlier round
            __syncthreads();
            if (valid) J[h] = (uint16_t)(p + 1);
            __syncthreads();
            const uint32_t t2 = valid ? J[h] : 0;          // this round's entry (a later position wins half the time)
            uint32_t best = 0, bd = 0;
            if (valid) {
                const uint32_t maxl = L - p < 258 ? L - p : 258;
                uint32_t c = 0xffffffffu;
                if (p >= 1 && df_ld32(dw, p - 1) == w) c = p - 1;
                else if (p >= 2 && df_ld32(dw, p - 2) == w) c = p - 2;
                else if (p >= 4 && df_ld32(dw, p - 4) == w) c = p - 4;
                if (c != 0xffffffffu) { best = df_match_len(dw, c, p, maxl); bd = p - c; }
                const uint32_t ct = (t2 && t2 - 1 < p) ? t2 - 1 : (t1 ? t1 - 1 : 0xffffffffu);
                if (ct != 0xffffffffu && ct != c && best < maxl) {
                    const uint32_t m = df_match_len(dw, ct, p, maxl);
                    if (m > best) { best = m; bd = p - ct; }
                }
            }
            if (p < L) { lenb[p] = (uint8_t)(best >= 4 ? best - 3 : 0); dist[p] = (uint16_t)bd; }
        }
        __syncthreads();

        // ---- P3: greedy parse by pointer doubling
        for (uint32_t k = 0; k < DF_PPT; k++) { const uint32_t p = tid * DF_PPT + k; if (p < L) J[p] = (uint16_t)(p + (lenb[p] ? lenb[p] + 3u : 1u)); }
        if (tid == 0) { J[L] = (uint16_t)L; path[0] = 1; }
        __syncthreads();
        for (;;) {
            // every marked position marks its successor (the path positions i < 2^(k+1) steps from 0 after round k)
            uint32_t bits = path[tid];
            while (bits) {
                const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
                const uint32_t p = tid * DF_PPT + k;
                if (p < L) { const uint32_t q = J[p]; if (q < L) atomicOr(&path[q >> 5], 1u << (q & 31)); }
            }
            __syncthreads();
            uint32_t nx[DF_PPT / 2];
#pragma unroll
            for (uint32_t k = 0; k < DF_PPT; k += 2) {
                const uint32_t p = tid * DF_PPT + k;
                const uint32_t lo = p < L ? J[J[p]] : 0, hi = p + 1 < L ? J[J[p + 1]] : 0;
                nx[k / 2] = lo | (hi << 16);
            }
            __syncthreads();
#pragma unroll
            for (uint32_t k = 0; k < DF_PPT; k += 2) {
                const uint32_t p = tid * DF_PPT + k;
                if (p < L) J[p] = (uint16_t)nx[k / 2];
                if (p + 1 < L) J[p + 1] = (uint16_t)(nx[k / 2] >> 16);
            }
            __syncthreads();
            if (J[0] == L) break;          // the path from 0 reaches the end within the steps already marked
            __syncthreads();
        }
        const uint32_t mine = path[tid] & (tid * DF_PPT + DF_PPT <= L ? 0xffffffffu : (tid * DF_PPT < L ? (1u << (L - tid * DF_PPT)) - 1 : 0u));

        // ---- P4: histograms
        uint32_t ext = 0;
        for (uint32_t bits = mine; bits;) {
            const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
            const uint32_t p = tid * DF_PPT + k, l = lenb[p];
            if (!l) { atomicAdd(&hl[db[p]], 1u); continue; }
            uint32_t s, eb, ev, ds, deb, dev;
            df_len_sym(l + 3, s, eb, ev); df_dist_sym(dist[p], ds, deb, dev);
            atomicAdd(&hl[s], 1u); atomicAdd(&hd[ds], 1u); ext += eb + deb;
        }
        if (tid == 0) atomicAdd(&hl[256], 1u);      // end of block
        uint32_t ext_total; block_excl_scan(ext, &ext_total, red);      // (also the barrier behind the histograms)

        // ---- P5: codes and the block choice
        const int nzd = __syncthreads_count(tid < 30 && hd[tid] > 0);
        if (tid < 288) { bw[tid] = tid < 286 ? hl[tid] : 0; ll_len[tid] = 0; }
        else if (tid < 320) {       // a distance code needs two symbols to be complete: pad the build weights when fewer are used
            const uint32_t i = tid - 288; uint32_t v = i < 30 ? hd[i] : 0;
            if (i < 30 && !v && ((nzd == 0 && i < 2) || (nzd == 1 && i == (hd[0] ? 1u : 0u)))) v = 1;
            bw[tid] = v; d_len[i] = 0;
        }
        __syncthreads();
        {   // rank sort of the used symbols by (weight, symbol)
            const bool ll = tid < 286, dd = tid >= 288 && tid < 318;
            if (ll || dd) {
                const uint32_t base = ll ? 0 : 288, n = ll ? 286 : 30, i = tid - base, v = bw[tid];
                if (v) {
                    uint32_t rank = 0;
                    for (uint32_t j = 0; j < n; j++) { const uint32_t u = bw[base + j]; rank += (u && (u < v || (u == v && j < i))) ? 1u : 0u; }
                    sw[base + rank] = v; ssym[base + rank] = (uint16_t)i;
                }
            }
        }
        const int nzl = __syncthreads_count(tid < 286 && hl[tid] > 0);
        if (tid == 0) df_huff_lengths(sw, ssym, nzl, 15, ll_len);
        if (tid == 32) df_huff_lengths(sw + 288, ssym + 288, nzd < 2 ? 2 : nzd, 15, d_len);
        __syncthreads();
        if (tid == 0) {
            // dynamic header: HLIT / HDIST trimmed, the lengths run-length coded with 16 / 17 / 18
            uint32_t hlit = 286; while (hlit > 257 && !ll_len[hlit - 1]) hlit--;
            uint32_t hdist = 30; while (hdist > 1 && !d_len[hdist - 1]) hdist--;
            const uint32_t N = hlit + hdist;
            auto lv = [&](uint32_t i) -> uint32_t { return i < hlit ? ll_len[i] : d_len[i - hlit]; };
            uint32_t nr = 0;
            for (uint32_t i = 0; i < N;) {
                const uint32_t v = lv(i); uint32_t run = 1;
                while (i + run < N && lv(i + run) == v) run++;
                i += run;
                if (v == 0) {
                    while (run >= 11) { const uint32_t r = run < 138 ? run : 138; rle[nr++] = (uint16_t)(18 | ((r - 11) << 8)); run -= r; }
                    if (run >= 3) { rle[nr++] = (uint16_t)(17 | ((run - 3) << 8)); run = 0; }
                } else {
                    rle[nr++] = (uint16_t)v; run--;
                    while (run >= 3) { const uint32_t r = run < 6 ? run : 6; rle[nr++] = (uint16_t)(16 | ((r - 3) << 8)); run -= r; }
                }
                while (run) { rle[nr++] = (uint16_t)v; run--; }
            }
            for (uint32_t k = 0; k < nr; k++) hc[rle[k] & 0xff]++;
            // code-length code: insertion sort of its used symbols (at least two), lengths limited to 7
            uint32_t n = 0;
            for (uint32_t s = 0; s < 19; s++) { c_len[s] = 0; if (hc[s]) { sw[n] = hc[s]; ssym[n] = (uint16_t)s; n++; } }
            for (uint32_t s = 0; n < 2; s++) if (!hc[s]) { sw[n] = 1; ssym[n] = (uint16_t)s; n++; }
            for (uint32_t i = 1; i < n; i++) {
                const uint32_t v = sw[i]; const uint16_t y = ssym[i]; int j = (int)i - 1;
                while (j >= 0 && (sw[j] > v || (sw[j] == v && ssym[j] > y))) { sw[j + 1] = sw[j]; ssym[j + 1] = ssym[j]; j--; }
                sw[j + 1] = v; ssym[j + 1] = y;
            }
            df_huff_lengths(sw, ssym, (int)n, 7, c_len);
            const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
            uint32_t hclen = 19; while (hclen > 4 && !c_len[order[hclen - 1]]) hclen--;
            uint64_t hdr = 14 + 3 * hclen;
            for (uint32_t s = 0; s < 19; s++) hdr += (uint64_t)hc[s] * (c_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0));
            uint64_t dyn = 3 + hdr + ext_total, fix = 3 + ext_total;
            for (uint32_t s = 0; s < 286; s++) { dyn += (uint64_t)hl[s] * ll_len[s]; fix += (uint64_t)hl[s] * df_fixed_len(s); }
            for (uint32_t s = 0; s < 30; s++) { dyn += (uint64_t)hd[s] * d_len[s]; fix += (uint64_t)hd[s] * 5; }
            const uint64_t by_dyn = (dyn + 3 + 7) / 8 + 4, by_fix = (fix + 3 + 7) / 8 + 4, by_sto = (uint64_t)L + DF_CHUNK_OVERHEAD;
            uint32_t bt = 2; uint64_t by = by_dyn;
            if (by_fix <= by) { bt = 1; by = by_fix; }
            if (by_sto <= by) { bt = 0; by = by_sto; }
            s_btype = bt; s_nbytes = (uint32_t)by; s_hdr_bits = bt == 2 ? (uint32_t)hdr : 0;
            s_nrle = nr; s_hlit = hlit; s_hdist = hdist; s_hclen = hclen;
            if (bt == 1) { for (uint32_t s = 0; s < 288; s++) ll_len[s] = (uint8_t)df_fixed_len(s); for (uint32_t s = 0; s < 30; s++) d_len[s] = 5; }
            if (bt != 0) { df_codes(ll_len, 288, ll_code); df_codes(d_len, 30, d_code); df_codes(c_len, 19, c_code); }
        }
        __syncthreads();
        const uint32_t btype = s_btype, nbytes = s_nbytes;
        for (uint32_t i = tid; i < (nbytes + 11) / 4; i += DF_THREADS) img[i] = 0;
        __syncthreads();

        // ---- P6: emit into the shared-memory image
        if (btype == 0) {       // stored: [BFINAL 0, BTYPE 00 | pad][LEN][NLEN][bytes], then the sync-flush marker
            uint8_t* ib = (uint8_t*)img;
            if (tid == 0) { ib[1] = (uint8_t)L; ib[2] = (uint8_t)(L >> 8); ib[3] = (uint8_t)~L; ib[4] = (uint8_t)(~L >> 8); ib[L + 8] = 0xff; ib[L + 9] = 0xff; }
            for (uint32_t i = tid; i < L; i += DF_THREADS) ib[5 + i] = db[i];
        } else {
            if (tid == 0) {
                df_put(img, 0, (uint32_t)btype << 1, 3);
                if (btype == 2) {
                    uint32_t at = 3;
                    df_put(img, at, s_hlit - 257, 5); df_put(img, at + 5, s_hdist - 1, 5); df_put(img, at + 10, s_hclen - 4, 4); at += 14;
                    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
                    for (uint32_t k = 0; k < s_hclen; k++) { df_put(img, at, c_len[order[k]], 3); at += 3; }
                    for (uint32_t k = 0; k < s_nrle; k++) {
                        const uint32_t s = rle[k] & 0xff, x = rle[k] >> 8;
                        df_put(img, at, c_code[s], c_len[s]); at += c_len[s];
                        const uint32_t xb = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
                        df_put(img, at, x, xb); at += xb;
                    }
                }
            }
            // bits of this thread's tokens, their offset by a block scan
            uint32_t my = 0;
            for (uint32_t bits = mine; bits;) {
                const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
                const uint32_t p = tid * DF_PPT + k, l = lenb[p];
                if (!l) { my += ll_len[db[p]]; continue; }
                uint32_t s, eb, ev, ds, deb, dev;
                df_len_sym(l + 3, s, eb, ev); df_dist_sym(dist[p], ds, deb, dev);
                my += ll_len[s] + eb + d_len[ds] + deb;
            }
            uint32_t tok_total; uint32_t at = 3 + s_hdr_bits + block_excl_scan(my, &tok_total, red);
            for (uint32_t bits = mine; bits;) {
                const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
                const uint32_t p = tid * DF_PPT + k, l = lenb[p];
                if (!l) { const uint32_t c = db[p]; df_put(img, at, ll_code[c], ll_len[c]); at += ll_len[c]; continue; }
                uint32_t s, eb, ev, ds, deb, dev;
                df_len_sym(l + 3, s, eb, ev); df_dist_sym(dist[p], ds, deb, dev);
                df_put(img, at, ll_code[s] | (ev << ll_len[s]), ll_len[s] + eb); at += ll_len[s] + eb;
                df_put(img, at, d_code[ds] | (dev << d_len[ds]), d_len[ds] + deb); at += d_len[ds] + deb;
            }
            if (tid == 0) {     // end of block, then the marker: 3 zero bits, pad, 00 00 ff ff
                const uint32_t e = 3 + s_hdr_bits + tok_total;
                df_put(img, e, ll_code[256], ll_len[256]);
                uint8_t* ib = (uint8_t*)img; ib[nbytes - 2] = 0xff; ib[nbytes - 1] = 0xff;
            }
        }
        if (tid == 0) *(volatile unsigned long long*)&a.pfx[f] = DF_FLAG_AGG | nbytes;      // the chunks behind can start summing
        __syncthreads();

        // ---- P7: look-back for the chunk's offset, then the image to its final place
        if (warp == 0) {
            const unsigned long long excl = df_lookback(a.pfx, a.st, f, lane);
            if (lane == 0) { *(volatile unsigned long long*)&a.pfx[f] = DF_FLAG_INCL | (excl + nbytes); s_off = excl; }
        }
        __syncthreads();
        uint8_t* G = a.out + (a.zlib ? sizeof(tfdf::ZLIB_HDR) : sizeof(tfdf::GZIP_HDR)) + s_off;
        const uint8_t* ib = (const uint8_t*)img;
        for (uint32_t i = tid; i < nbytes; i += DF_THREADS) G[i] = ib[i];
    }
}

// The container around the chunk bodies: header, the final empty fixed-Huffman block (03 00), the trailer with the chunk
// checksums combined in order (CRC-32 by GF(2) multiplication with x^(8 len), Adler-32 arithmetically). One CTA.
__global__ void __launch_bounds__(1024) k_deflate_finish(DeflateArgs a) {
    __shared__ uint32_t red[33];
    __shared__ unsigned long long red64[32];
    const uint32_t tid = threadIdx.x, n = a.nchunks;
    const uint64_t T = a.total;
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x, f0 = tid * per < n ? tid * per : n, f1 = f0 + per < n ? f0 + per : n;
    uint32_t sum;
    if (a.zlib) {
        uint64_t s1 = 0, s2 = 0;
        for (uint32_t f = f0; f < f1; f++) {
            const uint64_t end = (uint64_t)f * DF_CHUNK + DF_CHUNK < T ? (uint64_t)f * DF_CHUNK + DF_CHUNK : T;
            s1 += a.sums[2 * f]; s2 = (s2 + a.sums[2 * f + 1] + ((T - end) % tfdf::ADLER_MOD) * a.sums[2 * f]) % tfdf::ADLER_MOD;
        }
        s1 = df_block_sum64(s1 % tfdf::ADLER_MOD, red64) % tfdf::ADLER_MOD;
        s2 = df_block_sum64(s2, red64) % tfdf::ADLER_MOD;
        sum = (uint32_t)((((T % tfdf::ADLER_MOD) + s2) % tfdf::ADLER_MOD) << 16 | ((1 + s1) % tfdf::ADLER_MOD));
    } else {
        uint32_t acc = 0; uint64_t end = (uint64_t)f0 * DF_CHUNK;
        const uint32_t xc = tfdf::crc_xpow8(DF_CHUNK);
        for (uint32_t f = f0; f < f1; f++) {
            const uint64_t len = T - end < DF_CHUNK ? T - end : DF_CHUNK;
            acc = tfdf::crc_mulmod(len == DF_CHUNK ? xc : tfdf::crc_xpow8(len), acc) ^ a.sums[2 * f];
            end += len;
        }
        if (f1 > f0) acc = tfdf::crc_mulmod(tfdf::crc_xpow8(T - end), acc);
        sum = df_block_xor(acc, red);
    }
    if (tid == 0) {
        const uint32_t hdr = a.zlib ? sizeof(tfdf::ZLIB_HDR) : sizeof(tfdf::GZIP_HDR);
        const uint64_t body = n ? (a.pfx[n - 1] & DF_VAL_MASK) : 0;
        uint8_t* o = a.out;
        if (a.zlib) { o[0] = 0x78; o[1] = 0x9c; }         // tfdf::ZLIB_HDR / GZIP_HDR
        else { o[0] = 0x1f; o[1] = 0x8b; o[2] = 0x08; for (int i = 3; i < 9; i++) o[i] = 0; o[9] = 0xff; }
        o += hdr + body;
        *o++ = 0x03; *o++ = 0x00;
        if (a.zlib) { for (int i = 0; i < 4; i++) *o++ = (uint8_t)(sum >> (24 - 8 * i)); }
        else { for (int i = 0; i < 4; i++) *o++ = (uint8_t)(sum >> (8 * i)); for (int i = 0; i < 4; i++) *o++ = (uint8_t)(T >> (8 * i)); }
        a.st->wire_total = hdr + body + 2 + (a.zlib ? tfdf::ZLIB_TRAILER : tfdf::GZIP_TRAILER);
    }
}
#endif  // TF_KERNELS_DEFLATE

}  // namespace tfk
