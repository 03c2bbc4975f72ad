// zstd (RFC 8878) of the ClickHouse JSONEachRow text, the HTTP uploader's Content-Encoding: zstd (TF_WIRE_F_ZSTD).
//
// One frame: a fixed 14-byte header (no dictionary, no checksum, 8-byte Frame_Content_Size, a 32 KiB window), then one block per
// ZS_CHUNK-byte chunk of the text in text order. A chunk's matches may reach up to ZS_HIST bytes back into the text before it, so
// offsets stay below 32 KiB; a block never depends on an earlier block's encoder state (no repeat offsets, no treeless literals, no
// Repeat_Mode tables), so every chunk is encoded alone. One CTA encodes one chunk in shared memory at a time (persistent CTAs take
// chunks by ticket):
//   P1  stage the preceding ZS_HIST bytes and the chunk
//   P2  match finding in rounds of ZS_THREADS positions over history and chunk (hash table of an earlier round or this one, and the
//       same 4 bytes 1, 2 or 4 back); only the chunk's positions keep a match (4..ZS_MAX_MATCH bytes, inside the chunk)
//   P3  greedy parse by pointer doubling, as in k_deflate_chunks
//   P4  sequences (literal length, match length, offset) and the literals, placed by block scans; their code histograms
//   P5  literals: Huffman code lengths limited to 11 bits, the tree as direct 4-bit or FSE-compressed weights, 1 or 4 streams; sequence
//       tables: Predefined, RLE or FSE_Compressed per table; then Raw / RLE / Compressed block, every choice by exact byte count
//   P6  Huffman streams packed by every thread from prefix sums of code lengths (streams are read backward: the last literal first);
//       the sequence bitstream is one FSE state chain per block, written by one thread
//   P7  the block's size is published for the chunks behind it and the block is written at its final offset (decoupled look-back)
// k_zstd_finish writes the frame header, sets Last_Block on the last block and puts the frame's length into DState.
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "kernels_deflate.cuh"

namespace tfk {

#define ZS_CHUNK 16384          /* text bytes per block: chunk positions fit u16, history + chunk positions fit u16 (+1) */
#define ZS_HIST 16384           /* text bytes before the chunk that its matches may reach */
#define ZS_THREADS 512
#define ZS_PPT (ZS_CHUNK / ZS_THREADS)     /* 32 positions per thread: one word of the path bitmap */
#define ZS_HASH_BITS 12
#define ZS_MAX_MATCH 4096
#define ZS_HDR 14               /* magic, descriptor, window descriptor, 8-byte content size */
#define ZS_FHD 0xC0             /* Frame_Content_Size_flag 3 (8 bytes), no single segment, no checksum, no dictionary */
#define ZS_WD 0x28              /* Exponent 5, Mantissa 0: Window_Size 32 KiB, Block_Maximum_Size 32 KiB */
#define ZS_BLOCK_MAX 32768
#define ZS_HUF_MAXBITS 11

struct ZstdArgs {
    const uint8_t* text; uint64_t total;     // the row text and its byte count (the host read it before sizing the arena)
    uint8_t* out;                            // header | blocks
    unsigned long long* pfx;                 // [nchunks] decoupled look-back cells, zeroed before the launch
    uint32_t* ticket;                        // work counter, zeroed before the launch
    uint32_t nchunks;
    DState* st;                              // wire_total
};
__global__ void k_zstd_chunks(ZstdArgs a);
__global__ void k_zstd_finish(ZstdArgs a);

// shared-memory carve-up (byte offsets)
struct ZsSmem { uint32_t data, dist, lenm, work, path, hist, huf, fse, desc, total; };
__host__ __device__ inline ZsSmem zs_smem() {
    ZsSmem s; uint32_t o = 0;
    s.data = o; o += 16 + ZS_HIST + ZS_CHUNK + 32;         // zero guard words in front of and behind history + chunk
    s.dist = o; o += 2 * ZS_CHUNK;                         // P2-P4 u16 match offset per chunk position; P6 the block image
    s.lenm = o; o += 2 * ZS_CHUNK;                         // P2-P4 u16 match length per chunk position (0 = literal); P4+ the literals
    s.work = o; o += 2 * ZS_CHUNK + 64;                    // P2 hash table; P3 successors; P4+ sequences (3 x u16 x ZS_CHUNK / 4)
    s.path = o; o += (ZS_CHUNK / 32 + 4) * 4;              // bitmap of the parse's token starts
    s.hist = o; o += (256 + 36 + 53 + 32) * 4 + 12;        // literal, LL, ML, OF code histograms
    s.huf = o; o += 256 + 256 * 2 + 256 * 4 + 256 * 2;     // code lengths, codes, sorted weights, sorted symbols
    s.fse = o; o += 7 * (512 * 2 + 64 * 8) + 3 * 64 * 2 + 3 * 512 + 64;   // 7 encoding tables, 3 normalised counts, 4 spread scratch
    s.desc = o; o += 4 * 160;                              // LL, OF, ML table descriptions, Huffman tree description
    s.total = o; return s;
}

// ---- FSE (RFC 8878 §4.1), encoder side: host and device (the tables are small and built by one thread)
struct ZsFse { uint16_t* state; int32_t* dnb; int32_t* dfs; uint32_t log; };   // state table, per-symbol deltaNbBits / deltaFindState

__host__ __device__ inline uint32_t zs_hb(uint32_t v) {     // index of the highest set bit, v > 0
#ifdef __CUDA_ARCH__
    return 31u - (uint32_t)__clz((int)v);
#else
    return 31u - (uint32_t)__builtin_clz(v);
#endif
}
// normalised counts of cnt[0..n) summing to 1 << log; every used symbol gets at least 1
__host__ __device__ inline void zs_normalize(const uint32_t* cnt, int n, uint32_t total, uint32_t log, int16_t* norm) {
    const int32_t ts = 1 << log; int32_t sum = 0; int big = 0;
    for (int s = 0; s < n; s++) {
        int32_t v = 0;
        if (cnt[s]) { v = (int32_t)(((uint64_t)cnt[s] * ts + total / 2) / total); if (v < 1) v = 1; }
        norm[s] = (int16_t)v; sum += v;
        if (cnt[s] > cnt[big]) big = s;
    }
    while (sum > ts) {      // take one from the largest count that can give one
        int m = -1;
        for (int s = 0; s < n; s++) if (norm[s] > 1 && (m < 0 || norm[s] > norm[m])) m = s;
        norm[m]--; sum--;
    }
    norm[big] = (int16_t)(norm[big] + (ts - sum));
}
// table description (§4.1.1) of norm[0..n) into out; returns its byte count
__host__ __device__ inline uint32_t zs_write_ncount(const int16_t* norm, int n, uint32_t log, uint8_t* out) {
    uint64_t acc = log - 5; uint32_t nb = 4, o = 0;
    int32_t remaining = (1 << log) + 1, threshold = 1 << log; uint32_t nbits = log + 1;
    int s = 0; bool prev0 = false;
    auto flush = [&]() { while (nb >= 8) { out[o++] = (uint8_t)acc; acc >>= 8; nb -= 8; } };
    while (s < n && remaining > 1) {
        if (prev0) {
            int start = s;
            while (s < n && !norm[s]) s++;
            while (s >= start + 3) { acc |= (uint64_t)3 << nb; nb += 2; start += 3; flush(); }
            acc |= (uint64_t)(s - start) << nb; nb += 2; flush();
        }
        int32_t c = norm[s++];
        const int32_t mx = (2 * threshold - 1) - remaining;
        remaining -= c < 0 ? -c : c;
        c++;
        if (c >= threshold) c += mx;
        acc |= (uint64_t)c << nb; nb += nbits; if (c < mx) nb--;
        flush();
        prev0 = c == 1;
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    if (nb) { out[o++] = (uint8_t)acc; }
    return o;
}
// encoding table of norm[0..n) (no "less than 1" symbols); spread: 1 << log bytes of scratch
__host__ __device__ inline void zs_build(const int16_t* norm, int n, uint32_t log, uint8_t* spread, ZsFse& t) {
    const uint32_t ts = 1u << log, step = (ts >> 1) + (ts >> 3) + 3, mask = ts - 1;
    uint32_t pos = 0;
    for (int s = 0; s < n; s++) for (int i = 0; i < norm[s]; i++) { spread[pos] = (uint8_t)s; pos = (pos + step) & mask; }
    uint32_t cum[64]; uint32_t c = 0;
    for (int s = 0; s < n; s++) { cum[s] = c; c += (uint32_t)norm[s]; }
    for (uint32_t u = 0; u < ts; u++) t.state[cum[spread[u]]++] = (uint16_t)(ts + u);
    int32_t tot = 0;
    for (int s = 0; s < n; s++) {
        const int32_t k = norm[s];
        if (k == 0) { t.dnb[s] = 0; t.dfs[s] = 0; }
        else if (k == 1) { t.dnb[s] = (int32_t)(log << 16) - (int32_t)ts; t.dfs[s] = tot - 1; tot += 1; }
        else { const uint32_t mbo = log - zs_hb((uint32_t)k - 1); t.dnb[s] = (int32_t)(mbo << 16) - (k << mbo); t.dfs[s] = tot - k; tot += k; }
    }
    t.log = log;
}
__host__ __device__ inline uint32_t zs_init_state(const ZsFse& t, uint32_t s) {
    const uint32_t nbo = (uint32_t)((t.dnb[s] + (1 << 15)) >> 16);
    const uint32_t v = (nbo << 16) - (uint32_t)t.dnb[s];
    return t.state[(v >> nbo) + t.dfs[s]];
}
// one encode step: the bits to write (count, value) and the next state
__host__ __device__ inline uint32_t zs_step(const ZsFse& t, uint32_t& state, uint32_t s, uint32_t& val) {
    const uint32_t nbo = (state + (uint32_t)t.dnb[s]) >> 16;
    val = state & ((1u << nbo) - 1);
    state = t.state[(state >> nbo) + t.dfs[s]];
    return nbo;
}

// ---- sequence codes (§3.1.1.3.2.1)
__host__ __device__ inline uint32_t zs_ll_code(uint32_t ll) {
    if (ll < 16) return ll;
    if (ll < 24) return 16 + ((ll - 16) >> 1);
    if (ll < 64) return ll < 32 ? (ll < 28 ? 20 : 21) : (ll < 48 ? (ll < 40 ? 22 : 23) : 24);
    return 19 + zs_hb(ll);      // 64 -> 25, 128 -> 26, ...
}
__host__ __device__ inline uint32_t zs_ml_code(uint32_t ml) {
    const uint32_t m = ml - 3;
    if (m < 32) return m;
    if (m < 40) return 32 + ((m - 32) >> 1);
    if (m < 64) return m < 44 ? 36 : m < 48 ? 37 : m < 56 ? 38 : 39;
    if (m < 128) return m < 80 ? 40 : m < 96 ? 41 : 42;
    return 36 + zs_hb(m);       // 128 -> 43, 256 -> 44, ...
}
struct ZsCodeInfo { uint32_t base, bits; };
__host__ __device__ inline ZsCodeInfo zs_ll_info(uint32_t c) {
    const uint32_t B[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
    const uint8_t N[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
    return ZsCodeInfo{B[c], N[c]};
}
__host__ __device__ inline ZsCodeInfo zs_ml_info(uint32_t c) {
    if (c < 32) return ZsCodeInfo{c + 3, 0};
    const uint32_t B[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
    const uint8_t N[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
    return ZsCodeInfo{B[c - 32], N[c - 32]};
}
// predefined distributions (§3.1.1.3.2.2); every entry here is >= 1 except the "less than 1" cells, which only the decoder needs
// to place: this encoder uses a predefined table only when the block's codes avoid the symbols that have them
__host__ __device__ inline int16_t zs_predef(int t, int s) {
    const int8_t LL[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
    const int8_t OF[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
    const int8_t ML[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
    return t == 0 ? LL[s] : t == 1 ? OF[s] : ML[s];
}

#ifdef TF_KERNELS_ZSTD
// Predefined table t (0 LL, 1 OF, 2 ML) as an encoding table. Its "less than 1" symbols occupy the last cells of the decoding
// table, so the spread and the state table follow the format's rule for them: they are usable here, with one state each.
__device__ void zs_build_predef(int t, uint8_t* spread, ZsFse& f) {
    const int n = t == 0 ? 36 : t == 1 ? 29 : 53; const uint32_t log = t == 1 ? 5 : 6, ts = 1u << log;
    uint32_t high = ts - 1;
    for (int s = 0; s < n; s++) if (zs_predef(t, s) == -1) spread[high--] = (uint8_t)s;
    const uint32_t step = (ts >> 1) + (ts >> 3) + 3, mask = ts - 1; uint32_t pos = 0;
    for (int s = 0; s < n; s++) for (int i = 0; i < zs_predef(t, s); i++) { spread[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    uint32_t cum[64]; uint32_t c = 0;
    for (int s = 0; s < n; s++) { cum[s] = c; const int16_t k = zs_predef(t, s); c += k < 0 ? 1u : (uint32_t)k; }
    for (uint32_t u = 0; u < ts; u++) f.state[cum[spread[u]]++] = (uint16_t)(ts + u);
    int32_t tot = 0;
    for (int s = 0; s < n; s++) {
        const int32_t k = zs_predef(t, s);
        if (k == -1 || k == 1) { f.dnb[s] = (int32_t)(log << 16) - (int32_t)ts; f.dfs[s] = tot - 1; tot += 1; }
        else { const uint32_t mbo = log - zs_hb((uint32_t)k - 1); f.dnb[s] = (int32_t)(mbo << 16) - (k << mbo); f.dfs[s] = tot - k; tot += k; }
    }
    f.log = log;
}

// Exact FSE bits of the state chain of `n` codes read by code(i) (written from the last to the first), flush included.
template <typename F> __device__ uint32_t zs_chain_bits(const ZsFse& t, uint32_t n, F code) {
    if (!n) return 0;
    uint32_t st = zs_init_state(t, code(n - 1)), bits = t.log, v;
    for (int32_t i = (int32_t)n - 2; i >= 0; i--) bits += zs_step(t, st, code((uint32_t)i), v);
    return bits;
}

__global__ void __launch_bounds__(ZS_THREADS, 1) k_zstd_chunks(ZstdArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const ZsSmem S = zs_smem();
    uint8_t* db = smem + S.data + 16;                        // history + chunk; 16 zero bytes in front, 32 behind
    const uint32_t* dw = (const uint32_t*)db;
    uint16_t* dist = (uint16_t*)(smem + S.dist);
    uint16_t* lenm = (uint16_t*)(smem + S.lenm);
    uint32_t* img = (uint32_t*)(smem + S.dist);               // P6: the block
    uint8_t* lit = smem + S.lenm;                             // P4+: the literals
    uint16_t* J = (uint16_t*)(smem + S.work);
    uint16_t* sq_ll = (uint16_t*)(smem + S.work); uint16_t* sq_ml = sq_ll + ZS_CHUNK / 4; uint16_t* sq_of = sq_ml + ZS_CHUNK / 4;
    uint32_t* path = (uint32_t*)(smem + S.path);
    uint32_t* hlit = (uint32_t*)(smem + S.hist); uint32_t* hll = hlit + 256; uint32_t* hml = hll + 36; uint32_t* hof = hml + 53;
    uint8_t* hlen = smem + S.huf; uint16_t* hcode = (uint16_t*)(hlen + 256); uint32_t* sw = (uint32_t*)(hcode + 256); uint16_t* ssym = (uint16_t*)(sw + 256);
    uint8_t* F = smem + S.fse;
    auto fse_tab = [&](int k) { uint8_t* p = F + k * (512 * 2 + 64 * 8); return ZsFse{(uint16_t*)p, (int32_t*)(p + 1024), (int32_t*)(p + 1024 + 256), 0}; };
    int16_t* norms = (int16_t*)(F + 7 * (512 * 2 + 64 * 8));          // [3][64]
    uint8_t* spread = (uint8_t*)(norms + 3 * 64);                     // [3][512] sequence tables, [64] Huffman weights
    uint8_t* desc = smem + S.desc;                                    // [4][160]: LL, OF, ML, Huffman tree
    __shared__ ZsFse s_pre[3], s_tab[3];
    __shared__ uint32_t s_f, s_mode[3], s_dlen[3], s_bits[3], s_lmode, s_lsize, s_lhdr, s_hdesc, s_btype, s_nbytes;
    __shared__ uint32_t s_sbits[4], s_spos[5];
    __shared__ uint32_t red[33];
    __shared__ unsigned long long s_off;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int t = 0; t < 3; t++) {       // the predefined tables, once per CTA (tables 0..2); 3..5 are per block, 6 the Huffman weights'
        if (tid == (uint32_t)t) { ZsFse f = fse_tab(t); zs_build_predef(t, spread + 512 * t, f); s_pre[t] = f; }
    }
    for (;;) {
        __syncthreads();
        if (tid == 0) s_f = atomicAdd(a.ticket, 1u);
        __syncthreads();
        const uint32_t f = s_f;
        if (f >= a.nchunks) break;
        const uint64_t pos0 = (uint64_t)f * ZS_CHUNK;
        const uint32_t L = (uint32_t)((a.total - pos0 < ZS_CHUNK) ? a.total - pos0 : ZS_CHUNK);
        const uint32_t H = pos0 < ZS_HIST ? (uint32_t)pos0 : ZS_HIST, W = H + L;

        // ---- P1: stage history + chunk, clear
        {
            const int4* g = (const int4*)(a.text + pos0 - H);
            const uint32_t nv = (W + 15) >> 4;
            int4* d4 = (int4*)db;
            for (uint32_t i = tid; i < (ZS_HIST + ZS_CHUNK) / 16 + 2; i += ZS_THREADS) d4[i] = i < nv ? __ldg(g + i) : make_int4(0, 0, 0, 0);
            if (tid < 4) ((uint32_t*)(smem + S.data))[tid] = 0;
            int4* t4 = (int4*)J;
            for (uint32_t i = tid; i < (2u << ZS_HASH_BITS) / 16; i += ZS_THREADS) t4[i] = make_int4(0, 0, 0, 0);
            for (uint32_t i = tid; i < ZS_CHUNK / 32 + 4; i += ZS_THREADS) path[i] = 0;
            for (uint32_t i = tid; i < 256 + 36 + 53 + 32; i += ZS_THREADS) hlit[i] = 0;
        }
        __syncthreads();
        if (tid < 16 && W + tid < ((W + 15) & ~15u)) db[W + tid] = 0;     // the bytes the last 16-byte load brought in past the chunk
        __syncthreads();

        // ---- P2: match finding over history and chunk; matches kept for the chunk's positions
        const uint32_t nrounds = (W + ZS_THREADS - 1) / ZS_THREADS;
        for (uint32_t r = 0; r < nrounds; r++) {
            const uint32_t p = r * ZS_THREADS + tid;
            const bool valid = p + 4 <= W;
            const uint32_t w = valid ? df_ld32(dw, p) : 0, h = (w * 2654435761u) >> (32 - ZS_HASH_BITS);
            const uint32_t t1 = valid ? J[h] : 0;
            __syncthreads();
            if (valid) J[h] = (uint16_t)(p + 1);
            __syncthreads();
            const uint32_t t2 = valid ? J[h] : 0;
            uint32_t best = 0, bd = 0;
            if (valid && p >= H) {
                const uint32_t maxl = W - p < ZS_MAX_MATCH ? W - p : ZS_MAX_MATCH;
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
            if (p >= H && p < W) { lenm[p - H] = (uint16_t)(best >= 4 ? best : 0); dist[p - H] = (uint16_t)bd; }
        }
        __syncthreads();

        // ---- P3: greedy parse by pointer doubling over the chunk's positions
        for (uint32_t k = 0; k < ZS_PPT; k++) { const uint32_t p = tid * ZS_PPT + k; if (p < L) J[p] = (uint16_t)(p + (lenm[p] ? lenm[p] : 1u)); }
        if (tid == 0) { J[L] = (uint16_t)L; path[0] = 1; }
        __syncthreads();
        for (;;) {
            uint32_t bits = path[tid];
            while (bits) {
                const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
                const uint32_t p = tid * ZS_PPT + k;
                if (p < L) { const uint32_t q = J[p]; if (q < L) atomicOr(&path[q >> 5], 1u << (q & 31)); }
            }
            __syncthreads();
            uint32_t nx[ZS_PPT / 2];
#pragma unroll
            for (uint32_t k = 0; k < ZS_PPT; k += 2) {
                const uint32_t p = tid * ZS_PPT + k;
                const uint32_t lo = p < L ? J[J[p]] : 0, hi = p + 1 < L ? J[J[p + 1]] : 0;
                nx[k / 2] = lo | (hi << 16);
            }
            __syncthreads();
#pragma unroll
            for (uint32_t k = 0; k < ZS_PPT; k += 2) {
                const uint32_t p = tid * ZS_PPT + k;
                if (p < L) J[p] = (uint16_t)nx[k / 2];
                if (p + 1 < L) J[p + 1] = (uint16_t)(nx[k / 2] >> 16);
            }
            __syncthreads();
            if (J[0] == L) break;
            __syncthreads();
        }
        const uint32_t mine = path[tid] & (tid * ZS_PPT + ZS_PPT <= L ? 0xffffffffu : (tid * ZS_PPT < L ? (1u << (L - tid * ZS_PPT)) - 1 : 0u));

        // ---- P4: sequences and literals. A match's literal length reaches back to the end of the match before it (a max-scan of
        // match ends: positions only grow), its index and the literals' are block scans of the counts.
        uint32_t nm = 0, nl = 0, last_end = 0;
        for (uint32_t bits = mine; bits;) {
            const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
            const uint32_t p = tid * ZS_PPT + k;
            if (lenm[p]) { nm++; last_end = p + lenm[p]; } else nl++;
        }
        uint32_t nseq, nlit;
        const uint32_t m0 = block_excl_scan(nm, &nseq, red);
        const uint32_t l0 = block_excl_scan(nl, &nlit, red);
        uint32_t prev_end;          // the largest match end of the threads before this one
        {
            uint32_t v = last_end;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, v, d); if (lane >= (uint32_t)d && u > v) v = u; }
            if (lane == 31) red[warp] = v;
            __syncthreads();
            uint32_t before = 0;
            for (uint32_t w2 = 0; w2 < warp; w2++) before = red[w2] > before ? red[w2] : before;
            const uint32_t ex = __shfl_up_sync(0xffffffffu, v, 1);
            prev_end = lane ? (ex > before ? ex : before) : before;
            __syncthreads();
        }
        // sequence records (into the successor area, free now) and the code histograms; the literals wait until lenm is read
        uint8_t lits_mine[ZS_PPT]; uint32_t nlm = 0;
        {
            uint32_t si = m0, pe = prev_end;
            for (uint32_t bits = mine; bits;) {
                const uint32_t k = (uint32_t)__ffs((int)bits) - 1; bits &= bits - 1;
                const uint32_t p = tid * ZS_PPT + k, ml = lenm[p];
                if (!ml) { lits_mine[nlm++] = db[H + p]; continue; }
                const uint32_t ll = p - pe, of = dist[p];
                sq_ll[si] = (uint16_t)ll; sq_ml[si] = (uint16_t)ml; sq_of[si] = (uint16_t)of; si++;
                atomicAdd(&hll[zs_ll_code(ll)], 1u); atomicAdd(&hml[zs_ml_code(ml)], 1u); atomicAdd(&hof[zs_hb(of + 3)], 1u);
                pe = p + ml;
            }
        }
        __syncthreads();
        for (uint32_t i = 0; i < nlm; i++) { lit[l0 + i] = lits_mine[i]; atomicAdd(&hlit[lits_mine[i]], 1u); }
        __syncthreads();

        // ---- P5a: Huffman code lengths (rank sort of the used byte values by (count, value); lengths limited to 11 bits)
        const int nsym = __syncthreads_count(tid < 256 && hlit[tid] > 0);
        if (tid < 256) {
            hlen[tid] = 0;
            const uint32_t v = hlit[tid];
            if (v) {
                uint32_t rank = 0;
                for (uint32_t j = 0; j < 256; j++) { const uint32_t u = hlit[j]; rank += (u && (u < v || (u == v && j < tid))) ? 1u : 0u; }
                sw[rank] = v; ssym[rank] = (uint16_t)tid;
            }
        }
        __syncthreads();
        const bool try_huf = nsym >= 2 && nlit >= 32;
        if (tid == 0 && try_huf) df_huff_lengths(sw, ssym, nsym, ZS_HUF_MAXBITS, hlen);
        __syncthreads();

        // ---- P5b (three threads at once): sequence tables; the Huffman tree description and codes
        if (tid < 3 && nseq) {
            const int t = (int)tid, n = t == 0 ? 36 : t == 1 ? 32 : 53;
            const uint32_t* h = t == 0 ? hll : t == 1 ? hof : hml;
            int used = 0, one = 0, top = 0;
            for (int s = 0; s < n; s++) if (h[s]) { used++; one = s; top = s; }
            auto code = [&](uint32_t i) -> uint32_t { return t == 0 ? zs_ll_code(sq_ll[i]) : t == 1 ? zs_hb(sq_of[i] + 3u) : zs_ml_code(sq_ml[i]); };
            uint32_t mode = 0, dlen = 0, bits = 0;
            if (used == 1) { mode = 1; dlen = 1; desc[160 * t] = (uint8_t)one; bits = 0; }
            else {
                const uint32_t maxlog = t == 1 ? 8 : 9;
                uint32_t log = nseq > 1 ? zs_hb(nseq - 1) + 1 : 5;
                const uint32_t need = zs_hb((uint32_t)used) + 2;
                if (log < need) log = need;
                if (log < 5) log = 5;
                if (log > maxlog) log = maxlog;
                int16_t* nm16 = norms + 64 * t;
                zs_normalize(h, top + 1, nseq, log, nm16);
                ZsFse ft = fse_tab(3 + t);
                zs_build(nm16, top + 1, log, spread + 512 * t, ft);
                s_tab[t] = ft;
                const uint32_t fb = zs_chain_bits(ft, nseq, code);
                const uint32_t fd = zs_write_ncount(nm16, top + 1, log, desc + 160 * t);
                bool pre_ok = t != 1 || top <= 28;
                uint32_t pb = pre_ok ? zs_chain_bits(s_pre[t], nseq, code) : 0xffffffffu;
                if (pre_ok && (uint64_t)pb <= (uint64_t)fb + 8ull * fd) { mode = 0; dlen = 0; bits = pb; }
                else { mode = 2; dlen = fd; bits = fb; }
            }
            s_mode[t] = mode; s_dlen[t] = dlen; s_bits[t] = bits;
        }
        if (tid == 32 && try_huf) {
            // codes: by weight (longest code first), then by value; weight = maxbits + 1 - length
            uint32_t mb = 0; int last = 0;
            for (int s = 0; s < 256; s++) if (hlen[s]) { mb = hlen[s] > mb ? hlen[s] : mb; last = s; }
            uint32_t start[ZS_HUF_MAXBITS + 2], cnt[ZS_HUF_MAXBITS + 2];
            for (uint32_t w2 = 0; w2 <= mb + 1; w2++) cnt[w2] = 0;
            for (int s = 0; s < 256; s++) if (hlen[s]) cnt[mb + 1 - hlen[s]]++;
            uint32_t acc = 0;
            for (uint32_t w2 = 1; w2 <= mb; w2++) { start[w2] = acc; acc += cnt[w2] << (w2 - 1); }
            for (int s = 0; s < 256; s++) if (hlen[s]) { const uint32_t w2 = mb + 1 - hlen[s]; hcode[s] = (uint16_t)(start[w2] >> (w2 - 1)); start[w2] += 1u << (w2 - 1); }
            // tree description: the weights of symbols 0 .. last - 1 (the last one's is implied), direct or FSE-compressed
            uint8_t* dd = desc + 480;
            const uint32_t nw = (uint32_t)last;
            auto wt = [&](uint32_t i) -> uint32_t { return hlen[i] ? mb + 1 - hlen[i] : 0u; };
            uint32_t best = 0xffffffffu;
            uint32_t wc[ZS_HUF_MAXBITS + 1]; int wused = 0, wtop = 0;
            for (uint32_t k = 0; k <= ZS_HUF_MAXBITS; k++) wc[k] = 0;
            for (uint32_t i = 0; i < nw; i++) wc[wt(i)]++;
            for (uint32_t k = 0; k <= mb; k++) if (wc[k]) { wused++; wtop = (int)k; }
            if (nw >= 2 && wused >= 2) {
                // FSE-compressed weights: accuracy log 6, two interleaved states
                int16_t wn[16]; zs_normalize(wc, wtop + 1, nw, 6, wn);
                ZsFse ft = fse_tab(6);
                zs_build(wn, wtop + 1, 6, spread + 512 * 3, ft);
                uint32_t o = 1 + zs_write_ncount(wn, wtop + 1, 6, dd + 1);
                uint64_t acc2 = 0; uint32_t nb = 0; uint32_t st1 = 0, st2 = 0; bool u1 = false, u2 = false;
                bool fit = true;
                auto put = [&](uint32_t v, uint32_t n) {
                    acc2 |= (uint64_t)v << nb; nb += n;
                    while (nb >= 8) { if (o < 159) dd[o] = (uint8_t)acc2; else fit = false; o++; acc2 >>= 8; nb -= 8; }
                };
                for (int32_t i = (int32_t)nw - 1; i >= 0; i--) {
                    uint32_t& st = (i & 1) ? st2 : st1; bool& u = (i & 1) ? u2 : u1;
                    if (!u) { st = zs_init_state(ft, wt((uint32_t)i)); u = true; }
                    else { uint32_t v; const uint32_t n = zs_step(ft, st, wt((uint32_t)i), v); put(v, n); }
                }
                put(st2 & 63u, 6); put(st1 & 63u, 6); put(1, 1);
                if (nb) put(0, 8 - nb);
                if (fit && o - 1 < 128) { best = o; dd[0] = (uint8_t)(o - 1); }
            }
            if (nw <= 128 && 1 + (nw + 1) / 2 < best) {
                best = 1 + (nw + 1) / 2; dd[0] = (uint8_t)(127 + nw);
                for (uint32_t i = 0; i < nw; i += 2) dd[1 + i / 2] = (uint8_t)((wt(i) << 4) | (i + 1 < nw ? wt(i + 1) : 0u));
            }
            s_hdesc = best;
        }
        __syncthreads();

        // ---- P5c: Huffman stream sizes from a prefix sum of code lengths, then every choice by exact size
        const bool huf = try_huf && s_hdesc != 0xffffffffu;
        const uint32_t nstreams = nlit > 1023 ? 4 : 1, seg = nstreams == 4 ? (nlit + 3) / 4 : nlit;
        const uint32_t i0 = tid * ZS_PPT, i1 = i0 + ZS_PPT < nlit ? i0 + ZS_PPT : nlit;
        uint32_t mybits = 0;
        if (huf) for (uint32_t i = i0; i < i1; i++) mybits += hlen[lit[i]];
        uint32_t tb; const uint32_t b0 = block_excl_scan(huf ? mybits : 0, &tb, red);      // bits of the literals before i0
        if (huf) {
            // the bits before each stream start: the thread holding that literal knows them
            uint32_t run = b0;
            for (uint32_t i = i0; i < i1; i++) {
                for (uint32_t k = 1; k < nstreams; k++) if (k * seg == i) s_spos[k] = run;
                run += hlen[lit[i]];
            }
            if (tid == 0) { s_spos[0] = 0; s_spos[nstreams] = tb; }
        }
        __syncthreads();
        if (tid == 0) {
            // literals section
            auto raw_hdr = [](uint32_t n) -> uint32_t { return n < 32 ? 1u : n < 4096 ? 2u : 3u; };
            bool all_same = nlit > 0;
            uint32_t lmode = 0, lsize = raw_hdr(nlit) + nlit, lhdr = raw_hdr(nlit);
            if (nlit > 1) for (int s = 0; s < 256; s++) if (hlit[s] && hlit[s] != nlit) { all_same = false; break; }
            if (nlit >= 1 && all_same && raw_hdr(nlit) + 1 < lsize) { lmode = 1; lsize = raw_hdr(nlit) + 1; lhdr = raw_hdr(nlit); }
            if (huf && !all_same) {
                uint32_t body = s_hdesc + (nstreams == 4 ? 6 : 0);
                for (uint32_t k = 0; k < nstreams; k++) { const uint32_t bb = s_spos[k + 1] - s_spos[k]; s_sbits[k] = bb; body += (bb + 1 + 7) / 8; }
                const uint32_t h = nstreams == 1 ? 3u : (nlit < 16384 && body < 16384 ? 4u : 5u);
                const bool ok = nstreams == 4 || body <= 1023;
                if (ok && h + body < lsize) { lmode = 2; lsize = h + body; lhdr = h; }
            }
            s_lmode = lmode; s_lsize = lsize; s_lhdr = lhdr;
            // sequences section
            uint32_t seq = nseq < 128 ? 1 : nseq < 0x7F00 ? 2 : 3;
            uint64_t bits = 0;
            if (nseq) {
                seq += 1 + s_dlen[0] + s_dlen[1] + s_dlen[2];
                bits = (uint64_t)s_bits[0] + s_bits[1] + s_bits[2];
                for (uint32_t i = 0; i < nseq; i++)
                    bits += zs_ll_info(zs_ll_code(sq_ll[i])).bits + zs_ml_info(zs_ml_code(sq_ml[i])).bits + zs_hb(sq_of[i] + 3u);
                seq += (uint32_t)((bits + 1 + 7) / 8);
            }
            const uint32_t comp = 3 + lsize + seq;
            bool run = L > 0;
            for (uint32_t i = 1; i < L && run; i++) run = db[H + i] == db[H];
            uint32_t bt = 0, nb = 3 + L;
            if (run) { bt = 1; nb = 4; }
            else if (comp < nb && comp - 3 <= ZS_BLOCK_MAX) { bt = 2; nb = comp; }
            s_btype = bt; s_nbytes = nb;
        }
        __syncthreads();
        const uint32_t btype = s_btype, nbytes = s_nbytes;
        for (uint32_t i = tid; i < (nbytes + 11) / 4; i += ZS_THREADS) img[i] = 0;
        __syncthreads();

        // ---- P6: the block image
        uint8_t* ib = (uint8_t*)img;
        const uint32_t bsz = btype == 1 ? L : nbytes - 3;
        if (tid == 0) { const uint32_t bh = (btype << 1) | (bsz << 3); ib[0] = (uint8_t)bh; ib[1] = (uint8_t)(bh >> 8); ib[2] = (uint8_t)(bh >> 16); }
        if (btype == 0) { for (uint32_t i = tid; i < L; i += ZS_THREADS) ib[3 + i] = db[H + i]; }
        else if (btype == 1) { if (tid == 0) ib[3] = db[H]; }
        else {
            const uint32_t lmode = s_lmode, lhdr = s_lhdr, lsize = s_lsize;
            uint8_t* lp = ib + 3;
            if (lmode != 2) {
                if (tid == 0) {
                    const uint32_t v = lhdr == 1 ? (lmode | (nlit << 3)) : lhdr == 2 ? (lmode | (1u << 2) | (nlit << 4)) : (lmode | (3u << 2) | (nlit << 4));
                    for (uint32_t k = 0; k < lhdr; k++) lp[k] = (uint8_t)(v >> (8 * k));
                    if (lmode == 1) lp[lhdr] = lit[0];
                }
                if (lmode == 0) for (uint32_t i = tid; i < nlit; i += ZS_THREADS) lp[lhdr + i] = lit[i];
            } else {
                const uint32_t body = lsize - lhdr, hd = s_hdesc;
                const uint32_t jump = nstreams == 4 ? 6u : 0u;
                // stream byte offsets inside the literals section
                uint32_t sbyte[5]; sbyte[0] = lhdr + hd + jump;
                for (uint32_t k = 0; k < nstreams; k++) sbyte[k + 1] = sbyte[k] + (s_sbits[k] + 8) / 8;
                if (tid == 0) {
                    const uint32_t sf = nstreams == 1 ? 0u : lhdr == 4 ? 2u : 3u, nbts = nstreams == 1 ? 10u : lhdr == 4 ? 14u : 18u;
                    const uint64_t v = 2ull | ((uint64_t)sf << 2) | ((uint64_t)nlit << 4) | ((uint64_t)body << (4 + nbts));
                    for (uint32_t k = 0; k < lhdr; k++) lp[k] = (uint8_t)(v >> (8 * k));
                    for (uint32_t k = 0; k < hd; k++) lp[lhdr + k] = desc[480 + k];
                    if (nstreams == 4) for (uint32_t k = 0; k < 3; k++) { const uint32_t z = sbyte[k + 1] - sbyte[k]; lp[lhdr + hd + 2 * k] = (uint8_t)z; lp[lhdr + hd + 2 * k + 1] = (uint8_t)(z >> 8); }
                    for (uint32_t k = 0; k < nstreams; k++) {     // the end marker above each stream's last code
                        const uint32_t at = 8 * (3 + sbyte[k]) + s_sbits[k];
                        ib[at >> 3] |= (uint8_t)(1u << (at & 7));
                    }
                }
                __syncthreads();
                // literal i of stream k sits above the codes of the literals after it in the stream
                uint32_t run = b0;
                for (uint32_t i = i0; i < i1; i++) {
                    const uint32_t c = lit[i], n = hlen[c];
                    run += n;
                    const uint32_t k = nstreams == 4 ? i / seg : 0;
                    const uint32_t at = 8 * (3 + sbyte[k]) + (s_spos[k + 1] - run);
                    df_put(img, at, hcode[c], n);
                }
            }
            __syncthreads();
            if (tid == 0) {
                // sequences section header, table descriptions, then the bitstream: one state chain, written from the last sequence
                uint8_t* sp = lp + lsize; uint32_t o = 0;
                if (nseq < 128) sp[o++] = (uint8_t)nseq;
                else if (nseq < 0x7F00) { sp[o++] = (uint8_t)((nseq >> 8) + 128); sp[o++] = (uint8_t)nseq; }
                else { sp[o++] = 0xff; sp[o++] = (uint8_t)(nseq - 0x7F00); sp[o++] = (uint8_t)((nseq - 0x7F00) >> 8); }
                if (nseq) {
                    sp[o++] = (uint8_t)((s_mode[0] << 6) | (s_mode[1] << 4) | (s_mode[2] << 2));
                    const int order[3] = {0, 1, 2};     // LL, OF, ML
                    for (int q = 0; q < 3; q++) { const int t = order[q]; for (uint32_t k = 0; k < s_dlen[t]; k++) sp[o++] = desc[160 * t + k]; }
                    ZsFse tl = s_mode[0] == 0 ? s_pre[0] : s_tab[0], to = s_mode[1] == 0 ? s_pre[1] : s_tab[1], tm = s_mode[2] == 0 ? s_pre[2] : s_tab[2];
                    uint32_t at = 8 * (uint32_t)((sp + o) - ib);
                    auto put = [&](uint32_t v, uint32_t n) { df_put(img, at, v, n); at += n; };
                    const uint32_t n1 = nseq - 1;
                    uint32_t cl = zs_ll_code(sq_ll[n1]), cm = zs_ml_code(sq_ml[n1]), co = zs_hb(sq_of[n1] + 3u);
                    uint32_t sl = s_mode[0] == 1 ? 0 : zs_init_state(tl, cl), sm2 = s_mode[2] == 1 ? 0 : zs_init_state(tm, cm), so = s_mode[1] == 1 ? 0 : zs_init_state(to, co);
                    put(sq_ll[n1] - zs_ll_info(cl).base, zs_ll_info(cl).bits);
                    put(sq_ml[n1] - zs_ml_info(cm).base, zs_ml_info(cm).bits);
                    put(sq_of[n1] + 3u - (1u << co), co);
                    for (int32_t i = (int32_t)nseq - 2; i >= 0; i--) {
                        cl = zs_ll_code(sq_ll[i]); cm = zs_ml_code(sq_ml[i]); co = zs_hb(sq_of[i] + 3u);
                        uint32_t v, n;
                        if (s_mode[1] != 1) { n = zs_step(to, so, co, v); put(v, n); }
                        if (s_mode[2] != 1) { n = zs_step(tm, sm2, cm, v); put(v, n); }
                        if (s_mode[0] != 1) { n = zs_step(tl, sl, cl, v); put(v, n); }
                        put(sq_ll[i] - zs_ll_info(cl).base, zs_ll_info(cl).bits);
                        put(sq_ml[i] - zs_ml_info(cm).base, zs_ml_info(cm).bits);
                        put(sq_of[i] + 3u - (1u << co), co);
                    }
                    if (s_mode[2] != 1) put(sm2 & ((1u << tm.log) - 1), tm.log);
                    if (s_mode[1] != 1) put(so & ((1u << to.log) - 1), to.log);
                    if (s_mode[0] != 1) put(sl & ((1u << tl.log) - 1), tl.log);
                    put(1, 1);
                }
            }
        }
        if (tid == 0) *(volatile unsigned long long*)&a.pfx[f] = DF_FLAG_AGG | nbytes;
        __syncthreads();

        // ---- P7: look-back for the block's offset, then the image to its final place
        if (warp == 0) {
            const unsigned long long excl = df_lookback(a.pfx, a.st, f, lane);
            if (lane == 0) { *(volatile unsigned long long*)&a.pfx[f] = DF_FLAG_INCL | (excl + nbytes); s_off = excl; }
        }
        __syncthreads();
        uint8_t* G = a.out + ZS_HDR + s_off;
        for (uint32_t i = tid; i < nbytes; i += ZS_THREADS) G[i] = ib[i];
    }
}

// The frame header, Last_Block on the last block (or one empty last Raw_Block for an empty text), and the frame's length. One thread.
__global__ void __launch_bounds__(32) k_zstd_finish(ZstdArgs a) {
    if (threadIdx.x) return;
    uint8_t* o = a.out;
    o[0] = 0x28; o[1] = 0xB5; o[2] = 0x2F; o[3] = 0xFD; o[4] = ZS_FHD; o[5] = ZS_WD;
    for (int i = 0; i < 8; i++) o[6 + i] = (uint8_t)(a.total >> (8 * i));
    const uint32_t n = a.nchunks;
    uint64_t body;
    if (!n) { o[ZS_HDR] = 0x01; o[ZS_HDR + 1] = 0; o[ZS_HDR + 2] = 0; body = 3; }
    else {
        body = a.pfx[n - 1] & DF_VAL_MASK;
        const uint64_t last = n > 1 ? (a.pfx[n - 2] & DF_VAL_MASK) : 0;
        o[ZS_HDR + last] |= 1;
    }
    a.st->wire_total = ZS_HDR + body;
}
#endif  // TF_KERNELS_ZSTD

}  // namespace tfk
