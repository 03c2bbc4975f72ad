// mask_field: hex(HMAC-SHA256(salt, text(value))) fused with the ClickHouse String encode.
//   reference: pkg/transformer/registry/mask/hmac_hasher.go:29-33,52-74 (hash / Apply),
//              pkg/transformer/registry/to_string/to_string.go:145-171 (SerializeToString).
// The reference builds hmac.New(...) per value (two key-pad compressions each time); here the
// ipad/opad states are computed once per plan on the host and every value costs
// ceil((len+9)/64) + 1 compressions.  Integer-ALU bound, not HBM bound (SURVEY §8d).
#pragma once
#include "device_types.cuh"
#include "kernels_encode.cuh"
#include "kernels_fmt.cuh"

namespace tfk {

struct MaskKey { uint32_t istate[8]; uint32_t ostate[8]; };

__host__ __device__ inline uint32_t sha_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

#define TF_SHA_K_VALUES \
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, \
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, \
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, \
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2
__constant__ uint32_t d_sha_k[64] = {TF_SHA_K_VALUES};
static const uint32_t h_sha_k[64] = {TF_SHA_K_VALUES};
#ifdef __CUDA_ARCH__
#define SHA_K d_sha_k
#else
#define SHA_K h_sha_k
#endif

// one SHA-256 compression; w[16] is consumed (rolling schedule)
__host__ __device__ inline void sha256_compress(uint32_t st[8], uint32_t w[16]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll 8
    for (int i = 0; i < 64; i++) {
        uint32_t wi;
        if (i < 16) wi = w[i];
        else {
            const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            const uint32_t s0 = sha_rotr(w15, 7) ^ sha_rotr(w15, 18) ^ (w15 >> 3);
            const uint32_t s1 = sha_rotr(w2, 17) ^ sha_rotr(w2, 19) ^ (w2 >> 10);
            wi = w[i & 15] + s0 + w[(i - 7) & 15] + s1; w[i & 15] = wi;
        }
        const uint32_t S1 = sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25);
        const uint32_t ch = (e & f) ^ (~e & g);
        const uint32_t t1 = h + S1 + ch + SHA_K[i] + wi;
        const uint32_t S0 = sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22);
        const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + S0 + mj;
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// host: precompute the inner/outer pad states (crypto/hmac: keys longer than the block are hashed first)
inline MaskKey make_mask_key(const uint8_t* key, size_t klen) {
    static const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    uint8_t k[64]; memset(k, 0, 64);
    if (klen > 64) {
        uint32_t st[8]; memcpy(st, iv, 32);
        size_t full = klen / 64; uint32_t w[16];
        for (size_t b = 0; b < full; b++) { for (int i = 0; i < 16; i++) w[i] = (uint32_t)key[64 * b + 4 * i] << 24 | (uint32_t)key[64 * b + 4 * i + 1] << 16 | (uint32_t)key[64 * b + 4 * i + 2] << 8 | key[64 * b + 4 * i + 3]; sha256_compress(st, w); }
        uint8_t tail[128]; memset(tail, 0, 128); size_t rem = klen - full * 64; memcpy(tail, key + full * 64, rem); tail[rem] = 0x80;
        size_t tl = rem + 9 <= 64 ? 64 : 128; uint64_t bits = (uint64_t)klen * 8;
        for (int i = 0; i < 8; i++) tail[tl - 1 - i] = (uint8_t)(bits >> (8 * i));
        for (size_t b = 0; b < tl / 64; b++) { for (int i = 0; i < 16; i++) w[i] = (uint32_t)tail[64 * b + 4 * i] << 24 | (uint32_t)tail[64 * b + 4 * i + 1] << 16 | (uint32_t)tail[64 * b + 4 * i + 2] << 8 | tail[64 * b + 4 * i + 3]; sha256_compress(st, w); }
        for (int i = 0; i < 8; i++) { k[4 * i] = (uint8_t)(st[i] >> 24); k[4 * i + 1] = (uint8_t)(st[i] >> 16); k[4 * i + 2] = (uint8_t)(st[i] >> 8); k[4 * i + 3] = (uint8_t)st[i]; }
    } else memcpy(k, key, klen);
    MaskKey mk; uint32_t w[16];
    memcpy(mk.istate, iv, 32); memcpy(mk.ostate, iv, 32);
    for (int i = 0; i < 16; i++) w[i] = ((uint32_t)(k[4 * i] ^ 0x36) << 24) | ((uint32_t)(k[4 * i + 1] ^ 0x36) << 16) | ((uint32_t)(k[4 * i + 2] ^ 0x36) << 8) | (uint32_t)(k[4 * i + 3] ^ 0x36);
    sha256_compress(mk.istate, w);
    for (int i = 0; i < 16; i++) w[i] = ((uint32_t)(k[4 * i] ^ 0x5c) << 24) | ((uint32_t)(k[4 * i + 1] ^ 0x5c) << 16) | ((uint32_t)(k[4 * i + 2] ^ 0x5c) << 8) | (uint32_t)(k[4 * i + 3] ^ 0x5c);
    sha256_compress(mk.ostate, w);
    return mk;
}

// streaming message sink: bytes -> big-endian words -> compress
struct ShaSink {
    uint32_t st[8]; uint32_t w[16]; uint32_t n;   // n = message bytes so far (excluding the 64-byte pad block)
    __device__ __forceinline__ void init(const uint32_t* s) {
#pragma unroll
        for (int i = 0; i < 8; i++) st[i] = s[i];
#pragma unroll
        for (int i = 0; i < 16; i++) w[i] = 0;
        n = 0;
    }
    __device__ __forceinline__ void put(uint8_t b) {
        const uint32_t k = n & 63;
        w[k >> 2] |= (uint32_t)b << (24 - 8 * (k & 3));
        n++;
        if ((n & 63) == 0) {
            sha256_compress(st, w);
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = 0;
        }
    }
    __device__ __forceinline__ void finish(uint32_t prefix_bytes) {   // total length = prefix (pad block) + n
        const uint64_t bits = ((uint64_t)prefix_bytes + n) * 8;
        const uint32_t k = n & 63;
        w[k >> 2] |= 0x80u << (24 - 8 * (k & 3));
        if (k >= 56) {
            sha256_compress(st, w);
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = 0;
        }
        w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
        sha256_compress(st, w);
    }
};

struct MaskArgs { const DCol* cols; const int32_t* slots; const MaskKey* keys; const uint32_t* sel; const DState* st; uint8_t* raw; int columnar; };

// hex(HMAC-SHA256(salt, text(value))) of one value: 64 lowercase hex characters into out64
__device__ inline void mask_digest_hex(const DCol& c, uint64_t r, const MaskKey& mk, uint8_t* out64) {
    ShaSink s; s.init(mk.istate);
    fmt_value(s, c, r);       // to_string.SerializeToString(value, column type)
    s.finish(64);
    uint32_t o[8]; uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { o[i] = mk.ostate[i]; w[i] = s.st[i]; }
    w[8] = 0x80000000u;
#pragma unroll
    for (int i = 9; i < 15; i++) w[i] = 0;
    w[15] = (64 + 32) * 8;
    sha256_compress(o, w);
    const char* hex = "0123456789abcdef";
#pragma unroll
    for (int i = 0; i < 8; i++) {
#pragma unroll
        for (int b = 0; b < 4; b++) { const uint32_t by = (o[i] >> (24 - 8 * b)) & 0xff; out64[8 * i + 2 * b] = (uint8_t)hex[by >> 4]; out64[8 * i + 2 * b + 1] = (uint8_t)hex[by & 15]; }
    }
}

// one thread per (kept row, masked column): "\x40" + 64 hex chars into the block (or the bare digest, columnar output)
__global__ void k_mask_encode(MaskArgs a);
#ifdef TF_KERNELS_MASK
__global__ void __launch_bounds__(128) k_mask_encode(MaskArgs a) {
    const DCol c = a.cols[a.slots[blockIdx.y]];
    const uint64_t n = a.st->n_kept;
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint64_t r = a.sel ? a.sel[j] : j;
    uint8_t* out;
    if (a.columnar) {                                    // utf8 column: offsets 64 j, heap = hex digits
        out = a.raw + c.out_off + j * 64;
        ((uint32_t*)(a.raw + c.offs_off))[j] = (uint32_t)(64 * j);
    } else {
        out = a.raw + c.out_off + j * 65;
        if (c.nullable) a.raw[c.null_off + j] = 0;      // the digest of "<nil>" is a value, never NULL (hmac_hasher.go:60)
        *out++ = 64;
    }
    mask_digest_hex(c, r, a.keys[c.mask_slot], out);
}
#endif  // TF_KERNELS_MASK

// ------------------------------------------------------------------ sharder transformer
//   SharderTransformer.generatePartID pkg/transformer/registry/sharder/sharder.go:130-145:
//   PartID = decimal(crc32.ChecksumIEEE(join(".", SerializeToString(value, type) of the matched columns)) % uint32(ShardsNum)).
//   One thread per kept row streams the text forms through a table-driven CRC (table built per CTA in shared memory).
struct ShardCol { int32_t col, form, pad0, pad1; };       // form: 0 text of the input value, 1 mask digest, 3 converted datetime
struct ShardArgs { const DCol* cols; const ShardCol* sc; int nsc; const MaskKey* keys; const uint32_t* sel; DState* st; uint32_t shards; uint32_t* part; };
struct CrcSink { uint32_t c; const uint32_t* tab; __device__ __forceinline__ void put(uint8_t b) { c = tab[(c ^ b) & 0xffu] ^ (c >> 8); } };

__global__ void k_shard_ids(ShardArgs a);
#ifdef TF_KERNELS_MASK
__global__ void __launch_bounds__(256) k_shard_ids(ShardArgs a) {
    __shared__ uint32_t tab[256];
    { uint32_t c = threadIdx.x; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u))); tab[threadIdx.x] = c; }
    __syncthreads();
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.st->n_kept) return;
    const uint64_t r = a.sel ? a.sel[j] : j;
    CrcSink s{0xFFFFFFFFu, tab};
    for (int k = 0; k < a.nsc; k++) {
        const ShardCol sc = a.sc[k]; const DCol& c = a.cols[sc.col];
        if (k) s.put('.');
        if (sc.form == 1) { uint8_t hx[64]; mask_digest_hex(c, r, a.keys[c.mask_slot], hx); for (int i = 0; i < 64; i++) s.put(hx[i]); }
        else if (sc.form == 3) {           // SerializeToDateTime: nil -> time.Unix(0, 0) (to_datetime.go:137-151), then RFC3339Nano
            int64_t sec = 0; if (row_valid(c, r)) sec = c.type == TF_INT32 ? (int64_t)((const int32_t*)c.values)[r] : (int64_t)((const uint32_t*)c.values)[r];
            fmt_time(s, sec, 0, false);
        } else fmt_value(s, c, r);
    }
    a.part[j] = (~s.c) % a.shards;
}
#endif  // TF_KERNELS_MASK

}  // namespace tfk
