// The gzip / zlib containers of the deflate wire formats (TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB) and the checksum arithmetic their
// trailers need, shared by the device (per-chunk sums, combined across chunks by k_deflate_finish) and the host stream helper
// (tfgpu_deflate_stream_*, which joins several results into one member / stream).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define DF_HD __host__ __device__ __forceinline__
#else
#define DF_HD inline
#endif

namespace tfdf {

// Header bytes: what Go's gzip.NewWriter (no name, MTIME 0, XFL 0, OS 255) and zlib.NewWriter (default level) emit.
constexpr uint8_t GZIP_HDR[10] = {0x1f, 0x8b, 0x08, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0xff};
constexpr uint8_t ZLIB_HDR[2] = {0x78, 0x9c};
constexpr uint32_t GZIP_TRAILER = 8, ZLIB_TRAILER = 4;
constexpr uint32_t ADLER_MOD = 65521;
constexpr uint32_t CRC_POLY = 0xedb88320u;       // CRC-32/IEEE, reflected

// a * b modulo the CRC polynomial, both in the reflected representation (bit 31 = x^0)
DF_HD uint32_t crc_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}
// x^(8 n) modulo the polynomial: multiplying a CRC by it appends n zero bytes' worth of shift
DF_HD uint32_t crc_xpow8(uint64_t n) {
    uint32_t p = 0x80000000u, sq = 0x80000000u >> 8;      // x^0, x^8
    while (n) {
        if (n & 1) p = crc_mulmod(p, sq);
        n >>= 1;
        if (n) sq = crc_mulmod(sq, sq);
    }
    return p;
}
// CRC-32 of A || B from CRC-32(A), CRC-32(B) and |B| (the init and final xor of the standard CRC cancel out)
DF_HD uint32_t crc_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) { return crc_mulmod(crc_xpow8(len_b), crc_a) ^ crc_b; }
// Adler-32 of A || B from Adler-32(A), Adler-32(B) and |B|: a = a1 + a2 - 1, b = b1 + b2 + |B| (a1 - 1)
DF_HD uint32_t adler_combine(uint32_t ad_a, uint32_t ad_b, uint64_t len_b) {
    const uint64_t M = ADLER_MOD, n = len_b % M;
    const uint64_t a1 = ad_a & 0xffff, b1 = ad_a >> 16, a2 = ad_b & 0xffff, b2 = ad_b >> 16;
    const uint64_t a = (a1 + a2 + M - 1) % M;
    const uint64_t b = (b1 + b2 + n * ((a1 + M - 1) % M)) % M;
    return (uint32_t)(b << 16 | a);
}

}  // namespace tfdf
