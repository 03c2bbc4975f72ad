// ORACLE — test infrastructure only. Never linked into or called from the product path.
//
// LZ4 block format (lz4_Block_format.md, public) compressor/decompressor and the
// ClickHouse compressed-frame wrapper:
//     [16B CityHash128 v1.0.2 of the rest][0x82][u32 compressed_size+9][u32 raw_size][LZ4 block]
// Third-party in the reference: github.com/pierrec/lz4/v4 v4.1.25 (block compressor)
// under github.com/ClickHouse/ch-go v0.71.0 compress.Writer; call sites
// pkg/providers/clickhouse/conn/connection.go:46, async/streamer.go:196-245.
// PARITY UNPINNED for the compressed bytes: the LZ4 format admits many valid encodings
// and the reference pins none; parity is defined as "decodes with stock liblz4 to the
// bit-exact native block, header fields and checksum valid" (SURVEY §8c).
// This compressor is a plain greedy single-probe hash-chainless LZ4 ("fast" class, like
// the reference's default level) and doubles as the timed CPU baseline for the LZ4 stage.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>
#include "hashes.hpp"

namespace orc {

inline size_t lz4_bound(size_t n) { return n + n / 255 + 16; }

// Returns compressed size. dst must hold lz4_bound(n).
inline size_t lz4_compress(const uint8_t* src, size_t n, uint8_t* dst) {
    const int HLOG = 13;
    uint32_t table[1 << HLOG];
    std::memset(table, 0xFF, sizeof table);
    uint8_t* op = dst;
    size_t anchor = 0, ip = 0;
    const size_t MFLIMIT = 12, LASTLIT = 5;
    auto rd32 = [&](size_t p) { uint32_t v; std::memcpy(&v, src + p, 4); return v; };
    auto emit = [&](size_t lit_start, size_t lit_len, size_t mlen /*0 = last*/, size_t off) {
        uint8_t* tok = op++;
        if (lit_len >= 15) { *tok = 0xF0; size_t l = lit_len - 15; while (l >= 255) { *op++ = 255; l -= 255; } *op++ = (uint8_t)l; }
        else *tok = (uint8_t)(lit_len << 4);
        std::memcpy(op, src + lit_start, lit_len); op += lit_len;
        if (mlen) {
            *op++ = (uint8_t)off; *op++ = (uint8_t)(off >> 8);
            size_t m = mlen - 4;
            if (m >= 15) { *tok |= 15; m -= 15; while (m >= 255) { *op++ = 255; m -= 255; } *op++ = (uint8_t)m; }
            else *tok |= (uint8_t)m;
        }
    };
    if (n >= MFLIMIT + 1) {
        const size_t mflimit = n - MFLIMIT, matchlimit = n - LASTLIT;
        while (ip < mflimit) {
            uint32_t seq = rd32(ip);
            uint32_t h = (seq * 2654435761u) >> (32 - HLOG);
            uint32_t cand = table[h]; table[h] = (uint32_t)ip;
            if (cand != 0xFFFFFFFFu && ip - cand <= 65535 && rd32(cand) == seq) {
                size_t m = 4;
                while (ip + m < matchlimit && src[cand + m] == src[ip + m]) m++;
                emit(anchor, ip - anchor, m, ip - cand);
                ip += m; anchor = ip;
            } else ip++;
        }
    }
    emit(anchor, n - anchor, 0, 0);
    return (size_t)(op - dst);
}

// Strict decoder of one block of exactly rs raw bytes; returns rs, or (size_t)-1 when the block is malformed or breaks a
// rule of the block format that decoders copying in wide chunks rely on (lz4_Block_format.md, "End of block conditions"):
//   - the last sequence holds literals only (the block ends right behind a literal run, never behind a match);
//   - no match starts within the last 12 bytes (start <= rs - 12), so a block of fewer than 13 bytes has no match;
//   - no match reaches into the last 5 bytes (end <= rs - 5);
//   - offsets are in [1, bytes decoded so far]; length extensions and offsets are complete;
//   - the input is used up exactly when rs bytes have been decoded.
inline size_t lz4_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t rs) {
    const size_t MFLIMIT = 12, LASTLIT = 5;
    const size_t bad = (size_t)-1;
    size_t ip = 0, op = 0;
    if (n == 0) return bad;                                        // not even the token of the last sequence
    for (;;) {
        const uint8_t tok = src[ip++];
        size_t ll = tok >> 4;
        if (ll == 15) { uint8_t b; do { if (ip >= n) return bad; b = src[ip++]; ll += b; } while (b == 255); }
        if (ll > n - ip || ll > rs - op) return bad;
        std::memcpy(dst + op, src + ip, ll); ip += ll; op += ll;
        if (ip == n) break;                                       // literal-only last sequence
        if (op == rs) return bad;                                 // trailing input behind a complete block
        if (n - ip < 2) return bad;
        const size_t off = src[ip] | (src[ip + 1] << 8); ip += 2;
        if (off == 0 || off > op) return bad;
        size_t ml = tok & 15;
        if (ml == 15) { uint8_t b; do { if (ip >= n) return bad; b = src[ip++]; ml += b; } while (b == 255); }
        ml += 4;
        if (rs < MFLIMIT + 1 || op > rs - MFLIMIT) return bad;    // match starts within the last 12 bytes
        if (ml > rs - LASTLIT - op) return bad;                   // match reaches into the last 5 bytes
        for (size_t i = 0; i < ml; i++) dst[op + i] = dst[op + i - off];
        op += ml;
        if (ip == n) return bad;                                  // the block ends behind a match
    }
    return op == rs ? op : bad;
}

// Cut `raw` into frames of at most frame_bytes raw bytes and wrap each one.
inline std::vector<uint8_t> ch_compress_frames(const uint8_t* raw, size_t n, size_t frame_bytes) {
    std::vector<uint8_t> out;
    std::vector<uint8_t> tmp(lz4_bound(frame_bytes) + 25);
    for (size_t pos = 0; pos < n || (n == 0 && pos == 0); pos += frame_bytes) {
        size_t len = n - pos < frame_bytes ? n - pos : frame_bytes;
        size_t c = lz4_compress(raw + pos, len, tmp.data() + 25);
        uint8_t* f = tmp.data();
        f[16] = 0x82;
        uint32_t cs = (uint32_t)(c + 9), rs = (uint32_t)len;
        std::memcpy(f + 17, &cs, 4); std::memcpy(f + 21, &rs, 4);
        city::u128 h = city::hash128(f + 16, c + 9);
        std::memcpy(f, &h.first, 8); std::memcpy(f + 8, &h.second, 8);
        out.insert(out.end(), f, f + 25 + c);
        if (n == 0) break;
    }
    return out;
}

// Parse + verify + decode a frame stream. Returns false on any violation.
inline bool ch_decompress_frames(const uint8_t* wire, size_t n, std::vector<uint8_t>& raw, size_t* n_frames) {
    size_t pos = 0, frames = 0;
    while (pos < n) {
        if (pos + 25 > n) return false;
        const uint8_t* f = wire + pos;
        if (f[16] != 0x82) return false;
        uint32_t cs, rs; std::memcpy(&cs, f + 17, 4); std::memcpy(&rs, f + 21, 4);
        if (cs < 9 || pos + 16 + cs > n) return false;
        city::u128 h = city::hash128(f + 16, cs);
        uint64_t lo, hi; std::memcpy(&lo, f, 8); std::memcpy(&hi, f + 8, 8);
        if (lo != h.first || hi != h.second) return false;
        size_t o = raw.size(); raw.resize(o + rs);
        size_t d = lz4_decompress(f + 25, cs - 9, raw.data() + o, rs);
        if (d != rs) return false;
        pos += 16 + cs; frames++;
    }
    if (n_frames) *n_frames = frames;
    return true;
}

}  // namespace orc
