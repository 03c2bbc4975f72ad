// ORACLE — a strict inflater written from RFC 1950 (zlib), RFC 1951 (DEFLATE) and RFC 1952 (gzip), bit by bit, for checking the
// device's TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB containers. Besides the RFCs' own rules it refuses what lenient decoders accept:
// over-subscribed or incomplete codes (a single code of one bit excepted, as RFC 1951 §3.2.7 allows for distances), stored
// LEN / NLEN that disagree, a missing final block, bytes behind the trailer, a wrong CRC-32 / ISIZE / Adler-32, gzip header
// flags. With chunk > 0 it also checks the engine's layout (include/tfgpu.h): the exact header bytes of Go's default writers, a
// sync-flush marker (empty stored block) after every `chunk` bytes of output and after the last partial chunk, no distance
// reaching before the start of its chunk, and the empty final fixed block 03 00 behind them. Built on its own (oracle/pyinflate.py).
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace orcinf {

struct Fail { std::string what; };

struct Bits {
    const uint8_t* p; uint64_t n, pos = 0; uint32_t buf = 0, cnt = 0;
    uint32_t need(uint32_t k) {       // k <= 24 bits, LSB first
        while (cnt < k) { if (pos >= n) throw Fail{"truncated stream"}; buf |= (uint32_t)p[pos++] << cnt; cnt += 8; }
        const uint32_t v = buf & ((1u << k) - 1); buf >>= k; cnt -= k; return v;
    }
    void align() { buf = 0; cnt = 0; }     // drop the bits left in the current byte
};

struct Huff {
    uint16_t count[16] = {0}; std::vector<uint16_t> sym;
    int nsyms = 0;
    // canonical code from lengths; refuses over-subscribed codes, and incomplete ones unless single_ok and one code of one bit
    void build(const uint8_t* len, int n, int maxbits, bool single_ok, bool empty_ok, const char* what) {
        std::memset(count, 0, sizeof count); nsyms = 0;
        for (int s = 0; s < n; s++) { if (len[s] > maxbits) throw Fail{std::string(what) + ": code length over the limit"}; count[len[s]]++; }
        count[0] = 0;
        for (int l = 1; l < 16; l++) nsyms += count[l];
        if (!nsyms) { if (!empty_ok) throw Fail{std::string(what) + ": no codes"}; return; }
        int left = 1;
        for (int l = 1; l < 16; l++) { left <<= 1; left -= count[l]; if (left < 0) throw Fail{std::string(what) + ": over-subscribed code"}; }
        if (left > 0 && !(single_ok && nsyms == 1 && count[1] == 1)) throw Fail{std::string(what) + ": incomplete code"};
        uint16_t offs[16]; offs[1] = 0;
        for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + count[l];
        sym.assign(nsyms, 0);
        for (int s = 0; s < n; s++) if (len[s]) sym[offs[len[s]]++] = (uint16_t)s;
    }
    int decode(Bits& b) const {
        if (!nsyms) throw Fail{"symbol from an empty code"};
        int code = 0, first = 0, index = 0;
        for (int l = 1; l < 16; l++) {
            code |= (int)b.need(1);
            const int c = count[l];
            if (code - c < first) return sym[index + (code - first)];
            index += c; first += c; first <<= 1; code <<= 1;
        }
        throw Fail{"code not in the table"};
    }
};

struct Result { std::string out; uint64_t stored = 0, fixed = 0, dynamic = 0, markers = 0, max_len = 0; };   // max_len: longest literal/length code of a dynamic block

inline uint32_t crc32(const std::string& s) {
    uint32_t c = 0xffffffffu;
    for (unsigned char ch : s) { c ^= ch; for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1; }
    return ~c;
}
inline uint32_t adler32(const std::string& s) {
    uint64_t a = 1, b = 0;
    for (unsigned char ch : s) { a = (a + ch) % 65521; b = (b + a) % 65521; }
    return (uint32_t)(b << 16 | a);
}

// container: 0 raw DEFLATE, 1 zlib, 2 gzip
inline Result inflate(const uint8_t* src, uint64_t n, int container, uint64_t chunk) {
    static const uint16_t LBASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    static const uint8_t LEXT[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    static const uint16_t DBASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    static const uint8_t DEXT[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    static const uint8_t ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    Result r;
    uint64_t at = 0;
    if (container == 1) {
        if (n < 2) throw Fail{"truncated header"};
        if (chunk && (src[0] != 0x78 || src[1] != 0x9c)) throw Fail{"zlib header is not 78 9c"};
        if ((src[0] & 15) != 8 || (src[0] >> 4) > 7 || ((src[0] << 8) | src[1]) % 31 || (src[1] & 0x20)) throw Fail{"bad zlib header"};
        at = 2;
    } else if (container == 2) {
        static const uint8_t GO[10] = {0x1f, 0x8b, 0x08, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0xff};
        if (n < 10) throw Fail{"truncated header"};
        if (chunk && std::memcmp(src, GO, 10)) throw Fail{"gzip header is not 1f 8b 08 00 00000000 00 ff"};
        if (src[0] != 0x1f || src[1] != 0x8b || src[2] != 8 || src[3] != 0) throw Fail{"bad gzip header (or header flags)"};
        at = 10;
    }
    Bits b{src + at, n - at};
    uint64_t chunk_start = 0; bool last_partial = false, final = false;
    std::string& out = r.out;
    while (!final) {
        final = b.need(1);
        const uint32_t type = b.need(2);
        if (chunk && final) {
            if (type != 1 || out.size() != chunk_start) throw Fail{"layout: the final block is not the empty fixed block behind the last marker"};
        }
        if (chunk && out.size() - chunk_start >= chunk && !(type == 0)) throw Fail{"layout: a chunk runs past its size without a sync-flush marker"};
        if (type == 0) {
            b.align();
            const uint64_t q = b.pos;
            if (q + 4 > b.n) throw Fail{"truncated stored block"};
            const uint32_t len = b.p[q] | b.p[q + 1] << 8, nlen = b.p[q + 2] | b.p[q + 3] << 8;
            if ((len ^ 0xffff) != nlen) throw Fail{"stored LEN / NLEN disagree"};
            if (q + 4 + len > b.n) throw Fail{"truncated stored block"};
            out.append((const char*)b.p + q + 4, len);
            b.pos = q + 4 + len;
            if (len == 0 && !final) {
                r.markers++;
                if (chunk) {
                    const uint64_t got = out.size() - chunk_start;
                    if (got == 0 || got > chunk || last_partial) throw Fail{"layout: a sync-flush marker not at a chunk end"};
                    if (got < chunk) last_partial = true;
                    chunk_start = out.size();
                }
            } else r.stored++;
            continue;
        }
        if (type == 3) throw Fail{"reserved block type"};
        uint8_t lens[320];
        Huff lit, dst;
        if (type == 1) {
            for (int s = 0; s < 288; s++) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
            for (int s = 0; s < 30; s++) lens[288 + s] = 5;
            lit.build(lens, 288, 15, false, false, "fixed literal/length");
            // the fixed distance code has 30 of 32 five-bit codes: used as is (RFC 1951 §3.2.6)
            dst.nsyms = 30; std::memset(dst.count, 0, sizeof dst.count); dst.count[5] = 32; dst.sym.resize(32);
            for (int s = 0; s < 32; s++) dst.sym[s] = (uint16_t)s;
            r.fixed++;
        } else {
            const uint32_t hlit = b.need(5) + 257, hdist = b.need(5) + 1, hclen = b.need(4) + 4;
            if (hlit > 286 || hdist > 30) throw Fail{"HLIT / HDIST out of range"};
            uint8_t cl[19] = {0};
            for (uint32_t k = 0; k < hclen; k++) cl[ORDER[k]] = (uint8_t)b.need(3);
            Huff clh; clh.build(cl, 19, 7, false, false, "code-length code");
            uint32_t k = 0;
            while (k < hlit + hdist) {
                const int s = clh.decode(b);
                if (s < 16) { lens[k++] = (uint8_t)s; continue; }
                uint32_t rep; uint8_t v = 0;
                if (s == 16) { if (!k) throw Fail{"repeat with no previous length"}; v = lens[k - 1]; rep = 3 + b.need(2); }
                else if (s == 17) rep = 3 + b.need(3);
                else rep = 11 + b.need(7);
                if (k + rep > hlit + hdist) throw Fail{"code lengths overrun HLIT + HDIST"};
                while (rep--) lens[k++] = v;
            }
            if (!lens[256]) throw Fail{"no end-of-block code"};
            lit.build(lens, (int)hlit, 15, true, false, "literal/length");
            for (uint32_t s = 0; s < hlit; s++) if (lens[s] > r.max_len) r.max_len = lens[s];
            dst.build(lens + hlit, (int)hdist, 15, true, true, "distance");
            r.dynamic++;
        }
        for (;;) {
            if (chunk && out.size() - chunk_start > chunk) throw Fail{"layout: a chunk runs past its size without a sync-flush marker"};
            const int s = lit.decode(b);
            if (s < 256) { out.push_back((char)s); continue; }
            if (s == 256) break;
            if (s > 285) throw Fail{"invalid length symbol"};
            const uint32_t len = LBASE[s - 257] + b.need(LEXT[s - 257]);
            const int ds = dst.decode(b);
            if (ds > 29) throw Fail{"invalid distance symbol"};
            const uint32_t d = DBASE[ds] + b.need(DEXT[ds]);
            if (d > out.size()) throw Fail{"distance too far back"};
            if (chunk && out.size() - d < chunk_start) throw Fail{"layout: a distance reaches before its chunk"};
            const size_t from = out.size() - d;
            for (uint32_t i = 0; i < len; i++) out.push_back(out[from + i]);
        }
        if (chunk && out.size() - chunk_start > chunk) throw Fail{"layout: a chunk runs past its size without a sync-flush marker"};
        if (chunk && final && out.size() != chunk_start) throw Fail{"layout: the final block carries data"};
    }
    b.align();
    at += b.pos;
    if (container == 1) {
        if (at + 4 != n) throw Fail{at + 4 > n ? "truncated trailer" : "bytes behind the trailer"};
        const uint32_t want = (uint32_t)src[at] << 24 | (uint32_t)src[at + 1] << 16 | (uint32_t)src[at + 2] << 8 | src[at + 3];
        if (want != adler32(out)) throw Fail{"Adler-32 mismatch"};
    } else if (container == 2) {
        if (at + 8 != n) throw Fail{at + 8 > n ? "truncated trailer" : "bytes behind the trailer"};
        auto le = [&](uint64_t o) { return (uint32_t)src[o] | (uint32_t)src[o + 1] << 8 | (uint32_t)src[o + 2] << 16 | (uint32_t)src[o + 3] << 24; };
        if (le(at) != crc32(out)) throw Fail{"CRC-32 mismatch"};
        if (le(at + 4) != (uint32_t)out.size()) throw Fail{"ISIZE mismatch"};
    } else if (at != n) throw Fail{"bytes behind the final block"};
    return r;
}

}  // namespace orcinf

#ifdef ORC_INFLATE_EXPORT
// The C entry point of liboracle_inflate.so (oracle/pyinflate.py builds it from this header). container 0 raw DEFLATE, 1 zlib,
// 2 gzip; chunk > 0 also checks the engine's container layout. Returns the decoded length (the text goes to dst when it fits cap)
// or -1 with the broken rule in err; info = {stored blocks, fixed blocks, dynamic blocks, sync-flush markers, longest
// literal/length code of a dynamic block}.
extern "C" int64_t orc_inflate(const uint8_t* src, uint64_t n, int container, uint64_t chunk, uint8_t* dst, uint64_t cap, uint64_t info[5],
                               char* err, uint64_t errcap) {
    try {
        const orcinf::Result r = orcinf::inflate(src, n, container, chunk);
        if (dst && r.out.size() <= cap) std::memcpy(dst, r.out.data(), r.out.size());
        if (info) { info[0] = r.stored; info[1] = r.fixed; info[2] = r.dynamic; info[3] = r.markers; info[4] = r.max_len; }
        return (int64_t)r.out.size();
    } catch (const orcinf::Fail& f) {
        if (err && errcap) { std::strncpy(err, f.what.c_str(), errcap - 1); err[errcap - 1] = 0; }
        return -1;
    }
}
#endif
