// ORACLE — strict zstd frame decoder written from RFC 8878 (and the xxHash specification for XXH64), test infrastructure only.
// It decodes every block and table form of the format (raw / RLE / compressed blocks; raw, RLE, compressed and treeless literals
// with 1 or 4 streams; direct and FSE-compressed Huffman weights; predefined, RLE, FSE-compressed and repeat table modes; repeat
// offsets; windowed and single-segment frames; content checksums) and refuses what the format forbids: reserved bits, blocks past
// Block_Maximum_Size, offsets past the window or before the content start, Huffman weights that do not complete a power of two,
// accuracy logs past their limits, bitstreams with bits left over or without their end marker, a wrong content size or checksum and
// trailing bytes. Given the engine's chunk size it also checks TF_WIRE_F_ZSTD's layout (include/tfgpu.h).
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace orzstd {

struct Bad : std::runtime_error { using std::runtime_error::runtime_error; };
[[noreturn]] inline void bad(const std::string& m) { throw Bad(m); }
inline uint32_t hb(uint32_t v) { return 31u - (uint32_t)__builtin_clz(v); }

// ---- XXH64 (xxHash specification), seed 0
inline uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t xxh64(const uint8_t* p, size_t n) {
    const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull, P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
    auto rd64 = [](const uint8_t* q) { uint64_t v; std::memcpy(&v, q, 8); return v; };
    auto rd32 = [](const uint8_t* q) { uint32_t v; std::memcpy(&v, q, 4); return (uint64_t)v; };
    auto round = [&](uint64_t acc, uint64_t in) { acc += in * P2; acc = rotl(acc, 31); return acc * P1; };
    auto merge = [&](uint64_t acc, uint64_t v) { acc ^= round(0, v); return acc * P1 + P4; };
    const uint8_t* end = p + n; uint64_t h;
    if (n >= 32) {
        uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        while (p + 32 <= end) { v1 = round(v1, rd64(p)); v2 = round(v2, rd64(p + 8)); v3 = round(v3, rd64(p + 16)); v4 = round(v4, rd64(p + 24)); p += 32; }
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = merge(h, v1); h = merge(h, v2); h = merge(h, v3); h = merge(h, v4);
    } else h = P5;
    h += n;
    while (p + 8 <= end) { h ^= round(0, rd64(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p++) * P5; h = rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// ---- backward bitstream (§4.1: read from the last byte, whose highest set bit is the end marker)
struct BackBits {
    const uint8_t* p; size_t nbytes; int64_t pos;      // bits not yet read: [0, pos)
    BackBits(const uint8_t* src, size_t n, const char* what) : p(src), nbytes(n) {
        if (!n) bad(std::string(what) + ": empty bitstream");
        if (!src[n - 1]) bad(std::string(what) + ": no end marker in the last byte");
        pos = (int64_t)n * 8 - (8 - (int64_t)hb(src[n - 1]));
    }
    uint32_t peek_at(int64_t lo, uint32_t n) const {     // bits [lo, lo + n), lo >= 0
        uint64_t v = 0; const int64_t b = lo >> 3;
        for (int k = 0; k < 5; k++) if ((size_t)(b + k) < nbytes) v |= (uint64_t)p[b + k] << (8 * k);
        return (uint32_t)((v >> (lo & 7)) & ((1ull << n) - 1));
    }
    // n bits as a number; bits below the stream's start read as zero (overflow: pos goes negative)
    uint32_t read(uint32_t n) {
        if (!n) return 0;
        const int64_t lo = pos - (int64_t)n;
        uint32_t v;
        if (lo >= 0) v = peek_at(lo, n);
        else v = pos > 0 ? peek_at(0, (uint32_t)pos) << (uint32_t)(-lo) : 0;
        pos = lo;
        return v;
    }
    uint32_t read_strict(uint32_t n, const char* what) { if ((int64_t)n > pos) bad(std::string(what) + ": bitstream overread"); return read(n); }
};

// ---- FSE tables (§4.1)
struct Fse { uint32_t log = 0; std::vector<uint8_t> sym, nb; std::vector<uint16_t> base; };
inline Fse fse_table(const std::vector<int16_t>& norm, uint32_t log) {
    const uint32_t ts = 1u << log; Fse t; t.log = log; t.sym.assign(ts, 0); t.nb.assign(ts, 0); t.base.assign(ts, 0);
    std::vector<uint32_t> next(norm.size());
    uint32_t high = ts - 1;
    for (size_t s = 0; s < norm.size(); s++) if (norm[s] == -1) { t.sym[high--] = (uint8_t)s; next[s] = 1; } else next[s] = (uint32_t)norm[s];
    const uint32_t step = (ts >> 1) + (ts >> 3) + 3, mask = ts - 1; uint32_t pos = 0;
    for (size_t s = 0; s < norm.size(); s++) for (int i = 0; i < norm[s]; i++) { t.sym[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    if (pos != 0) bad("FSE: the spread does not close");
    for (uint32_t u = 0; u < ts; u++) {
        const uint32_t x = next[t.sym[u]]++;
        t.nb[u] = (uint8_t)(log - hb(x)); t.base[u] = (uint16_t)((x << t.nb[u]) - ts);
    }
    return t;
}
// table description (§4.1.1) at src[0, n); returns the bytes it took
inline size_t read_ncount(const uint8_t* src, size_t n, uint32_t max_log, uint32_t max_sym, std::vector<int16_t>& norm, uint32_t& log) {
    int64_t bit = 0; const int64_t total = (int64_t)n * 8;
    auto get = [&](uint32_t k) -> uint32_t {
        if (bit + k > total) bad("FSE table description: past its bytes");
        uint32_t v = 0; for (uint32_t i = 0; i < k; i++, bit++) v |= (uint32_t)((src[bit >> 3] >> (bit & 7)) & 1) << i;
        return v;
    };
    auto peek = [&](uint32_t k) -> uint32_t { const int64_t b0 = bit; uint32_t v = 0; for (uint32_t i = 0; i < k && b0 + i < total; i++) v |= (uint32_t)((src[(b0 + i) >> 3] >> ((b0 + i) & 7)) & 1) << i; return v; };
    log = get(4) + 5;
    if (log > max_log) bad("FSE table description: accuracy log " + std::to_string(log) + " past its limit " + std::to_string(max_log));
    norm.clear();
    int32_t remaining = (1 << log) + 1, threshold = 1 << log; uint32_t nbits = log + 1; bool prev0 = false;
    while (remaining > 1) {
        if (prev0) {
            uint32_t r;
            do { r = get(2); for (uint32_t k = 0; k < r; k++) norm.push_back(0); } while (r == 3);
            if (norm.size() > max_sym) bad("FSE table description: more symbols than the alphabet");
        }
        const int32_t mx = (2 * threshold - 1) - remaining;
        int32_t c;
        const uint32_t low = peek(nbits - 1);
        if ((int32_t)low < mx) { c = (int32_t)get(nbits - 1); }
        else { c = (int32_t)get(nbits); if (c >= threshold) c -= mx; }
        c--;
        remaining -= c < 0 ? -c : c;
        norm.push_back((int16_t)c);
        if (norm.size() > max_sym + 1) bad("FSE table description: more symbols than the alphabet");
        prev0 = c == 0;
        if (remaining < 1) bad("FSE table description: probabilities past the table size");
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    if (remaining != 1) bad("FSE table description: probabilities do not sum to the table size");
    return (size_t)((bit + 7) / 8);
}

struct Info { uint64_t raw = 0, rle = 0, compressed = 0, huf_lits = 0, fse_weights = 0, fse_tables = 0, predefined = 0, rle_tables = 0; };

struct Decoder {
    // state that outlives a block
    std::vector<uint8_t> hw_sym, hw_nb; uint32_t huf_bits = 0; bool have_huf = false;
    Fse last[3]; bool have_last[3] = {false, false, false};
    uint32_t rep[3] = {1, 4, 8};
    uint64_t window = 0, block_max = 0, chunk = 0;
    std::vector<uint8_t> out;
    Info info;

    static const Fse& predef(int t) {
        static const Fse T[3] = {
            fse_table({4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1}, 6),
            fse_table({1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1}, 5),
            fse_table({1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1}, 6)};
        return T[t];
    }

    // Huffman tree description (§4.2.1); returns its bytes
    size_t read_huf_tree(const uint8_t* src, size_t n) {
        if (!n) bad("Huffman tree: no header byte");
        const uint32_t h = src[0]; std::vector<uint8_t> w;
        size_t used;
        if (h >= 128) {
            const uint32_t nw = h - 127; used = 1 + (nw + 1) / 2;
            if (used > n) bad("Huffman tree: direct weights past the literals section");
            for (uint32_t i = 0; i < nw; i++) w.push_back((uint8_t)(i & 1 ? src[1 + i / 2] & 15 : src[1 + i / 2] >> 4));
        } else {
            used = 1 + h;
            if (used > n || !h) bad("Huffman tree: FSE-compressed weights past the literals section");
            std::vector<int16_t> norm; uint32_t log;
            const size_t nc = read_ncount(src + 1, h, 6, 12, norm, log);
            if (nc >= h) bad("Huffman tree: no weight bitstream");
            const Fse t = fse_table(norm, log);
            BackBits b(src + 1 + nc, h - nc, "Huffman weights");
            uint32_t s1 = b.read_strict(log, "Huffman weights"), s2 = b.read_strict(log, "Huffman weights");
            for (;;) {
                w.push_back(t.sym[s1]); s1 = t.base[s1] + b.read(t.nb[s1]);
                if (b.pos < 0) { w.push_back(t.sym[s2]); break; }
                w.push_back(t.sym[s2]); s2 = t.base[s2] + b.read(t.nb[s2]);
                if (b.pos < 0) { w.push_back(t.sym[s1]); break; }
                if (w.size() > 255) bad("Huffman weights: more than 255");
            }
            info.fse_weights++;
        }
        if (w.size() > 255) bad("Huffman weights: more than 255");
        uint64_t sum = 0;
        for (uint8_t x : w) { if (x > 11) bad("Huffman weight past 11"); if (x) sum += 1ull << (x - 1); }
        if (!sum) bad("Huffman weights: all zero");
        const uint32_t mb = hb((uint32_t)sum) + 1;
        if (mb > 11) bad("Huffman tree deeper than 11 bits");
        const uint64_t rest = (1ull << mb) - sum;
        if (rest & (rest - 1)) bad("Huffman weights do not complete a power of two");
        w.push_back((uint8_t)(hb((uint32_t)rest) + 1));
        // decoding table: by weight, then by symbol value
        huf_bits = mb; hw_sym.assign(1u << mb, 0); hw_nb.assign(1u << mb, 0);
        uint32_t p = 0;
        for (uint32_t wt = 1; wt <= mb; wt++) for (size_t s = 0; s < w.size(); s++) if (w[s] == wt) {
            for (uint32_t k = 0; k < (1u << (wt - 1)); k++) { hw_sym[p + k] = (uint8_t)s; hw_nb[p + k] = (uint8_t)(mb + 1 - wt); }
            p += 1u << (wt - 1);
        }
        have_huf = true;
        return used;
    }
    void huf_stream(const uint8_t* src, size_t n, size_t count, std::vector<uint8_t>& lit) {
        BackBits b(src, n, "Huffman stream");
        for (size_t i = 0; i < count; i++) {
            uint32_t v = b.pos >= (int64_t)huf_bits ? b.peek_at(b.pos - huf_bits, huf_bits) : (b.pos > 0 ? b.peek_at(0, (uint32_t)b.pos) << (huf_bits - b.pos) : 0);
            const uint32_t nb = hw_nb[v];
            if ((int64_t)nb > b.pos) bad("Huffman stream: overread");
            lit.push_back(hw_sym[v]); b.pos -= nb;
        }
        if (b.pos != 0) bad("Huffman stream: bits left over");
    }

    void block(const uint8_t* src, size_t n) {
        size_t o = 0;
        if (!n) bad("compressed block: empty");
        // literals section (§3.1.1.3.1)
        const uint32_t lt = src[0] & 3, sf = (src[0] >> 2) & 3;
        std::vector<uint8_t> lit; size_t regen;
        if (lt < 2) {
            size_t hl;
            if (!(sf & 1)) { regen = src[0] >> 3; hl = 1; }
            else if (sf == 1) { if (n < 2) bad("literals header"); regen = (src[0] >> 4) | ((size_t)src[1] << 4); hl = 2; }
            else { if (n < 3) bad("literals header"); regen = (src[0] >> 4) | ((size_t)src[1] << 4) | ((size_t)src[2] << 12); hl = 3; }
            o = hl;
            if (regen > block_max) bad("literals past Block_Maximum_Size");
            if (lt == 0) { if (o + regen > n) bad("raw literals past the block"); lit.assign(src + o, src + o + regen); o += regen; }
            else { if (o + 1 > n) bad("RLE literals past the block"); lit.assign(regen, src[o]); o += 1; }
        } else {
            const uint32_t nbts = sf < 2 ? 10 : sf == 2 ? 14 : 18, hl = sf < 2 ? 3 : sf == 2 ? 4 : 5;
            if (n < hl) bad("literals header");
            uint64_t v = 0; for (uint32_t k = 0; k < hl; k++) v |= (uint64_t)src[k] << (8 * k);
            regen = (size_t)((v >> 4) & ((1u << nbts) - 1)); const size_t comp = (size_t)((v >> (4 + nbts)) & ((1u << nbts) - 1));
            o = hl;
            if (regen > block_max) bad("literals past Block_Maximum_Size");
            if (o + comp > n) bad("compressed literals past the block");
            const uint8_t* c = src + o; size_t cn = comp;
            if (lt == 2) { const size_t t = read_huf_tree(c, cn); c += t; cn -= t; }
            else { if (!have_huf) bad("treeless literals without an earlier tree"); if (chunk) bad("layout: treeless literals"); }
            if (sf == 0) huf_stream(c, cn, regen, lit);
            else {
                if (cn < 6) bad("jump table past the literals");
                const size_t z1 = c[0] | c[1] << 8, z2 = c[2] | c[3] << 8, z3 = c[4] | c[5] << 8;
                if (6 + z1 + z2 + z3 > cn) bad("jump table past the literals");
                const size_t z4 = cn - 6 - z1 - z2 - z3, seg = (regen + 3) / 4;
                if (3 * seg > regen) bad("four streams with too few literals");
                const uint8_t* q = c + 6;
                huf_stream(q, z1, seg, lit); huf_stream(q + z1, z2, seg, lit); huf_stream(q + z1 + z2, z3, seg, lit);
                huf_stream(q + z1 + z2 + z3, z4, regen - 3 * seg, lit);
            }
            info.huf_lits++;
            o += comp;
        }
        // sequences section (§3.1.1.3.2)
        if (o >= n) bad("sequences section missing");
        size_t nseq = src[o++];
        if (nseq >= 128) {
            if (nseq < 255) { if (o >= n) bad("sequences header"); nseq = ((nseq - 128) << 8) + src[o++]; }
            else { if (o + 2 > n) bad("sequences header"); nseq = src[o] + ((size_t)src[o + 1] << 8) + 0x7F00; o += 2; }
        }
        const size_t start = out.size();
        size_t li = 0;
        if (nseq) {
            if (o >= n) bad("sequences header");
            const uint32_t modes = src[o++];
            if (modes & 3) bad("sequences header: reserved bits set");
            const uint32_t ms[3] = {modes >> 6, (modes >> 4) & 3, (modes >> 2) & 3};       // LL, OF, ML
            const uint32_t maxlog[3] = {9, 8, 9}, maxsym[3] = {35, 31, 52};
            Fse T[3]; uint32_t rsym[3] = {0, 0, 0};
            for (int t = 0; t < 3; t++) {
                if (ms[t] == 0) { T[t] = predef(t); info.predefined++; }
                else if (ms[t] == 1) { if (o >= n) bad("RLE table past the block"); rsym[t] = src[o++]; if (rsym[t] > maxsym[t]) bad("RLE table symbol past the alphabet"); info.rle_tables++; }
                else if (ms[t] == 2) { std::vector<int16_t> nm; uint32_t lg; o += read_ncount(src + o, n - o, maxlog[t], maxsym[t], nm, lg); T[t] = fse_table(nm, lg); info.fse_tables++; }
                else { if (!have_last[t]) bad("repeat table mode without an earlier table"); if (chunk) bad("layout: repeat table mode"); T[t] = last[t]; }
                if (ms[t] != 1 && ms[t] != 3) { last[t] = T[t]; have_last[t] = true; }
                if (ms[t] == 1) { Fse r; r.log = 0; r.sym.assign(1, (uint8_t)rsym[t]); r.nb.assign(1, 0); r.base.assign(1, 0); T[t] = r; last[t] = r; have_last[t] = true; }
            }
            BackBits b(src + o, n - o, "sequences");
            uint32_t sl = b.read_strict(T[0].log, "sequences"), so = b.read_strict(T[1].log, "sequences"), sm = b.read_strict(T[2].log, "sequences");
            static const uint32_t LLB[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
            static const uint8_t LLN[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
            static const uint32_t MLB[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
            static const uint8_t MLN[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
            uint32_t valid = 0;         // repeat slots this block has set itself (the engine layout's rule)
            for (size_t i = 0; i < nseq; i++) {
                const uint32_t oc = T[1].sym[so], mc = T[2].sym[sm], lc = T[0].sym[sl];
                if (oc > 31) bad("offset code past 31");
                if (mc > 52 || lc > 35) bad("sequence code past the alphabet");
                const uint32_t ofv = (1u << oc) + b.read_strict(oc, "sequences");
                const uint32_t ml = (mc < 32 ? mc + 3 : MLB[mc - 32]) + b.read_strict(mc < 32 ? 0 : MLN[mc - 32], "sequences");
                const uint32_t ll = LLB[lc] + b.read_strict(LLN[lc], "sequences");
                uint32_t off;
                if (ofv > 3) { off = ofv - 3; rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = off; valid = valid < 3 ? valid + 1 : 3; }
                else {
                    const uint32_t idx = ll == 0 ? ofv : ofv - 1;      // 0, 1, 2 = rep slot; 3 = rep[0] - 1
                    const uint32_t need = idx == 3 ? 1 : idx + 1;
                    if (chunk && valid < need) bad("layout: a repeat code names an offset the block did not set");
                    if (idx == 0) off = rep[0];
                    else if (idx == 1) { off = rep[1]; rep[1] = rep[0]; rep[0] = off; }
                    else {
                        off = idx == 2 ? rep[2] : rep[0] - 1;
                        if (!off) bad("repeat offset 0");
                        rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = off;
                    }
                    if (idx >= 2) valid = valid < 3 ? valid + 1 : 3;
                }
                if (i + 1 < nseq) { sl = T[0].base[sl] + b.read_strict(T[0].nb[sl], "sequences"); sm = T[2].base[sm] + b.read_strict(T[2].nb[sm], "sequences"); so = T[1].base[so] + b.read_strict(T[1].nb[so], "sequences"); }
                if (li + ll > lit.size()) bad("sequence past the literals");
                out.insert(out.end(), lit.begin() + li, lit.begin() + li + ll); li += ll;
                if (off > out.size()) bad("offset before the content start");
                if (off > window) bad("offset beyond the window");
                const size_t from = out.size() - off;
                for (uint32_t k = 0; k < ml; k++) out.push_back(out[from + k]);
                if (out.size() - start > block_max) bad("block regenerates past Block_Maximum_Size");
            }
            if (b.pos != 0) bad("sequences: bits left over");
        } else if (o != n) bad("bytes after an empty sequences section");
        out.insert(out.end(), lit.begin() + li, lit.end());
        if (out.size() - start > block_max) bad("block regenerates past Block_Maximum_Size");
    }

    void frame(const uint8_t* src, size_t n) {
        if (n < 5 || src[0] != 0x28 || src[1] != 0xB5 || src[2] != 0x2F || src[3] != 0xFD) bad("not a zstd frame (magic)");
        const uint32_t fhd = src[4];
        const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
        if (fhd & 8) bad("frame header: reserved bit set");
        size_t o = 5;
        if (!single) {
            if (o >= n) bad("frame header truncated");
            const uint32_t wd = src[o++], e = wd >> 3, m = wd & 7;
            const uint64_t wb = 1ull << (10 + e);
            window = wb + (wb / 8) * m;
        }
        const size_t did_len = did_flag == 0 ? 0 : did_flag == 1 ? 1 : did_flag == 2 ? 2 : 4;
        uint64_t did = 0; if (o + did_len > n) bad("frame header truncated");
        for (size_t k = 0; k < did_len; k++) did |= (uint64_t)src[o + k] << (8 * k);
        o += did_len;
        if (did) bad("frame needs a dictionary");
        const size_t fcs_len = fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
        if (o + fcs_len > n) bad("frame header truncated");
        uint64_t fcs = 0; for (size_t k = 0; k < fcs_len; k++) fcs |= (uint64_t)src[o + k] << (8 * k);
        if (fcs_len == 2) fcs += 256;
        o += fcs_len;
        const bool has_fcs = fcs_len > 0;
        if (single) window = fcs;
        block_max = window < 131072 ? window : 131072;
        if (chunk) {
            static const uint8_t H[6] = {0x28, 0xB5, 0x2F, 0xFD, 0xC0, 0x28};
            if (std::memcmp(src, H, 6) != 0 || o != 14) bad("layout: not the engine's frame header");
        }
        for (bool last = false; !last;) {
            if (o + 3 > n) bad("block header truncated");
            const uint32_t h = src[o] | src[o + 1] << 8 | src[o + 2] << 16; o += 3;
            last = h & 1; const uint32_t type = (h >> 1) & 3, size = h >> 3;
            if (type == 3) bad("reserved block type");
            if (size > block_max) bad("block larger than Block_Maximum_Size");
            const size_t before = out.size();
            if (type == 0) { if (o + size > n) bad("raw block truncated"); out.insert(out.end(), src + o, src + o + size); o += size; info.raw++; }
            else if (type == 1) { if (o + 1 > n) bad("RLE block truncated"); out.insert(out.end(), size, src[o]); o += 1; info.rle++; }
            else { if (o + size > n) bad("compressed block truncated"); block(src + o, size); o += size; info.compressed++; }
            if (chunk) {
                const uint64_t got = out.size() - before;
                if (has_fcs && fcs == 0) { if (!(last && type == 0 && size == 0)) bad("layout: an empty text is one empty last raw block"); }
                else {
                    const uint64_t want = fcs - before < chunk ? fcs - before : chunk;
                    if (got != want || !want) bad("layout: a block does not hold exactly one chunk");
                    if (last != (before + got == fcs)) bad("layout: Last_Block not on the last chunk only");
                }
            }
        }
        if (checksum) {
            if (chunk) bad("layout: content checksum present");
            if (o + 4 > n) bad("checksum truncated");
            const uint32_t want = src[o] | src[o + 1] << 8 | src[o + 2] << 16 | (uint32_t)src[o + 3] << 24; o += 4;
            if ((uint32_t)xxh64(out.data(), out.size()) != want) bad("content checksum mismatch");
        }
        if (has_fcs && fcs != out.size()) bad("Frame_Content_Size does not match the content");
        if (o != n) bad("trailing bytes after the frame");
    }
};

}  // namespace orzstd

#ifdef ORC_ZSTD_EXPORT
// Decodes src[0, n) (one frame). chunk > 0 also checks the engine's layout. Returns the content length (copied to dst when cap
// allows) or -1 with the broken rule in err. info[8]: raw, RLE, compressed blocks; Huffman-coded literal sections; FSE-compressed
// Huffman weights; FSE-compressed, predefined and RLE sequence tables.
extern "C" int64_t orc_zstd_decode(const uint8_t* src, uint64_t n, uint64_t chunk, uint8_t* dst, uint64_t cap, uint64_t* info, char* err, uint64_t errcap) {
    orzstd::Decoder d; d.chunk = chunk;
    try { d.frame(src, n); }
    catch (const orzstd::Bad& b) { if (errcap) { std::strncpy(err, b.what(), errcap - 1); err[errcap - 1] = 0; } return -1; }
    if (dst && d.out.size() <= cap) std::memcpy(dst, d.out.data(), d.out.size());
    if (info) { const orzstd::Info& i = d.info; const uint64_t v[8] = {i.raw, i.rle, i.compressed, i.huf_lits, i.fse_weights, i.fse_tables, i.predefined, i.rle_tables}; std::memcpy(info, v, sizeof v); }
    return (int64_t)d.out.size();
}
#endif
