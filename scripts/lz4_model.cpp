// CPU model of the round-synchronous GPU LZ4 frame compressor (k_lz4_frames): the same phases, executed
// phase by phase over all "threads", so that parse rules (segment size, probing stride, continuation merging)
// can be evaluated for compression ratio and validated against a decoder before they are written as a kernel.
// Development tool, not product code:  g++ -O2 -o /tmp/lz4_model scripts/lz4_model.cpp -ldl && /tmp/lz4_model block.bin
// (block.bin: the bench.py headline block from scripts/headline_block.py; key=value arguments override the rules below)
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <random>
#include <string>
#include <vector>

// The defaults are the rules k_lz4_frames runs with.
struct Cfg {
    uint32_t F = 15360, SEG = 60, ROUND = 1024, HASH_BITS = 11;
    int stride = 2;          // probe every stride-th position (inserts happen at every position)
    bool second_probe = true, period8 = true, merge = true, backext = true;
    int winner = 3; bool near_first = true; int ins_stride = 1; bool twoslot = false; bool recent_first = false;         // 0 lowest position wins an insert race, 1 highest, 2 random, 3 as in the kernel
    bool race = false, wmatch = false;
};

struct Seq { uint32_t p, ml, off; };

static uint32_t rd32(const uint8_t* d, uint32_t p) { uint32_t v; memcpy(&v, d + p, 4); return v; }

// returns the LZ4 block
static std::vector<uint8_t> compress_frame(const uint8_t* d, uint32_t len, const Cfg& c, std::mt19937& rng, uint64_t* stat_seq) {
    const uint32_t T = 1u << c.HASH_BITS;
    std::vector<uint32_t> table(T, 0xffffffffu);           // tag16 << 16 | pos ; 0xffffffff = empty
    std::vector<uint32_t> cand(len, 0xffffffffu);
    // ---- P2
    for (uint32_t r0 = 0; r0 < len; r0 += c.ROUND) {
        const uint32_t r1 = std::min(len, r0 + c.ROUND);
        std::vector<uint32_t> idx(r1 - r0), tag(r1 - r0);
        for (uint32_t p = r0; p < r1; p++) {
            if (p + 4 > len) { idx[p - r0] = 0; tag[p - r0] = 0; continue; }
            const uint32_t h = rd32(d, p) * 2654435761u;
            idx[p - r0] = h >> (32 - c.HASH_BITS); tag[p - r0] = (h << c.HASH_BITS) & 0xffff0000u;
        }
        if (c.race) {
            // one barrier per round: every warp (32 threads x 4 positions) probes and then inserts, and the warps of a round run in any
            // order, so a probe sees the inserts of the warps of this round that ran before it (accepted when they lie behind it)
            const uint32_t WP = 128, nw = (r1 - r0 + WP - 1) / WP;
            std::vector<uint32_t> worder(nw);
            for (uint32_t i = 0; i < nw; i++) worder[i] = i;
            std::shuffle(worder.begin(), worder.end(), rng);
            for (uint32_t w : worder) {
                const uint32_t w0 = r0 + w * WP, w1 = std::min(r1, w0 + WP);
                for (uint32_t p = w0; p < w1; p++) {
                    if (p % c.stride || p + 12 > len) continue;
                    if ((p & ~3u) >= 8) {
                        if (rd32(d, p) == rd32(d, p - 4)) { cand[p] = p - 4; continue; }
                        if (rd32(d, p) == rd32(d, p - 8)) { cand[p] = p - 8; continue; }
                    }
                    const uint32_t e = table[idx[p - r0]];
                    if (e != 0xffffffffu && (e & 0xffff0000u) == tag[p - r0] && (e & 0xffffu) < p) cand[p] = e & 0xffffu;
                    if (c.wmatch && cand[p] == 0xffffffffu)      // __match_any_sync: the nearest earlier lane of the warp with the same 4 bytes at the same offset mod 4
                        for (uint32_t q = p; q >= w0 + 4;) { q -= 4; if (rd32(d, q) == rd32(d, p)) { cand[p] = q; break; } }
                }
                std::vector<uint32_t> ord(w1 - w0);
                for (uint32_t i = 0; i < ord.size(); i++) ord[i] = w0 + i;
                std::shuffle(ord.begin(), ord.end(), rng);
                for (uint32_t p : ord) {
                    if (p + 4 > len || p % c.ins_stride) continue;
                    uint32_t& e = table[idx[p - r0]];
                    // winner 0 here: an insert of this round replaces an entry of an earlier round or one of this round behind it (atomicMax)
                    if (c.winner != 0 || e == 0xffffffffu || (e & 0xffffu) < r0 || (e & 0xffffu) > p) e = tag[p - r0] | p;
                }
            }
            continue;
        }
        // first probe: the table as it was before this round
        for (uint32_t p = r0; p < r1; p++) {
            if (p % c.stride || p + 12 > len) continue;
            const uint32_t e = table[idx[p - r0]];
            if (c.near_first && (p & ~3u) >= 8) {     // the kernel tests a thread's positions 4 / 8 back from its third word on
                if (rd32(d, p) == rd32(d, p - 4)) cand[p] = p - 4;
                else if (rd32(d, p) == rd32(d, p - 8)) cand[p] = p - 8;
            }
            if (cand[p] == 0xffffffffu && e != 0xffffffffu && (e & 0xffff0000u) == tag[p - r0]) cand[p] = e & 0xffffu;
            if (cand[p] == 0xffffffffu && c.period8 && p >= 8 && rd32(d, p) == rd32(d, p - 8)) cand[p] = p - 8;
        }
        // inserts (racing)
        std::vector<uint32_t> order(r1 - r0);
        for (uint32_t i = 0; i < order.size(); i++) order[i] = r0 + i;
        if (c.winner == 0) std::reverse(order.begin(), order.end());
        else if (c.winner == 2) std::shuffle(order.begin(), order.end(), rng);
        else if (c.winner == 3) {
            // the kernel: warps in any order; a warp stores its lanes' 4th, 3rd, 2nd, 1st positions. Which lane wins a store conflict
            // is undefined; the lowest lane winning reproduces the kernel's ratio on the bench.py block (1.687 here, 1.693 on the H100)
            std::vector<uint32_t> ws;
            for (uint32_t w0 = r0; w0 < r1; w0 += 128) ws.push_back(w0);
            std::shuffle(ws.begin(), ws.end(), rng);
            order.clear();
            for (uint32_t w0 : ws)
                for (int k = 3; k >= 0; k--)
                    for (int l = 31; l >= 0; l--) if (w0 + 4 * l + k < r1) order.push_back(w0 + 4 * l + k);
        }
        for (uint32_t p : order) if (p + 4 <= len && p % c.ins_stride == 0) table[idx[p - r0]] = tag[p - r0] | p;
        if (c.second_probe)
            for (uint32_t p = r0; p < r1; p++) {
                if (p % c.stride || p + 12 > len) continue;
                if (cand[p] != 0xffffffffu && !(c.recent_first && cand[p] + 8 < p)) continue;     // recent_first: a near candidate (4 / 8 back) stays
                const uint32_t e = table[idx[p - r0]];
                if ((e & 0xffff0000u) == tag[p - r0] && (e & 0xffffu) < p) cand[p] = e & 0xffffu;
            }
    }
    if (c.twoslot) {
        // one barrier per round: bucket = [slot of even rounds, slot of odd rounds]; round r probes both slots BEFORE inserting into
        // slot r % 2 (other threads' inserts of the same round may already be there), and positions of round r that found nothing
        // look at slot r % 2 again one round later, when it holds the round's final winner
        std::fill(cand.begin(), cand.end(), 0xffffffffu);
        const uint32_t NB = 1u << (c.HASH_BITS - 1);
        std::vector<uint32_t> t2(2 * NB, 0xffffffffu);
        auto hidx = [&](uint32_t p) { const uint32_t h = rd32(d, p) * 2654435761u; return h >> (32 - (c.HASH_BITS - 1)); };
        auto htag = [&](uint32_t p) { const uint32_t h = rd32(d, p) * 2654435761u; return (h << (c.HASH_BITS - 1)) & 0xffff0000u; };
        uint32_t rnd = 0;
        for (uint32_t r0 = 0; r0 < len + c.ROUND; r0 += c.ROUND, rnd++) {
            // late probe of the previous round
            if (r0 >= c.ROUND)
                for (uint32_t p = r0 - c.ROUND; p < std::min(len, r0); p += c.stride) {
                    if (p + 12 > len || cand[p] != 0xffffffffu) continue;
                    const uint32_t e = t2[2 * hidx(p) + ((rnd - 1) & 1)];
                    if (e != 0xffffffffu && (e & 0xffff0000u) == htag(p) && (e & 0xffffu) < p) cand[p] = e & 0xffffu;
                }
            if (r0 >= len) break;
            const uint32_t r1 = std::min(len, r0 + c.ROUND);
            std::vector<uint32_t> thr((r1 - r0 + 3) / 4);
            for (uint32_t i = 0; i < thr.size(); i++) thr[i] = i;
            std::shuffle(thr.begin(), thr.end(), rng);
            for (uint32_t ti : thr) {
                const uint32_t p0 = r0 + 4 * ti;
                for (uint32_t p = p0; p < std::min(r1, p0 + 4); p++) {
                    if (p % c.stride || p + 12 > len) continue;
                    if (p >= 4 && rd32(d, p) == rd32(d, p - 4)) { cand[p] = p - 4; continue; }
                    if (p >= 8 && rd32(d, p) == rd32(d, p - 8)) { cand[p] = p - 8; continue; }
                    uint32_t best = 0xffffffffu;
                    for (int sl = 0; sl < 2; sl++) {
                        const uint32_t e = t2[2 * hidx(p) + sl];
                        if (e != 0xffffffffu && (e & 0xffff0000u) == htag(p) && (e & 0xffffu) < p && (best == 0xffffffffu || (e & 0xffffu) > best)) best = e & 0xffffu;
                    }
                    cand[p] = best;
                }
                for (uint32_t p = p0; p < std::min(r1, p0 + 4); p++) if (p + 4 <= len && p % c.ins_stride == 0) t2[2 * hidx(p) + (rnd & 1)] = htag(p) | p;
            }
        }
    }
    // ---- P3: per segment greedy parse, matches cut at the segment end
    const uint32_t nseg = (len + c.SEG - 1) / c.SEG;
    const uint32_t lim5 = len >= 5 ? len - 5 : 0;
    std::vector<std::vector<Seq>> S(nseg);
    std::vector<uint8_t> reach(nseg, 0), pure(nseg, 0);
    for (uint32_t s = 0; s < nseg; s++) {
        const uint32_t a = s * c.SEG, b = std::min(len, a + c.SEG), limit = std::min(b, lim5);
        uint32_t cur = a, anchor = a;
        while (cur < b) {
            uint32_t p = cur; while (p < b && (p % c.stride || cand[p] == 0xffffffffu)) p++;
            if (p >= b || p + 4 > limit) break;
            uint32_t q = cand[p], ml = 0;
            while (p + ml < limit && d[q + ml] == d[p + ml]) ml++;
            if (ml < 4) { cur = p + 1; continue; }
            if (c.backext) while (p > anchor && q > 0 && d[p - 1] == d[q - 1]) { p--; q--; ml++; }
            S[s].push_back({p, ml, p - q});
            cur = anchor = p + ml;
            if (S[s].size() == c.SEG / 4) break;
        }
        if (!S[s].empty()) { const Seq& l = S[s].back(); reach[s] = (l.p + l.ml == a + c.SEG); }
        pure[s] = S[s].size() == 1 && S[s][0].p == a && S[s][0].ml == c.SEG;
    }
    // ---- P3b: continuation of a match that was cut at a segment end
    std::vector<uint32_t> cl(nseg, 0), D(nseg, 0), ext(nseg + 1, 0);
    std::vector<uint8_t> alive(nseg, 0), merged(nseg, 0), head(nseg, 0);
    if (c.merge) {
        std::vector<uint8_t> dvalid(nseg, 0);
        for (uint32_t t = 1; t < nseg; t++) {          // the kernel does this with a segmented scan
            if (!pure[t - 1]) { dvalid[t] = reach[t - 1]; D[t] = dvalid[t] ? S[t - 1].back().off : 0; }
            else { dvalid[t] = dvalid[t - 1]; D[t] = D[t - 1]; }
        }
        std::vector<uint32_t> clt(nseg, 0);
        for (uint32_t t = 1; t < nseg; t++) {
            if (!dvalid[t]) continue;
            const uint32_t a = t * c.SEG, b = std::min(len, a + c.SEG), limit = std::min(b, lim5);
            uint32_t n = 0; while (a + n < limit && d[a + n] == d[a + n - D[t]]) n++;
            clt[t] = n;
        }
        for (uint32_t t = 1; t < nseg; t++) {
            if (!dvalid[t]) continue;
            alive[t] = pure[t - 1] ? (clt[t - 1] == c.SEG && dvalid[t - 1]) : reach[t - 1];
            uint32_t n = clt[t];
            const uint32_t a = t * c.SEG;
            if (pure[t]) {
                if (!(alive[t] && n > 0) && n != c.SEG) n = 0;
                if (n && n < c.SEG && c.SEG - n < 4) n = c.SEG - 4;
            } else {
                if (!alive[t]) n = 0;
                if (reach[t] && n > c.SEG - 4) n = c.SEG - 4;
            }
            cl[t] = n;
            if (!n) continue;
            merged[t] = alive[t]; head[t] = !alive[t];
            // own sequences against the piece [a, a + n)
            std::vector<Seq> keep;
            for (const Seq& q : S[t]) {
                if (q.p + q.ml <= a + n) continue;
                if (q.p >= a + n) { keep.push_back(q); continue; }
                const uint32_t np = a + n, nml = q.p + q.ml - np;
                if (nml >= 4 && np + 12 <= len) keep.push_back({np, nml, q.off});
            }
            S[t] = keep;
        }
        for (uint32_t t = nseg; t-- > 1;) ext[t] = merged[t] ? cl[t] + (cl[t] == c.SEG ? ext[t + 1] : 0) : 0;
    }
    // ---- emit (sequentially here; the kernel computes the offsets with scans)
    std::vector<uint8_t> out;
    uint32_t anchor = 0;
    auto put_seq = [&](uint32_t p, uint32_t ml, uint32_t off) {
        const uint32_t ll = p - anchor, mt = ml - 4;
        out.push_back((uint8_t)(((ll < 15 ? ll : 15) << 4) | (mt < 15 ? mt : 15)));
        if (ll >= 15) { uint32_t x = ll - 15; while (x >= 255) { out.push_back(255); x -= 255; } out.push_back((uint8_t)x); }
        out.insert(out.end(), d + anchor, d + p);
        out.push_back((uint8_t)off); out.push_back((uint8_t)(off >> 8));
        if (mt >= 15) { uint32_t x = mt - 15; while (x >= 255) { out.push_back(255); x -= 255; } out.push_back((uint8_t)x); }
        anchor = p + ml; (*stat_seq)++;
    };
    for (uint32_t t = 0; t < nseg; t++) {
        const uint32_t a = t * c.SEG;
        if (merged[t]) anchor = a + cl[t];                       // bytes swallowed by the running match
        else if (head[t]) put_seq(a, cl[t] + ext[t + 1], D[t]);
        for (size_t k = 0; k < S[t].size(); k++) {
            const Seq& q = S[t][k];
            const bool last = k + 1 == S[t].size();
            put_seq(q.p, q.ml + ((last && q.p + q.ml == a + c.SEG && t + 1 < nseg) ? ext[t + 1] : 0), q.off);
        }
        if (merged[t] && cl[t] == c.SEG) anchor = a + c.SEG;
    }
    {
        const uint32_t ll = len - anchor;
        out.push_back((uint8_t)((ll < 15 ? ll : 15) << 4));
        if (ll >= 15) { uint32_t x = ll - 15; while (x >= 255) { out.push_back(255); x -= 255; } out.push_back((uint8_t)x); }
        out.insert(out.end(), d + anchor, d + len);
    }
    return out;
}

static bool decode(const std::vector<uint8_t>& in, std::vector<uint8_t>& out, uint32_t want) {
    size_t i = 0; out.clear();
    while (i < in.size()) {
        const uint8_t tok = in[i++];
        uint32_t ll = tok >> 4; if (ll == 15) { uint8_t b; do { if (i >= in.size()) return false; b = in[i++]; ll += b; } while (b == 255); }
        if (i + ll > in.size()) return false;
        out.insert(out.end(), in.begin() + i, in.begin() + i + ll); i += ll;
        if (i >= in.size()) break;
        if (i + 2 > in.size()) return false;
        const uint32_t off = in[i] | (in[i + 1] << 8); i += 2;
        uint32_t ml = tok & 15; if (ml == 15) { uint8_t b; do { if (i >= in.size()) return false; b = in[i++]; ml += b; } while (b == 255); }
        ml += 4;
        if (off == 0 || off > out.size()) return false;
        if (out.size() + 12 > want || out.size() + ml + 5 > want) return false;      // MFLIMIT / LASTLITERALS as stock liblz4 enforces them
        for (uint32_t k = 0; k < ml; k++) out.push_back(out[out.size() - off]);
    }
    return out.size() == want;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: lz4_model block.bin [key=value ...]\n"); return 2; }
    FILE* f = fopen(argv[1], "rb"); if (!f) return 2;
    fseek(f, 0, SEEK_END); const size_t n = ftell(f); fseek(f, 0, SEEK_SET);
    std::vector<uint8_t> blk(n); if (fread(blk.data(), 1, n, f) != n) return 2; fclose(f);
    Cfg c; size_t step = 1;
    for (int i = 2; i < argc; i++) {
        std::string kv = argv[i]; const size_t e = kv.find('='); const std::string k = kv.substr(0, e); const int v = atoi(kv.c_str() + e + 1);
        if (k == "F") c.F = v; else if (k == "SEG") c.SEG = v; else if (k == "ROUND") c.ROUND = v; else if (k == "HB") c.HASH_BITS = v;
        else if (k == "stride") c.stride = v; else if (k == "probe2") c.second_probe = v; else if (k == "p8") c.period8 = v;
        else if (k == "merge") c.merge = v; else if (k == "back") c.backext = v; else if (k == "winner") c.winner = v; else if (k == "step") step = v; else if (k == "near") c.near_first = v; else if (k == "ins") c.ins_stride = v; else if (k == "two") c.twoslot = v; else if (k == "recent") c.recent_first = v;
        else if (k == "race") c.race = v; else if (k == "wmatch") c.wmatch = v;
    }
    typedef int (*comp_t)(const char*, char*, int, int);
    comp_t stock = nullptr;
    if (void* h = dlopen("liblz4.so.1", RTLD_NOW)) stock = (comp_t)dlsym(h, "LZ4_compress_default");
    std::mt19937 rng(12345);
    uint64_t in_b = 0, out_b = 0, stock_b = 0, nseq = 0, frames = 0;
    std::vector<uint8_t> dec; std::vector<char> tmp(c.F + c.F / 255 + 64);
    for (size_t pos = 0; pos < n; pos += (size_t)c.F * step) {
        const uint32_t len = (uint32_t)std::min<size_t>(c.F, n - pos);
        const std::vector<uint8_t> o = compress_frame(blk.data() + pos, len, c, rng, &nseq);
        if (!decode(o, dec, len) || memcmp(dec.data(), blk.data() + pos, len)) { fprintf(stderr, "frame at %zu does not round-trip\n", pos); return 1; }
        in_b += len; out_b += o.size() + 25; frames++; if (getenv("PERFRAME")) printf("FR %zu %zu\n", pos, o.size());
        if (stock) { const int sb = stock((const char*)blk.data() + pos, tmp.data(), (int)len, (int)tmp.size()); stock_b += sb + 25; if (getenv("PERFRAME")) printf("ST %zu %d\n", pos, sb); }
    }
    printf("frames %llu in %llu out %llu ratio %.4f  stock %.4f  seq/frame %.1f\n", (unsigned long long)frames, (unsigned long long)in_b,
           (unsigned long long)out_b, (double)in_b / out_b, stock_b ? (double)in_b / stock_b : 0.0, (double)nseq / frames);
    return 0;
}
