// tfgpu_deflate_stream_*: one gzip member / zlib stream out of the results of several TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB pushes
// (include/tfgpu.h). Host only: every result already ends its chunks with a sync-flush marker, so its body (the bytes between
// the header and the final block) can follow another result's body as it is; only the trailer needs the checksums combined.
#include <cstring>
#include <new>

#include "../../include/tfgpu.h"
#include "deflate_sum.hpp"

struct tfgpu_deflate_stream {
    bool zlib = false, started = false;
    uint32_t crc = 0, adler = 1;          // of the text so far (CRC-32 / Adler-32 of nothing)
    uint64_t total = 0;
};

namespace {
uint32_t get_le32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
uint32_t get_be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | (uint32_t)p[3]; }
const uint8_t* header(const tfgpu_deflate_stream* s) { return s->zlib ? tfdf::ZLIB_HDR : tfdf::GZIP_HDR; }
uint32_t header_len(const tfgpu_deflate_stream* s) { return s->zlib ? sizeof(tfdf::ZLIB_HDR) : sizeof(tfdf::GZIP_HDR); }
uint32_t trailer_len(const tfgpu_deflate_stream* s) { return s->zlib ? tfdf::ZLIB_TRAILER : tfdf::GZIP_TRAILER; }
}  // namespace

extern "C" {

int tfgpu_deflate_stream_open(int container, tfgpu_deflate_stream** out) {
    if (!out) return TF_E_FATAL_ARG;
    *out = nullptr;
    if (container != TF_WIRE_F_GZIP && container != TF_WIRE_F_ZLIB) return TF_E_FATAL_ARG;
    tfgpu_deflate_stream* s = new (std::nothrow) tfgpu_deflate_stream();
    if (!s) return TF_E_FATAL_ARG;
    s->zlib = container == TF_WIRE_F_ZLIB;
    *out = s;
    return TF_OK;
}

int tfgpu_deflate_stream_append(tfgpu_deflate_stream* s, const uint8_t* bytes, uint64_t len, uint64_t raw_len, uint8_t* out, uint64_t cap,
                                uint64_t* written) {
    if (!s || !written || (!bytes && len)) return TF_E_FATAL_ARG;
    *written = 0;
    const uint32_t hl = header_len(s), tl = trailer_len(s);
    if (len < (uint64_t)hl + 2 + tl || std::memcmp(bytes, header(s), hl) != 0) return TF_E_FATAL_ARG;
    const uint8_t* fin = bytes + len - tl - 2;
    if (fin[0] != 0x03 || fin[1] != 0x00) return TF_E_FATAL_ARG;
    const uint64_t body = len - hl - tl - 2;
    static const uint8_t marker[4] = {0x00, 0x00, 0xff, 0xff};
    if (body && (body < 5 || std::memcmp(fin - 4, marker, 4) != 0)) return TF_E_FATAL_ARG;        // the last chunk's sync-flush marker
    const uint32_t sum = s->zlib ? get_be32(fin + 2) : get_le32(fin + 2);
    if (!s->zlib && get_le32(fin + 6) != (uint32_t)raw_len) return TF_E_FATAL_ARG;
    if (!body && (raw_len || sum != (s->zlib ? 1u : 0u))) return TF_E_FATAL_ARG;
    const uint64_t need = (s->started ? 0 : hl) + body;
    if (need > cap || (need && !out)) return TF_E_FATAL_ARG;
    uint8_t* o = out;
    if (!s->started) { std::memcpy(o, header(s), hl); o += hl; }
    if (body) std::memcpy(o, bytes + hl, body);
    s->started = true;
    if (s->zlib) s->adler = tfdf::adler_combine(s->adler, sum, raw_len);
    else s->crc = tfdf::crc_combine(s->crc, sum, raw_len);
    s->total += raw_len;
    *written = need;
    return TF_OK;
}

int tfgpu_deflate_stream_close(tfgpu_deflate_stream* s, uint8_t* out, uint64_t cap, uint64_t* written) {
    if (!s || !written) return TF_E_FATAL_ARG;
    *written = 0;
    const uint32_t hl = header_len(s), tl = trailer_len(s);
    const uint64_t need = (s->started ? 0 : hl) + 2 + tl;
    if (need > cap || !out) return TF_E_FATAL_ARG;
    uint8_t* o = out;
    if (!s->started) { std::memcpy(o, header(s), hl); o += hl; s->started = true; }
    *o++ = 0x03; *o++ = 0x00;
    if (s->zlib) { for (int i = 0; i < 4; i++) *o++ = (uint8_t)(s->adler >> (24 - 8 * i)); }
    else {
        for (int i = 0; i < 4; i++) *o++ = (uint8_t)(s->crc >> (8 * i));
        for (int i = 0; i < 4; i++) *o++ = (uint8_t)(s->total >> (8 * i));
    }
    *written = need;
    return TF_OK;
}

void tfgpu_deflate_stream_free(tfgpu_deflate_stream* s) { delete s; }

}  // extern "C"
