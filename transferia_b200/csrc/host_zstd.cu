// tfgpu_zstd_prefix: the INSERT line in front of a TF_WIRE_F_ZSTD result, inside the same frame (include/tfgpu.h). Host only: the
// engine's blocks never reach before the start of their own text, so raw blocks of other text may go in front of them as they are.
#include <cstring>

#include "../../include/tfgpu.h"

namespace {
constexpr uint32_t HDR = 14;                    // kernels_zstd.cuh: ZS_HDR
constexpr uint8_t MAGIC_FHD_WD[6] = {0x28, 0xB5, 0x2F, 0xFD, 0xC0, 0x28};
constexpr uint32_t BLOCK_MAX = 32768;           // Block_Maximum_Size of the 32 KiB window
}  // namespace

extern "C" {

int tfgpu_zstd_prefix(const uint8_t* text, uint64_t text_len, const uint8_t* frame, uint64_t frame_len, uint8_t* out, uint64_t cap,
                      uint64_t* written) {
    if (!frame || !out || !written || (text_len && !text)) return TF_E_FATAL_ARG;
    *written = 0;
    if (frame_len < HDR + 3 || std::memcmp(frame, MAGIC_FHD_WD, sizeof MAGIC_FHD_WD) != 0) return TF_E_FATAL_ARG;
    uint64_t content = 0;
    for (int i = 0; i < 8; i++) content |= (uint64_t)frame[6 + i] << (8 * i);
    // the block headers must walk exactly to the end, Last_Block on the last one only
    uint64_t at = HDR, regen = 0;
    for (bool last = false; !last;) {
        if (at + 3 > frame_len) return TF_E_FATAL_ARG;
        const uint32_t h = (uint32_t)frame[at] | (uint32_t)frame[at + 1] << 8 | (uint32_t)frame[at + 2] << 16;
        const uint32_t type = (h >> 1) & 3, size = h >> 3;
        last = h & 1;
        if (type == 3 || size > BLOCK_MAX) return TF_E_FATAL_ARG;
        at += 3 + (type == 1 ? 1 : size);
        if (type != 2) regen += size;
        if (at > frame_len) return TF_E_FATAL_ARG;
    }
    if (at != frame_len || regen > content) return TF_E_FATAL_ARG;
    const uint64_t nblocks = (text_len + BLOCK_MAX - 1) / BLOCK_MAX, need = HDR + text_len + 3 * nblocks;
    if (content + text_len < content || need > cap) return TF_E_FATAL_ARG;
    std::memcpy(out, MAGIC_FHD_WD, sizeof MAGIC_FHD_WD);
    const uint64_t total = content + text_len;
    for (int i = 0; i < 8; i++) out[6 + i] = (uint8_t)(total >> (8 * i));
    uint64_t o = HDR;
    for (uint64_t p = 0; p < text_len; p += BLOCK_MAX) {
        const uint32_t n = (uint32_t)(text_len - p < BLOCK_MAX ? text_len - p : BLOCK_MAX), h = n << 3;      // Raw_Block, not last
        out[o] = (uint8_t)h; out[o + 1] = (uint8_t)(h >> 8); out[o + 2] = (uint8_t)(h >> 16);
        std::memcpy(out + o + 3, text + p, n);
        o += 3 + n;
    }
    *written = o;
    return TF_OK;
}

}  // extern "C"
