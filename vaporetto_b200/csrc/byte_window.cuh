// Helpers of the line parsers that stream a line through one warp, 128 bytes per step, each lane holding one 4-byte word
// (`lo`, with the next word in `hi`): k_gold_parse (evaluate.cu) and k_part_parse (partial.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace vpt {
namespace bw {

constexpr unsigned kFull = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

// bit 7 of byte j set when byte addr + j lies in [b0, b1)
__device__ __forceinline__ uint32_t inside80(uint32_t addr, uint32_t b0, uint32_t b1) {
    const uint32_t from = b0 > addr ? b0 - addr : 0u;
    const uint32_t to = b1 - addr < 4u ? b1 - addr : 4u;
    return (from >= 4u ? 0u : 0x80808080u << (8 * from)) & (0x80808080u >> (8 * (4 - to)));
}

__device__ __forceinline__ uint32_t byte_of(uint32_t lo, uint32_t hi, int k) {
    return ((k < 4 ? lo >> (8 * k) : hi >> (8 * (k - 4)))) & 0xFFu;
}

// UTF-8 of the bytes of a lane's word inside the line [b0, b1): every non-continuation byte checks its own sequence and
// that no extra continuation byte follows it (str::from_utf8 once a warp has checked every byte of the line).
// k_gold_parse has the same check inline, where its compiled code stays as it was.
__device__ __forceinline__ bool utf8_word_bad(uint32_t lo, uint32_t hi, uint32_t addr, uint32_t b0, uint32_t b1,
                                              uint32_t in80) {
    bool bad = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (!(in80 & (0x80u << (8 * j)))) continue;
        const uint32_t c0 = byte_of(lo, hi, j);
        auto cont = [&](int k) { return addr + uint32_t(k) < b1 && (byte_of(lo, hi, k) & 0xC0u) == 0x80u; };
        if ((c0 & 0xC0u) == 0x80u) {
            if (addr + uint32_t(j) == b0) bad = true;  // a line cannot start inside a character
            continue;
        }
        const int len = c0 < 0x80u ? 1 : c0 < 0xC2u ? 0 : c0 < 0xE0u ? 2 : c0 < 0xF0u ? 3 : c0 < 0xF5u ? 4 : 0;
        if (len == 0) { bad = true; continue; }
        for (int k = 1; k < len; ++k) bad |= !cont(j + k);
        bad |= cont(j + len);
        if (len >= 3 && cont(j + 1)) {
            const uint32_t c1 = byte_of(lo, hi, j + 1);
            if ((c0 == 0xE0u && c1 < 0xA0u) || (c0 == 0xEDu && c1 >= 0xA0u) || (c0 == 0xF0u && c1 < 0x90u) ||
                (c0 == 0xF4u && c1 >= 0x90u))
                bad = true;
        }
    }
    return bad;
}

}  // namespace bw
}  // namespace vpt
