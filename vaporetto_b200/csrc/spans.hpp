// Per-window arithmetic of the token-span kernels (spans.cu): one lane's 4-byte word of a document's 128-byte window.
// Plain arithmetic on bit-7 byte masks (bit 7 of byte j of a word = bit 8 j + 7), compiled for the device by spans.cu
// and for the host by tests/native/spans_test.cpp, which runs the kernels' warp loops over it against a byte-by-byte
// restatement of SplitLinebreaksFilter (vaporetto_rules/src/sentence_filters/split_linebreaks.rs:9-37) and of
// `boundary_pos` (vaporetto_tantivy/src/lib.rs:179-188).
#pragma once
#include <cstdint>

#include "common.hpp"

namespace vpt {

VPT_HD uint32_t span_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return uint32_t(__popc(x));
#else
    return uint32_t(__builtin_popcount(x));
#endif
}

// bit 7 of the bytes of the word at `addr` that lie inside [b0, b1) (requires addr < b1, addr + 4 > b0)
VPT_HD uint32_t span_inside80(uint32_t addr, uint32_t b0, uint32_t b1) {
    const uint32_t from = b0 > addr ? b0 - addr : 0u;
    const uint32_t to = b1 - addr < 4u ? b1 - addr : 4u;
    return (from >= 4u ? 0u : 0x80808080u << (8 * from)) & (0x80808080u >> (8 * (4 - to)));
}

// bit 7 of the bytes of `in80` that start a character (every byte but 10xxxxxx)
VPT_HD uint32_t span_starts80(uint32_t w, uint32_t in80) { return ~(w & ~(w << 1)) & in80; }

// bit 7 of the bytes of `in80` that are '\n' (0x0A) or '\r' (0x0D): each is a whole character
VPT_HD uint32_t span_linebreaks80(uint32_t w, uint32_t in80) {
    const uint32_t n = w ^ 0x0A0A0A0Au, r = w ^ 0x0D0D0D0Du;
    const uint32_t zn = ~(((n & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | n);  // exact per byte: no carry between bytes
    const uint32_t zr = ~(((r & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | r);
    return (zn | zr) & in80;
}

// SplitLinebreaksFilter for the characters of one word: `st80` its character starts, `lb80` the line breaks among them,
// k0 the index of its first character in the document of n characters.  Boundary i lies between characters i and
// i + 1; the boundary on either side of every '\r' / '\n' becomes 1 (concurrent lanes may store 1 to the same byte).
VPT_HD void span_set_linebreaks(uint32_t st80, uint32_t lb80, uint32_t k0, uint32_t n, uint8_t* bnd) {
    uint32_t k = k0;
    for (int j = 0; j < 4; ++j) {
        const uint32_t bit = 0x80u << (8 * j);
        if (!(st80 & bit)) continue;
        if (lb80 & bit) {
            if (k > 0) bnd[k - 1] = 1;
            if (k + 1 < n) bnd[k] = 1;
        }
        ++k;
    }
}

// bit 7 of the character starts of `st80` that begin a token after the first one: the boundary before the character
// (index k - 1) is set.  k0: index of the word's first character in the document.
VPT_HD uint32_t span_token_starts80(uint32_t st80, uint32_t k0, const uint8_t* bnd) {
    uint32_t out = 0, k = k0;
    for (int j = 0; j < 4; ++j) {
        const uint32_t bit = 0x80u << (8 * j);
        if (!(st80 & bit)) continue;
        if (k > 0 && bnd[k - 1]) out |= bit;
        ++k;
    }
    return out;
}

// Stores the byte offsets (from the document's first byte, at b0 in the window coordinates) of the token starts of
// `ts80` in the word at `addr`, in text order: the exclusive ends of the tokens before them.  Returns how many.
VPT_HD uint32_t span_store_ends(uint32_t ts80, uint32_t addr, uint32_t b0, uint32_t* ends) {
    uint32_t r = 0;
    for (int j = 0; j < 4; ++j)
        if (ts80 & (0x80u << (8 * j))) ends[r++] = addr + uint32_t(j) - b0;
    return r;
}

}  // namespace vpt
