// lines.cu — the callers either side of the scoring path, on the device (SURVEY.md §8(f) rows 1 and 2):
//
//   * line splitting: raw file bytes -> sentence byte ranges, with the semantics of Rust's `BufRead::lines`
//     that the reference CLI loops over (predict/src/main.rs:126-130): a line ends at '\n', a '\r' directly
//     before it is dropped, a final line without '\n' still counts, a trailing '\n' adds no empty line;
//   * tokenised output: `Sentence::write_tokenized_text` (sentence.rs:850-886) for sentences without tags —
//     a ' ' between tokens, a '\' before each ' ', '\' and '/' of the surface — followed by the '\n' the CLI
//     writes after every line (predict/src/main.rs:140,149); rejected lines produce the bare '\n'.
//
// Both are byte-streaming work: SWAR byte tests on 32-bit words, warp prefix sums, no tables.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <mutex>
#include <type_traits>
#include <vector>

#include "device_model.hpp"
#include "grapheme.hpp"
#include "tag_rules.hpp"
#include "textnorm.hpp"

namespace vpt {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kGraphemeSubPages = 160;  // 256-entry sub-tables of the grapheme class table (145 in Unicode 16)

__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}
__device__ __forceinline__ uint64_t warp_incl_scan_u64(uint64_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}
// (the line writers' 32-bit lengths, the column writers' 64-bit ones)
template <class Len>
__device__ __forceinline__ Len warp_incl_scan_len(Len v, int lane) {
    if constexpr (sizeof(Len) == 8) return warp_incl_scan_u64(v, lane);
    else return warp_incl_scan_u32(v, lane);
}

// bit 7 of every byte of x that is zero (exact per byte: no borrow between bytes)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) {
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}
__device__ __forceinline__ uint32_t eq_bytes(uint32_t x, uint32_t c) { return zero_bytes(x ^ (c * 0x01010101u)); }

// bit 7 of the bytes of the word at `addr` that lie inside [b0, b1) (requires addr < b1, addr + 4 > b0)
__device__ __forceinline__ uint32_t inside80(uint32_t addr, uint32_t b0, uint32_t b1) {
    const uint32_t from = b0 > addr ? b0 - addr : 0u;
    const uint32_t to = b1 - addr < 4u ? b1 - addr : 4u;
    return (from >= 4u ? 0u : 0x80808080u << (8 * from)) & (0x80808080u >> (8 * (4 - to)));
}

// ------------------------------------------------------------------------------------------------
// line splitting
// ------------------------------------------------------------------------------------------------
constexpr int kSplitThreads = 256;
constexpr int kSplitBytesPerThread = kSplitBlockBytes / kSplitThreads;  // 32
static_assert(kSplitBytesPerThread == 32, "two 16-byte loads per thread");

// '\n' bytes of the thread's 32 bytes as a bit mask (bit i = byte i), bytes at or beyond n_bytes excluded
__device__ __forceinline__ uint32_t newline_mask(const uint8_t* __restrict__ text, uint64_t n_bytes, uint64_t pos) {
    uint32_t mask = 0;
    if (pos >= n_bytes) return 0;
    const uint4* p = reinterpret_cast<const uint4*>(text + pos);
    const uint4 v0 = __ldg(p);
    const uint4 v1 = pos + 16 < n_bytes ? __ldg(p + 1) : make_uint4(0, 0, 0, 0);
    const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t z = eq_bytes(w[i], 0x0Au);
        mask |= (((z >> 7) | (z >> 14) | (z >> 21) | (z >> 28)) & 15u) << (4 * i);
    }
    const uint64_t left = n_bytes - pos;
    if (left < 32) mask &= (1u << left) - 1u;
    return mask;
}

// pass 1: number of '\n' in every 8 KB block
__global__ void __launch_bounds__(kSplitThreads) k_nl_count(SplitArgs s) {
    __shared__ uint32_t s_w[kSplitThreads / 32];
    const uint64_t pos = uint64_t(blockIdx.x) * kSplitBlockBytes + uint64_t(threadIdx.x) * kSplitBytesPerThread;
    const uint32_t c = __popc(newline_mask(s.text, s.n_bytes, pos));
    const uint32_t w = __reduce_add_sync(kFull, c);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < kSplitThreads / 32; ++i) t += s_w[i];
        s.blk[blockIdx.x] = t;
    }
}

// pass 2 (one CTA): exclusive scan of the block counts; *n_lines = newlines (+1 for an unterminated last line)
__global__ void __launch_bounds__(1024) k_nl_scan(SplitArgs s, uint64_t nblk) {
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint64_t base = 0; base < nblk; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        const uint32_t v = i < nblk ? s.blk[i] : 0u;
        const uint32_t incl = warp_incl_scan_u32(v, lane);
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = s_w[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint64_t o = __shfl_up_sync(kFull, w, d);
                if (lane >= d) w += o;
            }
            s_w[lane] = w;
        }
        __syncthreads();
        const uint64_t excl = s_carry + (warp ? s_w[warp - 1] : 0) + incl - v;
        if (i < nblk) s.blk_base[i] = excl;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += s_w[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const bool open_tail = s.n_bytes > 0 && s.text[s.n_bytes - 1] != 0x0A;
        const uint64_t nl = s_carry + (open_tail ? 1 : 0);
        *s.n_lines = nl;
        if (s.n_lines_host) *s.n_lines_host = nl;
    }
}

// pass 3: line l ends at its '\n' (exclusive): offsets[l + 1] = position after it, trims[l] = 1 (+1 for "\r\n")
__global__ void __launch_bounds__(kSplitThreads) k_nl_write(SplitArgs s) {
    __shared__ uint32_t s_w[kSplitThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t pos = uint64_t(blockIdx.x) * kSplitBlockBytes + uint64_t(threadIdx.x) * kSplitBytesPerThread;
    uint32_t mask = newline_mask(s.text, s.n_bytes, pos);
    const uint32_t c = __popc(mask);
    const uint32_t incl = warp_incl_scan_u32(c, lane);
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t before = incl - c;
    for (int i = 0; i < warp; ++i) before += s_w[i];
    uint64_t line = s.blk_base[blockIdx.x] + before;
    while (mask) {
        const int b = __ffs(mask) - 1;
        mask &= mask - 1;
        const uint64_t p = pos + uint64_t(b);
        s.offsets[line + 1] = p + 1;
        s.trims[line] = (p > 0 && s.text[p - 1] == 0x0D) ? 2 : 1;
        ++line;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        s.offsets[0] = 0;
        if (s.n_bytes > 0 && s.text[s.n_bytes - 1] != 0x0A) {
            const uint64_t nl = *s.n_lines;
            s.offsets[nl] = s.n_bytes;
            s.trims[nl - 1] = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// tokenised output
// ------------------------------------------------------------------------------------------------
constexpr int kTokThreads = 256;

// Tokenised output in one pass.  One CTA per 64-sentence group (groups handed out by an atomic ticket, so a
// group's predecessors are always resident or done):
//   1. one warp per sentence counts its output bytes: surface + escapes + word boundaries + the '\n';
//   2. the group's total is published and the output offset of the group is found by a decoupled look-back
//      over the predecessors' published totals (state word = 2 flag bits | 62 value bits);
//   3. one warp per sentence writes: every byte of the surface goes to  base + index + (escapes and spaces
//      before it), preceded by its own ' ' (word boundary before this character) and '\' (escape).
// kCol: the column output of vpt_tokenize_dev (k_tok_write_col): one string per document, no '\n', a rejected document
// writes nothing; document d's output offset (group base + exclusive prefix in the group) goes to col.offsets[d], its
// status to col.status[d], and its bytes are written only when they end within col.capacity.  Lengths, in-group sums and output indexes are 64-bit there
// (a batch of 1 GiB documents); the line writers' 32-bit ones are safe for the line ring's chunks (kMaxLineChunk).
constexpr uint64_t kStAgg = 1ull << 62, kStIncl = 2ull << 62, kStMask = (1ull << 62) - 1;

template <bool kCol>
__device__ __forceinline__ void tok_write(const TokArgs& t, uint64_t ngroups, const ColOut& col) {
    using Len = std::conditional_t<kCol, uint64_t, uint32_t>;
    __shared__ uint64_t s_off[kGroup + 1], s_bo[kGroup];
    __shared__ uint32_t s_nch[kGroup];
    __shared__ Len s_len[kGroup], s_excl[kGroup];
    __shared__ uint8_t s_trim[kGroup], s_bad[kGroup];
    __shared__ uint64_t s_base;
    __shared__ uint32_t s_grp;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_grp = atomicAdd(t.ticket, 1u);
    __syncthreads();
    const uint64_t grp = s_grp;
    const uint64_t gbase = grp * kGroup;
    const int ns = int(min(uint64_t(kGroup), t.n_sent - gbase));
    if (threadIdx.x <= ns) s_off[threadIdx.x] = t.offsets[gbase + threadIdx.x];
    if (threadIdx.x < ns) {
        const uint64_t s = gbase + threadIdx.x;
        s_bo[threadIdx.x] = t.bound_offsets[s];
        s_nch[threadIdx.x] = t.n_chars[s];
        s_trim[threadIdx.x] = t.trims ? t.trims[s] : uint8_t(0);
        s_bad[threadIdx.x] = t.status[s] != 0;
    }
    __syncthreads();

    // ---- 1. output bytes per sentence -------------------------------------------------------------------
    // A sentence that fits one 128-byte window (the common case) is analysed once: its word, flag masks and
    // per-lane output index stay in registers for step 3.  Longer sentences are only counted here.
    constexpr int kPerWarp = kGroup / (kTokThreads / 32);
    uint32_t r_lo[kPerWarp], r_fl[kPerWarp], r_at[kPerWarp];
#pragma unroll
    for (int it = 0; it < kPerWarp; ++it) {
        const int i = warp + it * (kTokThreads / 32);
        Len len = 0;
        r_lo[it] = 0; r_fl[it] = 0; r_at[it] = 0;
        if (i < ns) {
            if constexpr (!kCol) len = 1;  // the '\n'
            if (!s_bad[i]) {
                const uint64_t o0 = s_off[i];
                const uint64_t a0 = o0 & ~3ull;
                const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(s_off[i + 1] - a0) - s_trim[i];
                const uint8_t* __restrict__ base = t.text + a0;
                if (b1 <= 128u) {
                    const uint32_t addr = 4u * uint32_t(lane);
                    uint32_t lo = 0, in80 = 0;
                    if (addr < b1) {
                        lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
                        in80 = inside80(addr, b0, b1);
                    }
                    const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;  // character starts (not 10xxxxxx)
                    const uint32_t nst = __popc(st80);
                    const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
                    const uint8_t* __restrict__ bnd = t.boundaries + s_bo[i];
                    uint32_t sp80 = 0, k = st_incl - nst;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (st80 & (0x80u << (8 * j))) {
                            if (k >= 1 && bnd[k - 1] == 1) sp80 |= 0x80u << (8 * j);
                            ++k;
                        }
                    }
                    const uint32_t esc80 = (eq_bytes(lo, 0x20u) | eq_bytes(lo, 0x2Fu) | eq_bytes(lo, 0x5Cu)) & in80;
                    const uint32_t nex = __popc(sp80) + __popc(esc80);
                    const uint32_t ex_incl = warp_incl_scan_u32(nex, lane);
                    r_lo[it] = lo;
                    r_fl[it] = in80 | (sp80 >> 1) | (esc80 >> 2);
                    r_at[it] = (addr - b0) + ex_incl - nex;
                    len += (b1 - b0) + __shfl_sync(kFull, ex_incl, 31);
                } else {
                    uint32_t cnt = 0;
                    for (uint32_t addr = 4u * uint32_t(lane); addr < b1; addr += 128) {
                        const uint32_t lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
                        cnt += __popc((eq_bytes(lo, 0x20u) | eq_bytes(lo, 0x2Fu) | eq_bytes(lo, 0x5Cu)) & inside80(addr, b0, b1));
                    }
                    const uint32_t nch = s_nch[i];
                    if (nch > 1) {
                        const uint64_t q0 = s_bo[i];
                        const uint64_t qa = q0 & ~3ull;
                        const uint32_t c0 = uint32_t(q0 - qa), c1 = c0 + nch - 1;
                        const uint8_t* __restrict__ bb = t.boundaries + qa;
                        for (uint32_t addr = 4u * uint32_t(lane); addr < c1; addr += 128) {
                            const uint32_t w = *reinterpret_cast<const uint32_t*>(bb + addr);
                            cnt += __popc(eq_bytes(w, 1u) & inside80(addr, c0, c1));
                        }
                    }
                    len += Len(b1 - b0) + __reduce_add_sync(kFull, cnt);
                }
            }
        }
        if (lane == 0) s_len[i] = len;
    }
    __syncthreads();

    // ---- 2. offsets: scan inside the group, look-back across groups -----------------------------------------
    if (warp == 0) {
        const Len v0 = s_len[2 * lane], v1 = s_len[2 * lane + 1];
        const Len iv = warp_incl_scan_len<Len>(v0 + v1, lane);
        s_excl[2 * lane] = iv - v0 - v1;
        s_excl[2 * lane + 1] = iv - v1;
        const uint64_t total = __shfl_sync(kFull, iv, 31);
        volatile uint64_t* state = t.tok_state;
        if (lane == 0) state[grp] = (grp == 0 ? kStIncl : kStAgg) | total;
        uint64_t prefix = 0;
        if (grp > 0) {
            int64_t idx = int64_t(grp) - 1;
            for (;;) {
                const int64_t j = idx - lane;
                uint64_t v = kStIncl;  // groups before the first: inclusive prefix 0
                if (j >= 0) {
                    do { v = state[j]; } while ((v >> 62) == 0);
                }
                // nearest predecessor (lowest lane) that already knows its inclusive prefix
                const unsigned incl = __ballot_sync(kFull, (v >> 62) == 2);
                const int stop = incl ? __ffs(incl) - 1 : 32;
                uint64_t add = lane <= stop ? (v & kStMask) : 0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
                prefix += add;
                if (incl) break;
                idx -= 32;
            }
            if (lane == 0) state[grp] = kStIncl | (prefix + total);
        }
        if (lane == 0) {
            s_base = prefix;
            if (grp + 1 == ngroups) {
                *t.total = prefix + total;
                if (t.total_host) *t.total_host = prefix + total;
            }
        }
    }
    __syncthreads();

    // ---- 3. write ---------------------------------------------------------------------------------------------
    const uint64_t gout = s_base;
#pragma unroll
    for (int it = 0; it < kPerWarp; ++it) {
        const int i = warp + it * (kTokThreads / 32);
        if (i >= ns) continue;
        if constexpr (kCol) {
            if (lane == 0) {
                col.offsets[gbase + i] = gout + s_excl[i];
                col.status[gbase + i] = uint8_t(t.status[gbase + i]);
            }
            if (s_bad[i] || gout + s_excl[i] + s_len[i] > col.capacity) continue;
        }
        uint8_t* __restrict__ out = t.out + gout + s_excl[i];
        if constexpr (!kCol) {
            if (s_bad[i]) {
                if (lane == 0) out[0] = 0x0A;
                continue;
            }
            if (lane == 0) out[s_len[i] - 1] = 0x0A;
        }
        const uint64_t o0 = s_off[i];
        const uint64_t a0 = o0 & ~3ull;
        const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(s_off[i + 1] - a0) - s_trim[i];
        if (b1 <= 128u) {
            const uint32_t lo = r_lo[it], fl = r_fl[it];
            uint32_t at = r_at[it];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (fl & bit) {
                    if (fl & (bit >> 1)) out[at++] = 0x20;
                    if (fl & (bit >> 2)) out[at++] = 0x5C;
                    out[at] = uint8_t(lo >> (8 * j));
                }
                ++at;
            }
            continue;
        }
        const uint8_t* __restrict__ base = t.text + a0;
        const uint8_t* __restrict__ bnd = t.boundaries + s_bo[i];
        uint32_t chars = 0;  // characters before this window
        Len extra = 0;       // inserted bytes before this window
        for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
            const uint32_t addr = w0 + 4u * uint32_t(lane);
            uint32_t lo = 0, in80 = 0;
            if (addr < b1) {
                lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
                in80 = inside80(addr, b0, b1);
            }
            const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;
            const uint32_t nst = __popc(st80);
            const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
            // a ' ' goes before character k >= 1 when boundary k-1 is a word boundary
            uint32_t sp80 = 0;
            {
                uint32_t k = chars + st_incl - nst;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (st80 & (0x80u << (8 * j))) {
                        if (k >= 1 && bnd[k - 1] == 1) sp80 |= 0x80u << (8 * j);
                        ++k;
                    }
                }
            }
            const uint32_t esc80 = (eq_bytes(lo, 0x20u) | eq_bytes(lo, 0x2Fu) | eq_bytes(lo, 0x5Cu)) & in80;
            const uint32_t nex = __popc(sp80) + __popc(esc80);
            const uint32_t ex_incl = warp_incl_scan_u32(nex, lane);
            Len at = Len(addr) - b0 + extra + ex_incl - nex;  // output index of byte 0 of this word (if inside)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (in80 & bit) {
                    if (sp80 & bit) out[at++] = 0x20;
                    if (esc80 & bit) out[at++] = 0x5C;
                    out[at] = uint8_t(lo >> (8 * j));
                }
                ++at;
            }
            chars += __shfl_sync(kFull, st_incl, 31);
            extra += __shfl_sync(kFull, ex_incl, 31);
        }
    }
}

__global__ void __launch_bounds__(kTokThreads) k_tok_write(TokArgs t, uint64_t ngroups) { tok_write<false>(t, ngroups, ColOut()); }
// (one resident block per SM as the bound: ptxas then keeps the 64-bit indexes in registers instead of spilling them)
__global__ void __launch_bounds__(kTokThreads, 1) k_tok_write_col(TokArgs t, uint64_t ngroups, ColOut col) {
    tok_write<true>(t, ngroups, col);
}

// ---- tokenised output with tags (the CLI's --predict-tags: main.rs:130-136,159-166 + sentence.rs:850-886) ------------------
// Same three steps as k_tok_write; every token's surface is followed by '/' + tag for its tag slots up to the last one
// that has a tag (an empty string for a slot without one), the strings escaped like the surface.  The suffix of the
// token that ends in front of a character travels with that character's ' ' (it is written right before it); the last
// token's suffix goes in front of the '\n'.  A token's record is tok_base[sentence] + (word boundaries before it).
// kRules: PatternMatchTagger's rules fill the slots the model left empty (tag_rules.hpp); without them the code is the
// model-only writer.
template <bool kRules>
__device__ __forceinline__ uint32_t tag_suffix_len(const TokArgs& t, const TagRuleArgs& ra, uint64_t rec) {
    if constexpr (kRules)
        return merged_suffix_len(t.n_tags, t.tok_ids[rec], t.tok_cands + rec * t.n_tags, t.ts_slot, t.ts_cand, t.ts_ref,
                                 ra.tok_rule[rec], ra.rules);
    const int32_t tid = t.tok_ids[rec];
    if (tid < 0) return 0;
    const uint32_t sb = __ldg(t.ts_slot + tid);
    uint32_t len = 0, run = 0;
    for (uint32_t k = 0; k < t.n_tags; ++k) {
        const uint32_t c = t.tok_cands[rec * t.n_tags + k];
        ++run;  // the '/'
        if (c != 255u) {
            run += __ldg(t.ts_ref + __ldg(t.ts_cand + sb + k) + c).y;
            len += run;  // slots up to this one count
            run = 0;
        }
    }
    return len;
}
template <bool kRules>
__device__ __forceinline__ void tag_suffix_write(const TokArgs& t, const TagRuleArgs& ra, uint64_t rec, uint8_t* __restrict__ out) {
    if constexpr (kRules) {
        merged_suffix_write(t.n_tags, t.tok_ids[rec], t.tok_cands + rec * t.n_tags, t.ts_slot, t.ts_cand, t.ts_ref,
                            t.ts_bytes, ra.tok_rule[rec], ra.rules, out);
        return;
    }
    const int32_t tid = t.tok_ids[rec];
    if (tid < 0) return;
    const uint32_t sb = __ldg(t.ts_slot + tid);
    int last = -1;
    for (uint32_t k = 0; k < t.n_tags; ++k) if (t.tok_cands[rec * t.n_tags + k] != 255u) last = int(k);
    uint32_t at = 0;
    for (int k = 0; k <= last; ++k) {
        out[at++] = 0x2F;
        const uint32_t c = t.tok_cands[rec * t.n_tags + k];
        if (c == 255u) continue;
        const uint2 ref = __ldg(t.ts_ref + __ldg(t.ts_cand + sb + k) + c);
        for (uint32_t j = 0; j < ref.y; ++j) out[at++] = __ldg(t.ts_bytes + ref.x + j);
    }
}

// One sentence by one warp: returns the output length without the '\n'; writes the bytes when kWrite.  Len: the type of
// the sentence's output indexes (uint64_t for the column writers).
template <bool kWrite, bool kRules, class Len>
__device__ __forceinline__ Len tagged_sentence(const TokArgs& t, const TagRuleArgs& ra, uint64_t s, uint64_t o0, uint64_t o1, uint32_t trim, uint32_t nch,
                                                    uint8_t* __restrict__ out, int lane) {
    const uint64_t a0 = o0 & ~3ull;
    const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(o1 - a0) - trim;
    const uint8_t* __restrict__ base = t.text + a0;
    const uint8_t* __restrict__ bnd = t.boundaries + t.bound_offsets[s];
    const uint64_t rec0 = t.tok_base[s];
    // characters / inserted bytes / tokens that ended before this window
    uint32_t chars = 0;
    Len extra = 0;
    uint32_t toks = 0;
    for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t lo = 0, in80 = 0;
        if (addr < b1) {
            lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
            in80 = inside80(addr, b0, b1);
        }
        const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;
        const uint32_t nst = __popc(st80);
        const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
        // a ' ' (and the suffix of the token that just ended) goes before character k >= 1 when boundary k-1 is set
        uint32_t sp80 = 0;
        {
            uint32_t k = chars + st_incl - nst;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (st80 & (0x80u << (8 * j))) {
                    if (k >= 1 && bnd[k - 1] == 1) sp80 |= 0x80u << (8 * j);
                    ++k;
                }
            }
        }
        const uint32_t nsp = __popc(sp80);
        const uint32_t sp_incl = warp_incl_scan_u32(nsp, lane);
        uint32_t sl[4] = {0, 0, 0, 0}, sl_sum = 0;
        {
            uint64_t rec = rec0 + toks + sp_incl - nsp;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (sp80 & (0x80u << (8 * j))) {
                    sl[j] = tag_suffix_len<kRules>(t, ra, rec);
                    sl_sum += sl[j];
                    ++rec;
                }
            }
        }
        const uint32_t esc80 = (eq_bytes(lo, 0x20u) | eq_bytes(lo, 0x2Fu) | eq_bytes(lo, 0x5Cu)) & in80;
        const uint32_t nex = nsp + __popc(esc80) + sl_sum;
        const uint32_t ex_incl = warp_incl_scan_u32(nex, lane);
        if (kWrite) {
            Len at = Len(addr) - b0 + extra + ex_incl - nex;  // output index of byte 0 of this word (if inside)
            uint64_t rec = rec0 + toks + sp_incl - nsp;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (in80 & bit) {
                    if (sp80 & bit) {
                        tag_suffix_write<kRules>(t, ra, rec, out + at);
                        at += sl[j];
                        ++rec;
                        out[at++] = 0x20;
                    }
                    if (esc80 & bit) out[at++] = 0x5C;
                    out[at] = uint8_t(lo >> (8 * j));
                }
                ++at;
            }
        }
        extra += __shfl_sync(kFull, ex_incl, 31);
        chars += __shfl_sync(kFull, st_incl, 31);
        toks += __shfl_sync(kFull, sp_incl, 31);
    }
    Len len = Len(b1 - b0) + extra;
    if (nch > 0) {
        const uint32_t last = tag_suffix_len<kRules>(t, ra, rec0 + toks);
        if (kWrite && lane == 0) tag_suffix_write<kRules>(t, ra, rec0 + toks, out + len);
        len += last;
    }
    return len;
}

// kCol: the column output, as tok_write<true>
template <bool kRules, bool kCol>
__device__ __forceinline__ void tok_write_tags(const TokArgs& t, uint64_t ngroups, const TagRuleArgs& ra, const ColOut& col) {
    using Len = std::conditional_t<kCol, uint64_t, uint32_t>;
    __shared__ uint64_t s_off[kGroup + 1];
    __shared__ uint32_t s_nch[kGroup];
    __shared__ Len s_len[kGroup], s_excl[kGroup];
    __shared__ uint8_t s_trim[kGroup], s_bad[kGroup];
    __shared__ uint64_t s_base;
    __shared__ uint32_t s_grp;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_grp = atomicAdd(t.ticket, 1u);
    __syncthreads();
    const uint64_t grp = s_grp;
    const uint64_t gbase = grp * kGroup;
    const int ns = int(min(uint64_t(kGroup), t.n_sent - gbase));
    if (threadIdx.x <= ns) s_off[threadIdx.x] = t.offsets[gbase + threadIdx.x];
    if (threadIdx.x < kGroup) s_len[threadIdx.x] = 0;
    if (threadIdx.x < ns) {
        const uint64_t s = gbase + threadIdx.x;
        s_nch[threadIdx.x] = t.n_chars[s];
        s_trim[threadIdx.x] = t.trims ? t.trims[s] : uint8_t(0);
        s_bad[threadIdx.x] = t.status[s] != 0;
    }
    __syncthreads();
    // 1. output bytes per sentence
    for (int i = warp; i < ns; i += kTokThreads / 32) {
        Len len = kCol ? 0 : 1;  // the '\n'
        if (!s_bad[i]) len += tagged_sentence<false, kRules, Len>(t, ra, gbase + i, s_off[i], s_off[i + 1], s_trim[i], s_nch[i], nullptr, lane);
        if (lane == 0) s_len[i] = len;
    }
    __syncthreads();
    // 2. offsets: scan inside the group, look-back across groups (as k_tok_write)
    if (warp == 0) {
        const Len v0 = s_len[2 * lane], v1 = s_len[2 * lane + 1];
        const Len iv = warp_incl_scan_len<Len>(v0 + v1, lane);
        s_excl[2 * lane] = iv - v0 - v1;
        s_excl[2 * lane + 1] = iv - v1;
        const uint64_t total = __shfl_sync(kFull, iv, 31);
        volatile uint64_t* state = t.tok_state;
        if (lane == 0) state[grp] = (grp == 0 ? kStIncl : kStAgg) | total;
        uint64_t prefix = 0;
        if (grp > 0) {
            int64_t idx = int64_t(grp) - 1;
            for (;;) {
                const int64_t j = idx - lane;
                uint64_t v = kStIncl;
                if (j >= 0) {
                    do { v = state[j]; } while ((v >> 62) == 0);
                }
                const unsigned incl = __ballot_sync(kFull, (v >> 62) == 2);
                const int stop = incl ? __ffs(incl) - 1 : 32;
                uint64_t add = lane <= stop ? (v & kStMask) : 0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
                prefix += add;
                if (incl) break;
                idx -= 32;
            }
            if (lane == 0) state[grp] = kStIncl | (prefix + total);
        }
        if (lane == 0) {
            s_base = prefix;
            if (grp + 1 == ngroups) {
                *t.total = prefix + total;
                if (t.total_host) *t.total_host = prefix + total;
            }
        }
    }
    __syncthreads();
    // 3. write
    const uint64_t gout = s_base;
    for (int i = warp; i < ns; i += kTokThreads / 32) {
        if constexpr (kCol) {
            if (lane == 0) {
                col.offsets[gbase + i] = gout + s_excl[i];
                col.status[gbase + i] = uint8_t(t.status[gbase + i]);
            }
            if (s_bad[i] || gout + s_excl[i] + s_len[i] > col.capacity) continue;
        }
        uint8_t* __restrict__ out = t.out + gout + s_excl[i];
        if constexpr (!kCol) {
            if (lane == 0) out[s_len[i] - 1] = 0x0A;
        }
        if (!s_bad[i]) tagged_sentence<true, kRules, Len>(t, ra, gbase + i, s_off[i], s_off[i + 1], s_trim[i], s_nch[i], out, lane);
    }
}

// (kRules: one resident block per SM is enough for ptxas to keep the merge in registers; min blocks 0 is the bound
// without a minimum, so the path without rules compiles as before)
template <bool kRules>
__global__ void __launch_bounds__(kTokThreads, kRules ? 1 : 0) k_tok_write_tags(TokArgs t, uint64_t ngroups, TagRuleArgs ra) {
    tok_write_tags<kRules, false>(t, ngroups, ra, ColOut());
}
template <bool kRules>
__global__ void __launch_bounds__(kTokThreads, kRules ? 1 : 0) k_tok_write_tags_col(TokArgs t, uint64_t ngroups, TagRuleArgs ra,
                                                                                     ColOut col) {
    tok_write_tags<kRules, true>(t, ngroups, ra, col);
}

// KyteaWsConstFilter (vaporetto_rules/src/sentence_filters/kytea_wsconst.rs:27-44) for a set of character types —
// the CLI's --wsconst D/R/H/T/K/O options, applied after prediction (predict/src/main.rs:100-106,157): boundary i
// becomes NotWordBoundary when characters i and i+1 have the same type and that type is in `mask` (bit t = type t).
// The types are those of the text the predictor saw, i.e. of the full-width filtered characters when norm != 0.
// One warp per sentence, 128 bytes per step; only zeros are written, the scores stay as they are.
__global__ void __launch_bounds__(kTokThreads) k_wsconst(TokArgs t, uint8_t* __restrict__ boundaries, uint32_t mask, int norm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t gbase = uint64_t(blockIdx.x) * kGroup;
    const int ns = int(min(uint64_t(kGroup), t.n_sent - gbase));
    for (int i = warp; i < ns; i += kTokThreads / 32) {
        const uint64_t s = gbase + i;
        if (t.status[s] != 0 || t.n_chars[s] < 2) continue;
        const uint64_t o0 = t.offsets[s];
        const uint64_t a0 = o0 & ~3ull;
        const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(t.offsets[s + 1] - a0) - (t.trims ? t.trims[s] : 0);
        const uint8_t* __restrict__ base = t.text + a0;
        uint8_t* __restrict__ bnd = boundaries + t.bound_offsets[s];
        uint32_t chars = 0;    // characters before this window
        uint32_t prev_ty = 0;  // type of the last character before this window (0: none yet)
        for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
            const uint32_t addr = w0 + 4u * uint32_t(lane);
            uint32_t lo = 0, hi = 0, in80 = 0;
            if (addr < b1) {
                lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
                if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(base + addr + 4));
                in80 = inside80(addr, b0, b1);
            }
            const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;  // character starts (not 10xxxxxx)
            const uint32_t nst = __popc(st80);
            const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
            // types of this lane's characters in order, 3 bits each
            uint32_t tys = 0, cnt = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (st80 & (0x80u << (8 * j))) {
                    uint32_t c = decode_cp(__funnelshift_r(lo, hi, 8 * j));
                    if (norm) c = kytea_fullwidth(c);
                    tys |= char_type(c) << (3 * cnt);
                    ++cnt;
                }
            }
            // f = type of the first character at or after this lane inside the window (0: none)
            uint32_t f = cnt ? (tys & 7u) : 0u;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t v = __shfl_down_sync(kFull, f, d);
                if (f == 0 && lane + d < 32) f = v;
            }
            uint32_t next_first = __shfl_down_sync(kFull, f, 1);
            if (lane == 31) next_first = 0;
            const uint32_t k = chars + st_incl - nst;  // index of this lane's first character
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (uint32_t(q) < cnt) {
                    const uint32_t ta = (tys >> (3 * q)) & 7u;
                    const uint32_t tb = uint32_t(q) + 1 < cnt ? (tys >> (3 * (q + 1))) & 7u : next_first;
                    if (tb != 0 && ta == tb && ((mask >> ta) & 1u)) bnd[k + q] = 0;
                }
            }
            // the pair across the window edge: last character before this window / first character of it
            const uint32_t f0 = __shfl_sync(kFull, f, 0);
            if (lane == 0 && prev_ty != 0 && f0 == prev_ty && ((mask >> f0) & 1u)) bnd[chars - 1] = 0;
            const unsigned has = __ballot_sync(kFull, cnt > 0);
            if (has) {
                const uint32_t last = cnt ? (tys >> (3 * (cnt - 1))) & 7u : 0u;
                prev_ty = __shfl_sync(kFull, last, 31 - __clz(has));
            }
            chars += __shfl_sync(kFull, st_incl, 31);
        }
    }
}

// ConcatGraphemeClustersFilter (vaporetto_rules/src/sentence_filters/concat_grapheme_clusters.rs:10-35) — the CLI's
// `--wsconst G`: every boundary inside an extended grapheme cluster (UAX #29, grapheme.hpp) becomes NotWordBoundary.
// One warp per sentence, 128 bytes per step: the lanes decode their characters and look their classes up in a two-level
// table; a window whose characters all have the default class (Japanese text: almost every window) has a cluster
// boundary before each of its characters and leaves the rule state clean, so only windows with marks, emoji, Hangul
// jamo, regional indicators ... run the rule engine, all lanes in step over the window's class words in shared memory.
__device__ uint16_t g_gr_page[0x1100];              // page c >> 8: 0x8000 | class for a uniform page, else sub-table index
__device__ uint8_t g_gr_cls[kGraphemeSubPages * 256];

__device__ __forceinline__ uint32_t grapheme_class_dev(uint32_t c) {
    const uint32_t pg = g_gr_page[c >> 8];
    return (pg & 0x8000u) ? (pg & 0x7Fu) : uint32_t(g_gr_cls[(pg << 8) + (c & 255u)]);
}

__global__ void __launch_bounds__(kTokThreads) k_grapheme(TokArgs t, uint8_t* __restrict__ boundaries, int norm) {
    __shared__ uint8_t s_cw[kTokThreads / 32][128];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t gbase = uint64_t(blockIdx.x) * kGroup;
    const int ns = int(min(uint64_t(kGroup), t.n_sent - gbase));
    for (int i = warp; i < ns; i += kTokThreads / 32) {
        const uint64_t s = gbase + i;
        if (t.status[s] != 0 || t.n_chars[s] < 2) continue;
        const uint64_t o0 = t.offsets[s];
        const uint64_t a0 = o0 & ~3ull;
        const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(t.offsets[s + 1] - a0) - (t.trims ? t.trims[s] : 0);
        const uint8_t* __restrict__ base = t.text + a0;
        uint8_t* __restrict__ bnd = boundaries + t.bound_offsets[s];
        uint32_t chars = 0;  // characters before this window
        GraphemeState st;    // (the same in every lane)
        for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
            const uint32_t addr = w0 + 4u * uint32_t(lane);
            uint32_t lo = 0, hi = 0, in80 = 0;
            if (addr < b1) {
                lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
                if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(base + addr + 4));
                in80 = inside80(addr, b0, b1);
            }
            const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;  // character starts (not 10xxxxxx)
            const uint32_t nst = __popc(st80);
            const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
            const uint32_t nwin = __shfl_sync(kFull, st_incl, 31);
            uint32_t k = st_incl - nst, any = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (st80 & (0x80u << (8 * j))) {
                    uint32_t c = decode_cp(__funnelshift_r(lo, hi, 8 * j));
                    if (norm) c = kytea_fullwidth(c);
                    const uint32_t cw = grapheme_class_dev(c);
                    s_cw[warp][k++] = uint8_t(cw);
                    any |= cw;
                }
            }
            // (a default-class character still joins a Prepend character in front of it: GB9b)
            if (__any_sync(kFull, any != 0) || (st.started && (st.prev & 15u) == kGcbPrepend)) {
                __syncwarp();
                for (uint32_t q = 0; q < nwin; ++q) {
                    const bool brk = grapheme_step(st, s_cw[warp][q]);
                    if (!brk && chars + q > 0 && lane == 0) bnd[chars + q - 1] = 0;
                }
                __syncwarp();
            } else if (nwin) {
                st = GraphemeState();
                st.started = 1;
            }
            chars += nwin;
        }
    }
}

}  // namespace

namespace {
// two-level class table from the sorted ranges of grapheme_tables.hpp (built once, uploaded once per device)
struct GraphemeHostTable {
    std::vector<uint16_t> page;
    std::vector<uint8_t> cls;
    GraphemeHostTable() : page(0x1100, uint16_t(0x8000)) {
        std::vector<uint8_t> flat(0x110000, 0);
        for (int r = 0; r < kGraphemeRanges; ++r)
            for (uint32_t c = kGraphemeTable[r].lo; c <= kGraphemeTable[r].hi; ++c) flat[c] = uint8_t(kGraphemeTable[r].cls);
        for (uint32_t p = 0; p < 0x1100; ++p) {
            bool uniform = true;
            for (uint32_t c = 1; c < 256 && uniform; ++c) uniform = flat[(p << 8) + c] == flat[p << 8];
            if (uniform) { page[p] = uint16_t(0x8000u | flat[p << 8]); continue; }
            page[p] = uint16_t(cls.size() >> 8);
            cls.insert(cls.end(), flat.begin() + (p << 8), flat.begin() + (p << 8) + 256);
        }
    }
};
}  // namespace

cudaError_t launch_grapheme(const TokArgs& t, uint8_t* boundaries, bool norm, cudaStream_t stream) {
    if (t.n_sent == 0) return cudaSuccess;
    static std::mutex mu;
    static bool uploaded[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    {
        std::lock_guard<std::mutex> lock(mu);
        if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
        if (!uploaded[dev]) {
            static const GraphemeHostTable tab;
            if (tab.cls.size() > size_t(kGraphemeSubPages) * 256) return cudaErrorInvalidValue;
            // (synchronous copies: the table is in place before any kernel of any stream reads it)
            e = cudaMemcpyToSymbol(g_gr_page, tab.page.data(), tab.page.size() * 2);
            if (e != cudaSuccess) return e;
            e = cudaMemcpyToSymbol(g_gr_cls, tab.cls.data(), tab.cls.size());
            if (e != cudaSuccess) return e;
            uploaded[dev] = true;
        }
    }
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    k_grapheme<<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, boundaries, norm ? 1 : 0);
    return cudaGetLastError();
}

cudaError_t launch_wsconst(const TokArgs& t, uint8_t* boundaries, uint32_t mask, bool norm, cudaStream_t stream) {
    if (t.n_sent == 0 || (mask & 0x7Eu) == 0) return cudaSuccess;
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    k_wsconst<<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, boundaries, mask, norm ? 1 : 0);
    return cudaGetLastError();
}

cudaError_t launch_split_count(const SplitArgs& s, cudaStream_t stream) {
    const uint64_t nblk = (s.n_bytes + kSplitBlockBytes - 1) / kSplitBlockBytes;
    if (nblk) k_nl_count<<<unsigned(nblk), kSplitThreads, 0, stream>>>(s);
    k_nl_scan<<<1, 1024, 0, stream>>>(s, nblk);
    return cudaGetLastError();
}

cudaError_t launch_split_write(const SplitArgs& s, cudaStream_t stream) {
    const uint64_t nblk = (s.n_bytes + kSplitBlockBytes - 1) / kSplitBlockBytes;
    if (nblk == 0) return cudaSuccess;
    k_nl_write<<<unsigned(nblk), kSplitThreads, 0, stream>>>(s);
    return cudaGetLastError();
}

cudaError_t launch_tokenize(const TokArgs& t, cudaStream_t stream) { return launch_tokenize_rules(t, TagRuleArgs(), stream); }

cudaError_t launch_tokenize_rules(const TokArgs& t, const TagRuleArgs& ra, cudaStream_t stream) {
    if (t.n_sent == 0) return cudaMemsetAsync(t.total, 0, 8, stream);
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    // look-back state words + the ticket that follows them
    cudaError_t e = cudaMemsetAsync(t.tok_state, 0, 8 * (ngroups + 1), stream);
    if (e != cudaSuccess) return e;
    if (t.tok_base && ra.tok_rule) k_tok_write_tags<true><<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups, ra);
    else if (t.tok_base) k_tok_write_tags<false><<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups, ra);
    else k_tok_write<<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups);
    return cudaGetLastError();
}

cudaError_t launch_tokenize_column(const TokArgs& t, const TagRuleArgs& ra, const ColOut& col, cudaStream_t stream) {
    if (t.n_sent == 0) return cudaMemsetAsync(col.offsets, 0, 8, stream);
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    cudaError_t e = cudaMemsetAsync(t.tok_state, 0, 8 * (ngroups + 1), stream);
    if (e != cudaSuccess) return e;
    if (t.tok_base && ra.tok_rule) k_tok_write_tags_col<true><<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups, ra, col);
    else if (t.tok_base) k_tok_write_tags_col<false><<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups, ra, col);
    else k_tok_write_col<<<unsigned(ngroups), kTokThreads, 0, stream>>>(t, ngroups, col);
    return cudaGetLastError();
}

}  // namespace vpt
