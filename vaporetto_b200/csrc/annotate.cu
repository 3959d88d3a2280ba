// annotate.cu — partially annotated output on the device (vpt_annotate_lines): the line path's predicted sentences,
// with every boundary whose score lies strictly inside (-margin, margin) left Unknown, written in the format of the
// reference's `Sentence::write_partial_annotation_text` (sentence.rs:907-944):
//
//   * k_pa_margin (before the post-filters): boundary byte 2 (Unknown) where -margin < score < margin; the wsconst and
//     grapheme post-filters then clear what they clear, as the reference's filters overwrite Unknown;
//   * k_pa_marks (after the post-filters): the marker of every boundary ('-', '|', ' ') into its own array, and the
//     predicted boundary (score > 0) back into every byte that still holds 2, so the tag, rule and count kernels run
//     unchanged on the full segmentation;
//   * k_pa_untag (after the tag records): every token next to or across a ' ' marker loses its model tags and its rule,
//     as fill_tags (predictor.rs:567-570) and iter_tokens (sentence.rs:1273-1299) skip such tokens;
//   * k_pa_write<kTags, kRules>: the output lines, as k_tok_write / k_tok_write_tags (lines.cu) write theirs
//     (separate kernels, so that those keep their compiled code): one warp per sentence, 128 bytes per step, one CTA per 64-sentence group with a decoupled look-back for
//     the group's output offset.  A marker goes before every character after the first; a token's "/tag" suffix goes
//     in front of the marker after its last character (the last token's in front of the '\n').  Nothing is escaped:
//     the tag strings, stored escaped (tags_build.cpp, tag_rules.hpp), are copied without their '\' escapes;
//   * k_pa_rewrite<kTags, kRules> (vpt_reannotate_lines): k_pa_write's body with the caller's input tags, which go after
//     any character that carries them (k_part_tags, partial.cu, found where in the chunk's input), in place of the
//     suffix of the token it ends.
#include <cuda_runtime.h>

#include <cstdint>

#include "byte_window.cuh"
#include "device_model.hpp"
#include "tag_rules.hpp"

namespace vpt {

namespace {

using bw::inside80;
using bw::kFull;
using bw::warp_incl_scan_u32;

constexpr int kAnThreads = 256;
constexpr int kWarps = kAnThreads / 32;
constexpr uint64_t kStAgg = 1ull << 62, kStIncl = 2ull << 62, kStMask = (1ull << 62) - 1;

// One warp per sentence, 32 boundaries per step
__global__ void __launch_bounds__(kAnThreads) k_pa_margin(AnnArgs a) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t l = uint64_t(blockIdx.x) * kWarps + warp;
    if (l >= a.n_sent || a.status[l] != 0) return;
    const uint32_t nb = a.n_chars[l] - 1;
    const uint64_t bo = a.bound_offsets[l];
    const int32_t m = a.margin;
    for (uint32_t j = lane; j < nb; j += 32) {
        const int32_t sc = a.scores[bo + j];
        if (-m < sc && sc < m) a.boundaries[bo + j] = 2;
    }
}

__global__ void __launch_bounds__(kAnThreads) k_pa_marks(AnnArgs a) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t l = uint64_t(blockIdx.x) * kWarps + warp;
    if (l >= a.n_sent || a.status[l] != 0) return;
    const uint32_t nb = a.n_chars[l] - 1;
    const uint64_t bo = a.bound_offsets[l];
    for (uint32_t j = lane; j < nb; j += 32) {
        const uint8_t b = a.boundaries[bo + j];
        a.marks[bo + j] = b == 0 ? uint8_t('-') : b == 1 ? uint8_t('|') : uint8_t(' ');
        if (b == 2) a.boundaries[bo + j] = a.scores[bo + j] > 0 ? 1 : 0;
    }
}

// Token t of a sentence spans the characters between its t-th and (t+1)-th word boundaries; a ' ' at boundary j touches
// the token of character j and that of character j + 1 (the same token unless boundary j is a word boundary).
__global__ void __launch_bounds__(kAnThreads) k_pa_untag(AnnArgs a) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t l = uint64_t(blockIdx.x) * kWarps + warp;
    if (l >= a.n_sent || a.status[l] != 0) return;
    const uint32_t nb = a.n_chars[l] - 1;
    const uint64_t bo = a.bound_offsets[l], rec0 = a.tok_base[l];
    uint32_t toks = 0;  // word boundaries before this step
    for (uint32_t j0 = 0; j0 < nb; j0 += 32) {
        const uint32_t j = j0 + uint32_t(lane);
        const uint8_t b = j < nb ? a.boundaries[bo + j] : uint8_t(0);
        const unsigned wb = __ballot_sync(kFull, b == 1);
        if (j < nb && a.marks[bo + j] == ' ') {
            const uint64_t rec = rec0 + toks + __popc(wb & ((1u << lane) - 1u));
            a.tok_ids[rec] = -1;
            a.tok_ids[rec + b] = -1;
            if (a.tok_rule) {
                a.tok_rule[rec] = -1;
                a.tok_rule[rec + b] = -1;
            }
        }
        toks += __popc(wb);
    }
}

// vpt_reannotate_lines: the chunk's input and the input tag region of every character (k_part_tags)
struct InTags {
    const uint8_t* input = nullptr;
    const uint2* regions = nullptr;
    const uint64_t* char_offsets = nullptr;
};

// The bytes of a stored (escaped) tag string without its escapes
__device__ __forceinline__ uint32_t unescaped_len(const uint8_t* __restrict__ src, uint2 ref) {
    uint32_t n = 0;
    for (uint32_t j = 0; j < ref.y; ++j, ++n)
        if (__ldg(src + ref.x + j) == 0x5Cu) ++j;
    return n;
}
__device__ __forceinline__ uint32_t unescaped_copy(const uint8_t* __restrict__ src, uint2 ref, uint8_t* __restrict__ out) {
    uint32_t n = 0;
    for (uint32_t j = 0; j < ref.y; ++j) {
        uint8_t c = __ldg(src + ref.x + j);
        if (c == 0x5Cu) c = __ldg(src + ref.x + ++j);
        out[n++] = c;
    }
    return n;
}

// The token's "/tag/.." suffix as write_partial_annotation_text writes it: '/' + tag for every slot up to the last one
// that has a tag (merged_slot: the model's tag, else with kRules the rule's), the tags unescaped.  kWrite: writes it at
// `out`.  Returns its length.
template <bool kWrite, bool kRules>
__device__ __forceinline__ uint32_t pa_suffix(const TokArgs& t, const TagRuleArgs& ra, uint64_t rec, uint8_t* __restrict__ out) {
    const int32_t tid = t.tok_ids[rec];
    const int32_t rid = kRules ? ra.tok_rule[rec] : -1;
    if (tid < 0 && rid < 0) return 0;
    uint32_t at = 0, pending = 0;  // '/' of the slots since the last one with a tag
    for (uint32_t k = 0; k < t.n_tags; ++k) {
        uint2 ref;
        const int from = merged_slot(k, tid, t.tok_cands[rec * t.n_tags + k], t.ts_slot, t.ts_cand, t.ts_ref, rid,
                                     ra.rules, ref);
        ++pending;
        if (!from) continue;
        const uint8_t* src = from == 1 ? t.ts_bytes : ra.rules.tag_bytes;
        if (kWrite) {
            for (; pending; --pending) out[at++] = 0x2F;
            at += unescaped_copy(src, ref, out + at);
        } else {
            at += pending + unescaped_len(src, ref);
            pending = 0;
        }
    }
    return at;
}

// One sentence by one warp: returns its output length without the '\n'; writes the bytes when kWrite.  Byte x of
// character k of the sentence goes to x + k + (suffix bytes of the tokens that ended before character k); the marker of
// character k >= 1 goes right before its first byte, and the suffix of the token that ends at character k - 1 right
// before that marker.
// kIn (vpt_reannotate_lines): a character whose input tag region (`in`) is not empty gets it, unescaped, right after
// it, in place of the suffix of the token it ends; the suffix bytes in front of character k are then those of character
// k - 1, of either kind.
template <bool kWrite, bool kTags, bool kRules, bool kIn = false>
__device__ __forceinline__ uint32_t pa_sentence(const TokArgs& t, const TagRuleArgs& ra, const uint8_t* __restrict__ marks,
                                                uint64_t s, uint64_t o0, uint64_t o1, uint32_t trim, uint32_t nch,
                                                uint8_t* __restrict__ out, int lane, const InTags& in = InTags()) {
    const uint64_t a0 = o0 & ~3ull;
    const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(o1 - a0) - trim;
    if (!kWrite && !kTags && !kIn) return (b1 - b0) + nch - 1;
    const uint8_t* __restrict__ base = t.text + a0;
    const uint64_t bo = t.bound_offsets[s];
    const uint8_t* __restrict__ bnd = t.boundaries + bo;
    const uint8_t* __restrict__ mk = marks + bo;
    const uint64_t rec0 = kTags ? t.tok_base[s] : 0;
    const uint2* __restrict__ reg = kIn ? in.regions + in.char_offsets[s] : nullptr;
    uint32_t chars = 0, extra = 0, toks = 0;  // characters / suffix bytes / tokens ended, before this window
    for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t lo = 0, in80 = 0;
        if (addr < b1) {
            lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
            in80 = inside80(addr, b0, b1);
        }
        const uint32_t st80 = ~(lo & ~(lo << 1)) & in80;  // character starts (not 10xxxxxx)
        const uint32_t nst = __popc(st80);
        const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
        // word boundaries before this lane's characters: a token ended there
        uint32_t wb80 = 0;
        if (kTags) {
            uint32_t k = chars + st_incl - nst;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (st80 & (0x80u << (8 * j))) {
                    if (k >= 1 && bnd[k - 1] == 1) wb80 |= 0x80u << (8 * j);
                    ++k;
                }
            }
        }
        const uint32_t nwb = __popc(wb80);
        const uint32_t wb_incl = kTags ? warp_incl_scan_u32(nwb, lane) : 0u;
        uint32_t sl[4] = {0, 0, 0, 0}, sl_sum = 0;
        uint32_t in80s = 0;  // kIn: the character starts whose previous character has input tags
        uint2 rg[4];
        if (kIn) {
            uint32_t k = chars + st_incl - nst;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (st80 & (0x80u << (8 * j))) {
                    rg[j] = k >= 1 ? reg[k - 1] : make_uint2(0, 0);
                    if (rg[j].y) {
                        in80s |= 0x80u << (8 * j);
                        sl[j] = unescaped_len(in.input, rg[j]);
                        sl_sum += sl[j];
                    }
                    ++k;
                }
            }
        }
        if (kTags) {
            uint64_t rec = rec0 + toks + wb_incl - nwb;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (wb80 & (0x80u << (8 * j))) {
                    if (!(kIn && (in80s & (0x80u << (8 * j))))) {
                        sl[j] = pa_suffix<false, kRules>(t, ra, rec, nullptr);
                        sl_sum += sl[j];
                    }
                    ++rec;
                }
            }
        }
        const uint32_t sl_incl = (kTags || kIn) ? warp_incl_scan_u32(sl_sum, lane) : 0u;
        if (kWrite) {
            uint32_t k = chars + st_incl - nst;        // the next character that starts in this word
            uint32_t e = extra + sl_incl - sl_sum;     // suffix bytes in front of character k - 1
            uint64_t rec = rec0 + toks + wb_incl - nwb;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (!(in80 & bit)) continue;
                const uint32_t x = addr + uint32_t(j) - b0;
                if (st80 & bit) {
                    if (k >= 1) {
                        if (kIn && (in80s & bit)) {
                            e += sl[j];
                            unescaped_copy(in.input, rg[j], out + x + k + e - 1 - sl[j]);
                            if (kTags && (wb80 & bit)) ++rec;
                        } else if (kTags && (wb80 & bit)) {
                            e += sl[j];
                            pa_suffix<true, kRules>(t, ra, rec, out + x + k + e - 1 - sl[j]);
                            ++rec;
                        }
                        out[x + k + e - 1] = mk[k - 1];
                    }
                    ++k;
                }
                out[x + (k - 1) + e] = uint8_t(lo >> (8 * j));  // a byte of character k - 1
            }
        }
        chars += __shfl_sync(kFull, st_incl, 31);
        if (kTags || kIn) extra += __shfl_sync(kFull, sl_incl, 31);
        if (kTags) toks += __shfl_sync(kFull, wb_incl, 31);
    }
    uint32_t len = (b1 - b0) + nch - 1 + extra;
    const uint2 last_in = kIn && nch > 0 ? reg[nch - 1] : make_uint2(0, 0);
    if (kIn && last_in.y) {
        const uint32_t last = unescaped_len(in.input, last_in);
        if (kWrite && lane == 0) unescaped_copy(in.input, last_in, out + len);
        len += last;
    } else if (kTags && nch > 0) {
        const uint32_t last = pa_suffix<false, kRules>(t, ra, rec0 + toks, nullptr);
        if (kWrite && lane == 0) pa_suffix<true, kRules>(t, ra, rec0 + toks, out + len);
        len += last;
    }
    return len;
}

template <bool kTags, bool kRules, bool kIn>
__device__ __forceinline__ void pa_write(const TokArgs& t, uint64_t ngroups, const TagRuleArgs& ra,
                                         const uint8_t* __restrict__ marks, const InTags& in) {
    __shared__ uint64_t s_off[kGroup + 1];
    __shared__ uint32_t s_nch[kGroup];
    __shared__ uint32_t s_len[kGroup], s_excl[kGroup];
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
    for (int i = warp; i < ns; i += kWarps) {
        uint32_t len = 1;  // the '\n'
        if (!s_bad[i])
            len += pa_sentence<false, kTags, kRules, kIn>(t, ra, marks, gbase + i, s_off[i], s_off[i + 1], s_trim[i],
                                                          s_nch[i], nullptr, lane, in);
        if (lane == 0) s_len[i] = len;
    }
    __syncthreads();
    // 2. offsets: scan inside the group, look-back across groups (as k_tok_write)
    if (warp == 0) {
        const uint32_t v0 = s_len[2 * lane], v1 = s_len[2 * lane + 1];
        const uint32_t iv = warp_incl_scan_u32(v0 + v1, lane);
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
    for (int i = warp; i < ns; i += kWarps) {
        uint8_t* __restrict__ out = t.out + gout + s_excl[i];
        if (lane == 0) out[s_len[i] - 1] = 0x0A;
        if (!s_bad[i])
            pa_sentence<true, kTags, kRules, kIn>(t, ra, marks, gbase + i, s_off[i], s_off[i + 1], s_trim[i], s_nch[i],
                                                  out, lane, in);
    }
}

template <bool kTags, bool kRules>
__global__ void __launch_bounds__(kAnThreads, 1) k_pa_write(TokArgs t, uint64_t ngroups, TagRuleArgs ra, const uint8_t* __restrict__ marks) {
    pa_write<kTags, kRules, false>(t, ngroups, ra, marks, InTags());
}

// k_pa_write with the input tags of vpt_reannotate_lines
template <bool kTags, bool kRules>
__global__ void __launch_bounds__(kAnThreads, 1) k_pa_rewrite(TokArgs t, uint64_t ngroups, TagRuleArgs ra,
                                                              const uint8_t* __restrict__ marks, InTags in) {
    pa_write<kTags, kRules, true>(t, ngroups, ra, marks, in);
}

unsigned warp_blocks(uint64_t n) { return unsigned((n + kWarps - 1) / kWarps); }

}  // namespace

cudaError_t launch_pa_margin(const AnnArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0 || a.margin == 0) return cudaSuccess;
    k_pa_margin<<<warp_blocks(a.n_sent), kAnThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_pa_marks(const AnnArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    k_pa_marks<<<warp_blocks(a.n_sent), kAnThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_pa_untag(const AnnArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0 || a.margin == 0) return cudaSuccess;
    k_pa_untag<<<warp_blocks(a.n_sent), kAnThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_pa_write(const TokArgs& t, const TagRuleArgs& ra, const uint8_t* marks, cudaStream_t stream) {
    if (t.n_sent == 0) return cudaMemsetAsync(t.total, 0, 8, stream);
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    // look-back state words + the ticket that follows them
    cudaError_t e = cudaMemsetAsync(t.tok_state, 0, 8 * (ngroups + 1), stream);
    if (e != cudaSuccess) return e;
    if (t.tok_base && ra.tok_rule) k_pa_write<true, true><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks);
    else if (t.tok_base) k_pa_write<true, false><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks);
    else k_pa_write<false, false><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks);
    return cudaGetLastError();
}

cudaError_t launch_pa_rewrite(const TokArgs& t, const TagRuleArgs& ra, const uint8_t* marks, const uint8_t* input,
                              const uint2* regions, const uint64_t* char_offsets, cudaStream_t stream) {
    if (t.n_sent == 0) return cudaMemsetAsync(t.total, 0, 8, stream);
    const uint64_t ngroups = (t.n_sent + kGroup - 1) / kGroup;
    cudaError_t e = cudaMemsetAsync(t.tok_state, 0, 8 * (ngroups + 1), stream);
    if (e != cudaSuccess) return e;
    InTags in;
    in.input = input;
    in.regions = regions;
    in.char_offsets = char_offsets;
    if (t.tok_base && ra.tok_rule) k_pa_rewrite<true, true><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks, in);
    else if (t.tok_base) k_pa_rewrite<true, false><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks, in);
    else k_pa_rewrite<false, false><<<unsigned(ngroups), kAnThreads, 0, stream>>>(t, ngroups, ra, marks, in);
    return cudaGetLastError();
}

}  // namespace vpt
