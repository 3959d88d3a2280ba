// vaporetto_b200 — k_tags: Predictor::predict_tags on the device (reference predictor.rs:546-637).
//
// One warp per sentence walks its characters 32 at a time (the same window decoder as the sentence-warp scorer: it
// yields the byte position of every character).  A lane whose character ends a token (final boundary after it, or the
// last character) takes the byte position of the token's first character from the ring when the token began in the same
// 32-character step, and otherwise from a warp-uniform carry that the step closing the previous token read from the ring
// (tokens of any length are located: the ring itself reaches back only ~100 characters), hashes the token's bytes and
// looks it up in the token table; for a known token it starts from the tag model's bias, adds the weight vectors keyed
// by (pattern id at characters last .. last + rel, token, rel) of both scorers -- the pattern's own vector plus those of
// its suffix patterns with the reference's truncation (tags.hpp) -- and takes the first strict maximum of every tag slot
// with at least two candidates (predictor.rs:286-304).  Integer adds wrap as in the reference's release build.
#include <algorithm>
#include <atomic>

#include "kernels_common.cuh"
#include "tag_rules.hpp"
#include "tags.hpp"
#include "tags_token.hpp"

namespace vpt {

namespace {

constexpr int kTagWarps = 8;

// kLocateOnly: phase 1 of the per-token path (descriptors for k_tok_lookup / k_tok_score); otherwise the kernel predicts the tags itself.
template <bool kLocateOnly>
__global__ void __launch_bounds__(kTagWarps * 32, kLocateOnly ? 8 : 1) k_tags(DevTags t, TagArgs a) {
    __shared__ Rings s_rings[kTagWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // (the work list of the per-token kernels starts empty: they run behind this kernel on the stream)
    if (kLocateOnly && a.tok_work && blockIdx.x == 0 && threadIdx.x == 0) a.tok_work[0] = 0;
    const uint64_t s = uint64_t(blockIdx.x) * kTagWarps + warp;
    if (s >= a.n_sent) return;
    Rings& r = s_rings[warp];
    const uint64_t b0 = a.offsets[s], b1 = a.offsets[s + 1] - (a.trims ? a.trims[s] : 0);
    const uint64_t cb = a.char_offsets[s] - a.char_base;
    const uint32_t n = uint32_t(a.char_offsets[s + 1] - a.char_offsets[s]);
    const uint64_t bo = a.bound_offsets[s] - a.bound_base;
    const uint32_t nt = t.n_tags;
    if (a.status[s] != 0) {
        if (a.tok_base) return;  // a rejected sentence has no tokens
        for (uint32_t i = lane; i < n; i += 32) {
            a.tag_token[cb + i] = -1;
            for (uint32_t k = 0; k < nt; ++k) a.tag_cand[(cb + i) * nt + k] = -1;
        }
        return;
    }
    uint64_t wpos = b0 & ~3ull;
    uint32_t nd = 0;
    uint32_t tok_rank = 0;  // tokens that end before this chunk of characters
    uint32_t open_sb = 0;   // byte position (from b0) of the first character of the token open at the start of the chunk
    for (uint32_t c0 = 0; c0 < n; c0 += 32) {
        // byte positions of the characters up to c0 + 32 (one more: the end of the chunk's last character)
        const uint32_t need = min(n, c0 + 33u);
        while (nd < need && wpos < b1) {
            nd += decode_window(a.text, wpos, b0, b1, nd, r, lane, false);
            wpos += 128;
        }
        __syncwarp();
        const uint32_t i = c0 + lane;
        int32_t tok = -1;
        int32_t cand[kTagMaxSlots];
#pragma unroll
        for (int k = 0; k < kTagMaxSlots; ++k) cand[k] = -1;
        const bool ends = i < n && (i + 1 == n || a.boundaries[bo + i] == 1);
        const unsigned endm_all = __ballot_sync(kFull, ends);
        uint32_t desc_x = 0, desc_y = 0, desc_z = 0, desc_w = 0;
        if (i < n) {
            if (ends) {
                // the token starts behind the previous token end: in this chunk (ballot; the ring holds it) or before it (carried)
                const unsigned before = endm_all & ((1u << lane) - 1u);
                const uint32_t sb = before ? r.bp[(c0 + 32u - uint32_t(__clz(before))) & kRingMask] : open_sb;
                const uint32_t eb = i + 1 < n ? r.bp[(i + 1) & kRingMask] : uint32_t(b1 - b0);
                if (kLocateOnly) {
                    // phase 1 of the per-token path: where the token is; k_tok_lookup and k_tok_score do the rest, one thread per token
                    const uint64_t off = b0 + sb - a.text_base;
                    desc_x = uint32_t(off);
                    desc_y = uint32_t(off >> 32) | (min(n - i, 0xFFFFu) << 16);
                    desc_z = uint32_t(cb + i);
                    desc_w = eb - sb;
                } else {
                    tok = tag_token_at(t, a.text + b0 + sb, eb - sb, a.char_states ? a.char_states + cb : nullptr,
                                       a.type_states ? a.type_states + cb : nullptr, i, n, cand, a.n_unserved, a.norm);
                }
            }
        }
        __syncwarp();
        if (endm_all) {
            // The token after this chunk's last token end starts at character `next` <= c0 + 32.  Its ring slot is live
            // now and is overwritten by a later chunk's decoding: decoding stops once nd >= min(n, c0 + 33) and appends
            // at most 128 characters per window, so next < nd <= c0 + 160 and the ring holds [nd - 256, nd) with
            // nd - 256 <= c0 - 96 < next.  (next == n: no token follows.)
            const uint32_t next = c0 + 32u - uint32_t(__clz(endm_all));
            if (next < n) open_sb = r.bp[next & kRingMask];
        }
        if (a.tok_base) {
            // per-token records: the token's rank is the number of boundaries before its last character
            const unsigned endm = endm_all;
            if (ends) {
                const uint64_t rec = a.tok_base[s] + tok_rank + __popc(endm & ((1u << lane) - 1u));
                if (kLocateOnly) {
                    a.tok_desc[rec] = make_uint4(desc_x, desc_y, desc_z, desc_w);
                } else {
                    a.tok_ids[rec] = tok;
                    for (uint32_t k = 0; k < nt; ++k) a.tok_cands[rec * nt + k] = (tok >= 0 && cand[k] >= 0) ? uint8_t(cand[k]) : uint8_t(255);
                }
            }
            tok_rank += __popc(endm);
        } else if (i < n) {
            a.tag_token[cb + i] = tok;
            for (uint32_t k = 0; k < nt; ++k) a.tag_cand[(cb + i) * nt + k] = tok >= 0 ? cand[k] : -1;
        }
        __syncwarp();
    }
}

// Phase 2 of the per-token path, one thread per token record (descriptor written by k_tags): consecutive lanes read
// consecutive text.  Two kernels, because only some tokens have a tag model (41 % on the config-3 workload) and the work
// behind the lookup is 5-10 x the lookup: with both in one kernel a warp runs the long path at the lane density of the
// tokens that have a model.
//   k_tok_lookup  every token: hash + table lookup; the token id (or -1) is final here; tokens with a model are appended
//                 to a work list (one atomic per warp)
//   k_tok_score   the listed tokens, dense lanes: bias + tag weights + arg-max
// Both are grid-stride loops over a resident grid (the token count is known on the device only).
// kScores (TagScoreArgs, tags.hpp): the lookup also writes every record's score count, k_score_block / k_score_scan turn
// the counts into offsets, and k_tok_score stores each listed token's score vector at its record's offset.  Without it
// the kernels are the ones of the path without scores.
constexpr int kTokTagThreads = 128;
constexpr int kTokWorkHead = 4;  // words in front of the work list: [0] = entries
template <bool kScores>
__global__ void __launch_bounds__(kTokTagThreads) k_tok_lookup(DevTags t, TagArgs a, TagScoreArgs sc) {
    const uint64_t ntok = a.tok_base[a.n_sent];
    const uint32_t nt = t.n_tags;
    const int lane = threadIdx.x & 31;
    const uint64_t stride = uint64_t(gridDim.x) * kTokTagThreads;
    // (warp-uniform trip count: the list append is a warp operation)
    for (uint64_t rec0 = uint64_t(blockIdx.x) * kTokTagThreads + (threadIdx.x & ~31u); rec0 < ntok; rec0 += stride) {
        const uint64_t rec = rec0 + uint32_t(lane);
        bool listed = false;
        if (rec < ntok) {
            const uint4 d = a.tok_desc[rec];
            int32_t tok = -1;
            uint32_t tid = 0;
            if (token_lookup(t, a.text + a.text_base + ((uint64_t(d.y & 0xFFFFu) << 32) | d.x), d.w, a.norm, tid)) {
                if (__ldg(&t.tok_info[tid].usable)) {
                    tok = int32_t(tid);
                    listed = true;
                } else if (a.n_unserved) {
                    atomicAdd(a.n_unserved, 1u);
                }
            }
            a.tok_ids[rec] = tok;
            if (!listed)
                for (uint32_t k = 0; k < nt; ++k) a.tok_cands[rec * nt + k] = uint8_t(255);
            if (kScores) sc.rec_off[rec] = listed ? tag_score_count(t.tok_info[tid], nt) : 0u;
        }
        const unsigned m = __ballot_sync(kFull, listed);
        if (m) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(a.tok_work, uint32_t(__popc(m)));
            base = __shfl_sync(kFull, base, 0);
            if (listed) a.tok_work[kTokWorkHead + base + __popc(m & ((1u << lane) - 1u))] = uint32_t(rec);
        }
    }
}

template <bool kScores>
__global__ void __launch_bounds__(kTokTagThreads) k_tok_score(DevTags t, TagArgs a, TagScoreArgs sc) {
    const uint32_t nw = a.tok_work[0];
    const uint32_t nt = t.n_tags;
    for (uint32_t w = blockIdx.x * kTokTagThreads + threadIdx.x; w < nw; w += gridDim.x * kTokTagThreads) {
        const uint32_t rec = a.tok_work[kTokWorkHead + w];
        const uint4 d = a.tok_desc[rec];
        int32_t cand[kTagMaxSlots];
#pragma unroll
        for (int k = 0; k < kTagMaxSlots; ++k) cand[k] = -1;
        // (characters [d.z, d.z + n_after) are the token's last character and what follows it in its sentence)
        int32_t* out = nullptr;
        if (kScores) out = sc.scores + sc.blk[rec / kScoreScanBlock] + sc.rec_off[rec];
        const int32_t tok = tag_score_token<kScores>(t, uint32_t(a.tok_ids[rec]), a.char_states ? a.char_states + d.z : nullptr,
                                                     a.type_states ? a.type_states + d.z : nullptr, 0, d.y >> 16, cand,
                                                     a.n_unserved, out);
        if (tok < 0) a.tok_ids[rec] = -1;
        for (uint32_t k = 0; k < nt; ++k) a.tok_cands[uint64_t(rec) * nt + k] = (tok >= 0 && cand[k] >= 0) ? uint8_t(cand[k]) : uint8_t(255);
    }
}

// Offsets of the score vectors, step 1: exclusive prefix of the records' score counts inside each block of
// kScoreScanBlock records (grid over max_tokens: the record count is known on the device only) and the block's total.
__global__ void __launch_bounds__(kScoreScanBlock) k_score_block(TagArgs a, TagScoreArgs sc) {
    __shared__ uint32_t s_w[kScoreScanBlock / 32];
    const uint64_t ntok = a.tok_base[a.n_sent];
    const uint64_t rec = uint64_t(blockIdx.x) * kScoreScanBlock + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (uint64_t(blockIdx.x) * kScoreScanBlock >= ntok) {
        if (threadIdx.x == 0) sc.blk[blockIdx.x] = 0;
        return;
    }
    const uint32_t v = rec < ntok ? sc.rec_off[rec] : 0u;
    const uint32_t incl = warp_incl_scan(v, lane);
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kScoreScanBlock / 32; ++w) {
        if (w < warp) base += s_w[w];
        tot += s_w[w];
    }
    if (rec < ntok) sc.rec_off[rec] = base + incl - v;
    if (threadIdx.x == 0) sc.blk[blockIdx.x] = tot;
}

// step 2: exclusive prefix of the block totals (one block, 1024 totals per round); the chunk's total behind them and in
// the pinned host word
__global__ void __launch_bounds__(1024) k_score_scan(TagScoreArgs sc, uint64_t nblk) {
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint64_t lo = 0; lo < nblk; lo += 1024) {
        const uint64_t i = lo + threadIdx.x;
        const uint64_t v = i < nblk ? sc.blk[i] : 0;
        uint64_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t o = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl += o;
        }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        uint64_t base = s_carry;
        for (int w = 0; w < warp; ++w) base += s_w[w];
        if (i < nblk) sc.blk[i] = base + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = base + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        sc.blk[nblk] = s_carry;
        if (sc.total_host) *sc.total_host = s_carry;
    }
}

// PatternMatchTagger's rule lookup, one thread per token record, behind k_tok_lookup: every token is looked up, unknown
// tokens included (they are what rules are for), by the surface bytes k_tok_lookup hashed.  A kernel of its own keeps
// the path without rules as it was; the lookup costs one more pass over the descriptors and the token bytes.
__global__ void __launch_bounds__(kTokTagThreads) k_rule_lookup(DevTagRules r, TagArgs a, int32_t* __restrict__ tok_rule,
                                                                unsigned long long* __restrict__ suffix_sum) {
    const uint64_t ntok = a.tok_base[a.n_sent];
    const uint64_t stride = uint64_t(gridDim.x) * kTokTagThreads;
    unsigned long long sum = 0;
    for (uint64_t rec = uint64_t(blockIdx.x) * kTokTagThreads + threadIdx.x; rec < ntok; rec += stride) {
        const uint4 d = a.tok_desc[rec];
        const int32_t rid = rule_lookup(r, a.text + a.text_base + ((uint64_t(d.y & 0xFFFFu) << 32) | d.x), d.w, a.norm);
        tok_rule[rec] = rid;
        if (rid >= 0) sum += __ldg(r.suffix + rid);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
    if ((threadIdx.x & 31) == 0 && sum) atomicAdd(suffix_sum, sum);
}

// ---- compact outputs -----------------------------------------------------------------------------------------------------

constexpr int kPackThreads = 256;

// boundaries (one byte each) -> one bit each; thread per output word
__global__ void __launch_bounds__(kPackThreads) k_pack_bits(CompactArgs c) {
    const uint64_t w = uint64_t(blockIdx.x) * kPackThreads + threadIdx.x;
    const uint64_t nwords = (uint64_t(c.bit_base) + c.n_bound + 31) / 32;
    if (w >= nwords) return;
    // word w holds the boundaries [32 w - bit_base, 32 w - bit_base + 32)
    const int64_t first = int64_t(32 * w) - int64_t(c.bit_base);
    uint32_t v = 0;
    if (first >= 0 && uint64_t(first) + 32 <= c.n_bound && ((reinterpret_cast<uintptr_t>(c.boundaries) + first) & 3) == 0) {
        const uint32_t* q = reinterpret_cast<const uint32_t*>(c.boundaries + first);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t x = __ldg(q + j) & 0x01010101u;  // bytes are 0 / 1
            v |= (((x * 0x01020408u) >> 24) & 15u) << (4 * j);
        }
    } else {
        for (int j = 0; j < 32; ++j) {
            const int64_t i = first + j;
            if (i >= 0 && uint64_t(i) < c.n_bound && c.boundaries[i]) v |= 1u << j;
        }
    }
    c.bits[w] = v;
}

// status as one byte, tokens per sentence (boundaries set + 1 for a scored sentence), their prefix inside the block of
// 256 sentences and the block's total
__global__ void __launch_bounds__(kPackThreads) k_sentence_info(CompactArgs c) {
    __shared__ uint32_t s_w[kPackThreads / 32];
    const uint64_t s = uint64_t(blockIdx.x) * kPackThreads + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ntok = 0;
    if (s < c.n_sent) {
        const int32_t st = c.status[s];
        c.status8[s] = uint8_t(st);
        if (c.n_tokens) {
            const uint32_t n = c.n_chars[s];
            if (st == 0 && n > 0) {
                const uint8_t* b = c.boundaries + (c.bound_offsets[s] - c.bound_base);
                ntok = 1;
                for (uint32_t i = 0; i + 1 < n; ++i) ntok += b[i];
            }
            c.n_tokens[s] = ntok;
        }
    }
    if (!c.n_tokens) return;
    const uint32_t incl = warp_incl_scan(ntok, lane);
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kPackThreads / 32; ++w) {
        if (w < warp) base += s_w[w];
        tot += s_w[w];
    }
    if (s < c.n_sent) c.tok_local[s] = base + incl - ntok;
    if (threadIdx.x == 0) c.tok_blk[blockIdx.x] = tot;
}

// exclusive prefix of the block totals (one block; 1024 totals per round), the grand total behind them
__global__ void __launch_bounds__(1024) k_token_scan(CompactArgs c) {
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const uint64_t nblk = (c.n_sent + kPackThreads - 1) / kPackThreads;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint64_t lo = 0; lo < nblk; lo += 1024) {
        const uint64_t i = lo + threadIdx.x;
        const uint64_t v = i < nblk ? c.tok_blk[i] : 0;
        uint64_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t o = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl += o;
        }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        uint64_t base = s_carry;
        for (int w = 0; w < warp; ++w) base += s_w[w];
        if (i < nblk) c.tok_blk[i] = base + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = base + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        c.tok_blk[nblk] = s_carry;
        c.tok_base[c.n_sent] = s_carry;
        if (c.tok_total_host) *c.tok_total_host = s_carry;
    }
}

__global__ void __launch_bounds__(kPackThreads) k_token_base(CompactArgs c) {
    const uint64_t s = uint64_t(blockIdx.x) * kPackThreads + threadIdx.x;
    if (s < c.n_sent) c.tok_base[s] = c.tok_blk[blockIdx.x] + c.tok_local[s];
}

}  // namespace

cudaError_t launch_compact(const CompactArgs& c, cudaStream_t stream) {
    const uint64_t nwords = (uint64_t(c.bit_base) + c.n_bound + 31) / 32;
    if (nwords) k_pack_bits<<<unsigned((nwords + kPackThreads - 1) / kPackThreads), kPackThreads, 0, stream>>>(c);
    if (c.n_sent) {
        k_sentence_info<<<unsigned((c.n_sent + kPackThreads - 1) / kPackThreads), kPackThreads, 0, stream>>>(c);
        if (c.n_tokens) {
            k_token_scan<<<1, 1024, 0, stream>>>(c);
            k_token_base<<<unsigned((c.n_sent + kPackThreads - 1) / kPackThreads), kPackThreads, 0, stream>>>(c);
        }
    }
    return cudaGetLastError();
}

cudaError_t launch_rule_lookup(const DevTagRules& r, const TagArgs& a, int32_t* tok_rule, unsigned long long* suffix_sum,
                               cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(suffix_sum, 0, sizeof *suffix_sum, stream);
    if (e != cudaSuccess) return e;
    if (a.n_sent == 0 || a.max_tokens == 0) return cudaSuccess;
    if (!a.tok_desc || !a.tok_base) return cudaErrorInvalidValue;
    // (grid-stride: the number of tokens is known on the device only; 2048 blocks fill an H100 at 16 per SM)
    const uint64_t want = (a.max_tokens + kTokTagThreads - 1) / kTokTagThreads;
    k_rule_lookup<<<unsigned(std::min<uint64_t>(want, 2048)), kTokTagThreads, 0, stream>>>(r, a, tok_rule, suffix_sum);
    return cudaGetLastError();
}

cudaError_t launch_tags(const DevTags& t, const TagArgs& a, cudaStream_t stream, const TagScoreArgs* scores) {
    if (a.n_sent == 0) return cudaSuccess;
    if (scores && (!a.tok_desc || !a.tok_base || !scores->rec_off || !scores->blk || !scores->scores)) return cudaErrorInvalidValue;
    const uint64_t nblocks = (a.n_sent + kTagWarps - 1) / kTagWarps;
    if (a.tok_desc && a.tok_base) k_tags<true><<<unsigned(nblocks), kTagWarps * 32, 0, stream>>>(t, a);
    else k_tags<false><<<unsigned(nblocks), kTagWarps * 32, 0, stream>>>(t, a);
    if (a.tok_desc && a.tok_base && a.max_tokens) {
        // (the number of tokens is known on the device only: resident grids, grid-stride loops)
        if (!a.tok_work || a.max_tokens > 0xFFFFFFFFull) return cudaErrorInvalidValue;
        static std::atomic<int> sm_count[64] = {};  // (written with the same value by whoever comes first)
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
        if (sm_count[dev] == 0) {
            int v = 0;
            e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
            if (e != cudaSuccess) return e;
            sm_count[dev] = v;
        }
        const uint64_t want = (a.max_tokens + kTokTagThreads - 1) / kTokTagThreads;
        // (resident blocks per SM: 16 x 128 threads at 32 registers, 8 x 128 at 56)
        const unsigned lookup_grid = unsigned(std::min<uint64_t>(want, uint64_t(sm_count[dev]) * 16));
        const unsigned score_grid = unsigned(std::min<uint64_t>(want, uint64_t(sm_count[dev]) * 8));
        if (scores) {
            const uint64_t nblk = (a.max_tokens + kScoreScanBlock - 1) / kScoreScanBlock;
            k_tok_lookup<true><<<lookup_grid, kTokTagThreads, 0, stream>>>(t, a, *scores);
            k_score_block<<<unsigned(nblk), kScoreScanBlock, 0, stream>>>(a, *scores);
            k_score_scan<<<1, 1024, 0, stream>>>(*scores, nblk);
            k_tok_score<true><<<score_grid, kTokTagThreads, 0, stream>>>(t, a, *scores);
        } else {
            k_tok_lookup<false><<<lookup_grid, kTokTagThreads, 0, stream>>>(t, a, TagScoreArgs{});
            k_tok_score<false><<<score_grid, kTokTagThreads, 0, stream>>>(t, a, TagScoreArgs{});
        }
    }
    return cudaGetLastError();
}

}  // namespace vpt
