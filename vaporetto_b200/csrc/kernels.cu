// vaporetto_b200 — sm_90a kernels for the Predictor::predict hot path.
//
// Replaces (reference, vaporetto/src): predictor.rs:518-543 (predict), char_scorer/boundary_scorer.rs:93-113
// and char_scorer/boundary_tag_scorer.rs:121-147 (pattern walk + weight add), predictor.rs:176-213
// (PositionalWeight::add_score), type_scorer/boundary_scorer_cache.rs:59-81 (type table),
// type_scorer/boundary_scorer.rs:64-80 / boundary_tag_scorer.rs:95-116 (type automaton variants),
// sentence.rs:50-67,160-196 (get_type / parse_raw: done on device from raw UTF-8).
//
// Pipeline per batch (DESIGN.md §4):
//   k_count        one warp per sentence: chars per sentence, validation (empty / NUL / bad UTF-8),
//                  group-local exclusive offsets (64 sentences per CTA)
//   k_scan_groups  one CTA: exclusive scan of the per-group totals
//   k_tile_fast    one CTA per group of 64 sentences: the group's UTF-8 bytes are staged into shared memory
//                  with one TMA bulk copy (cp.async.bulk + mbarrier); characters of all sentences are laid
//                  out as one flat slot stream (zero separators between sentences) so every lane of every
//                  warp owns one character: decode, longest-suffix lookup in the perfect-hash node table
//                  (one 32-byte record per probe), warp-shuffle gather of the 6-wide weight rows
//                  into per-boundary sums, type-table add, bias, threshold, coalesced stores.
//   (fast_sentence_warp: one warp per sentence — fallback for groups too large for the tile buffers)
//   k_score_general  same skeleton for models whose rows do not fit the inline window, for the type
//                  automaton variant and for tag-state output: rows scatter with global atomics.
// No tensor cores: integer indexing + scatter/gather add.
#include <atomic>
#include <algorithm>
#include <cstdint>

#include <cuda_runtime.h>

#include "device_model.hpp"
#include "kernel_plan.hpp"
#include "keys.hpp"
#include "textnorm.hpp"

#include "kernels_common.cuh"

namespace vpt {

namespace {


// ------------------------------------------------------------------------------------------------
// k_count
// ------------------------------------------------------------------------------------------------
constexpr int kCountTextCap = 24576;  // bytes of one group staged in shared memory by k_count

// One CTA per group of 64 sentences.  The group's bytes are staged in shared memory with one TMA bulk copy
// (groups larger than the buffer are read from global memory instead); each warp then counts and validates
// its sentences: characters, NUL, malformed UTF-8.
__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_count(BatchArgs a) {
    __shared__ __align__(128) uint8_t s_text[kCountTextCap];
    __shared__ uint64_t s_off[kGroup + 1];
    __shared__ uint32_t s_nout[kGroup], s_nch[kGroup];
    __shared__ uint8_t s_trim[kGroup];
    __shared__ __align__(8) uint64_t s_bar;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t gbase = uint64_t(blockIdx.x) * kGroup;
    const int ns = int(min(uint64_t(kGroup), a.n_sent - gbase));
    const uint8_t* __restrict__ text = a.text;
    if (threadIdx.x <= ns) s_off[threadIdx.x] = a.offsets[gbase + threadIdx.x];
    if (threadIdx.x < kGroup) s_trim[threadIdx.x] = (a.trims && threadIdx.x < ns) ? a.trims[gbase + threadIdx.x] : uint8_t(0);
    if (threadIdx.x == 0) mbar_init(&s_bar, 1);
    __syncthreads();
    const uint64_t a0 = s_off[0] & ~15ull;
    const uint64_t span = (s_off[ns] - a0 + 15) & ~15ull;
    const bool staged = span + 16 <= uint64_t(kCountTextCap);
    if (staged && span) {
        if (threadIdx.x == 0) {
            mbar_expect_tx(&s_bar, uint32_t(span));
            tma_bulk_g2s(s_text, text + a0, uint32_t(span), &s_bar);
        }
        mbar_wait(&s_bar, 0);
    }
    // each warp scores 4 sentences at a time: 8 lanes per sentence, 32 bytes per sentence per iteration
    const int quad = lane >> 3, l8 = lane & 7;
    for (int it = 0; it < kGroup / (kWarpsPerBlock * 4); ++it) {
        const int i = (warp * (kGroup / kWarpsPerBlock)) + it * 4 + quad;
        uint32_t nch = 0, nout = 0;
        {
            // lanes of a quad beyond the group's last sentence run an empty range (all 32 lanes must reach
            // the shuffles below)
            // 32-bit byte offsets relative to a0 (a group's text is far below 4 GB)
            const uint32_t b0 = i < ns ? uint32_t(s_off[i] - a0) : 0u, b1 = i < ns ? uint32_t(s_off[i + 1] - a0) - s_trim[i] : 0u;
            const uint8_t* __restrict__ gtext = text + a0;
            uint32_t starts = 0, conts = 0, expect = 0, flags = 0;  // flags: 1 NUL, 2 malformed
            for (uint32_t wpos = b0 & ~3u; wpos < b1; wpos += 32) {
                const uint32_t addr = wpos + 4u * uint32_t(l8);
                if (addr < b1) {
                    uint32_t lo, hi = 0;
                    if (staged) {
                        lo = *reinterpret_cast<const uint32_t*>(s_text + addr);
                        if (addr + 4 < b1) hi = *reinterpret_cast<const uint32_t*>(s_text + addr + 4);
                    } else {
                        lo = __ldg(reinterpret_cast<const uint32_t*>(gtext + addr));
                        if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(gtext + addr + 4));
                    }
                    // ---- SWAR fast path over the 4 bytes of this word (V = the word and the 4 bytes after it) ----
                    const uint32_t from = b0 > addr ? b0 - addr : 0u;                     // first byte inside
                    const uint32_t to = b1 - addr < 4u ? b1 - addr : 4u;                  // one past the last
                    const uint32_t im = (from >= 4 ? 0u : 0xFFFFFFFFu << (8 * from)) & (0xFFFFFFFFu >> (8 * (4 - to)));
                    const uint32_t im80 = im & 0x80808080u;
                    const uint32_t top2 = lo & (lo << 1);                                  // bit7 = b7&b6
                    const uint32_t cont80 = lo & ~(lo << 1) & 0x80808080u;                 // 10xxxxxx
                    const uint32_t l2 = top2 & im80;                                        // 11xxxxxx (any lead)
                    const uint32_t l3 = top2 & (lo << 2) & im80;                            // 111xxxxx
                    const uint32_t l4 = top2 & (lo << 2) & (lo << 3) & im80;                // 1111xxxx
                    const uint32_t lz = (lo & im) | (0x20202020u & ~im);
                    if ((lz - 0x01010101u) & ~lz & 0x80808080u) flags |= 1;                 // a NUL inside
                    // bytes that need the exact per-byte rules: C0/C1, E0, ED, F0..FF (rare in real text)
                    const uint32_t xe0 = lo ^ 0xE0E0E0E0u, xed = lo ^ 0xEDEDEDEDu, xc0 = (lo & 0xFEFEFEFEu) ^ 0xC0C0C0C0u;
                    const uint32_t special = (l4 | ((xe0 - 0x01010101u) & ~xe0) | ((xed - 0x01010101u) & ~xed) |
                                              ((xc0 - 0x01010101u) & ~xc0)) & im80;
                    if (special == 0) {
                        starts += __popc(im80 & ~cont80);
                        conts += __popc(im80 & cont80);
                        expect += __popc(l2) + __popc(l3);
                        // every lead must be followed, inside the sentence, by its continuation bytes
                        const uint64_t c64 = (uint64_t(hi & ~(hi << 1) & 0x80808080u) << 32) | cont80;
                        const uint64_t avail = b1 - addr >= 8 ? ~0ull : (~0ull >> (8 * (8 - (b1 - addr))));
                        const uint64_t okc = c64 & avail;
                        const uint64_t need = (uint64_t(l2) << 8) | (uint64_t(l3) << 16);
                        if (need & ~okc) flags |= 2;
                    } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t p = addr + j;
                        if (p < b0 || p >= b1) continue;
                        const uint32_t x = __funnelshift_r(lo, hi, 8 * j);
                        const uint32_t b = x & 0xFF;
                        if ((b & 0xC0) == 0x80) { ++conts; continue; }
                        ++starts;
                        if (b < 0x80) continue;
                        const uint32_t c1 = (x >> 8) & 0xFF, c2 = (x >> 16) & 0xFF, c3 = x >> 24;
                        uint32_t len;
                        bool ok;
                        if (b < 0xC2) { len = 1; ok = false; }
                        else if (b < 0xE0) { len = 2; ok = (c1 & 0xC0) == 0x80; }
                        else if (b < 0xF0) {
                            len = 3;
                            ok = (c1 & 0xC0) == 0x80 && (c2 & 0xC0) == 0x80 && !(b == 0xE0 && c1 < 0xA0) &&
                                 !(b == 0xED && c1 > 0x9F);
                        } else if (b < 0xF5) {
                            len = 4;
                            ok = (c1 & 0xC0) == 0x80 && (c2 & 0xC0) == 0x80 && (c3 & 0xC0) == 0x80 &&
                                 !(b == 0xF0 && c1 < 0x90) && !(b == 0xF4 && c1 > 0x8F);
                        } else { len = 1; ok = false; }
                        if (p + len > b1) ok = false;
                        if (!ok) flags |= 2;
                        expect += len - 1;
                    }
                    }
                }
            }
#pragma unroll
            for (int d = 4; d > 0; d >>= 1) {
                starts += __shfl_xor_sync(kFull, starts, d);
                conts += __shfl_xor_sync(kFull, conts, d);
                expect += __shfl_xor_sync(kFull, expect, d);
                flags |= __shfl_xor_sync(kFull, flags, d);
            }
            if (conts != expect) flags |= 2;
            nch = i < ns ? starts : 0;
            nout = nch > 0 ? nch - 1 : 0;
            const int st = (flags & 2) ? 3 : (flags & 1) ? 2 : (nch == 0 ? 1 : 0);
            if (l8 == 0 && i < ns) {
                a.n_chars[gbase + i] = nch;
                a.status[gbase + i] = st;
            }
        }
        if (l8 == 0) { s_nout[i] = nout; s_nch[i] = nch; }
    }
    __syncthreads();
    if (warp == 0) {
        const uint32_t v0 = s_nout[2 * lane], v1 = s_nout[2 * lane + 1];
        const uint32_t u0 = s_nch[2 * lane], u1 = s_nch[2 * lane + 1];
        const uint32_t iv = warp_incl_scan(v0 + v1, lane), iu = warp_incl_scan(u0 + u1, lane);
        const uint64_t s0 = gbase + 2 * lane;
        if (s0 < a.n_sent) { a.local_bound[s0] = iv - v0 - v1; a.local_char[s0] = iu - u0 - u1; }
        if (s0 + 1 < a.n_sent) { a.local_bound[s0 + 1] = iv - v1; a.local_char[s0 + 1] = iu - u1; }
        if (lane == 31) { a.group_bound[blockIdx.x] = iv; a.group_char[blockIdx.x] = iu; }
    }
}

// Exclusive scan of the per-group totals (in place); element [ngroups] receives the grand total.
__global__ void __launch_bounds__(1024) k_scan_groups(uint64_t* gb, uint64_t* gc, uint64_t ngroups, uint32_t* ticket,
                                                     uint64_t* totals_host) {
    __shared__ uint64_t s_wb[32], s_wc[32];
    __shared__ uint64_t s_carry[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_carry[0] = 0; s_carry[1] = 0; }
    __syncthreads();
    for (uint64_t base = 0; base < ngroups; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        const uint64_t vb = i < ngroups ? gb[i] : 0, vc = i < ngroups ? gc[i] : 0;
        uint64_t ib = vb, ic = vc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t ob = __shfl_up_sync(kFull, ib, d), oc = __shfl_up_sync(kFull, ic, d);
            if (lane >= d) { ib += ob; ic += oc; }
        }
        if (lane == 31) { s_wb[warp] = ib; s_wc[warp] = ic; }
        __syncthreads();
        if (warp == 0) {
            uint64_t wb = s_wb[lane], wc = s_wc[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint64_t ob = __shfl_up_sync(kFull, wb, d), oc = __shfl_up_sync(kFull, wc, d);
                if (lane >= d) { wb += ob; wc += oc; }
            }
            s_wb[lane] = wb;
            s_wc[lane] = wc;
        }
        __syncthreads();
        const uint64_t pb = (warp ? s_wb[warp - 1] : 0) + s_carry[0], pc = (warp ? s_wc[warp - 1] : 0) + s_carry[1];
        if (i < ngroups) { gb[i] = pb + ib - vb; gc[i] = pc + ic - vc; }
        __syncthreads();
        if (threadIdx.x == 0) { s_carry[0] += s_wb[31]; s_carry[1] += s_wc[31]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        gb[ngroups] = s_carry[0];
        gc[ngroups] = s_carry[1];
        *ticket = 0;
        if (totals_host) { totals_host[0] = s_carry[0]; totals_host[1] = s_carry[1]; }
    }
}


__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_score_fast(DevModel m, BatchArgs a) {
    __shared__ Rings s_rings[kWarpsPerBlock];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t s = uint64_t(blockIdx.x) * kWarpsPerBlock + warp;
    if (s >= a.n_sent) return;
    fast_sentence_warp(m, a, s, s_rings[warp], lane);
}


// ------------------------------------------------------------------------------------------------
// k_score_general (one warp per sentence)
// ------------------------------------------------------------------------------------------------
template <bool kTypes>
__device__ __forceinline__ void scatter_general(const DevTable& t, const Rings& r, const uint8_t* __restrict__ text,
                                                const SentInfo& si, uint32_t g, int32_t* scores, uint32_t* states,
                                                bool norm) {
    Rec32 rec;
    uint32_t slot;
    uint32_t pid = kNoPattern;
    if (find_node<kTypes>(t, r, text, si.b0, g, rec, slot, norm)) {
        pid = rec.v[2];
        const uint32_t row = rec.v[3];
        if (row != kNoPattern) {
            const int32_t off = int32_t(rec.v[4]);
            const uint32_t len = rec.v[5];
            for (uint32_t k = 0; k < len; ++k) {
                const int64_t i = int64_t(g) + off + int64_t(k);
                if (i >= 0 && i < int64_t(si.nout)) atomicAdd(scores + si.obase + i, __ldg(t.pool + row + k));
            }
        }
    }
    if (states) states[si.cbase + g] = pid;
}

// One warp scores one sentence with the general (pooled-row) tables: rows of any length scatter with global
// atomics, pattern-id states are emitted, the type automaton variant is supported.  Used by k_score_general and
// as the fallback of k_tile for single sentences larger than the tile buffers.
__device__ __forceinline__ void general_sentence_warp(const DevModel& m, const BatchArgs& a, uint64_t s, Rings& r, int lane) {
    const SentInfo si = sentence_info(a, s, lane);
    const uint8_t* __restrict__ text = a.text;
    const uint32_t n = si.n;
    uint32_t* cstates = a.char_states;
    uint32_t* tstates = a.type_states;
    if (si.status != 0) {
        for (uint32_t i = lane; i < si.nout; i += 32) { if (a.scores) a.scores[si.obase + i] = 0; a.boundaries[si.obase + i] = 0; }
        if (cstates) for (uint32_t i = lane; i < n; i += 32) cstates[si.cbase + i] = kNoPattern;
        if (tstates) for (uint32_t i = lane; i < n; i += 32) tstates[si.cbase + i] = kNoPattern;
        return;
    }
    const int tw = m.type_cache_window;
    // pass 1: scores = bias + type table; states = none
    {
        uint64_t wpos = si.b0 & ~3ull;
        uint32_t nd = 0;
        for (uint32_t cb = 0; cb < n; cb += 32) {
            const uint32_t need = min(n, cb + 32u + uint32_t(tw));
            while (nd < need && wpos < si.b1) {
                nd += decode_window(text, wpos, si.b0, si.b1, nd, r, lane, m.kytea_norm != 0);
                wpos += 128;
            }
            __syncwarp();
            const uint32_t g = cb + lane;
            if (g + 1 < n) {
                int32_t v = m.bias;
                if (tw > 0) v += __ldg(m.type_cache + type_index(r, int64_t(g), n, tw));
                if (a.scores) a.scores[si.obase + g] = v;
            }
            if (g < n) {
                if (cstates) cstates[si.cbase + g] = kNoPattern;
                if (tstates) {
                    uint32_t ts = kNoPattern;
                    if (m.emit_states && m.type_state3) {  // tag variant with short type patterns: direct table
                        const uint32_t t2 = g >= 1 ? r.ty[(g - 1) & kRingMask] : 0u;
                        const uint32_t t1 = (g >= 2 && t2) ? r.ty[(g - 2) & kRingMask] : 0u;
                        ts = __ldg(m.type_state3 + ((t1 << 6) | (t2 << 3) | r.ty[g & kRingMask]));
                    }
                    tstates[si.cbase + g] = ts;
                }
            }
            __syncwarp();
        }
    }
    __threadfence();
    __syncwarp();
    // pass 2: pattern rows
    if (m.ct.present || m.tt.present) {
        uint64_t wpos = si.b0 & ~3ull;
        uint32_t nd = 0;
        for (uint32_t cb = 0; cb < n; cb += 32) {
            const uint32_t need = min(n, cb + 32u);
            while (nd < need && wpos < si.b1) {
                nd += decode_window(text, wpos, si.b0, si.b1, nd, r, lane, m.kytea_norm != 0);
                wpos += 128;
            }
            __syncwarp();
            const uint32_t g = cb + lane;
            if (g < n) {
                if (m.ct.present)
                    scatter_general<false>(m.ct, r, text, si, g, a.scores, m.emit_states ? cstates : nullptr, m.kytea_norm != 0);
                if (m.tt.present)
                    scatter_general<true>(m.tt, r, text, si, g, a.scores, m.emit_states ? tstates : nullptr, m.kytea_norm != 0);
            }
            __syncwarp();
        }
    }
    __threadfence();
    __syncwarp();
    // pass 3: threshold
    for (uint32_t i = lane; i < si.nout; i += 32) {
        const int32_t v = __ldcg(a.scores + si.obase + i);
        a.boundaries[si.obase + i] = v > 0 ? 1 : 0;
    }
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_score_general(DevModel m, BatchArgs a) {
    __shared__ Rings s_rings[kWarpsPerBlock];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t s = uint64_t(blockIdx.x) * kWarpsPerBlock + warp;
    if (s >= a.n_sent) return;
    general_sentence_warp(m, a, s, s_rings[warp], lane);
}

// ------------------------------------------------------------------------------------------------
// k_tile_fast — persistent: one 1024-thread CTA per SM = 4 independent 256-thread sub-blocks that pull
// 64-sentence groups from a global ticket.  Shared by the 4 sub-blocks: the perfect-hash seed bytes and the
// split type tables (staged once per CTA); private to each sub-block: the tile buffers below.
// ------------------------------------------------------------------------------------------------
constexpr int kSubThreads = 256;
constexpr int kSubBlocks = 4;
constexpr int kTileThreads = kSubThreads * kSubBlocks;
constexpr int kTextCap = 12288;   // bytes of text staged per tile
constexpr int kSlotCap = 3072;    // character slots (characters + separators) per tile
constexpr int kSeedCap = 37632;   // seed bytes kept in shared memory (one per 8 nodes: ~300 K nodes)
constexpr int kTypeSub = 4096;    // entries of each split type table
constexpr uint32_t kSepPos = 0xFFFFu;

struct TileTables {
    uint64_t off[kGroup + 1];
    uint64_t obase[kGroup];
    uint64_t cbase[kGroup];
    uint32_t lc[kGroup + 1];  // chars before sentence k inside the group
    int64_t odelta[kGroup];   // output index of a boundary = its slot + odelta[sentence]
    int64_t cdelta[kGroup];   // state index of a character = its slot + cdelta[sentence]
    uint32_t nch[kGroup];
    int8_t st[kGroup];
    uint8_t trim[kGroup];     // separator bytes after sentence k (BatchArgs::trims)
    uint32_t ticket;
    int32_t k1;               // end of the current sentence range
    uint32_t pad[2];
};

// per-sub-block shared memory layout (bytes)
constexpr int kOffText = 0;                              // text bytes, later per-slot partial sums (sc)
constexpr int kOffCp = kOffText + kTextCap;              // code point per slot
constexpr int kOffPos = kOffCp + 4 * kSlotCap;           // byte position per slot (u16), later spill arrays
constexpr int kOffTy = kOffPos + 2 * kSlotCap;           // char type per slot (+ 32 guard bytes each side)
constexpr int kOffKk = kOffTy + kSlotCap + 64;           // sentence-in-group per slot
constexpr int kOffTab = kOffKk + kSlotCap;               // TileTables
constexpr int kOffBar = kOffTab + ((int(sizeof(TileTables)) + 15) & ~15);
constexpr int kSubBytes = (kOffBar + 16 + 15) & ~15;
// CTA-shared part
constexpr int kOffSeeds = 0;
constexpr int kOffTypeA = kOffSeeds + kSeedCap;
constexpr int kOffTypeB = kOffTypeA + 4 * kTypeSub;
constexpr int kOffTyTab = kOffTypeB + 4 * kTypeSub;  // character-type page table (256 B) + 4 sub-tables (textnorm.hpp)
constexpr int kOffSub = kOffTyTab + kTypeTableBytes;
constexpr int kTileSmem = kOffSub + kSubBlocks * kSubBytes;
static_assert(4 * kSlotCap <= kTextCap, "sc aliases the text buffer");
static_assert(2 * (kSlotCap / 32) * 8 * 4 <= 2 * kSlotCap, "spill arrays alias the position buffer");
static_assert(int(sizeof(Rings)) * (kSubThreads / 32) <= kOffPos, "fallback rings alias text+cp");
static_assert(kTileSmem <= 227 * 1024, "shared memory budget");
// what plan() reports (kernel_plan.hpp) is what the kernel is built with
static_assert(kTextCap == plan_detail::kTileTextCap && kSlotCap == plan_detail::kTileSlotCap, "tile buffers differ from the plan");
static_assert(kSubBlocks == plan_detail::kTileSubBlocks && kSeedCap == fused_detail::kSeedCap, "tile geometry differs from the plan");

__device__ __forceinline__ void sub_sync(int sub) {
    asm volatile("bar.sync %0, %1;" ::"r"(sub + 1), "r"(kSubThreads) : "memory");
}

template <bool kSeedsSmem>
__device__ __forceinline__ uint32_t slot_of_t(const DevTable& t, const uint8_t* s_seeds, uint64_t key) {
    uint32_t ha, hb;
    key_hashes(key, t.hk, ha, hb);
    const uint32_t b = bucket_of(ha, t.nbuckets);
    const uint32_t seed = kSeedsSmem ? uint32_t(s_seeds[b])
                                     : t.seed16 ? uint32_t(__ldg(reinterpret_cast<const uint16_t*>(t.seeds) + b))
                                                : uint32_t(__ldg(t.seeds + b));
    // (staged seeds: read the spill seed unconditionally, beside the primary one; index nbuckets, in the buffer, without
    //  a spill table)
    const uint32_t sb = spill_bucket_of(hb, t.nbuckets, t.spill_buckets);
    if (kSeedsSmem) return slot_of_seeds<true>(ha, hb, seed, uint32_t(s_seeds[sb]), t.nslots, t.spill_slots, t.spill_mul);
    if (!t.spill_buckets) return slot_of_seeds<false>(ha, hb, seed, 0u, t.nslots, 0u, 0u);
    return slot_of_seeds<true>(ha, hb, seed, uint32_t(__ldg(t.seeds + sb)), t.nslots, t.spill_slots, t.spill_mul);
}

__device__ __forceinline__ bool rec_matches(const Rec32& rec, uint64_t key) {
    const uint64_t k = (uint64_t(rec.v[1]) << 32) | rec.v[0];
    // (records of 2-symbol nodes hold a child mask in the unused c1 field: not part of the key)
    return (k & ~((key >> 42) ? kExtFlag : (kExtFlag | kChildMaskField))) == key;
}

// Continues a depth-3 hit backwards through the text for patterns longer than three characters (rare).
template <bool kSeedsSmem>
__device__ __forceinline__ bool deep_walk(const DevTable& t, const uint8_t* s_seeds, const uint32_t* __restrict__ cp, int p,
                                          uint32_t& slot, Rec32& rec) {
    bool deep_hit = false;
    uint32_t node = __ldg(t.slot_node + slot);
    for (int i = p - 3; cp[i] != 0; --i) {
        const uint64_t key = deep_key(node, cp[i]);
        const uint32_t nslot = slot_of_t<kSeedsSmem>(t, s_seeds, key);
        const Rec32 nrec = load_record(t.records, nslot);
        const uint64_t k = (uint64_t(nrec.v[1]) << 32) | nrec.v[0];
        if ((k & ~(kExtFlag | kOvfFlag)) != key) break;
        rec = nrec;
        slot = nslot;
        deep_hit = true;
        if (!(rec.v[1] >> 31)) break;
        node = __ldg(t.slot_node + nslot);
    }
    return deep_hit;
}

// Adds the part of a long row that lies outside the inline window (record flagged kOvfFlag) to the per-slot sums,
// clipped to the boundary slots [lo_slot, hi_slot) of the character's sentence.
__device__ __forceinline__ void apply_overflow(const DevTable& t, uint32_t slot, int p, int lo_slot, int hi_slot, int32_t* s_sc) {
    const uint64_t dsc = __ldg(t.slot_ovf + slot);
    const uint32_t ptr = uint32_t(dsc);
    const int off = int(int16_t(uint16_t(dsc >> 32))), len = int(uint16_t(dsc >> 48));
    int k_lo = lo_slot - (p + off), k_hi = hi_slot - (p + off);
    if (k_lo < 0) k_lo = 0;
    if (k_hi > len) k_hi = len;
    for (int k = k_lo; k < k_hi; ++k) {
        const int32_t w = __ldg(t.pool + ptr + k);
        if (w != 0) atomicAdd(s_sc + p + off + k, w);
    }
}

// gather of the 6-wide rows of one 32-slot warp chunk: boundary (lane) <- row entry j of lane - r0 - j
// (kR0 = compile-time window start for the common char-window-3 model, kRuntimeR0 = use the argument)
constexpr int kRuntimeR0 = 99;
template <int kR0, bool kAtomic = false>
__device__ __forceinline__ void gather_store(const int32_t (&d)[kInlineWidth], int r0_arg, int lane, int p, int32_t* s_sc,
                                             int32_t* s_spill_prev, int32_t* s_spill_next) {
    const int r0 = kR0 == kRuntimeR0 ? r0_arg : kR0;
    int32_t mainv = 0, to_prev = 0, to_next = 0;
#pragma unroll
    for (int j = 0; j < kInlineWidth; ++j) {
        const int src = lane - r0 - j;
        const int32_t v = __shfl_sync(kFull, d[j], src & 31);
        if (src < 0) to_next += v;
        else if (src >= 32) to_prev += v;
        else mainv += v;
    }
    if (kAtomic) atomicAdd(s_sc + p, mainv);  // overflow rows of other characters may target this slot concurrently
    else s_sc[p] = mainv;
    const int wc = p >> 5;
    if (lane >= 24) s_spill_prev[wc * 8 + lane - 24] = to_prev;
    if (lane < 8) s_spill_next[wc * 8 + lane] = to_next;
}

// General-table lookup + scatter for slot p of the flat slot stream: the row of the longest pattern ending at p
// adds w[k] to boundary slot p + off + k, restricted to the boundary slots [lo_slot, hi_slot) of p's sentence
// (what falls outside lands in the reference's strip padding or is clipped: predictor.rs:181-201).
template <bool kSeedsSmem, bool kTypes>
__device__ __forceinline__ void tile_scatter(const DevTable& t, const uint8_t* s_seeds, const uint32_t* __restrict__ cp,
                                             const uint8_t* __restrict__ ty, int p, int lo_slot, int hi_slot, int32_t* s_sc,
                                             uint32_t* state_out) {
    auto sym = [&](int i) -> uint32_t { return kTypes ? uint32_t(ty[i]) : cp[i]; };
    const uint32_t c3 = sym(p), c2 = sym(p - 1);
    const uint32_t c1 = c2 ? sym(p - 2) : 0u;
    uint64_t key = shallow_key(c1, c2, c3);
    Rec32 rec = load_record(t.records, slot_of_t<kSeedsSmem>(t, s_seeds, key));
    bool found = rec_matches(rec, key);
    const bool depth3 = found && c1 != 0;
    if (!found && c1 != 0) {
        key = shallow_key(0, c2, c3);
        rec = load_record(t.records, slot_of_t<kSeedsSmem>(t, s_seeds, key));
        found = rec_matches(rec, key);
    }
    if (!found && c2 != 0) {
        key = shallow_key(0, 0, c3);
        rec = load_record(t.records, slot_of_t<kSeedsSmem>(t, s_seeds, key));
        found = rec_matches(rec, key);
    }
    if (depth3 && (rec.v[1] >> 31)) {
        for (int i = p - 3; sym(i) != 0; --i) {
            key = deep_key(rec.v[6], sym(i));  // general records carry their node id
            const Rec32 nrec = load_record(t.records, slot_of_t<kSeedsSmem>(t, s_seeds, key));
            if (!rec_matches(nrec, key)) break;
            rec = nrec;
            if (!(rec.v[1] >> 31)) break;
        }
    }
    uint32_t pid = kNoPattern;
    if (found) {
        pid = rec.v[2];
        const uint32_t row = rec.v[3];
        if (row != kNoPattern) {
            const int off = int(rec.v[4]);
            const int len = int(rec.v[5]);
            int k_lo = lo_slot - (p + off), k_hi = hi_slot - (p + off);
            if (k_lo < 0) k_lo = 0;
            if (k_hi > len) k_hi = len;
            for (int k = k_lo; k < k_hi; ++k) atomicAdd(s_sc + p + off + k, __ldg(t.pool + row + k));
        }
    }
    if (state_out) *state_out = pid;
}

// kSplit3: type window 3 with the split tables in shared memory (compile-time type window: the common model shape)
// kOverflow: inline-format table whose deep records may carry rows wider than the window (dictionary words)
template <bool kSeedsSmem, int kR0, bool kGeneral, bool kSplit3, bool kOverflow>
__global__ void __launch_bounds__(kTileThreads, 1) k_tile_fast(DevModel m, BatchArgs a, int gap) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_seeds = smem + kOffSeeds;
    int32_t* s_type_a = reinterpret_cast<int32_t*>(smem + kOffTypeA);
    int32_t* s_type_b = reinterpret_cast<int32_t*>(smem + kOffTypeB);
    const int sub = threadIdx.x / kSubThreads;
    const int tid = threadIdx.x % kSubThreads, warp = tid >> 5, lane = tid & 31;
    uint8_t* sb = smem + kOffSub + sub * kSubBytes;
    uint8_t* s_text = sb + kOffText;
    int32_t* s_sc = reinterpret_cast<int32_t*>(sb + kOffText);
    uint32_t* s_cp = reinterpret_cast<uint32_t*>(sb + kOffCp);
    uint16_t* s_pos = reinterpret_cast<uint16_t*>(sb + kOffPos);
    int32_t* s_spill_prev = reinterpret_cast<int32_t*>(sb + kOffPos);
    int32_t* s_spill_next = s_spill_prev + (kSlotCap / 32) * 8;
    uint8_t* s_ty = sb + kOffTy + 32;  // 32 guard bytes in front
    uint8_t* s_kk = sb + kOffKk;
    TileTables& T = *reinterpret_cast<TileTables*>(sb + kOffTab);
    uint64_t* s_bar = reinterpret_cast<uint64_t*>(sb + kOffBar);
    const uint8_t* __restrict__ text = a.text;

    // ---- CTA-shared tables ----------------------------------------------------------------------------
    const bool tsplit = kSplit3;
    if (kSeedsSmem) {
        const uint32_t nwords = (m.ct.nbuckets + m.ct.spill_buckets + 3) / 4;
        const uint32_t* src = reinterpret_cast<const uint32_t*>(m.ct.seeds);
        for (uint32_t i = threadIdx.x; i < nwords; i += kTileThreads) reinterpret_cast<uint32_t*>(s_seeds)[i] = __ldg(src + i);
    }
    if (tsplit) {
        for (int i = threadIdx.x; i < kTypeSub; i += kTileThreads) {
            s_type_a[i] = __ldg(m.type_a + i);
            s_type_b[i] = __ldg(m.type_b + i);
        }
    }
    // character types by table: page table over c >> 8 (entries >= 0x80 select a 256-entry sub-table)
    uint8_t* s_tytab = smem + kOffTyTab;
    for (int i = threadIdx.x; i < kTypeTableBytes; i += kTileThreads) s_tytab[i] = uint8_t(type_table_entry(uint32_t(i)));
    if (tid == 0) mbar_init(s_bar, 1);
    if (tid < 8) reinterpret_cast<uint32_t*>(sb + kOffTy)[tid] = 0;  // front guard of s_ty
    __syncthreads();

    const uint64_t ngroups = (a.n_sent + kGroup - 1) / kGroup;
    const int r0 = m.ct.r0;
    const int tw = m.type_cache_window;
    uint32_t phase = 0;

    for (;;) {
        if (tid == 0) T.ticket = atomicAdd(a.ticket, 1u);
        sub_sync(sub);
        const uint64_t grp = T.ticket;
        if (grp >= ngroups) break;
        const uint64_t s0 = grp * kGroup;
        const int ns = int(min(uint64_t(kGroup), a.n_sent - s0));

        // ---- per-sentence tables -----------------------------------------------------------------------
        if (tid <= ns) T.off[tid] = a.offsets[s0 + tid];
        if (tid < ns) {
            const uint64_t s = s0 + tid;
            const uint32_t n = a.n_chars[s];
            const uint32_t lc = a.local_char[s], lb = a.local_bound[s];
            const uint64_t ob = a.group_bound[grp] + lb, cb = a.group_char[grp] + lc;
            T.nch[tid] = n;
            T.lc[tid] = lc;
            T.st[tid] = int8_t(a.status[s]);
            T.trim[tid] = a.trims ? a.trims[s] : uint8_t(0);
            T.obase[tid] = ob;
            T.cbase[tid] = cb;
            a.bound_offsets[s] = a.bound_base + ob;
            if (a.char_offsets) a.char_offsets[s] = a.char_base + cb;
            if (s + 1 == a.n_sent) {
                a.bound_offsets[s + 1] = a.bound_base + ob + (n > 0 ? n - 1 : 0);
                if (a.char_offsets) a.char_offsets[s + 1] = a.char_base + cb + n;
            }
        }
        if (tid == 0) T.lc[ns] = uint32_t(a.group_char[grp + 1] - a.group_char[grp]);
        sub_sync(sub);

        for (int k0 = 0; k0 < ns;) {
            // ---- choose the longest sentence range [k0, k1) that fits the tile buffers ---------------------
            // (the fit test is monotone in the range end: the first sentence that does not fit ends the range)
            if (tid == 0) T.k1 = ns;
            sub_sync(sub);
            if (tid >= k0 && tid < ns) {
                const uint64_t ra0 = T.off[k0] & ~15ull;
                const uint64_t rspan = (T.off[tid + 1] - ra0 + 15) & ~15ull;
                const int slots = gap + int(T.lc[tid + 1] - T.lc[k0]) + gap * (tid + 1 - k0);
                if (rspan + 16 > uint64_t(kTextCap) || ((slots + 8 + 255) & ~255) > kSlotCap) atomicMin(&T.k1, tid);
            }
            sub_sync(sub);
            const bool single = T.k1 == k0;
            const int k1 = single ? k0 + 1 : T.k1;
            if (single) {
                // a single sentence larger than the tile buffers: one warp walks it in 32-character steps
                Rings* rings = reinterpret_cast<Rings*>(sb);
                if (warp == 0) {
                    if (kGeneral) general_sentence_warp(m, a, s0 + k0, rings[0], lane);
                    else fast_sentence_warp(m, a, s0 + k0, rings[0], lane);
                }
                sub_sync(sub);
                k0 = k1;
                continue;
            }
            const uint64_t a0 = T.off[k0] & ~15ull;
            const uint32_t span = uint32_t((T.off[k1] - a0 + 15) & ~15ull);
            const int S = gap + int(T.lc[k1] - T.lc[k0]) + gap * (k1 - k0);
            const int Sround = (S + 8 + 255) & ~255;
            const uint32_t lc0 = T.lc[k0];

            // ---- stage the range's bytes: one TMA bulk copy --------------------------------------------------
            if (tid == 0 && span) {
                mbar_expect_tx(s_bar, span);
                tma_bulk_g2s(s_text, text + a0, span, s_bar);
            }
            for (int i = tid; i < Sround / 2; i += kSubThreads) reinterpret_cast<uint32_t*>(s_pos)[i] = 0xFFFFFFFFu;
            if (tid >= k0 && tid < k1) {
                const int64_t slot0 = int64_t(gap) + int64_t(T.lc[tid] - lc0) + int64_t(gap) * (tid - k0);
                T.odelta[tid] = int64_t(T.obase[tid]) - slot0;
                T.cdelta[tid] = int64_t(T.cbase[tid]) - slot0;
            }
            sub_sync(sub);
            if (span) {
                mbar_wait(s_bar, phase);
                phase ^= 1;
            }

            // ---- pass A: byte position and sentence of every character slot ---------------------------------
            for (int k = k0 + warp; k < k1; k += kSubThreads / 32) {
                if (T.st[k] != 0) {
                    const uint32_t nout = T.nch[k] > 0 ? T.nch[k] - 1 : 0;
                    for (uint32_t i = lane; i < nout; i += 32) { if (a.scores) a.scores[T.obase[k] + i] = 0; a.boundaries[T.obase[k] + i] = 0; }
                    if (a.char_states) for (uint32_t i = lane; i < T.nch[k]; i += 32) a.char_states[T.cbase[k] + i] = kNoPattern;
                    if (a.type_states) for (uint32_t i = lane; i < T.nch[k]; i += 32) a.type_states[T.cbase[k] + i] = kNoPattern;
                    continue;
                }
                const uint32_t rb0 = uint32_t(T.off[k] - a0), rb1 = uint32_t(T.off[k + 1] - a0) - T.trim[k];
                uint32_t idx = uint32_t(gap) + (T.lc[k] - lc0) + uint32_t(gap) * uint32_t(k - k0);
                for (uint32_t w = rb0 & ~3u; w < rb1; w += 128) {
                    const uint32_t addr = w + 4u * uint32_t(lane);
                    const uint32_t lo = addr < rb1 ? *reinterpret_cast<const uint32_t*>(s_text + addr) : 0u;
                    // start-of-character bytes of this word that lie inside the sentence (SWAR: bit 7 of byte j)
                    uint32_t smask = 0;
                    if (addr < rb1) {
                        const uint32_t from = rb0 > addr ? rb0 - addr : 0u;
                        const uint32_t to = rb1 - addr < 4u ? rb1 - addr : 4u;
                        const uint32_t im80 = (from >= 4u ? 0u : 0x80808080u << (8 * from)) & (0x80808080u >> (8 * (4 - to)));
                        const uint32_t st80 = ~(lo & ~(lo << 1)) & im80;       // not 10xxxxxx
                        smask = ((st80 >> 7) | (st80 >> 14) | (st80 >> 21) | (st80 >> 28)) & 15u;
                    }
                    const uint32_t cnt = __popc(smask);
                    const uint32_t incl = warp_incl_scan(cnt, lane);
                    uint32_t at = idx + incl - cnt;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (smask & (1u << j)) {
                            s_pos[at] = uint16_t(addr + j);
                            s_kk[at] = uint8_t(k);
                            ++at;
                        }
                    }
                    idx += __shfl_sync(kFull, incl, 31);
                }
            }
            sub_sync(sub);

            // ---- pass B: one thread per slot: decode the code point and its type -----------------------------
            for (int p = tid; p < Sround; p += kSubThreads) {
                const uint32_t pos = s_pos[p];
                uint32_t c = 0, ty = 0;
                if (pos != kSepPos) {
                    const uint32_t al = pos & ~3u;
                    const uint32_t lo = *reinterpret_cast<const uint32_t*>(s_text + al);
                    const uint32_t hi = *reinterpret_cast<const uint32_t*>(s_text + al + 4);
                    c = decode_cp(__funnelshift_r(lo, hi, 8 * (pos & 3u)));
                    if (c < 0x10000u) {
                        ty = type_from_table(s_tytab, c);
                    } else {
                        ty = char_type(c);
                    }
                }
                s_cp[p] = c;
                s_ty[p] = uint8_t(ty);
            }
            sub_sync(sub);
            if (m.kytea_norm) {
                // KyteaFullwidthFilter (textnorm.hpp) as its own pass, so that the common path above stays as it is:
                // the few characters the filter changes get their code point and type rewritten in place
                for (int p = tid; p < Sround; p += kSubThreads) {
                    const uint32_t c = s_cp[p];
                    const uint32_t f = kytea_fullwidth(c);
                    if (f != c) {
                        s_cp[p] = f;
                        s_ty[p] = uint8_t(char_type(f));
                    }
                }
                sub_sync(sub);
            }

            if constexpr (kGeneral) {
                // ---- pass C (general tables): rows of any offset/length scatter into the per-slot sums with
                //      shared-memory atomics; pattern-id states go straight to global memory ----------------------
                for (int p = tid; p < Sround; p += kSubThreads) s_sc[p] = 0;
                sub_sync(sub);
                uint32_t* cst = m.emit_states ? a.char_states : nullptr;
                uint32_t* tst = m.emit_states ? a.type_states : nullptr;
                for (int p = tid; p < Sround; p += kSubThreads) {
                    if (s_cp[p] == 0) continue;
                    const int k = s_kk[p];
                    const int lo_slot = int(int64_t(T.obase[k]) - T.odelta[k]);       // first slot of the sentence
                    const int hi_slot = lo_slot + int(T.nch[k]) - 1;                  // boundary slots [lo, hi)
                    if (m.ct.present)
                        tile_scatter<kSeedsSmem, false>(m.ct, s_seeds, s_cp, s_ty, p, lo_slot, hi_slot, s_sc,
                                                        cst ? cst + (int64_t(p) + T.cdelta[k]) : nullptr);
                    if (m.tt.present)
                        tile_scatter<false, true>(m.tt, s_seeds, s_cp, s_ty, p, lo_slot, hi_slot, s_sc,
                                                  tst ? tst + (int64_t(p) + T.cdelta[k]) : nullptr);
                }
            } else {
                if constexpr (kOverflow) {
                    for (int p = tid; p < Sround; p += kSubThreads) s_sc[p] = 0;
                    sub_sync(sub);
                }
                // ---- pass C: node lookup + warp-shuffle gather, two slots per thread in flight ----------------
                for (int base = 0; base < Sround; base += 2 * kSubThreads) {
                    const int pA = base + tid, pB = pA + kSubThreads;
                    const bool hasB = pB < Sround;  // uniform: Sround is a multiple of 256
                    int32_t dA[kInlineWidth], dB[kInlineWidth];
    #pragma unroll
                    for (int j = 0; j < kInlineWidth; ++j) dA[j] = dB[j] = 0;
                    uint32_t a1 = 0, a2 = 0, b1 = 0, b2 = 0, slA = 0, slB = 0;
                    const uint32_t a3 = m.ct.present ? s_cp[pA] : 0u;
                    const uint32_t b3 = (m.ct.present && hasB) ? s_cp[pB] : 0u;
                    Rec32 rA, rB;
                    if (a3) {
                        a2 = s_cp[pA - 1];
                        a1 = a2 ? s_cp[pA - 2] : 0u;
                        slA = slot_of_t<kSeedsSmem>(m.ct, s_seeds, shallow_key(a1, a2, a3));
                        rA = load_record(m.ct.records, slA);
                    }
                    if (b3) {
                        b2 = s_cp[pB - 1];
                        b1 = b2 ? s_cp[pB - 2] : 0u;
                        slB = slot_of_t<kSeedsSmem>(m.ct, s_seeds, shallow_key(b1, b2, b3));
                        rB = load_record(m.ct.records, slB);
                    }
                    // resolve both slots level by level so that the fallback probes of A and B are in flight together
                    bool fA = a3 != 0 && rec_matches(rA, shallow_key(a1, a2, a3));
                    bool fB = b3 != 0 && rec_matches(rB, shallow_key(b1, b2, b3));
                    const bool deepA = fA && a1 != 0 && (rA.v[1] >> 31), deepB = fB && b1 != 0 && (rB.v[1] >> 31);
                    {   // two-character suffixes
                        const bool nA = a3 != 0 && !fA && a1 != 0, nB = b3 != 0 && !fB && b1 != 0;
                        const uint64_t kA = shallow_key(0, a2, a3), kB = shallow_key(0, b2, b3);
                        // (a slot that still needs a probe has no use for its previous record: load in place)
                        if (nA) { slA = slot_of_t<kSeedsSmem>(m.ct, s_seeds, kA); rA = load_record(m.ct.records, slA); }
                        if (nB) { slB = slot_of_t<kSeedsSmem>(m.ct, s_seeds, kB); rB = load_record(m.ct.records, slB); }
                        if (nA) fA = rec_matches(rA, kA);
                        if (nB) fB = rec_matches(rB, kB);
                    }
                    {   // single characters
                        const bool nA = a3 != 0 && !fA && a2 != 0, nB = b3 != 0 && !fB && b2 != 0;
                        const uint64_t kA = shallow_key(0, 0, a3), kB = shallow_key(0, 0, b3);
                        // (a slot that still needs a probe has no use for its previous record: load in place)
                        if (nA) { slA = slot_of_t<kSeedsSmem>(m.ct, s_seeds, kA); rA = load_record(m.ct.records, slA); }
                        if (nB) { slB = slot_of_t<kSeedsSmem>(m.ct, s_seeds, kB); rB = load_record(m.ct.records, slB); }
                        if (nA) fA = rec_matches(rA, kA);
                        if (nB) fB = rec_matches(rB, kB);
                    }
                    bool dhA = false, dhB = false;
                    if (deepA) dhA = deep_walk<kSeedsSmem>(m.ct, s_seeds, s_cp, pA, slA, rA);
                    if (deepB) dhB = deep_walk<kSeedsSmem>(m.ct, s_seeds, s_cp, pB, slB, rB);
                    if constexpr (kOverflow) {
                        if (dhA && (rA.v[1] & (1u << 29))) {
                            const int k = s_kk[pA], lo_slot = int(int64_t(T.obase[k]) - T.odelta[k]);
                            apply_overflow(m.ct, slA, pA, lo_slot, lo_slot + int(T.nch[k]) - 1, s_sc);
                        }
                        if (dhB && (rB.v[1] & (1u << 29))) {
                            const int k = s_kk[pB], lo_slot = int(int64_t(T.obase[k]) - T.odelta[k]);
                            apply_overflow(m.ct, slB, pB, lo_slot, lo_slot + int(T.nch[k]) - 1, s_sc);
                        }
                    }
                    if (m.emit_states && a.char_states) {
                        // pattern id of the longest match (tag prediction input): side array indexed by the final slot
                        if (a3) a.char_states[int64_t(pA) + T.cdelta[s_kk[pA]]] = fA ? __ldg(m.ct.slot_pid + slA) : kNoPattern;
                        if (b3) a.char_states[int64_t(pB) + T.cdelta[s_kk[pB]]] = fB ? __ldg(m.ct.slot_pid + slB) : kNoPattern;
                    }
    #pragma unroll
                    for (int j = 0; j < kInlineWidth; ++j) {
                        dA[j] = fA ? int32_t(rA.v[2 + j]) : 0;
                        dB[j] = fB ? int32_t(rB.v[2 + j]) : 0;
                    }
                    gather_store<kR0, kOverflow>(dA, r0, lane, pA, s_sc, s_spill_prev, s_spill_next);
                    if (hasB) gather_store<kR0, kOverflow>(dB, r0, lane, pB, s_sc, s_spill_prev, s_spill_next);
                }
            }
            sub_sync(sub);

            // ---- pass D: one thread per boundary: spills, type table, bias, threshold, store ------------------
            const int nwc = Sround >> 5;
            for (int p = tid; p < Sround - 1; p += kSubThreads) {
                if (s_cp[p] == 0) continue;
                const int k = s_kk[p];
                // states not produced by pass C: "no pattern" (non-tag predictors), or the direct type-state table
                if (a.char_states && !(m.emit_states && m.ct.present)) a.char_states[int64_t(p) + T.cdelta[k]] = kNoPattern;
                if (a.type_states && !(kGeneral && m.emit_states && m.tt.present)) {
                    uint32_t ts = kNoPattern;
                    if (m.emit_states && m.type_state3) {
                        const uint32_t t2 = s_ty[p - 1], t1 = t2 ? uint32_t(s_ty[p - 2]) : 0u;
                        ts = __ldg(m.type_state3 + ((t1 << 6) | (t2 << 3) | s_ty[p]));
                    }
                    a.type_states[int64_t(p) + T.cdelta[k]] = ts;
                }
                if (s_cp[p + 1] == 0) continue;
                const int wc = p >> 5, ln = p & 31;
                int32_t v = s_sc[p] + m.bias;
                if (!kGeneral) {
                    if (ln >= 24 && wc + 1 < nwc) v += s_spill_prev[(wc + 1) * 8 + ln - 24];
                    if (ln < 8 && wc > 0) v += s_spill_next[(wc - 1) * 8 + ln];
                }
                if (kSplit3) {
                    const uint32_t ia = (uint32_t(s_ty[p - 2]) << 9) | (uint32_t(s_ty[p - 1]) << 6) | (uint32_t(s_ty[p]) << 3) | s_ty[p + 1];
                    const uint32_t ib = ((ia & 63u) << 6) | (uint32_t(s_ty[p + 2]) << 3) | s_ty[p + 3];
                    v += s_type_a[ia] + s_type_b[ib];
                } else if (tw > 0) {
                    uint32_t idx = 0;
                    for (int q = p - tw + 1; q <= p + tw; ++q) idx = (idx << 3) | s_ty[q];
                    v += __ldg(m.type_cache + idx);
                }
                const int64_t o = int64_t(p) + T.odelta[k];
                if (a.scores) a.scores[o] = v;
                a.boundaries[o] = v > 0 ? 1 : 0;
            }
            sub_sync(sub);
            k0 = k1;
        }
    }
}

}  // namespace

cudaError_t launch_count_only(const BatchArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    const uint64_t ngroups = (a.n_sent + kGroup - 1) / kGroup;
    k_count<<<unsigned(ngroups), kWarpsPerBlock * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_scan_only(const BatchArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    const uint64_t ngroups = (a.n_sent + kGroup - 1) / kGroup;
    k_scan_groups<<<1, 1024, 0, stream>>>(a.group_bound, a.group_char, ngroups, a.ticket, a.totals_host);
    return cudaGetLastError();
}

cudaError_t launch_count(const BatchArgs& a, cudaStream_t stream) {
    cudaError_t e = launch_count_only(a, stream);
    return e != cudaSuccess ? e : launch_scan_only(a, stream);
}

constexpr int kMaxDevices = 64;

template <bool kSeeds, int kR0, bool kGeneral, bool kSplit3, bool kOverflow>
static cudaError_t launch_tile_t(const KernelPlan& pl, const DevModel& m, const BatchArgs& a, cudaStream_t stream, int dev, int n_sm) {
    static std::atomic<bool> attr_set[kMaxDevices] = {};  // the opt-in shared memory size is a per-device function attribute
    if (!attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_tile_fast<kSeeds, kR0, kGeneral, kSplit3, kOverflow>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileSmem);
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    const uint64_t ngroups = (a.n_sent + kGroup - 1) / kGroup;
    const unsigned grid = unsigned(std::min<uint64_t>(uint64_t(n_sm), (ngroups + kSubBlocks - 1) / kSubBlocks));
    k_tile_fast<kSeeds, kR0, kGeneral, kSplit3, kOverflow><<<grid, kTileThreads, kTileSmem, stream>>>(m, a, pl.gap);
    return cudaGetLastError();
}

template <bool kSeeds, int kR0, bool kGeneral>
static cudaError_t launch_tile(const KernelPlan& pl, const DevModel& m, const BatchArgs& a, cudaStream_t stream, int dev, int n_sm) {
    if (pl.overflow)
        return pl.split3 ? launch_tile_t<kSeeds, kR0, false, true, true>(pl, m, a, stream, dev, n_sm)
                         : launch_tile_t<kSeeds, kR0, false, false, true>(pl, m, a, stream, dev, n_sm);
    return pl.split3 ? launch_tile_t<kSeeds, kR0, kGeneral, true, false>(pl, m, a, stream, dev, n_sm)
                     : launch_tile_t<kSeeds, kR0, kGeneral, false, false>(pl, m, a, stream, dev, n_sm);
}

cudaError_t launch_batch(const DevModel& m, const BatchArgs& a, cudaStream_t stream) {
    if (fused_ok(m)) return launch_fused(m, a, stream);
    cudaError_t e = launch_count(a, stream);
    return e != cudaSuccess ? e : launch_score(m, a, stream);
}

cudaError_t launch_score(const DevModel& m, const BatchArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    const KernelPlan pl = plan(m, a.char_states != nullptr || a.type_states != nullptr);
    if (pl.kernel == kPlanFused) return launch_fused(m, a, stream);  // self-contained: does not need the count pass
    if (pl.kernel == kPlanTileFast) {
        static std::atomic<int> sm_count[kMaxDevices] = {};  // (idempotent cache: every writer stores the same value)
        int dev = 0;
        cudaError_t e0 = cudaGetDevice(&dev);
        if (e0 != cudaSuccess) return e0;
        if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
        if (sm_count[dev] == 0) {
            int v = 0;
            e0 = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
            if (e0 != cudaSuccess) return e0;
            sm_count[dev] = v;
        }
        const int n_sm = sm_count[dev];
        if (pl.general) return pl.seeds_smem ? launch_tile<true, kRuntimeR0, true>(pl, m, a, stream, dev, n_sm)
                                             : launch_tile<false, kRuntimeR0, true>(pl, m, a, stream, dev, n_sm);
        if (pl.seeds_smem && pl.r0_fixed) return launch_tile<true, -3, false>(pl, m, a, stream, dev, n_sm);
        if (pl.seeds_smem) return launch_tile<true, kRuntimeR0, false>(pl, m, a, stream, dev, n_sm);
        if (pl.r0_fixed) return launch_tile<false, -3, false>(pl, m, a, stream, dev, n_sm);
        return launch_tile<false, kRuntimeR0, false>(pl, m, a, stream, dev, n_sm);
    }
    const uint64_t nblocks = (a.n_sent + kWarpsPerBlock - 1) / kWarpsPerBlock;
    if (pl.kernel == kPlanScoreFast) k_score_fast<<<unsigned(nblocks), kWarpsPerBlock * 32, 0, stream>>>(m, a);
    else k_score_general<<<unsigned(nblocks), kWarpsPerBlock * 32, 0, stream>>>(m, a);
    return cudaGetLastError();
}

int launches_per_batch(const DevModel& m) { return fused_ok(m) ? 1 : 3; }

// The paths that accumulate into the score array itself (general rows, overflow rows of long sentences) need
// it; the inline-row tile kernel keeps the sums in shared memory and can skip the score stores.
bool scores_optional(const DevModel& m) {
    const KernelPlan pl = plan(m, false);
    return (pl.kernel == kPlanFused || (pl.kernel == kPlanTileFast && !pl.general)) && !m.ct.has_overflow;
}

}  // namespace vpt
