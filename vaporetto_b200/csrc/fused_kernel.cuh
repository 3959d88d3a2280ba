// vaporetto_b200 — k_fused: the whole Predictor::predict hot path of a batch in ONE launch.
//
// Replaces (reference, vaporetto/src): sentence.rs:160-196 (parse_raw: validation, character count),
// predictor.rs:518-543 (predict), char_scorer/boundary_scorer.rs:93-113 and boundary_tag_scorer.rs:121-147 (pattern
// walk + weight add), predictor.rs:176-213 (PositionalWeight::add_score), type_scorer/boundary_scorer_cache.rs:59-81
// (type table), threshold predictor.rs:531-541.  Same results as k_count + k_scan_groups + k_tile_fast (kernels.cu),
// which stay for the model shapes this kernel does not take (DESIGN.md §4).
//
// One persistent CTA per SM = up to 4 independent 256-thread sub-blocks; a sub-block pulls 64-sentence groups from a
// global ticket and, per group:
//   load    every thread reads its 32-byte units of the group's UTF-8 bytes from global memory into registers
//           (L1::no_allocate, evict-first in L2), where they stay until the scatter step: no shared-memory staging,
//           so the shared memory is small enough for the 196 KB carve-out and the L1 it leaves (60 KB) holds the
//           node records of frequent characters and pairs
//   count   byte space, one thread per 32 bytes: SWAR masks of character starts, structural UTF-8 validation
//           (continuation bytes == bytes the leads ask for), NUL; one block scan gives every thread the number of
//           characters and sentence starts before its bytes -> group totals
//   publish the group's totals go to a descriptor; its output offset comes from a decoupled look-back over the
//           predecessors (no separate count / scan kernels, no second read of the text)
//   scatter every character's raw 4-byte window goes to its slot of the flat slot stream (`gap` zero slots between
//           sentences) together with its output index
//   stream  slot space, each warp owns a contiguous range of slots and walks it in 32-slot chunks with everything in
//           registers: decode + character type, left neighbours by shuffle (carried across chunks), longest-suffix
//           lookup as TWO probes (2-character node first; then the 3-character node if that node has extensions,
//           or the 1-character node if it does not exist) whose hashes share their partial sums (keys.hpp), a
//           software pipeline that keeps the record loads of three chunks in flight, shuffle gather of the 6-wide
//           rows (lagging so that every source lies to the left), type tables from a packed type history, bias,
//           threshold, coalesced stores.
// Groups the fast path cannot take (text or slots beyond the tile buffers, NUL / malformed UTF-8, zero-width
// sentences) run the same stream stage behind an exact per-sentence count (slow_*), a range at a time.
// No tensor cores: integer indexing + gather-add.
#pragma once
#include <atomic>
#include <type_traits>

#include "fused_launch.hpp"
#include "kernel_plan.hpp"
#include "kernels_common.cuh"
#include "utf8_window.hpp"

namespace vpt {

namespace {

constexpr int kFGroup = fused_detail::kGroupSentences;  // sentences per tile
constexpr int kFSubThreads = 256;
constexpr int kFWarps = kFSubThreads / 32;
// Tile buffers: bytes of text per tile (multiple of 32: a bound on the group's span, which the threads hold in registers)
// and character slots (characters + separators) per tile.
// 64 sentences of 40 characters need 7.4 KB and 2 760 slots; the buffers are sized so that 64 sentences of ragged
// natural-length text (log-normal, mean 41 characters: 7.6 +- 0.6 KB, 2 840 +- 220 slots) still fit -- a group that does
// not fit takes the slow path, and every later group waits in its look-back for the slow group's totals (with 8 192 B /
// 2 816 slots, ragged text took about twice as long per step as with 10 240 B / 3 840 slots, while the fixed-length batch
// gained about 1 %).  The variants with 4-byte slot words (pattern-id states) get the largest buffers
// that keep four sub-blocks per SM.
// (With the overflow sums -- 4 more bytes per slot -- the buffers are what keeps four sub-blocks per SM when the seeds
// live in global memory, the large-dictionary case, and three when they take 37 KB of shared memory.)
template <bool kSeedsSmem, bool kStates, bool kOverflow>
struct FCaps {
    static constexpr int kText = (kStates || (kOverflow && !kSeedsSmem)) ? 9216 : 10240;
    static constexpr int kSlots = !kOverflow ? (kStates ? 3328 : 3840)
                                  : kSeedsSmem ? (kStates ? 3264 : 3840)
                                               : (kStates ? 2944 : 3584);
};
constexpr int kFPadFront = 8;      // zero slots in front of slot 0 (halo of the first warp range)
constexpr int kFPadBack = 64;      // zero slots behind the last slot (lagging outputs of the last range)
constexpr int kFSeedCap = fused_detail::kSeedCap;   // seed bytes kept in shared memory
constexpr int kFTypeSub = 4096;    // entries of each split type table
constexpr int kFHalo = 8;          // slots a warp range re-reads in front of its first output

// decoupled look-back descriptors: 2-bit state + 62-bit value
constexpr uint64_t kDescAgg = 1ull << 62, kDescIncl = 2ull << 62, kDescVal = (1ull << 62) - 1;

struct FTab {
    uint64_t off[kFGroup + 1];
    uint32_t first[kFGroup + 1];  // group-local index of a sentence's first character; [ns] = characters of the group
    uint32_t lb[kFGroup + 1];     // group-local index of a sentence's first boundary; [ns] = boundaries of the group
    uint8_t st[kFGroup];         // slow path: status per sentence
    uint8_t trim[kFGroup];
    uint32_t wsum[kFWarps];
    uint64_t obase, cbase;       // output index of the group's first boundary / character (without bound_base)
    uint32_t ticket;
    int32_t anomaly;
    int32_t bad_chars;
    int32_t k1;
    uint32_t bytes_want, bytes_have;  // fast path: bytes of the group's characters, expected / summed by the stream stage
};

template <bool kSeedsSmem, bool kCommon, int kDeep, bool kStates>
struct FLayout {
    static constexpr bool kOverflow = kDeep == 2;
    using MetaT = typename std::conditional<kStates, uint32_t, uint16_t>::type;
    static constexpr int kFTextCap = FCaps<kSeedsSmem, kStates, kDeep == 2>::kText;
    static constexpr int kFSlotCap = FCaps<kSeedsSmem, kStates, kDeep == 2>::kSlots;
    static constexpr int kFSlotAlloc = kFPadFront + kFSlotCap + kFPadBack;
    static_assert(kFSlotCap < 4096, "output indices inside a tile are 12-bit");
    // CTA-shared part
    static constexpr int kOffSeeds = 0;
    static constexpr int kOffTypeA = kOffSeeds + (kSeedsSmem ? kFSeedCap : 0);
    static constexpr int kOffTypeB = kOffTypeA + (kCommon ? 4 * kFTypeSub : 0);
    static constexpr int kOffTyTab = kOffTypeB + (kCommon ? 4 * kFTypeSub : 0);
    static constexpr int kOffSub = kOffTyTab + kTypeTableBytes;
    // per sub-block (the group's text is read into registers, not staged here)
    static constexpr int kSRaw = 0;
    static constexpr int kSMeta = kSRaw + 4 * kFSlotAlloc;
    static constexpr int kSAcc = kSMeta + int(sizeof(MetaT)) * kFSlotAlloc;
    static constexpr int kSBitsS = kSAcc + (kOverflow ? 4 * kFSlotAlloc : 0);
    static constexpr int kSBitsX = kSBitsS + kFTextCap / 8 + 16;
    static constexpr int kSTab = kSBitsX + kFTextCap / 8 + 16;
    static constexpr int kSubBytes = (kSTab + int(sizeof(FTab)) + 127) & ~127;
    // four sub-blocks per SM (three with the overflow sums next to the seed table: kernel_plan.hpp)
    static constexpr int kSubBlocks = plan_detail::fused_sub_blocks(kSeedsSmem, kOverflow);
    static constexpr int kThreads = kSubBlocks * kFSubThreads;
    static constexpr int kSmem = kOffSub + kSubBlocks * kSubBytes;
    static_assert(kSmem <= 227 * 1024, "shared memory budget: more than a CTA may have");
    // Shared memory and L1 are one 256 KB array per SM: the L1 is what the shared-memory carve-out leaves (H100
    // carve-outs: ... 132, 164, 196, 228 KB), and it holds the node records of frequent characters and pairs.  With the
    // 1 KB the system reserves per CTA, every variant fits the 196 KB carve-out (60 KB of L1 or more) except the two
    // with overflow sums next to the seed table (three sub-blocks; 197 and 199 KB: the 228 KB carve-out).  The launch
    // asks for the smallest carve-out that fits.
    static constexpr int kCarveoutKB = (kOverflow && kSeedsSmem) ? 228 : 196;
    static_assert(kSmem + 1024 <= kCarveoutKB * 1024, "shared memory exceeds the carve-out this variant is built for");
    static_assert(int(sizeof(Rings)) <= 4 * kFSlotAlloc, "fallback ring aliases the slot array");
    // what plan() reports (kernel_plan.hpp) is what this variant is built with
    static_assert(kFTextCap == plan_detail::fused_text_cap(kSeedsSmem, kStates, kOverflow), "text buffer differs from the plan");
    static_assert(kFSlotCap == plan_detail::fused_slot_cap(kSeedsSmem, kStates, kOverflow), "slot buffer differs from the plan");
    static_assert(kSubBlocks == plan_detail::fused_sub_blocks(kSeedsSmem, kOverflow), "sub-blocks differ from the plan");
};

__device__ __forceinline__ void fsub_sync(int sub) {
    asm volatile("bar.sync %0, %1;" ::"r"(sub + 1), "r"(kFSubThreads) : "memory");
}

__device__ __forceinline__ uint64_t ld_relaxed(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
    return v;
}

// Exclusive prefixes of group `grp` over the two descriptor arrays at once (called by a full warp).  Every
// predecessor has at least published its aggregate or is being processed by a resident sub-block (tickets are handed
// out in order).  The two arrays are written independently (each word carries its own state), so the two scans may
// stop at different predecessors.
__device__ __forceinline__ void lookback2(const uint64_t* desc_b, const uint64_t* desc_c, uint64_t grp, int lane, uint64_t& sum_b,
                                          uint64_t& sum_c) {
    sum_b = 0;
    sum_c = 0;
    bool done_b = false, done_c = false;
    for (int64_t j = int64_t(grp) - 1; j >= 0 && !(done_b && done_c); j -= 32) {
        const int64_t idx = j - lane;
        uint64_t vb = kDescIncl, vc = kDescIncl;  // before the first group: an inclusive prefix of zero
        if (idx >= 0) {
            vb = ld_relaxed(desc_b + idx);
            vc = ld_relaxed(desc_c + idx);
            while ((vb >> 62) == 0 || (vc >> 62) == 0) {
                __nanosleep(20);
                vb = ld_relaxed(desc_b + idx);
                vc = ld_relaxed(desc_c + idx);
            }
        }
        if (!done_b) {
            const unsigned incl = __ballot_sync(kFull, (vb >> 62) == 2);
            const int first = incl ? __ffs(incl) - 1 : 32;
            sum_b += warp_sum64(lane <= first ? (vb & kDescVal) : 0ull);
            done_b = incl != 0;
        }
        if (!done_c) {
            const unsigned incl = __ballot_sync(kFull, (vc >> 62) == 2);
            const int first = incl ? __ffs(incl) - 1 : 32;
            sum_c += warp_sum64(lane <= first ? (vc & kDescVal) : 0ull);
            done_c = incl != 0;
        }
    }
}

// value of lane (lane - d) of the 64-lane sequence [prev chunk | this chunk] (shfl takes the source lane modulo 32)
__device__ __forceinline__ uint32_t up_u(uint32_t cur, uint32_t prev, int d, int lane) {
    const uint32_t src = lane >= 32 - d ? prev : cur;
    return __shfl_sync(kFull, src, lane - d);
}
__device__ __forceinline__ int32_t up_i(int32_t cur, int32_t prev, int d, int lane) {
    return int32_t(up_u(uint32_t(cur), uint32_t(prev), d, lane));
}

// (decode_any / decode_ascii_or_three: utf8_window.hpp -- plain arithmetic, also compiled and tested on the host)
// The decoder of a warp: Japanese text is three-byte characters and ASCII; the general decoder runs only for a chunk
// that holds another lead byte.
__device__ __forceinline__ uint32_t decode_checked(uint32_t x, bool& bad, uint32_t& len) {
    const bool ascii = (x & 0x80u) == 0, three = (x & 0xF0u) == 0xE0u;
    if (__any_sync(kFull, !(ascii || three))) return decode_any(x, bad, len);
    return decode_ascii_or_three(x, ascii, three, bad, len);
}

__device__ __forceinline__ uint32_t type_of(uint32_t c, const uint8_t* s_tytab) {
    if (c >= 0x10000u) return char_type(c);
    return type_from_table(s_tytab, c);
}

// The text goes from global memory straight into registers.  It is read once, so it is not allocated in L1 (which
// holds the hot node records) and it is evict-first in L2 (which must keep the node table while the text and the
// outputs stream through it).
__device__ __forceinline__ uint4 ldg_text16(const uint8_t* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(l2_policy_evict_first()));
    return v;
}
__device__ __forceinline__ uint32_t ldg_text4(const uint8_t* p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(l2_policy_evict_first()));
    return v;
}

// the bytes of word x whose bits are set in the 4-bit mask `keep` stay, the others read as spaces
__device__ __forceinline__ uint32_t keep_bytes(uint32_t x, uint32_t keep) {
    const uint32_t bm = ((keep * 0x00204081u) & 0x01010101u) * 0xFFu;  // bit j of `keep` -> byte j
    return (x & bm) | (0x20202020u & ~bm);
}

// Exact validation + character count of one sentence by one warp, from global memory (slow path; the rules of
// k_count's per-byte branch: reference sentence.rs:160-196 + str::from_utf8).
__device__ __forceinline__ void slow_validate(const uint8_t* __restrict__ text, uint64_t b0, uint64_t b1, int lane,
                                              uint32_t& nch, int& status) {
    uint32_t starts = 0, conts = 0, expect = 0, flags = 0;
    for (uint64_t pos = b0 + uint64_t(lane); pos < b1; pos += 32) {
        const uint32_t b = __ldg(text + pos);
        if ((b & 0xC0u) == 0x80u) { ++conts; continue; }
        ++starts;
        if (b == 0) flags |= 1;
        if (b < 0x80u) continue;
        const uint32_t c1 = pos + 1 < b1 ? __ldg(text + pos + 1) : 0u, c2 = pos + 2 < b1 ? __ldg(text + pos + 2) : 0u,
                       c3 = pos + 3 < b1 ? __ldg(text + pos + 3) : 0u;
        uint32_t len;
        bool ok;
        if (b < 0xC2u) { len = 1; ok = false; }
        else if (b < 0xE0u) { len = 2; ok = (c1 & 0xC0u) == 0x80u; }
        else if (b < 0xF0u) {
            len = 3;
            ok = (c1 & 0xC0u) == 0x80u && (c2 & 0xC0u) == 0x80u && !(b == 0xE0u && c1 < 0xA0u) && !(b == 0xEDu && c1 > 0x9Fu);
        } else if (b < 0xF5u) {
            len = 4;
            ok = (c1 & 0xC0u) == 0x80u && (c2 & 0xC0u) == 0x80u && (c3 & 0xC0u) == 0x80u && !(b == 0xF0u && c1 < 0x90u) &&
                 !(b == 0xF4u && c1 > 0x8Fu);
        } else { len = 1; ok = false; }
        if (pos + len > b1) ok = false;
        if (!ok) flags |= 2;
        expect += len - 1;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        starts += __shfl_xor_sync(kFull, starts, d);
        conts += __shfl_xor_sync(kFull, conts, d);
        expect += __shfl_xor_sync(kFull, expect, d);
        flags |= __shfl_xor_sync(kFull, flags, d);
    }
    if (conts != expect) flags |= 2;
    nch = starts;
    status = (flags & 2) ? 3 : (flags & 1) ? 2 : (starts == 0 ? 1 : 0);
}

// Characters (bytes that are not continuation bytes) of the sentence [b0, b1): one 4-byte word per lane and 128-byte step.
// The text buffer is readable up to a multiple of 16 bytes (include/vaporetto_b200.h), and an address has the alignment of
// its offset (the batch's text pointer is biased that way).
__device__ __forceinline__ uint32_t slow_count(const uint8_t* __restrict__ text, uint64_t b0, uint64_t b1, int lane) {
    uint32_t cnt = 0;
    for (uint64_t addr = (b0 & ~3ull) + 4u * uint64_t(lane); addr < b1; addr += 128) {
        const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(text + addr));
        uint32_t in80 = 0x80808080u;  // bit 7 of the bytes of this word that lie inside [b0, b1)
        if (addr < b0) in80 &= 0xFFFFFFFFu << (8u * uint32_t(b0 - addr));
        if (addr + 4 > b1) in80 &= 0xFFFFFFFFu >> (8u * uint32_t(addr + 4 - b1));
        cnt += __popc(~(w & ~(w << 1)) & in80);  // not 10xxxxxx
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_xor_sync(kFull, cnt, d);
    return cnt;
}

// Zero outputs of a rejected sentence (the reference never scores it: Sentence::from_raw fails).
__device__ __forceinline__ void zero_sentence(const BatchArgs& a, uint64_t ob, uint64_t cb, uint32_t n, int lane) {
    const uint32_t nout = n > 0 ? n - 1 : 0;
    for (uint32_t i = lane; i < nout; i += 32) {
        if (a.scores) a.scores[ob + i] = 0;
        a.boundaries[ob + i] = 0;
    }
    if (a.char_states) for (uint32_t i = lane; i < n; i += 32) a.char_states[cb + i] = kNoPattern;
    if (a.type_states) for (uint32_t i = lane; i < n; i += 32) a.type_states[cb + i] = kNoPattern;
}

// ---- rare paths of the stream stage -----------------------------------------------------------------------------------

// Continues a 3-character hit backwards through the slot stream for patterns longer than three characters.
template <bool kSeedsSmem>
__device__ __forceinline__ bool deep_walk_f(const DevTable& t, const uint32_t* s_raw, int p, bool norm, uint32_t& slot, Rec32& rec) {
    bool deep_hit = false;
    uint32_t node = __ldg(t.slot_node + slot);
    for (int i = p - 3;; --i) {
        const uint32_t x = s_raw[i];
        if (x == 0) break;
        bool bad;
        uint32_t len;
        uint32_t c = decode_any(x, bad, len);  // (not the warp-wide decoder: only some lanes walk)
        if (norm) c = kytea_fullwidth(c);
        const uint64_t key = deep_key(node, c);
        const uint32_t nslot = slot_of<kSeedsSmem>(t, key);
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

// Adds the part of a long row outside the inline window to the per-slot sums, clipped to the boundary slots of the
// character's sentence (found by looking for the separator slots around p).
__device__ __forceinline__ void apply_overflow_f(const DevTable& t, uint32_t slot, int p, const uint32_t* s_raw, int32_t* s_acc) {
    const uint64_t dsc = __ldg(t.slot_ovf + slot);
    const uint32_t ptr = uint32_t(dsc);
    const int off = int(int16_t(uint16_t(dsc >> 32))), len = int(uint16_t(dsc >> 48));
    int lo = p + off, hi = p + off + len;  // boundary slots [lo, hi) the row wants
    if (lo < p) {
        int q = p;
        while (q > lo && s_raw[q - 1] != 0) --q;  // first slot of the sentence, if inside the row's reach
        lo = q > lo ? q : lo;
    }
    {
        int q = p;  // last valid boundary slot is the one before the sentence's last character
        while (q < hi && s_raw[q + 1] != 0) ++q;
        hi = q < hi ? q : hi;
    }
    for (int b = lo; b < hi; ++b) {
        const int32_t w = __ldg(t.pool + ptr + (b - p - off));
        if (w != 0) atomicAdd(s_acc + b, w);
    }
}

template <bool kSeedsSmem>
__device__ __forceinline__ uint32_t seed_of(const DevTable& t, const uint8_t* s_seeds, uint32_t b) {
    return kSeedsSmem ? uint32_t(s_seeds[b])
                      : t.seed16 ? uint32_t(__ldg(reinterpret_cast<const uint16_t*>(t.seeds) + b)) : uint32_t(__ldg(t.seeds + b));
}

// Slot of `key hashes (h, g)` in the node table, and its record.  The spill seed is read beside the primary one (no
// dependent load); only tables whose seeds are staged in shared memory have a spill table (validate_blob_header).
template <bool kSeedsSmem>
__device__ __forceinline__ Rec32 probe_load(const DevTable& ct, const uint8_t* s_seeds, uint32_t h, uint32_t g, uint32_t& slot) {
    const uint32_t seed = seed_of<kSeedsSmem>(ct, s_seeds, mulhi32(h, ct.nbuckets));
    const uint32_t spill_seed = kSeedsSmem ? uint32_t(s_seeds[spill_bucket_of(g, ct.nbuckets, ct.spill_buckets)]) : 0u;
    slot = slot_of_seeds<kSeedsSmem>(h, g, seed, spill_seed, ct.nslots, ct.spill_slots, ct.spill_mul);
    // (as PTX: the compiler otherwise folds "slot times 32" into a 64-bit shift/mask sequence of ALU-pipe instructions;
    //  this is IMAD.WIDE on the FMA pipe -- the kernel's ALU pipe is its busiest unit)
    uint64_t addr;
    asm("mad.wide.u32 %0, %1, 32, %2;" : "=l"(addr) : "r"(slot), "l"(ct.records));
    return load_record(reinterpret_cast<const void*>(addr), 0);
}

// ---- the stream stage: slots [0, S) of the tile's flat slot stream -> scores / boundaries / states ----------------
// kCommon: the usual model shape (char window 3: inline window r0 = -3; type window 3 with the split tables in shared
// memory): lag and shuffle distances are compile-time constants.  Otherwise they come from cfg and the type table is
// read from global memory.
template <bool kSeedsSmem, bool kCommon, int kDeep, bool kStates, typename MetaT>
__device__ __forceinline__ void stream_stage(const DevModel& m, const BatchArgs& a, const StreamCfg cfg, const uint32_t* s_raw,
                                             MetaT* s_meta, int32_t* s_acc, const uint8_t* s_seeds, const int32_t* s_ta,
                                             const int32_t* s_tb, const uint8_t* s_tytab, FTab& T, int S, uint64_t obase,
                                             uint64_t cbase, int warp, int lane) {
    // obase / cbase: output index of the tile's first boundary / character (the meta indices are tile-local)
    constexpr bool kOverflow = kDeep == 2;
    const int R = (S + kFWarps - 1) / kFWarps;
    const int ra = warp * R, rb = min(S, ra + R);
    if (ra >= rb) return;
    const int L = kCommon ? 3 : cfg.lag;
    const int dist0 = kCommon ? 0 : L + cfg.r0;  // shuffle distance of row entry 0 (entry j: dist0 + j)
    const int tw = kCommon ? 3 : cfg.tw;
    const int p0 = ra - kFHalo;
    const int nchunk = (rb + L - p0 + 31) >> 5;
    const DevTable& ct = m.ct;
    const bool have_ct = kCommon || ct.present != 0;  // (the common shape has a char scorer: fused.cu)
    const uint32_t ka0 = ct.hk.a[0], ka1 = ct.hk.a[1], ka2 = ct.hk.a[2], kb0 = ct.hk.b[0], kb1 = ct.hk.b[1], kb2 = ct.hk.b[2];
    int32_t* const scores = a.scores ? a.scores + obase : nullptr;
    uint8_t* const bounds = a.boundaries + obase;
    const bool want_cst = kStates && a.char_states != nullptr, want_tst = kStates && a.type_states != nullptr;
    const bool emit_c = m.emit_states && have_ct;

    // Software pipeline over the 32-slot chunks of the range: three chunks are in flight, so that the record loads of
    // the first probe (chunk it) and of the second probe (chunk it-1) are outstanding while chunk it-2 is finished.
    //   state A: chunk it-1 after stage 1 (first probe issued)
    uint32_t cA = 0, c2A = 0, c1A = 0, HA = 0, slA = 0;
    Rec32 rA;
    //   state B: chunk it-2 after stage 2 (second probe issued)
    uint32_t kloB = 0, khiB = 0, HB = 0, flB = 0, slB = 0, sl1B = 0;  // slB / sl1B: slots of the second / first probe  // flB: 1 first probe hit, 2 second probe issued, 4 .. for 3 characters
    int32_t dB[kInlineWidth];
    Rec32 rB;
    //   carried from chunk to chunk
    uint32_t pcc = 0, pH3 = 0;
    int32_t pd[kInlineWidth];
    uint32_t nbytes = 0;  // bytes of the characters of this warp's range (structural check: the tile's must add up)
#pragma unroll
    for (int j = 0; j < kInlineWidth; ++j) { pd[j] = 0; dB[j] = 0; }
#pragma unroll
    for (int j = 0; j < 8; ++j) { rA.v[j] = 0; rB.v[j] = 0; }

    // one pipeline step; d3 / d2 / d1 select the stages at compile time (prologue, steady state, epilogue)
    auto step = [&](const int it, auto d3, auto d2, auto d1) {
        // ================= stage 3: chunk it-2 — second probe result, gather, type table, output ========================
        if constexpr (decltype(d3)::value) {
            const int p = p0 + ((it - 2) << 5) + lane;
            bool f2 = (flB & 2u) && rB.v[0] == kloB && (rB.v[1] & 0x7FFFFFFFu) == khiB;
            if (kDeep > 0) {
                if (f2 && (flB & 4u) && (rB.v[1] >> 31)) {
                    // a 3-character node with longer extensions: walk on (patterns longer than 3: dictionary words)
                    const bool dh = deep_walk_f<kSeedsSmem>(ct, s_raw, p, cfg.norm, slB, rB);
                    // (the slots of the halo and behind the range end are walked by two warps: only the owner adds)
                    if (kOverflow) { if (dh && (rB.v[1] & (1u << 29)) && p >= ra && p < rb) apply_overflow_f(ct, slB, p, s_raw, s_acc); }
                }
            }
            int32_t d[kInlineWidth];
#pragma unroll
            for (int j = 0; j < kInlineWidth; ++j) d[j] = f2 ? int32_t(rB.v[2 + j]) : dB[j];
            if (kStates) {
                if ((want_cst || want_tst) && (HB & 7u) != 0 && p >= ra && p < rb) {
                    const uint64_t ci = cbase + (uint32_t(s_meta[p]) >> 12);
                    if (want_cst) a.char_states[ci] = (emit_c && (f2 || (flB & 1u))) ? __ldg(ct.slot_pid + (f2 ? slB : sl1B)) : kNoPattern;
                    if (want_tst) a.type_states[ci] = (m.emit_states && m.type_state3) ? __ldg(m.type_state3 + (HB & 0x1FFu)) : kNoPattern;
                }
            }
            // gather: boundary b = p - L takes entry j of the row found at slot p - (dist0 + j)
            int32_t v = m.bias;
#pragma unroll
            for (int j = 0; j < kInlineWidth; ++j) {
                const int dist = dist0 + j;
                v += dist == 0 ? d[j] : up_i(d[j], pd[j], dist, lane);
                pd[j] = d[j];
            }
            // type table of the 2*tw types around b: H holds t[p-5 .. p], 3 bits each, t[p] lowest
            if (kCommon) {
                v += s_ta[(HB >> 6) & 0xFFFu] + s_tb[HB & 0xFFFu];
            } else if (m.type_a != nullptr && tw == 3) {
                v += __ldg(m.type_a + ((HB >> (3 * (L - 1))) & 0xFFFu)) + __ldg(m.type_b + ((HB >> (3 * (L - 3))) & 0xFFFu));
            } else if (tw > 0) {
                v += __ldg(m.type_cache + ((HB >> (3 * (L - tw))) & ((1u << (6 * tw)) - 1u)));
            }
            const int b = p - L;
            const bool ok = ((HB >> (3 * L)) & 7u) != 0 && ((HB >> (3 * (L - 1))) & 7u) != 0 && b >= ra && b < rb;
            if (kOverflow) {
                // rows of long dictionary words add into s_acc from any slot of the tile: finish in a later pass
                constexpr MetaT kValid = MetaT(1u << (8 * sizeof(MetaT) - 1));
                if (ok) { atomicAdd(s_acc + b, v); s_meta[b] = MetaT(s_meta[b] | kValid); }
            } else if (ok) {
                const uint32_t ol = uint32_t(s_meta[b]) & 0xFFFu;
                // (streaming stores: the outputs are not read again by this kernel)
                if (scores) __stcs(scores + ol, v);
                __stcs(bounds + ol, uint8_t(v > 0 ? 1 : 0));
            }
        }
        // ================= stage 2: chunk it-1 — first probe result, second probe =====================================
        if constexpr (decltype(d2)::value) {
            const uint32_t klo = cA | (c2A << 21), khi = c2A >> 11;
            const bool act = cA != 0 && have_ct;
            // (bits 10..28 of the second key word of a 2-character record: the mask of its 3-character extensions)
            // bits 29 / 30 of the word (61 / 62 of the key) are clear in a 2-symbol record and the deep-key marker sets
            // bit 30: a (parent node, symbol) record whose parent id equals c2 as a number has the same low 42 bits and
            // must not pass for the 2-character node when that node does not exist (found by the fuzzer: 1 case in 1 300
            // random models; tests/golden/fuzz_cases/)
            const bool f1 = act && rA.v[0] == klo && (rA.v[1] & 0x600003FFu) == khi;
            // the 3-character node if the 2-character node may have this extension, the 1-character node if the
            // 2-character node does not exist
            const bool w3 = f1 && c1A != 0 && ((rA.v[1] >> (10u + child_bit(c1A))) & 1u) != 0, w1 = act && !f1 && c2A != 0;
            slB = slA;
            if (kStates) sl1B = slA;
            if (w3 || w1) {
                const uint32_t h2 = cA * ka0 + c2A * ka1, g2 = cA * kb0 + c2A * kb1;
                rB = probe_load<kSeedsSmem>(ct, s_seeds, w3 ? h2 + c1A * ka2 : cA * ka0, w3 ? g2 + c1A * kb2 : cA * kb0, slB);
            }
            kloB = w3 ? klo : cA;
            khiB = w3 ? (khi | (c1A << 10)) : 0u;
            flB = (f1 ? 1u : 0u) | ((w3 || w1) ? 2u : 0u) | (w3 ? 4u : 0u);
#pragma unroll
            for (int j = 0; j < kInlineWidth; ++j) dB[j] = f1 ? int32_t(rA.v[2 + j]) : 0;
            HB = HA;
        }
        // ================= stage 1: chunk it — decode, type, neighbours, first probe ====================================
        if constexpr (decltype(d1)::value) {
            const int p = p0 + (it << 5) + lane;
            bool bad;
            uint32_t len;
            uint32_t c = decode_checked(s_raw[p], bad, len);
            if (p >= ra && p < rb) nbytes += len;
            if (cfg.norm) c = kytea_fullwidth(c);
            if (__any_sync(kFull, bad)) { if (bad) T.bad_chars = 1; }
            const uint32_t ty = c ? type_of(c, s_tytab) : 0u;
            // left neighbours: code point | type << 24 travels as one value
            const uint32_t cc = c | (ty << 24);
            const uint32_t n1 = up_u(cc, pcc, 1, lane), n2 = up_u(cc, pcc, 2, lane);
            pcc = cc;
            cA = c;
            c2A = n1 & 0x1FFFFFu;
            c1A = n2 & 0x1FFFFFu;
            // packed type history t[p-5 .. p]
            const uint32_t h3 = ty + (n1 >> 24) * 8u + (n2 >> 24) * 64u;
            HA = h3 | (up_u(h3, pH3, 3, lane) << 9);
            pH3 = h3;
            // first probe: the node of the last two characters (one character at a sentence start)
            if (c != 0 && have_ct) rA = probe_load<kSeedsSmem>(ct, s_seeds, c * ka0 + c2A * ka1, c * kb0 + c2A * kb1, slA);
        }
    };
    using Yes = std::true_type;
    using No = std::false_type;
    step(0, No{}, No{}, Yes{});
    if (nchunk >= 2) {
        step(1, No{}, Yes{}, Yes{});
        // Unrolled by two where it fits the register budget: the copies of the carried pipeline state between steps
        // then become register renames (the variants without deep patterns or states: fewer spills, and config 2's
        // step 3 % shorter).  The others spill more when unrolled and keep the one-step loop.
        if constexpr (kDeep == 0 && !kStates) {
#pragma unroll 2
            for (int it = 2; it < nchunk; ++it) step(it, Yes{}, Yes{}, Yes{});
        } else {
#pragma unroll 1
            for (int it = 2; it < nchunk; ++it) step(it, Yes{}, Yes{}, Yes{});
        }
        step(nchunk, Yes{}, Yes{}, No{});
        step(nchunk + 1, Yes{}, No{}, No{});
    } else {
        step(1, No{}, Yes{}, No{});
        step(2, Yes{}, No{}, No{});
    }
#pragma unroll
    for (int dd = 16; dd > 0; dd >>= 1) nbytes += __shfl_xor_sync(kFull, nbytes, dd);
    if (lane == 0) atomicAdd(&T.bytes_have, nbytes);
}

// one tile's final pass of the overflow variant: per-slot sums -> outputs
template <typename MetaT>
__device__ __forceinline__ void finish_overflow(const BatchArgs& a, MetaT* s_meta, const int32_t* s_acc, uint64_t obase, int S, int tid) {
    constexpr MetaT kValid = MetaT(1u << (8 * sizeof(MetaT) - 1));
    for (int p = tid; p < S; p += kFSubThreads) {
        const MetaT mt = s_meta[p];
        if (!(mt & kValid)) continue;
        const uint32_t ol = uint32_t(mt) & 0xFFFu;
        const int32_t v = s_acc[p];
        if (a.scores) a.scores[obase + ol] = v;
        a.boundaries[obase + ol] = v > 0 ? 1 : 0;
    }
}

template <bool kSeedsSmem, bool kCommon, int kDeep, bool kStates>
__global__ void __launch_bounds__((FLayout<kSeedsSmem, kCommon, kDeep, kStates>::kThreads), 1)
k_fused(DevModel m, BatchArgs a, StreamCfg cfg) {
    using Lay = FLayout<kSeedsSmem, kCommon, kDeep, kStates>;
    using MetaT = typename Lay::MetaT;
    constexpr bool kOverflow = kDeep == 2;
    constexpr int kFTextCap = Lay::kFTextCap, kFSlotCap = Lay::kFSlotCap, kFSlotAlloc = Lay::kFSlotAlloc;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* s_seeds = smem + Lay::kOffSeeds;
    int32_t* s_ta = reinterpret_cast<int32_t*>(smem + Lay::kOffTypeA);
    int32_t* s_tb = reinterpret_cast<int32_t*>(smem + Lay::kOffTypeB);
    uint8_t* s_tytab = smem + Lay::kOffTyTab;
    const int sub = threadIdx.x / kFSubThreads;
    const int tid = threadIdx.x % kFSubThreads, warp = tid >> 5, lane = tid & 31;
    uint8_t* sb = smem + Lay::kOffSub + sub * Lay::kSubBytes;
    uint32_t* s_raw_alloc = reinterpret_cast<uint32_t*>(sb + Lay::kSRaw);
    uint32_t* s_raw = s_raw_alloc + kFPadFront;
    MetaT* s_meta = reinterpret_cast<MetaT*>(sb + Lay::kSMeta) + kFPadFront;
    int32_t* s_acc = reinterpret_cast<int32_t*>(sb + Lay::kSAcc) + kFPadFront;
    uint32_t* s_sbits = reinterpret_cast<uint32_t*>(sb + Lay::kSBitsS);
    uint32_t* s_xbits = reinterpret_cast<uint32_t*>(sb + Lay::kSBitsX);
    FTab& T = *reinterpret_cast<FTab*>(sb + Lay::kSTab);
    const uint8_t* __restrict__ text = a.text;
    uint64_t* const desc_b = a.group_bound;  // look-back descriptors (zeroed by the launcher, with the ticket)
    uint64_t* const desc_c = a.group_char;

    // ---- CTA-shared tables -------------------------------------------------------------------------------------
    if (kSeedsSmem) {
        const uint32_t nwords = (m.ct.nbuckets + m.ct.spill_buckets + 3) / 4;
        const uint32_t* src = reinterpret_cast<const uint32_t*>(m.ct.seeds);
        for (uint32_t i = threadIdx.x; i < nwords; i += Lay::kThreads) reinterpret_cast<uint32_t*>(s_seeds)[i] = __ldg(src + i);
    }
    if (kCommon) {
        for (int i = threadIdx.x; i < kFTypeSub; i += Lay::kThreads) {
            s_ta[i] = __ldg(m.type_a + i);
            s_tb[i] = __ldg(m.type_b + i);
        }
    }
    // character types by table: page table over c >> 8 + the sub-tables of the mixed pages (textnorm.hpp)
    for (int i = threadIdx.x; i < kTypeTableBytes; i += Lay::kThreads) s_tytab[i] = uint8_t(type_table_entry(uint32_t(i)));
    __syncthreads();

    const uint64_t ngroups = (a.n_sent + kFGroup - 1) / kFGroup;
    // (the common shape separates sentences by two slots -- fused.cu checks it --: the separator loop of the scatter step,
    //  which a whole warp walks for the one lane that sees a sentence start, unrolls to two stores)
    const int gap = kCommon ? fused_detail::kCommonGap : cfg.gap;

    for (;;) {
        if (tid == 0) T.ticket = atomicAdd(a.ticket, 1u);
        fsub_sync(sub);
        const uint64_t grp = T.ticket;
        if (grp >= ngroups) break;
        // (the per-group flags are cleared behind the barrier: the other threads read them after the last barrier of
        //  the previous group, bytes_have / bad_chars below; their first use in this group is two barriers away)
        if (tid == 0) {
            T.anomaly = 0;
            T.bad_chars = 0;
            T.bytes_want = 0;  // (first: the sum of the excluded bytes)
            T.bytes_have = 0;
        }
        const uint64_t s0 = grp * kFGroup;
        const int ns = int(min(uint64_t(kFGroup), a.n_sent - s0));
        if (tid <= ns) T.off[tid] = a.offsets[s0 + tid];
        if (tid < ns) T.trim[tid] = a.trims ? a.trims[s0 + tid] : uint8_t(0);
        fsub_sync(sub);

        const uint64_t a0 = T.off[0] & ~15ull;
        const uint64_t end = T.off[ns];
        // (the text cap is a bound on the group's span, rounded up to 16 bytes: the geometry plan() reports)
        bool fast = end >= T.off[0] && ((end - a0 + 15) & ~15ull) + 16 <= uint64_t(kFTextCap);
        const uint32_t lo_byte = uint32_t(T.off[0] - a0), hi_byte = fast ? uint32_t(end - a0) : 0u;
        int S = 0;

        if (fast) {
            // ---- load the group's bytes; meanwhile clear the slot stream and mark sentence starts / excluded bytes ----
            // Thread tid holds unit tid and unit 256 + tid (32 bytes each) in registers from the count step to the
            // scatter step.  The bytes up to the next multiple of 16 behind the group's end are readable (the text buffer
            // is padded to 16 bytes and an address has the alignment of its offset); bytes outside the group's
            // [lo_byte, hi_byte) read as spaces (count step): never a continuation byte, never NUL.  The first word behind
            // a unit (`halo`) comes from the next lane; the last lane of a warp loads its own.
            auto load_unit = [&](uint32_t ub, uint32_t (&v)[8], uint32_t& h) {
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = 0x20202020u;
                h = 0x20202020u;
                if (ub < hi_byte) {
                    const uint4 q0 = ldg_text16(text + a0 + ub);
                    v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w;
                    if (ub + 16 < hi_byte) {
                        const uint4 q1 = ldg_text16(text + a0 + ub + 16);
                        v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w;
                    }
                    if (lane == 31 && ub + 32 < hi_byte) h = ldg_text4(text + a0 + ub + 32);
                }
            };
            // bytes of the unit at ub that lie inside the group's range
            auto range_mask = [&](uint32_t ub) {
                uint32_t rm = 0xFFFFFFFFu;
                if (ub < lo_byte) rm &= lo_byte - ub >= 32 ? 0u : 0xFFFFFFFFu << (lo_byte - ub);
                if (ub + 32 > hi_byte) rm &= 0xFFFFFFFFu >> (ub + 32 - hi_byte);
                return rm;
            };
            auto patch_unit = [&](uint32_t ub, uint32_t rm, uint32_t (&v)[8], uint32_t& h) {
                if (rm != 0xFFFFFFFFu) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = keep_bytes(v[i], (rm >> (4 * i)) & 15u);
                }
                if (lane == 31 && ub + 32 < hi_byte && hi_byte - ub - 32 < 4) h = keep_bytes(h, (1u << (hi_byte - ub - 32)) - 1u);
            };
            uint32_t w[2][8], halo[2];
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) load_unit(uint32_t(pass * kFSubThreads + tid) << 5, w[pass], halo[pass]);
            // (the separator slots of the slot stream are cleared by the scatter step itself; the front padding here)
            if (tid < kFPadFront) s_raw_alloc[tid] = 0;
            if (kOverflow)
                for (int i = tid; i < kFSlotAlloc / 4; i += kFSubThreads) reinterpret_cast<uint4*>(s_acc - kFPadFront)[i] = make_uint4(0, 0, 0, 0);
            // (the finishing pass of the overflow variant trusts the per-slot "valid boundary" flags: none may be stale)
            if (kOverflow)
                for (int i = tid; i < kFSlotAlloc; i += kFSubThreads) (s_meta - kFPadFront)[i] = MetaT(0);
            for (int i = tid; i < kFTextCap / 32 + 4; i += kFSubThreads) { s_sbits[i] = 0; s_xbits[i] = 0; }
            fsub_sync(sub);
            if (tid < ns) {
                const uint64_t o0 = T.off[tid], o1 = T.off[tid + 1];
                const uint32_t tr = T.trim[tid];
                if (o1 < o0 || o1 - o0 < tr || o0 < T.off[0] || o1 > end) {
                    T.anomaly = 1;  // offsets out of order
                } else {
                    const uint32_t b = uint32_t(o0 - a0);
                    atomicOr(&s_sbits[b >> 5], 1u << (b & 31));
                    for (uint32_t t = 0; t < tr; ++t) {
                        const uint32_t x = uint32_t(o1 - a0) - 1 - t;
                        atomicOr(&s_xbits[x >> 5], 1u << (x & 31));
                    }
                    if (tr) atomicAdd(&T.bytes_want, tr);
                }
            }
            fsub_sync(sub);

            // ---- count: one thread per 32-byte unit (two passes cover the tile buffer): character starts, NUL ------------
            // (whether the continuation bytes are where the lead bytes want them is checked by the stream stage, per
            //  character; the counts do not depend on it)
            const int nunits = int((hi_byte + 31) >> 5);
            uint32_t u_starts[2] = {0, 0}, u_sbits[2] = {0, 0}, u_excl[2] = {0, 0};
            uint32_t carry = 0;  // packed totals of the earlier pass: chars | sentence starts << 14 | non-empty starts << 22
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                const int u = pass * kFSubThreads + tid;
                uint32_t packed = 0;
                if (pass == 0 || nunits > kFSubThreads) {
                    if (u < nunits) {
                        const uint32_t ub = uint32_t(u) << 5;
                        // bytes outside the group's range and excluded bytes (line terminators) are not characters
                        const uint32_t rm = range_mask(ub);
                        patch_unit(ub, rm, w[pass], halo[pass]);
                        uint32_t starts = 0, nul = 0;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const uint32_t x = w[pass][i];
                            nul |= (x - 0x01010101u) & ~x;                           // bit 7 of a byte: the byte is zero
                            const uint32_t st80 = ~(x & ~(x << 1)) & 0x80808080u;    // not 10xxxxxx
                            starts |= ((((st80 >> 7) * 0x00204081u) >> 21) & 15u) << (4 * i);
                        }
                        if (nul & 0x80808080u) T.anomaly = 1;
                        const uint32_t ex = s_xbits[u], sbt = s_sbits[u] & rm;
                        // a sentence must not start on a continuation byte (with the structural check of the stream
                        // stage this makes every sentence valid on its own)
                        if (sbt & ~starts) T.anomaly = 1;
                        starts &= rm & ~ex;
                        u_starts[pass] = starts;
                        u_sbits[pass] = sbt;
                        packed = __popc(starts) | (__popc(sbt) << 14) | (__popc(sbt & starts) << 22);
                    }
                    {
                        const uint32_t next = __shfl_down_sync(kFull, w[pass][0], 1);
                        if (lane != 31) halo[pass] = next;
                    }
                    // block scan of the packed counts
                    const uint32_t incl = warp_incl_scan(packed, lane);
                    if (lane == 31) T.wsum[warp] = incl;
                    fsub_sync(sub);
                    uint32_t base = carry, tot = carry;
#pragma unroll
                    for (int wv = 0; wv < kFWarps; ++wv) {
                        const uint32_t sw = T.wsum[wv];
                        if (wv < warp) base += sw;
                        tot += sw;
                    }
                    u_excl[pass] = base + incl - packed;
                    carry = tot;
                    fsub_sync(sub);
                }
            }
            const uint32_t g_tot = carry & 0x3FFFu, k_tot = (carry >> 14) & 0xFFu, ne_tot = carry >> 22;
            S = gap + int(g_tot) + gap * int(k_tot);
            // every sentence must have its own start byte (zero-width sentences share one) and the slots must fit
            if (int(k_tot) != ns || S > kFSlotCap) fast = false;
            if (T.anomaly) fast = false;  // (uniform: read after the barrier that ends the scan)

            if (fast) {
                // ---- publish the group's totals; scatter characters to their slots ------------------------------------
                if (tid == 0) {
                    st_relaxed(desc_c + grp, kDescAgg | uint64_t(g_tot));
                    st_relaxed(desc_b + grp, kDescAgg | uint64_t(g_tot - ne_tot));
                    T.first[ns] = g_tot;
                    T.lb[ns] = g_tot - ne_tot;
                    // bytes the characters of the group must add up to (stream stage: structural check)
                    T.bytes_want = hi_byte - lo_byte - T.bytes_want;
                }
                // the separator slots behind the last sentence and the padding the lagging outputs read
                if (tid < gap + kFPadBack) s_raw[S - gap + tid] = 0;
#pragma unroll
                for (int pass = 0; pass < 2; ++pass) {
                    const uint32_t mset = u_starts[pass] | u_sbits[pass];
                    if (mset == 0) continue;
                    uint32_t G = u_excl[pass] & 0x3FFFu, K = (u_excl[pass] >> 14) & 0xFFu, NE = u_excl[pass] >> 22;
                    uint32_t slot = G + uint32_t(gap) * K;  // slot of the next character
                    uint32_t ol = G - NE + 1;               // its boundary index (valid once its sentence has started)
                    // a character's four-byte window is a funnel shift of two of the unit's registers
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        uint32_t nib = (mset >> (4 * k)) & 15u;
                        while (nib) {
                            const int jj = __ffs(nib) - 1;
                            nib &= nib - 1;
                            const uint32_t bit = 1u << (4 * k + jj);
                            const bool is_start = (u_starts[pass] & bit) != 0;
                            if (u_sbits[pass] & bit) {
                                // a sentence starts here: `gap` more separator slots; a non-empty one loses one boundary index
                                T.first[K] = G;
                                T.lb[K] = G - NE;
                                ++K;
                                for (int g = 0; g < gap; ++g) s_raw[slot + uint32_t(g)] = 0;  // the separator slots in front of it
                                slot += uint32_t(gap);
                                if (is_start) { ++NE; --ol; }
                            }
                            if (is_start) {
                                s_raw[slot] = __funnelshift_r(w[pass][k], k < 7 ? w[pass][k + 1] : halo[pass], 8 * jj);
                                s_meta[slot] = kStates ? MetaT(ol | (G << 12)) : MetaT(ol);
                                ++G; ++slot; ++ol;
                            }
                        }
                    }
                }
                (void)u_excl;
                fsub_sync(sub);
                // ---- output offsets of the group (look-back), per-sentence outputs -----------------------------------
                if (warp == 0) {
                    uint64_t pb, pcv;
                    lookback2(desc_b, desc_c, grp, lane, pb, pcv);
                    if (lane == 0) {
                        st_relaxed(desc_c + grp, kDescIncl | (pcv + g_tot));
                        st_relaxed(desc_b + grp, kDescIncl | (pb + (g_tot - ne_tot)));
                        T.obase = pb;
                        T.cbase = pcv;
                    }
                }
                fsub_sync(sub);
                if (tid < ns) {
                    const uint64_t s = s0 + tid;
                    const uint32_t n = T.first[tid + 1] - T.first[tid];
                    a.n_chars[s] = n;
                    a.status[s] = n == 0 ? 1 : 0;
                    a.bound_offsets[s] = a.bound_base + T.obase + T.lb[tid];
                    if (a.char_offsets) a.char_offsets[s] = a.char_base + T.cbase + T.first[tid];
                    if (s + 1 == a.n_sent) {
                        a.bound_offsets[s + 1] = a.bound_base + T.obase + T.lb[ns];
                        if (a.char_offsets) a.char_offsets[s + 1] = a.char_base + T.cbase + T.first[ns];
                        if (a.totals_host) { a.totals_host[0] = T.obase + T.lb[ns]; a.totals_host[1] = T.cbase + T.first[ns]; }
                    }
                }
                // ---- stream ------------------------------------------------------------------------------------------
                stream_stage<kSeedsSmem, kCommon, kDeep, kStates, MetaT>(m, a, cfg, s_raw, s_meta, s_acc, s_seeds, s_ta, s_tb,
                                                                             s_tytab, T, S, T.obase, T.cbase, warp, lane);
                fsub_sync(sub);
                if (kOverflow) { finish_overflow<MetaT>(a, s_meta, s_acc, T.obase, S, tid); fsub_sync(sub); }
                if (T.bad_chars || T.bytes_have != T.bytes_want) {
                    // malformed UTF-8 (a lead byte without its continuation bytes, stray continuation bytes, overlong
                    // forms, surrogates, > U+10FFFF): find the sentences exactly and take their outputs back
                    for (int k = warp; k < ns; k += kFWarps) {
                        uint32_t nch;
                        int st;
                        slow_validate(text, T.off[k], T.off[k + 1] - T.trim[k], lane, nch, st);
                        if (st >= 2) {
                            if (lane == 0) a.status[s0 + k] = st;
                            zero_sentence(a, T.obase + T.lb[k], T.cbase + T.first[k], nch, lane);
                        }
                    }
                    fsub_sync(sub);
                }
                continue;
            }
        }

        // ================= slow path: exact per-sentence count, then the stream stage a sentence range at a time ========
        // The character counts come first, from word loads (one round trip per 128 bytes of a sentence): every group
        // behind this one waits in its look-back for this group's totals, the byte-exact validation can follow them.
        for (int k = warp; k < ns; k += kFWarps) {
            uint64_t b0 = T.off[k], b1 = T.off[k + 1];
            const uint32_t tr = T.trim[k];
            b1 = (b1 >= b0 && b1 - b0 >= tr) ? b1 - tr : b0;  // offsets out of order: an empty sentence
            const uint32_t nch = slow_count(text, b0, b1, lane);
            if (lane == 0) T.first[k] = nch;
        }
        fsub_sync(sub);
        if (warp == 0) {
            const uint32_t n0 = 2 * lane < ns ? T.first[2 * lane] : 0u, n1 = 2 * lane + 1 < ns ? T.first[2 * lane + 1] : 0u;
            const uint32_t o0 = n0 ? n0 - 1 : 0u, o1 = n1 ? n1 - 1 : 0u;
            const uint32_t ic = warp_incl_scan(n0 + n1, lane), io = warp_incl_scan(o0 + o1, lane);
            const uint32_t gc = __shfl_sync(kFull, ic, 31), go = __shfl_sync(kFull, io, 31);
            __syncwarp();
            if (2 * lane < ns) { T.first[2 * lane] = ic - n0 - n1; T.lb[2 * lane] = io - o0 - o1; }
            if (2 * lane + 1 < ns) { T.first[2 * lane + 1] = ic - n1; T.lb[2 * lane + 1] = io - o1; }
            if (lane == 0) {
                T.first[ns] = gc;
                T.lb[ns] = go;
                st_relaxed(desc_c + grp, kDescAgg | uint64_t(gc));
                st_relaxed(desc_b + grp, kDescAgg | uint64_t(go));
            }
            uint64_t pb, pcv;
            lookback2(desc_b, desc_c, grp, lane, pb, pcv);
            if (lane == 0) {
                st_relaxed(desc_c + grp, kDescIncl | (pcv + gc));
                st_relaxed(desc_b + grp, kDescIncl | (pb + go));
                T.obase = pb;
                T.cbase = pcv;
            }
        }
        for (int k = warp; k < ns; k += kFWarps) {
            uint64_t b0 = T.off[k], b1 = T.off[k + 1];
            const uint32_t tr = T.trim[k];
            b1 = (b1 >= b0 && b1 - b0 >= tr) ? b1 - tr : b0;
            uint32_t nch;
            int st;
            slow_validate(text, b0, b1, lane, nch, st);  // (nch: the count the totals were built from)
            if (lane == 0) T.st[k] = uint8_t(st);
        }
        fsub_sync(sub);
        if (tid < ns) {
            const uint64_t s = s0 + tid;
            a.n_chars[s] = T.first[tid + 1] - T.first[tid];
            a.status[s] = T.st[tid];
            a.bound_offsets[s] = a.bound_base + T.obase + T.lb[tid];
            if (a.char_offsets) a.char_offsets[s] = a.char_base + T.cbase + T.first[tid];
            if (s + 1 == a.n_sent) {
                a.bound_offsets[s + 1] = a.bound_base + T.obase + T.lb[ns];
                if (a.char_offsets) a.char_offsets[s + 1] = a.char_base + T.cbase + T.first[ns];
                if (a.totals_host) { a.totals_host[0] = T.obase + T.lb[ns]; a.totals_host[1] = T.cbase + T.first[ns]; }
            }
        }
        for (int k0 = 0; k0 < ns;) {
            // the longest sentence range [k0, k1) that fits the tile buffers (the fit test is monotone in the range end)
            if (tid == 0) T.k1 = ns;
            fsub_sync(sub);
            if (tid >= k0 && tid < ns) {
                const uint64_t ra0 = T.off[k0] & ~15ull;
                const uint64_t e = T.off[tid + 1] >= T.off[k0] ? T.off[tid + 1] : T.off[k0];
                const uint64_t rspan = (e - ra0 + 15) & ~15ull;
                const int slots = gap + int(T.first[tid + 1] - T.first[k0]) + gap * (tid + 1 - k0);
                if (rspan + 16 > uint64_t(kFTextCap) || slots > kFSlotCap || T.off[tid + 1] < T.off[tid]) atomicMin(&T.k1, tid);
            }
            fsub_sync(sub);
            const bool single = T.k1 == k0;
            const int k1 = single ? k0 + 1 : T.k1;
            if (single) {
                // one sentence larger than the tile buffers (or with unusable offsets): one warp walks it from global memory
                if (warp == 0) {
                    SentInfo si;
                    si.b0 = T.off[k0];
                    const uint64_t e1 = T.off[k0 + 1];
                    si.b1 = (e1 >= si.b0 && e1 - si.b0 >= T.trim[k0]) ? e1 - T.trim[k0] : si.b0;
                    si.n = T.first[k0 + 1] - T.first[k0];
                    si.nout = si.n > 0 ? si.n - 1 : 0;
                    si.status = T.st[k0];
                    si.obase = T.obase + T.lb[k0];
                    si.cbase = T.cbase + T.first[k0];
                    fast_sentence_warp_si(m, a, si, *reinterpret_cast<Rings*>(s_raw_alloc), lane);
                }
                fsub_sync(sub);
                k0 = k1;
                continue;
            }
            const int Sr = gap + int(T.first[k1] - T.first[k0]) + gap * (k1 - k0);
            for (int i = tid; i < kFSlotAlloc / 4; i += kFSubThreads) reinterpret_cast<uint4*>(s_raw_alloc)[i] = make_uint4(0, 0, 0, 0);
            if (kOverflow)
                for (int i = tid; i < kFSlotAlloc / 4; i += kFSubThreads) reinterpret_cast<uint4*>(s_acc - kFPadFront)[i] = make_uint4(0, 0, 0, 0);
            // (the finishing pass of the overflow variant trusts the per-slot "valid boundary" flags: none may be stale)
            if (kOverflow)
                for (int i = tid; i < kFSlotAlloc; i += kFSubThreads) (s_meta - kFPadFront)[i] = MetaT(0);
            fsub_sync(sub);
            // scatter, one warp per sentence, from global memory: a lane reads one word per 128-byte step and takes the
            // word behind it from the next lane (the last lane reads its own)
            for (int k = k0 + warp; k < k1; k += kFWarps) {
                const uint32_t n = T.first[k + 1] - T.first[k];
                if (T.st[k] != 0) {
                    zero_sentence(a, T.obase + T.lb[k], T.cbase + T.first[k], n, lane);
                    continue;
                }
                const uint8_t* const st = text + (T.off[k] & ~3ull);  // offsets below are relative to it
                const uint32_t rb0 = uint32_t(T.off[k] & 3u), rb1 = rb0 + uint32_t(T.off[k + 1] - T.off[k]) - T.trim[k];
                uint32_t idx = uint32_t(gap) + (T.first[k] - T.first[k0]) + uint32_t(gap) * uint32_t(k - k0);
                uint32_t ci = 0;  // characters of this sentence already placed
                for (uint32_t wpos = 0; wpos < rb1; wpos += 128) {
                    const uint32_t addr = wpos + 4u * uint32_t(lane);
                    uint32_t lo = 0, hi = 0;
                    if (addr < rb1) {
                        lo = ldg_text4(st + addr);
                        if (lane == 31 && addr + 4 < rb1) hi = ldg_text4(st + addr + 4);
                    }
                    {
                        const uint32_t next = __shfl_down_sync(kFull, lo, 1);
                        if (lane != 31) hi = next;
                    }
                    uint32_t smask = 0;
                    if (addr < rb1) {
                        const uint32_t from = rb0 > addr ? rb0 - addr : 0u;
                        const uint32_t to = rb1 - addr < 4u ? rb1 - addr : 4u;
                        const uint32_t im80 = (from >= 4u ? 0u : 0x80808080u << (8 * from)) & (0x80808080u >> (8 * (4 - to)));
                        const uint32_t st80 = ~(lo & ~(lo << 1)) & im80;
                        smask = ((st80 >> 7) | (st80 >> 14) | (st80 >> 21) | (st80 >> 28)) & 15u;
                    }
                    const uint32_t cnt = __popc(smask);
                    const uint32_t incl = warp_incl_scan(cnt, lane);
                    uint32_t at = incl - cnt;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (smask & (1u << j)) {
                            const uint32_t gi = T.first[k] - T.first[k0] + ci + at;  // range-local character index
                            const uint32_t ol = T.lb[k] - T.lb[k0] + ci + at;        // range-local boundary index
                            s_raw[idx + at] = __funnelshift_r(lo, hi, 8u * uint32_t(j));
                            s_meta[idx + at] = kStates ? MetaT(ol | (gi << 12)) : MetaT(ol);
                            ++at;
                        }
                    }
                    const uint32_t tot = __shfl_sync(kFull, incl, 31);
                    idx += tot;
                    ci += tot;
                }
            }
            fsub_sync(sub);
            stream_stage<kSeedsSmem, kCommon, kDeep, kStates, MetaT>(m, a, cfg, s_raw, s_meta, s_acc, s_seeds, s_ta, s_tb, s_tytab,
                                                                         T, Sr, T.obase + T.lb[k0], T.cbase + T.first[k0], warp, lane);
            fsub_sync(sub);
            if (kOverflow) { finish_overflow<MetaT>(a, s_meta, s_acc, T.obase + T.lb[k0], Sr, tid); fsub_sync(sub); }
            k0 = k1;
        }
    }
    if (a.self_clean) {
        // single-CTA launch of the one-sentence call: the descriptors and the ticket are left zeroed for the next call
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint64_t ng = (a.n_sent + kFGroup - 1) / kFGroup;
            for (uint64_t g = 0; g < ng; ++g) { st_relaxed(desc_b + g, 0); st_relaxed(desc_c + g, 0); }
            *a.ticket = 0;
        }
    }
}

}  // namespace


// ---- launch of one (seeds, shape) group of kernel variants: instantiated in its own translation unit (fused_*.cu) ----
namespace fused_detail {

template <bool kSeeds, bool kCommon, int kDeep, bool kStates>
cudaError_t launch_fused_t(const DevModel& m, const BatchArgs& a, const StreamCfg& cfg, cudaStream_t stream, int dev, int n_sm) {
    using Lay = FLayout<kSeeds, kCommon, kDeep, kStates>;
    static std::atomic<bool> attr_set[kMaxDevices] = {};  // (idempotent: set after the attribute call succeeded)
    if (!attr_set[dev]) {
        auto* k = k_fused<kSeeds, kCommon, kDeep, kStates>;
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, Lay::kSmem);
        if (e != cudaSuccess) return e;
        // The smallest shared-memory carve-out that holds the CTA (with the 1 KB reserved per CTA), so that the rest of
        // the SM's array is L1 for the node records.  The attribute is a percentage of the SM's shared memory, which the
        // driver rounds up to the next carve-out it supports.
        int smem_sm = 0;
        e = cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
        if (e != cudaSuccess) return e;
        const int carveout = std::min(100, int(((int64_t(Lay::kSmem) + 1024) * 100 + smem_sm - 1) / smem_sm));
        e = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    const uint64_t ngroups = (a.n_sent + kFGroup - 1) / kFGroup;
    const unsigned grid = unsigned(std::min<uint64_t>(uint64_t(n_sm), (ngroups + Lay::kSubBlocks - 1) / Lay::kSubBlocks));
    k_fused<kSeeds, kCommon, kDeep, kStates><<<grid, Lay::kThreads, Lay::kSmem, stream>>>(m, a, cfg);
    return cudaGetLastError();
}

template <bool kSeeds, bool kCommon>
cudaError_t launch_fused_group(const KernelPlan& pl, const DevModel& m, const BatchArgs& a, const StreamCfg& cfg, cudaStream_t stream, int dev, int n_sm) {
    if (pl.deep == 2) return pl.states ? launch_fused_t<kSeeds, kCommon, 2, true>(m, a, cfg, stream, dev, n_sm)
                                       : launch_fused_t<kSeeds, kCommon, 2, false>(m, a, cfg, stream, dev, n_sm);
    if (pl.deep == 1) return pl.states ? launch_fused_t<kSeeds, kCommon, 1, true>(m, a, cfg, stream, dev, n_sm)
                                       : launch_fused_t<kSeeds, kCommon, 1, false>(m, a, cfg, stream, dev, n_sm);
    return pl.states ? launch_fused_t<kSeeds, kCommon, 0, true>(m, a, cfg, stream, dev, n_sm)
                     : launch_fused_t<kSeeds, kCommon, 0, false>(m, a, cfg, stream, dev, n_sm);
}

}  // namespace fused_detail

}  // namespace vpt
