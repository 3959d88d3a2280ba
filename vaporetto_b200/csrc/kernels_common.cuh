// Device helpers shared by the scoring kernels (kernels.cu: count / general / tile kernels; fused.cu: the one-pass
// streaming kernel): record loads, the perfect-hash probe, UTF-8 window decoding, TMA bulk copy + mbarrier,
// and the warp-per-sentence scorer used for sentences larger than a tile.
#pragma once
#include <algorithm>
#include <cstdint>

#include <cuda_runtime.h>

#include "device_model.hpp"
#include "keys.hpp"
#include "textnorm.hpp"

namespace vpt {

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kRing = 256;          // per-warp ring of decoded characters (power of two)
constexpr int kRingMask = kRing - 1;
constexpr unsigned kFull = 0xFFFFFFFFu;

struct Rec32 {
    uint32_t v[8];
};

// One 32-byte node record.  sm_90 has no 256-bit global load: the record is two 128-bit loads of the same 32-byte sector.
// The loads allocate in L1.  Natural text is Zipf-like, so the nodes of frequent characters and character pairs are
// probed again while they are still in the L1 that k_fused's shared memory leaves (60 KB per SM in the 196 KB
// carve-out; k_fused reads its text around L1).  A config-2 step took 1.087 ms against 1.442 ms with L1::no_allocate
// when 28 KB of L1 were left (H100 80GB HBM3, 700 W power limit; DESIGN §4).  The records are re-used from L2, which
// on an H100 (50 MB) is smaller than the text and the outputs a batch streams through it, so they are loaded with an
// evict-last policy and the text with an evict-first one.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

__device__ __forceinline__ Rec32 load_record(const void* base, uint32_t slot) {
    Rec32 r;
    const char* p = static_cast<const char*>(base) + (size_t(slot) << 5);
    const uint64_t pol = l2_policy_evict_last();
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3])
                 : "l"(p), "l"(pol));
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4+16], %5;"
                 : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
                 : "l"(p), "l"(pol));
    return r;
}

// kMaySpill = false: the caller knows the table has no spill table (its seeds are not staged in shared memory:
// validate_blob_header)
template <bool kMaySpill = true>
__device__ __forceinline__ uint32_t slot_of(const DevTable& t, uint64_t key) {
    uint32_t ha, hb;
    key_hashes(key, t.hk, ha, hb);
    const uint32_t b = bucket_of(ha, t.nbuckets);
    const uint32_t seed = t.seed16 ? uint32_t(__ldg(reinterpret_cast<const uint16_t*>(t.seeds) + b)) : uint32_t(__ldg(t.seeds + b));
    if (!kMaySpill || !t.spill_buckets) return slot_of_seeds<false>(ha, hb, seed, 0u, t.nslots, 0u, 0u);
    const uint32_t spill_seed = __ldg(t.seeds + spill_bucket_of(hb, t.nbuckets, t.spill_buckets));
    return slot_of_seeds<true>(ha, hb, seed, spill_seed, t.nslots, t.spill_slots, t.spill_mul);
}

// One probe: returns true when the node with `key` exists; rec/slot are valid then.
__device__ __forceinline__ bool probe(const DevTable& t, uint64_t key, Rec32& rec, uint32_t& slot, bool deep = false) {
    slot = slot_of(t, key);
    rec = load_record(t.records, slot);
    const uint64_t k = (uint64_t(rec.v[1]) << 32) | rec.v[0];
    // (records of 2-symbol nodes hold a child mask in the unused c1 field: not part of the key)
    const uint64_t flags = deep ? (kExtFlag | kOvfFlag) : ((key >> 42) ? kExtFlag : (kExtFlag | kChildMaskField));
    return (k & ~flags) == key;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

struct Rings {
    uint32_t cp[kRing];  // code points
    uint32_t bp[kRing];  // byte position of the character relative to the sentence start
    uint8_t ty[kRing];   // character types
};

// Decodes the 128-byte window starting at the 4-byte aligned position `wpos`, appends its characters
// (those whose lead byte lies in [b0, b1)) to the ring at index nd.., returns how many were appended.
__device__ __forceinline__ uint32_t decode_window(const uint8_t* __restrict__ text, uint64_t wpos, uint64_t b0,
                                                  uint64_t b1, uint32_t nd, Rings& r, int lane, bool norm) {
    const uint64_t addr = wpos + 4u * uint32_t(lane);
    uint32_t lo = 0, hi = 0;
    if (addr < b1) {
        lo = __ldg(reinterpret_cast<const uint32_t*>(text + addr));
        if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(text + addr + 4));
    }
    uint32_t smask = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint64_t p = addr + j;
        const uint32_t b = (lo >> (8 * j)) & 0xFF;
        if (p >= b0 && p < b1 && (b & 0xC0) != 0x80) smask |= 1u << j;
    }
    const uint32_t cnt = __popc(smask);
    const uint32_t incl = warp_incl_scan(cnt, lane);
    uint32_t idx = nd + incl - cnt;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (smask & (1u << j)) {
            const uint32_t x = __funnelshift_r(lo, hi, 8 * j);
            uint32_t c = decode_cp(x);
            if (norm) c = kytea_fullwidth(c);
            r.cp[idx & kRingMask] = c;
            r.bp[idx & kRingMask] = uint32_t(addr + j - b0);
            r.ty[idx & kRingMask] = uint8_t(char_type(c));
            ++idx;
        }
    }
    return __shfl_sync(kFull, incl, 31);
}

// Steps back from byte position `pos` (a character start, > b0) to the previous character; returns its
// code point and updates pos.
__device__ __forceinline__ uint32_t prev_char(const uint8_t* __restrict__ text, uint64_t b0, uint64_t& pos, bool norm) {
    uint64_t q = pos - 1;
    uint32_t x = __ldg(text + q);
    uint32_t bytes = x;
    while ((x & 0xC0) == 0x80 && q > b0) {
        --q;
        x = __ldg(text + q);
        bytes = (bytes << 8) | x;
    }
    pos = q;
    const uint32_t c = decode_cp(bytes);
    return norm ? kytea_fullwidth(c) : c;
}

// ------------------------------------------------------------------------------------------------
// TMA bulk copy + mbarrier helpers (PTX; SASS: UBLKCP / SYNCS)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(l2_policy_evict_first())
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// shared per-sentence prologue
// ------------------------------------------------------------------------------------------------
struct SentInfo {
    uint64_t b0, b1, obase, cbase;
    uint32_t n, nout;
    int status;
};

__device__ __forceinline__ SentInfo sentence_info(const BatchArgs& a, uint64_t s, int lane) {
    SentInfo si;
    si.b0 = a.offsets[s];
    si.b1 = a.offsets[s + 1] - (a.trims ? a.trims[s] : 0);
    si.n = a.n_chars[s];
    si.status = a.status[s];
    si.nout = si.n > 0 ? si.n - 1 : 0;
    const uint64_t grp = s / kGroup;
    si.obase = a.group_bound[grp] + a.local_bound[s];
    si.cbase = a.group_char[grp] + a.local_char[s];
    if (lane == 0) {
        a.bound_offsets[s] = a.bound_base + si.obase;
        if (a.char_offsets) a.char_offsets[s] = a.char_base + si.cbase;
        if (s + 1 == a.n_sent) {
            a.bound_offsets[s + 1] = a.bound_base + si.obase + si.nout;
            if (a.char_offsets) a.char_offsets[s + 1] = a.char_base + si.cbase + si.n;
        }
    }
    return si;
}

// Type-table index of boundary g: the 2W character types around it, zero outside the sentence
// (reference type_scorer/boundary_scorer_cache.rs:59-81).
__device__ __forceinline__ uint32_t type_index(const Rings& r, int64_t g, uint32_t n, int w) {
    uint32_t idx = 0;
    for (int k = 0; k < 2 * w; ++k) {
        const int64_t i = g - w + 1 + k;
        const uint32_t t = (i >= 0 && i < int64_t(n)) ? r.ty[i & kRingMask] : 0u;
        idx = (idx << 3) | t;
    }
    return idx;
}

// Longest-suffix lookup for the text ending at ring index g.  Symbols are code points (types=false)
// or character types (types=true).  Returns true and the record of the deepest existing node.
template <bool kTypes>
__device__ __forceinline__ bool find_node(const DevTable& t, const Rings& r, const uint8_t* __restrict__ text,
                                          uint64_t b0, uint32_t g, Rec32& rec, uint32_t& slot, bool norm,
                                          bool* deep_hit = nullptr) {
    if (deep_hit) *deep_hit = false;
    uint32_t c3, c2 = 0, c1 = 0;
    if (kTypes) {
        c3 = r.ty[g & kRingMask];
        if (g >= 1) c2 = r.ty[(g - 1) & kRingMask];
        if (g >= 2) c1 = r.ty[(g - 2) & kRingMask];
    } else {
        c3 = r.cp[g & kRingMask];
        if (g >= 1) c2 = r.cp[(g - 1) & kRingMask];
        if (g >= 2) c1 = r.cp[(g - 2) & kRingMask];
    }
    bool found = probe(t, shallow_key(c1, c2, c3), rec, slot);
    const bool depth3 = found && c1 != 0;
    if (!found && c1 != 0) found = probe(t, shallow_key(0, c2, c3), rec, slot);
    if (!found && c2 != 0) found = probe(t, shallow_key(0, 0, c3), rec, slot);
    if (depth3 && (rec.v[1] >> 31) && g >= 3) {
        // deeper nodes exist: keep walking backwards through the text (rare: patterns longer than 3)
        uint64_t pos = b0 + r.bp[(g - 2) & kRingMask];
        uint32_t node = __ldg(t.slot_node + slot);
        while (pos > b0) {
            uint32_t sym = prev_char(text, b0, pos, norm);
            if (kTypes) sym = char_type(sym);
            Rec32 nrec;
            uint32_t nslot;
            if (!probe(t, deep_key(node, sym), nrec, nslot, true)) break;
            rec = nrec;
            slot = nslot;
            if (deep_hit) *deep_hit = true;
            if (!(rec.v[1] >> 31)) break;
            node = __ldg(t.slot_node + slot);
        }
    }
    return found;
}

// ------------------------------------------------------------------------------------------------
// k_score_fast
// ------------------------------------------------------------------------------------------------
// One warp scores one sentence, 32 characters per iteration (used by k_score_fast and as the fallback of
// k_tile_fast for groups that do not fit the tile buffers).
__device__ __forceinline__ void fast_sentence_warp_si(const DevModel& m, const BatchArgs& a, const SentInfo& si, Rings& r, int lane) {
    const uint8_t* __restrict__ text = a.text;
    const uint32_t n = si.n;
    if (si.status != 0) {
        for (uint32_t i = lane; i < si.nout; i += 32) { if (a.scores) a.scores[si.obase + i] = 0; a.boundaries[si.obase + i] = 0; }
        if (a.char_states) for (uint32_t i = lane; i < n; i += 32) a.char_states[si.cbase + i] = kNoPattern;
        if (a.type_states) for (uint32_t i = lane; i < n; i += 32) a.type_states[si.cbase + i] = kNoPattern;
        return;
    }
    const int tw = m.type_cache_window;
    const int r0 = m.ct.r0;
    uint64_t wpos = si.b0 & ~3ull;
    uint32_t nd = 0;
    int32_t prev_main = 0, carry_r = 0;
    uint32_t prev_g = 0;
    bool have_prev = false;
    for (uint32_t cb = 0; cb < n; cb += 32) {
        const uint32_t need = min(n, cb + 32u + uint32_t(tw));
        while (nd < need && wpos < si.b1) {
            nd += decode_window(text, wpos, si.b0, si.b1, nd, r, lane, m.kytea_norm != 0);
            wpos += 128;
        }
        __syncwarp();
        const uint32_t g = cb + lane;
        const bool active = g < n;
        int32_t d[kInlineWidth];
#pragma unroll
        for (int j = 0; j < kInlineWidth; ++j) d[j] = 0;
        uint32_t cstate = kNoPattern;
        if (active && m.ct.present) {
            Rec32 rec;
            uint32_t slot;
            if (find_node<false>(m.ct, r, text, si.b0, g, rec, slot, m.kytea_norm != 0)) {
#pragma unroll
                for (int j = 0; j < kInlineWidth; ++j) d[j] = int32_t(rec.v[2 + j]);
                if (m.emit_states && a.char_states) cstate = __ldg(m.ct.slot_pid + slot);
            }
        }
        // gather: boundary (lane) <- row entry j of the source lane (lane - r0 - j); sources that fall
        // into the neighbouring 32-character chunks are carried in registers (same lane index).
        int32_t mainv = 0, to_prev = 0, to_next = 0;
#pragma unroll
        for (int j = 0; j < kInlineWidth; ++j) {
            const int src = lane - r0 - j;
            const int32_t v = __shfl_sync(kFull, d[j], src & 31);
            if (src < 0) to_next += v;
            else if (src >= 32) to_prev += v;
            else mainv += v;
        }
        int32_t tsc = 0;
        if (tw > 0 && g + 1 < n) tsc = __ldg(m.type_cache + type_index(r, int64_t(g), n, tw));
        mainv += m.bias + tsc + carry_r;
        if (have_prev && prev_g + 1 < n) {
            const int32_t fin = prev_main + to_prev;
            if (a.scores) a.scores[si.obase + prev_g] = fin;
            a.boundaries[si.obase + prev_g] = fin > 0 ? 1 : 0;
        }
        if (a.char_states && active) a.char_states[si.cbase + g] = cstate;
        if (a.type_states && active) {
            uint32_t ts = kNoPattern;
            if (m.emit_states && m.type_state3) {
                const uint32_t t2 = g >= 1 ? r.ty[(g - 1) & kRingMask] : 0u, t1 = (g >= 2 && t2) ? r.ty[(g - 2) & kRingMask] : 0u;
                ts = __ldg(m.type_state3 + ((t1 << 6) | (t2 << 3) | r.ty[g & kRingMask]));
            }
            a.type_states[si.cbase + g] = ts;
        }
        prev_main = mainv;
        prev_g = g;
        have_prev = true;
        carry_r = to_next;
        __syncwarp();
    }
    if (have_prev && prev_g + 1 < n) {
        if (a.scores) a.scores[si.obase + prev_g] = prev_main;
        a.boundaries[si.obase + prev_g] = prev_main > 0 ? 1 : 0;
    }
    if (m.ct.present && m.ct.has_overflow) {
        // rows of long dictionary words stick out of the inline window: add the outside parts with atomics in a
        // second sweep and redo the thresholds (only sentences larger than a tile come through here)
        __threadfence();
        __syncwarp();
        uint64_t wpos2 = si.b0 & ~3ull;
        uint32_t nd2 = 0;
        for (uint32_t cb = 0; cb < n; cb += 32) {
            const uint32_t need = min(n, cb + 32u);
            while (nd2 < need && wpos2 < si.b1) {
                nd2 += decode_window(text, wpos2, si.b0, si.b1, nd2, r, lane, m.kytea_norm != 0);
                wpos2 += 128;
            }
            __syncwarp();
            const uint32_t g = cb + lane;
            if (g < n) {
                Rec32 rec;
                uint32_t slot;
                bool deep_hit;
                if (find_node<false>(m.ct, r, text, si.b0, g, rec, slot, m.kytea_norm != 0, &deep_hit) && deep_hit && (rec.v[1] & (1u << 29))) {
                    const uint64_t dsc = __ldg(m.ct.slot_ovf + slot);
                    const uint32_t ptr = uint32_t(dsc);
                    const int off = int(int16_t(uint16_t(dsc >> 32))), len = int(uint16_t(dsc >> 48));
                    for (int k = 0; k < len; ++k) {
                        const int64_t i = int64_t(g) + off + k;
                        if (i >= 0 && i < int64_t(si.nout)) atomicAdd(a.scores + si.obase + i, __ldg(m.ct.pool + ptr + k));
                    }
                }
            }
            __syncwarp();
        }
        __threadfence();
        __syncwarp();
        for (uint32_t i = lane; i < si.nout; i += 32) a.boundaries[si.obase + i] = __ldcg(a.scores + si.obase + i) > 0 ? 1 : 0;
    }
}

__device__ __forceinline__ void fast_sentence_warp(const DevModel& m, const BatchArgs& a, uint64_t s, Rings& r, int lane) {
    const SentInfo si = sentence_info(a, s, lane);
    fast_sentence_warp_si(m, a, si, r, lane);
}

}  // namespace

}  // namespace vpt
