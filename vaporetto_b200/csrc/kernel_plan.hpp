// vaporetto_b200 — which scoring kernel, which template variant of it, and which tile geometry a batch runs.
// Host code only (no device code): launch_score / launch_fused dispatch on plan(), vpt_predictor_kernel_plan reports
// it, and the kernels tie their buffer sizes to the numbers below with static_asserts (fused_kernel.cuh, kernels.cu).
#pragma once
#include <algorithm>
#include <cstdint>

#include "device_model.hpp"
#include "fused_launch.hpp"

namespace vpt {

enum PlanKernel : int32_t { kPlanNone = 0, kPlanFused = 1, kPlanTileFast = 2, kPlanScoreFast = 3, kPlanScoreGeneral = 4 };

struct KernelPlan {
    int32_t kernel = kPlanNone;
    // template switches of k_fused (seeds_smem is k_tile_fast's too)
    bool seeds_smem = false;  // perfect-hash seed bytes staged in shared memory
    bool common = false;      // char window 3 + type window 3 with split tables: lag and gap are compile-time constants
    int32_t deep = 0;         // 0: patterns of <= 3 characters; 1: longer ones (backward walk); 2: and rows outside the window
    bool states = false;      // pattern-id states are written
    // template switches of k_tile_fast
    bool r0_fixed = false;    // inline window start -3 compiled in (otherwise a run-time value)
    bool general = false;     // general rows (scattered with atomics) instead of inline rows
    bool split3 = false;      // type window 3 with the split tables in shared memory
    bool overflow = false;    // inline rows plus the long rows of dictionary words
    // tile geometry (zero for the one-warp-per-sentence kernels)
    int32_t text_cap = 0;     // bytes of text a tile stages
    int32_t slot_cap = 0;     // character slots (characters + separator slots) per tile
    int32_t gap = 0;          // separator slots in front of every sentence of a tile
    int32_t lag = 0;          // k_fused: a boundary is finished `lag` slots after its own slot
    int32_t sub_blocks = 0;   // independent 256-thread sub-blocks per CTA
    int32_t group = 0;        // sentences per group
};

namespace plan_detail {

// k_fused (fused_kernel.cuh FCaps / FLayout)
constexpr int fused_text_cap(bool seeds_smem, bool states, bool overflow) {
    return (states || (overflow && !seeds_smem)) ? 9216 : 10240;
}
constexpr int fused_slot_cap(bool seeds_smem, bool states, bool overflow) {
    return !overflow ? (states ? 3328 : 3840) : seeds_smem ? (states ? 3264 : 3840) : (states ? 2944 : 3584);
}
constexpr int fused_sub_blocks(bool seeds_smem, bool overflow) { return (overflow && seeds_smem) ? 3 : 4; }

// k_tile_fast (kernels.cu)
constexpr int kTileTextCap = 12288;
constexpr int kTileSlotCap = 3072;
constexpr int kTileSubBlocks = 4;

inline bool inline_rows(const DevModel& m) { return (!m.ct.present || m.ct.fast) && !m.tt.present; }

inline bool seeds_smem(const DevModel& m) {
    return m.ct.present && !m.ct.seed16 && m.ct.nbuckets + m.ct.spill_buckets <= uint32_t(fused_detail::kSeedCap);
}

// separator slots between the sentences of a tile, so that neither the weight-row gather (window [r0, r0 + 6)) nor the
// type window reaches a neighbouring sentence (general tables clip their rows per sentence)
inline int tile_gap(const DevModel& m) {
    const int tw = std::max(2, m.type_cache_window - 1);
    if (!inline_rows(m)) return tw;
    const int r0 = m.ct.present ? m.ct.r0 : 0;
    return std::max(tw, std::max(-r0 - 1, r0 + kInlineWidth - 1));
}

inline int fused_lag(const DevModel& m) {
    const int r0 = m.ct.present ? m.ct.r0 : 0;
    return std::max(std::max(-r0, m.type_cache_window), 1);
}

inline bool fused_shape_ok(const DevModel& m) {
    if (!inline_rows(m)) return false;
    const int r0 = m.ct.present ? m.ct.r0 : 0;
    const int tw = m.type_cache_window;
    if (r0 < -5 || r0 > 0 || tw < 0 || tw > 3) return false;
    if (tile_gap(m) > 8) return false;
    if (m.emit_states && m.ct.present && m.ct.max_depth == 0) return false;
    return fused_lag(m) + std::max(tw, 1) <= 6;  // the packed type history holds t[p-5 .. p]
}

inline bool tile_shape_ok(const DevModel& m) {
    if (!inline_rows(m)) return false;
    const int r0 = m.ct.present ? m.ct.r0 : 0;
    return r0 >= -8 && r0 <= 2 && tile_gap(m) <= 8 && m.type_cache_window <= 3;
}

}  // namespace plan_detail

// `states`: the batch asks for pattern-id states (BatchArgs::char_states or type_states set).
inline KernelPlan plan(const DevModel& m, bool states) {
    using namespace plan_detail;
    KernelPlan p;
    if (fused_shape_ok(m)) {
        p.kernel = kPlanFused;
        p.seeds_smem = seeds_smem(m);
        p.gap = tile_gap(m);
        p.lag = fused_lag(m);
        // the usual shape: char window 3 (inline window starts at -3) + type window 3 with split tables
        p.common = m.type_a != nullptr && m.type_cache_window == 3 && m.ct.present && m.ct.r0 == -3 &&
                   p.gap == fused_detail::kCommonGap;
        // patterns longer than three symbols (dictionary words) need the backward walk; their rows may stick out of the window
        p.deep = !m.ct.present || m.ct.max_depth <= 3 ? 0 : (m.ct.has_overflow ? 2 : 1);
        p.states = states;
        p.text_cap = fused_text_cap(p.seeds_smem, p.states, p.deep == 2);
        p.slot_cap = fused_slot_cap(p.seeds_smem, p.states, p.deep == 2);
        p.sub_blocks = fused_sub_blocks(p.seeds_smem, p.deep == 2);
        p.group = fused_detail::kGroupSentences;
        return p;
    }
    // general tables through the tile kernel pay off for shallow pattern sets (n-gram models with tags); deep
    // dictionaries (long rows, backward walks, seed array too large for shared memory) are faster one warp per sentence
    const bool tile_general = !inline_rows(m) && m.type_cache_window <= 3 && m.ct.max_depth <= 3 && m.tt.max_depth <= 4;
    if (tile_shape_ok(m) || tile_general) {
        p.kernel = kPlanTileFast;
        p.seeds_smem = seeds_smem(m);
        p.r0_fixed = !tile_general && m.ct.present && m.ct.r0 == -3;
        p.general = tile_general;
        p.split3 = m.type_a != nullptr && m.type_cache_window == 3;
        p.overflow = !tile_general && m.ct.present && m.ct.has_overflow;
        p.text_cap = kTileTextCap;
        p.slot_cap = kTileSlotCap;
        p.gap = tile_gap(m);
        p.sub_blocks = kTileSubBlocks;
        p.group = kGroup;
        return p;
    }
    // inline rows with an unusual window, or deep general tables: one warp per sentence
    p.kernel = inline_rows(m) ? kPlanScoreFast : kPlanScoreGeneral;
    return p;
}

}  // namespace vpt
