// PatternMatchTagger (vaporetto_rules/src/sentence_filters/pattern_match_tagger.rs:21-41) in the tagged line path: a
// user's table of rules surface -> [Option<tag>; k] fills the tag slots the model left empty.
//
// Table (one device allocation per vpt_tag_rules, built by build_tag_rules):
//   * rule table   open addressing over the token table's 64-bit surface hash (tag_hash_step / tag_hash_finish); an
//                  entry holds the hash, the rule id and where the surface's bytes live (compared byte by byte)
//   * slots        per rule id, slot_first[r] .. slot_first[r + 1]: its tag slots, clipped to the predictor's n_tags;
//                  a slot is (offset, length) into tag_bytes, offset kRuleNone = None; length 0 is Some("")
//   * tag bytes    escaped as write_tokenized_text writes them (' ', '\\', '/' behind a '\\'), like ts_bytes
//   * suffix       per rule id, an upper bound on the bytes the rule adds behind a token: 1 + length per slot
// The merge (merged_suffix_len / merged_suffix_write) is the per-thread code of k_tok_write_tags<true> (lines.cu); it
// has no warp operations, so tests/native/tag_rules_test.cpp runs it on the host.
#pragma once
#include <cstdint>
#include <vector>

#include "tags.hpp"
#include "tags_token.hpp"

namespace vpt {

constexpr uint32_t kRuleNone = 0xFFFFFFFFu;

struct TagRulesHost {
    uint32_t n_rules = 0;
    uint32_t mask = 0;         // rule table capacity - 1 (power of two)
    uint32_t max_bytes = 0;    // longest surface
    std::vector<TagTokenEntry> tab;
    std::vector<uint8_t> surf;
    std::vector<uint32_t> slot_first;  // [n_rules + 1]
    std::vector<uint32_t> slot_ref;    // pairs (offset, length)
    std::vector<uint8_t> tag_bytes;
    std::vector<uint32_t> suffix;      // [n_rules]
};

// The rules of vpt_tag_rules_new (include/vaporetto_b200.h), checked: throws Error(kInvalidArgument) naming the rule.
TagRulesHost build_tag_rules(uint64_t n_rules, const uint8_t* surfaces, const uint64_t* surface_offsets,
                             const uint64_t* slot_offsets, const uint32_t* slots, const uint8_t* tags, uint64_t tags_len,
                             uint32_t n_tags);

struct DevTagRules {
    const TagTokenEntry* tab = nullptr;
    const uint8_t* surf = nullptr;
    const uint32_t* slot_first = nullptr;
    const uint2* slot_ref = nullptr;
    const uint8_t* tag_bytes = nullptr;
    const uint32_t* suffix = nullptr;
    uint32_t mask = 0, max_bytes = 0;
};

// What the tagged writer needs besides TokArgs: the rules and the rule id of every token record
struct TagRuleArgs {
    DevTagRules rules;
    const int32_t* tok_rule = nullptr;  // [n_tokens] rule id or -1; nullptr = no rules
};

// k_rule_lookup (tags.cu): every token record of `a` (the per-token path: tok_base, tok_desc, text_base, norm; after
// launch_tags) gets its rule id in tok_rule; *suffix_sum (zeroed here) receives the sum of TagRulesHost::suffix over the
// records that matched, which bounds the bytes the rules add to the output.
cudaError_t launch_rule_lookup(const DevTagRules& r, const TagArgs& a, int32_t* tok_rule, unsigned long long* suffix_sum,
                               cudaStream_t stream);
struct TokArgs;
// launch_tokenize (lines.cu) with rules (ra.tok_rule != nullptr): k_tok_write_tags<true>
cudaError_t launch_tokenize_rules(const TokArgs& t, const TagRuleArgs& ra, cudaStream_t stream);
struct ColOut;
// launch_tokenize_rules writing the column output `col` (device_model.hpp) instead of '\n'-terminated lines:
// k_tok_write_col, k_tok_write_tags_col<kRules>; with n_sent == 0 it writes col.offsets[0] = 0
cudaError_t launch_tokenize_column(const TokArgs& t, const TagRuleArgs& ra, const ColOut& col, cudaStream_t stream);

// rule id of a token (its KyteaFullwidthFilter image when norm != 0), or -1: the token table's probe over the rule table
VPT_HD int32_t rule_lookup(const DevTagRules& r, const uint8_t* __restrict__ bytes, uint32_t len, int norm) {
    DevTags t;
    t.tok_tab = r.tab;
    t.tok_bytes = r.surf;
    t.tok_mask = r.mask;
    t.max_token_bytes = r.max_bytes;
    uint32_t id = 0;
    return token_lookup(t, bytes, len, norm, id) ? int32_t(id) : -1;
}

// Tag of slot k after the filter: the model's candidate c (255 = none; tid >= 0 when c != 255), else the rule's slot k.
// Returns 0 for None, 1 for a model tag (ref indexes ts_bytes), 2 for a rule tag (ref indexes r.tag_bytes).
VPT_HD int merged_slot(uint32_t k, int32_t tid, uint32_t c, const uint32_t* __restrict__ ts_slot,
                       const uint32_t* __restrict__ ts_cand, const uint2* __restrict__ ts_ref, int32_t rid,
                       const DevTagRules& r, uint2& ref) {
    if (c != 255u) {
        ref = VPT_LDG(ts_ref + VPT_LDG(ts_cand + VPT_LDG(ts_slot + tid) + k) + c);
        return 1;
    }
    if (rid >= 0) {
        const uint32_t first = VPT_LDG(r.slot_first + rid);
        if (k < VPT_LDG(r.slot_first + rid + 1) - first) {
            ref = VPT_LDG(r.slot_ref + first + k);
            if (ref.x != kRuleNone) return 2;
        }
    }
    return 0;
}

// Bytes of the token's "/tag/.." suffix: one '/' per slot up to the last slot that has a tag, plus the tags.
VPT_HD uint32_t merged_suffix_len(uint32_t n_tags, int32_t tid, const uint8_t* cands, const uint32_t* ts_slot,
                                  const uint32_t* ts_cand, const uint2* ts_ref, int32_t rid, const DevTagRules& r) {
    if (tid < 0 && rid < 0) return 0;  // (most tokens: no tag model, no rule)
    uint32_t len = 0, run = 0;
    for (uint32_t k = 0; k < n_tags; ++k) {
        uint2 ref;
        ++run;  // the '/'
        if (merged_slot(k, tid, cands[k], ts_slot, ts_cand, ts_ref, rid, r, ref)) {
            run += ref.y;
            len += run;
            run = 0;
        }
    }
    return len;
}
VPT_HD void merged_suffix_write(uint32_t n_tags, int32_t tid, const uint8_t* cands, const uint32_t* ts_slot,
                                const uint32_t* ts_cand, const uint2* ts_ref, const uint8_t* ts_bytes, int32_t rid,
                                const DevTagRules& r, uint8_t* __restrict__ out) {
    if (tid < 0 && rid < 0) return;
    uint32_t at = 0, pending = 0;  // '/' of the slots since the last one with a tag
    for (uint32_t k = 0; k < n_tags; ++k) {
        uint2 ref;
        const int from = merged_slot(k, tid, cands[k], ts_slot, ts_cand, ts_ref, rid, r, ref);
        ++pending;
        if (!from) continue;
        for (; pending; --pending) out[at++] = 0x2F;
        const uint8_t* src = from == 1 ? ts_bytes : r.tag_bytes;
        for (uint32_t j = 0; j < ref.y; ++j) out[at++] = VPT_LDG(src + ref.x + j);
    }
}

}  // namespace vpt
