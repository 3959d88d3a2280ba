// Device-side tag prediction (reference Predictor::predict_tags, predictor.rs:546-637; add_tag_scores,
// char_scorer/boundary_tag_scorer.rs:154-174 and type_scorer/boundary_tag_scorer.rs:123-143; TagPredictor::predict,
// predictor.rs:286-304): flat tables built on the host from the predictor's tag models, and the launch interface.
//
// Tables (one device allocation per predictor, built by build_tag_tables):
//   * token table   open addressing over a 64-bit hash of the token's bytes; an entry holds the hash, the token id and
//                   where the token's bytes live (compared byte by byte: the lookup is exact)
//   * token info    per token id: bias vector (i32 pool), number of tag slots, candidates per slot, and where the
//                   token's KEY LIST lives
//   * key lists     per token, contiguous: one 16-byte entry per (pattern id, rel position) that carries an OWN weight
//                   vector for this token -- the char scorer's entries first, then the type scorer's; each part sorted by
//                   rel position and, within one rel position, by pattern length (suffix-chain depth), longest first.
//                   The reference merges the vectors of a pattern's suffix patterns into it at build time
//                   (PositionalWeightWithTag +=, predictor.rs:242-262, along char_scorer.rs:50-78); here the kernel
//                   adds, for the pattern found at a position, the own vectors of the patterns on its suffix chain with
//                   the same truncation rule (element k of a shorter suffix's vector counts only while every longer
//                   pattern on the chain has an own vector longer than k) -- identical sums, no 300-second
//                   materialisation.  Scanning the token's short list in this order visits the chain members longest
//                   first, which is the order the rule needs.
//   * chain tables  per pattern id: the next four patterns on its suffix chain (16 bytes, one load); longer chains
//                   (dictionary words) continue through `link`
#pragma once
#include <cstdint>
#include <vector>

#include <cuda_runtime.h>

#include "predictor_build.hpp"

namespace vpt {

constexpr int kTagMaxScores = 64;  // score entries a token's tag model may have on the device path
constexpr int kTagMaxSlots = 8;    // tag slots (n_tags) on the device path

struct TagTokenEntry {   // 24 bytes
    uint64_t hash;       // 0 = empty
    uint32_t tid;
    uint32_t str_off;
    uint32_t len;
    uint32_t pad;
};
struct alignas(16) TagTokenInfo {    // per token id, 32 bytes
    uint32_t bias_off;   // into the i32 pool
    uint16_t bias_len;
    uint8_t n_slots;     // tags.size() (slots beyond n_tags never exist)
    uint8_t usable;      // 0: the token's model exceeds the device limits (never happens for the reference's models)
    uint8_t cand[kTagMaxSlots];  // candidates per slot (255 = too many)
    uint32_t key_off;    // first entry of the token's key list
    uint8_t ckeys[4];    // char scorer entries with rel position 0 .. 3, then
    uint8_t tkeys[4];    // type scorer entries with rel position 0 .. 3 (after all char entries)
    uint16_t c_rest;     // char scorer entries with rel position >= 4 (windows wider than 3), after ckeys
    uint16_t t_rest;     // type scorer entries with rel position >= 4
};
static_assert(sizeof(TagTokenInfo) == 32, "TagTokenInfo layout");
struct TagKey {          // 16 bytes
    uint32_t pid;        // pattern id
    uint32_t off;        // the own weight vector, into the i32 pool
    uint32_t len;
    uint32_t rel;        // rel position
};
struct TagChain {        // 16 bytes: patterns 1..4 steps down the suffix chain of a pattern (kNoPattern = end)
    uint32_t next[4];
};

struct TagTablesHost {
    bool usable = false;           // false: some limit is exceeded -> only the host path (vpt_fill_tags) serves the model
    bool all_tokens_usable = false;  // every TagTokenInfo::usable is set: the device serves every token of the model
    uint32_t n_tags = 0, n_tokens = 0;
    uint32_t tok_mask = 0;         // token table capacity - 1 (power of two)
    uint32_t char_rels = 0, type_rels = 0;   // rel positions 0 .. rels-1 carry weights (window + 1)
    uint32_t max_token_bytes = 0;
    std::vector<TagTokenEntry> tok_tab;
    std::vector<uint8_t> tok_bytes;
    std::vector<TagTokenInfo> tok_info;
    std::vector<int32_t> pool;
    // tag strings, escaped as write_tokenized_text writes them (' ', '\\', '/' behind a '\\'): ts_slot[tid] -> first slot
    // entry, ts_cand[slot entry] -> first string reference, ts_ref = (offset, length) into ts_bytes
    std::vector<uint32_t> ts_slot, ts_cand;
    std::vector<uint32_t> ts_ref;              // pairs
    std::vector<uint8_t> ts_bytes;
    uint32_t max_suffix = 0;                   // longest "/tag/tag..." suffix a token can get
    std::vector<TagKey> keys;
    std::vector<TagChain> c_chain, t_chain;
    std::vector<uint32_t> c_link, t_link;      // suffix links by pattern id
};

TagTablesHost build_tag_tables(const HostPredictor& hp);

struct DevTags {
    const TagTokenEntry* tok_tab = nullptr;
    const uint8_t* tok_bytes = nullptr;
    const TagTokenInfo* tok_info = nullptr;
    const int32_t* pool = nullptr;
    const uint32_t* ts_slot = nullptr;
    const uint32_t* ts_cand = nullptr;
    const uint2* ts_ref = nullptr;
    const uint8_t* ts_bytes = nullptr;
    uint32_t max_suffix = 0;
    const TagKey* keys = nullptr;
    const TagChain* c_chain = nullptr;
    const TagChain* t_chain = nullptr;
    const uint32_t* c_link = nullptr;
    const uint32_t* t_link = nullptr;
    uint32_t tok_mask = 0;
    uint32_t n_tags = 0, char_rels = 0, type_rels = 0, max_token_bytes = 0;
    uint32_t n_char_patterns = 0, n_type_patterns = 0;
};

struct TagArgs {
    const uint8_t* text = nullptr;
    const uint64_t* offsets = nullptr;      // [n_sent + 1] byte offsets
    const uint8_t* trims = nullptr;         // nullable
    uint64_t n_sent = 0;
    const int32_t* status = nullptr;        // from the scoring pass
    const uint8_t* boundaries = nullptr;    // final boundaries (0 / 1)
    const uint64_t* bound_offsets = nullptr;  // [n_sent + 1] (values include bound_base)
    const uint64_t* char_offsets = nullptr;   // [n_sent + 1] (values include char_base)
    uint64_t bound_base = 0, char_base = 0;
    const uint32_t* char_states = nullptr;  // nullable when the char scorer has no tag weights
    const uint32_t* type_states = nullptr;
    int32_t* tag_token = nullptr;           // [n_chars] out: token id of the token ending at the character, or -1
    int32_t* tag_cand = nullptr;            // [n_chars * n_tags] out: chosen candidate per slot, or -1
    uint32_t* n_unserved = nullptr;         // nullable device counter: tokens whose own model exceeds the device limits
                                            // (TagTokenInfo::usable == 0) or is malformed; tokens of any length are served
    // per-TOKEN output (vpt_predict_batch_compact) instead of the per-character arrays above: token r of sentence s
    // (in text order) is record tok_base[s] + r
    const uint64_t* tok_base = nullptr;     // [n_sent + 1] exclusive prefix of the tokens per sentence; selects this mode
    int32_t* tok_ids = nullptr;             // [n_tokens] token id or -1
    uint8_t* tok_cands = nullptr;           // [n_tokens * n_tags] chosen candidate per slot, 255 = none
    // with tok_desc the sentence-warp kernel only LOCATES the tokens (16 bytes each: x = low 32 bits of the byte offset
    // from text + text_base, y = its bits 32..47 | characters left in the sentence (saturated at 0xFFFF) << 16, z = index
    // of the last character, w = byte length) and two more kernels, one thread per token, look the tokens up and predict
    // the tags of those that have a model: full lanes and short dependent-load chains instead of one sentence per warp.
    // (The offsets index a host buffer's bytes, below 2^47 on every 64-bit host.)
    uint4* tok_desc = nullptr;              // [max_tokens] scratch; nullable (then k_tags does everything itself)
    uint64_t max_tokens = 0;                // bound on the number of tokens (e.g. the number of characters)
    uint32_t* tok_work = nullptr;           // [4 + max_tokens] scratch, needed with tok_desc: [0] counts the tokens that have a
                                            // tag model, their record indices follow from [4] on (k_tok_lookup -> k_tok_score)
    uint64_t text_base = 0;                 // byte offset the descriptors are relative to (keeps them below 2^64 safely)
    int norm = 0;                           // tokens are looked up by their KyteaFullwidthFilter image (the CLI default:
                                            // fill_tags runs on the pre-filtered sentence, predict/src/main.rs:153-166)
};

// Compact outputs (vpt_predict_batch_compact): boundaries as one bit each, tokens per sentence and their prefix.
struct CompactArgs {
    uint64_t n_sent = 0;
    const int32_t* status = nullptr;          // [n_sent] from the scoring pass
    const uint32_t* n_chars = nullptr;        // [n_sent]
    const uint8_t* boundaries = nullptr;      // [n_bound] 0 / 1
    const uint64_t* bound_offsets = nullptr;  // [n_sent + 1], values include bound_base
    uint64_t bound_base = 0;
    uint64_t n_bound = 0;
    uint32_t bit_base = 0;                    // the chunk's first boundary is bit `bit_base` (0..31) of bits[0]
    uint32_t* bits = nullptr;                 // [(bit_base + n_bound + 31) / 32]
    uint8_t* status8 = nullptr;               // [n_sent]
    uint32_t* n_tokens = nullptr;             // [n_sent] tokens per sentence (0 for a rejected sentence); nullable
    uint64_t* tok_base = nullptr;             // [n_sent + 1]; nullable with n_tokens
    uint32_t* tok_local = nullptr;            // [n_sent] scratch: prefix inside a block of 256 sentences
    uint64_t* tok_blk = nullptr;              // [n_sent / 256 + 2] scratch: block totals, then their prefix
    uint64_t* tok_total_host = nullptr;       // nullable: pinned host word that receives the number of tokens
};
cudaError_t launch_compact(const CompactArgs& c, cudaStream_t stream);

// 64-bit hash of a token's bytes (host builder and kernel)
#if defined(__CUDACC__)
#define VPT_TAG_HD __host__ __device__ __forceinline__
#else
#define VPT_TAG_HD inline
#endif
VPT_TAG_HD uint64_t tag_hash_step(uint64_t h, uint32_t byte) {
    h ^= byte;
    h *= 0x100000001B3ull;  // FNV-1a
    return h;
}
VPT_TAG_HD uint64_t tag_hash_finish(uint64_t h) {
    h ^= h >> 32;
    h *= 0x9E3779B97F4A7C15ull;
    h ^= h >> 29;
    return h | 1ull;  // never 0 (0 marks an empty entry)
}
constexpr uint64_t kTagHashInit = 0xCBF29CE484222325ull;

// Tag candidate scores of the per-token path (vpt_predict_batch_compact_tag_scores, vpt_token_spans_tag_scores): record r
// with token id >= 0 gets its token's whole score vector (tag_score_count entries), the vectors of the chunk concatenated
// in record order.  k_tok_lookup writes each record's count, a block scan + a one-block scan of the block totals turn
// the counts into offsets, k_tok_score stores the vectors there.
constexpr int kScoreScanBlock = 1024;   // records per block of the offset scan
struct TagScoreArgs {
    uint32_t* rec_off = nullptr;        // [max_tokens] scratch: score count of the record, then its offset inside its block
    uint64_t* blk = nullptr;            // [max_tokens / kScoreScanBlock + 2] scratch: block totals, then their prefix
    int32_t* scores = nullptr;          // [max_tokens x the longest vector] out: the chunk's score vectors
    uint64_t* total_host = nullptr;     // pinned host word that receives the number of scores of the chunk
};

// scores: nullable; with it (and the per-token path: tok_desc) the score vectors come out as well
cudaError_t launch_tags(const DevTags& t, const TagArgs& a, cudaStream_t stream, const TagScoreArgs* scores = nullptr);

}  // namespace vpt
