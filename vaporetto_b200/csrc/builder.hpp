// Builds the flat, device-resident form of a predictor from a Model.
//
// What the reference does at `Predictor::new` (vaporetto/src/predictor.rs:450-508):
//   * CharScorer::new (char_scorer.rs:92-124) / TypeScorer::new (type_scorer.rs:104-143) select the
//     scorer variants, merge weights per pattern string and suffix-sum them
//     (CharWeightMerger, char_scorer.rs:29-79) and build a daachorse automaton.
// What this build does instead (GPU-first, see DESIGN.md §3):
//   * the same merged weight rows, but no automaton.  Matching is position-parallel on the GPU:
//     for the text ending at a character the kernel looks up the longest suffix that is a suffix of
//     some pattern in a *perfect-hash table of reversed-pattern trie nodes*; every node record carries
//     the merged weight row of the longest pattern that is a suffix of the node string, so one probe
//     yields what `find_overlapping_no_suffix_iter` + `weights[id]` yield in the reference.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "keys.hpp"
#include "model.hpp"

namespace vpt {


// One merged weight row: adds w[k] to boundary (last_char_index + off + k).
struct Row {
    bool present = false;
    int off = 0;
    std::vector<int32_t> w;
};

// Per-pattern tag weights (PositionalWeightWithTag::tag_info, predictor.rs:217-262): (token_id, rel_position) ->
// weights.  The reference suffix-merges them at build time; here the merge is evaluated at lookup time along
// `suffix_link` (same result, without copying a short pattern's entries into every longer pattern).
using TagInfo = std::vector<std::pair<std::pair<uint32_t, uint8_t>, std::vector<int32_t>>>;

struct PatternSet {
    bool utf8 = true;                          // char patterns (code points) or type patterns (bytes)
    std::vector<std::string> raw;              // pattern bytes, sorted byte-lexicographically; index = pattern id
    std::vector<std::vector<uint32_t>> syms;   // the same patterns as symbol sequences
    std::vector<Row> rows;                     // merged boundary rows (zero-trimmed)
    std::vector<TagInfo> tags;                 // the pattern's OWN tag weights (tag variant only; not suffix-merged)
    std::vector<uint32_t> suffix_link;         // longest proper suffix that is a pattern, or kNoPattern
    bool tag_variant = false;
    size_t max_len = 0;                        // longest pattern in symbols
};

struct NodeTable {
    bool present = false;
    bool fast = false;          // records are FastRecord (all rows fit the inline window)
    int r0 = 0;                 // inline window start (fast) — relative position of w[0]
    TableGeom geom;
    uint32_t n_nodes = 0;
    uint32_t max_depth = 0;
    std::vector<uint8_t> records;       // (nslots + spill_slots) * 32 bytes
    std::vector<uint8_t> seeds;         // nbuckets (x 2 for 16-bit seeds), then spill_buckets
    std::vector<uint32_t> slot_node;    // per slot: node id of the record in the slot (deep keys)
    std::vector<uint32_t> slot_pid;     // per slot: best pattern id (tag states); fast tables only
    std::vector<int32_t> pool;          // general rows / overflow rows (full row with the inline part zeroed)
    std::vector<uint64_t> slot_ovf;     // fast tables with overflow: ptr | (off & 0xFFFF) << 32 | len << 48 per slot
                                        // (the spill slots follow the primary ones in all four per-slot arrays)
    bool has_overflow = false;
    int rel_min = 0, rel_max = 0;       // union extent of all rows: [rel_min, rel_max)
};

// Builds merged pattern rows.  `dict` may be null (type scorer).
PatternSet build_patterns(const std::vector<NgramEntry>& ngrams, const std::vector<DictEntry>* dict, uint8_t window,
                          const std::vector<const std::vector<TagNgramEntry>*>& tag_ngrams, bool utf8);

// Reversed-pattern trie -> perfect-hash table.  `force_general` disables the inline format; `bucket_cap` is the
// number of seed bytes the kernel can keep in shared memory (0 = no preference).
NodeTable build_node_table(const PatternSet& ps, bool force_general, uint32_t bucket_cap = 0);

// Tag variant of the type scorer with patterns of at most 3 types: pattern id of the longest pattern ending at
// a character as a direct table over the 9-bit code (t[-2] t[-1] t[0]), zero = before the sentence start.
bool build_type_state3(const PatternSet& tps, std::vector<uint32_t>& table);

// Type score table of TypeScorerBoundaryCache::new (type_scorer/boundary_scorer_cache.rs:22-56).
std::vector<int32_t> build_type_cache(const std::vector<NgramEntry>& type_ngrams, uint8_t window);

// For window 3 and n-grams of at most 3 types the 8^6-entry table splits exactly into two 8^4-entry
// tables: T[t0..t5] = A[t0..t3] + B[t2..t5] (A: occurrences inside positions 0..3, B: the others, which all
// lie inside positions 2..5).  Returns false if the model does not qualify.  Both tables fit in shared memory.
bool build_type_split(const std::vector<NgramEntry>& type_ngrams, uint8_t window, std::vector<int32_t>& a,
                      std::vector<int32_t>& b);

uint32_t table_slot(const TableGeom& g, const uint8_t* seeds, uint64_t key);

}  // namespace vpt
