// Host-side construction of a predictor (no CUDA): variant selection, merged rows, node tables, the flat
// model blob and the host tag tables.  `Predictor::new` of the reference (vaporetto/src/predictor.rs:450-508).
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "builder.hpp"
#include "model.hpp"

namespace vpt {

constexpr char kBlobMagic[8] = {'V', 'P', 'T', 'B', '2', '0', '0', '\6'};

struct BlobTable {
    uint64_t rec_off, seeds_off, node_off, pid_off, pool_off;
    uint64_t salt;
    uint32_t nslots, nbuckets;
    int32_t r0;
    uint32_t max_depth;
    int32_t present, fast;
    uint32_t n_nodes, n_patterns;
    uint32_t seed_bits, has_overflow;
    uint64_t ovf_off;
    // spill table (keys.hpp: spill_slots_of / spill_buckets_of of the primary geometry): its records and side-array
    // entries follow the nslots primary ones, its seeds the nbuckets primary ones; 0 / 0 = none
    uint32_t spill_slots, spill_buckets;
};
struct BlobHeader {
    char magic[8];
    uint64_t total_bytes;
    int32_t bias, char_window, type_window, type_cache_window;
    int32_t emit_states, char_variant, type_variant, max_char_pattern_len;
    uint64_t type_cache_off;
    uint64_t type_a_off, type_b_off;  // split tables (0 = absent)
    uint64_t type_state3_off;         // 512-entry type state table (0 = absent)
    BlobTable ct, tt;
};


struct TagPredictorHost {  // reference TagPredictor (predictor.rs:264-304)
    std::vector<std::vector<std::string>> tags;
    std::vector<int32_t> bias;  // zero-padded to >= 8 like WeightVector::from (predictor.rs:118-135)
};

using TagWeightMap = std::vector<std::vector<std::unordered_map<uint32_t, std::vector<int32_t>>>>;


struct HostPredictor {
    bool predict_tags = false;
    BlobHeader hdr{};
    std::vector<uint8_t> blob;  // flat model image: BlobHeader + 256-byte aligned sections
    // tags (host)
    size_t n_tags = 0;
    std::unordered_map<std::string, uint32_t> token_ids;
    std::vector<TagPredictorHost> tag_preds;
    TagWeightMap char_tag_weight, type_tag_weight;      // own (un-merged) entries per pattern id
    std::vector<uint32_t> char_suffix_link, type_suffix_link;
    bool char_tags = false, type_tags = false;
};

HostPredictor build_host_predictor(const Model& m, bool predict_tags);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace vpt
