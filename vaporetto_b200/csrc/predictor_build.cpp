#include "predictor_build.hpp"

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.hpp"

namespace vpt {

namespace {

struct BlobWriter {
    std::vector<uint8_t> buf;
    uint64_t add(const void* p, size_t n) {
        size_t off = align_up(buf.size(), 256);
        buf.resize(off + n);
        if (n) memcpy(buf.data() + off, p, n);
        return off;
    }
};

void write_table(BlobWriter& w, const NodeTable& t, size_t n_patterns, BlobTable& bt) {
    memset(&bt, 0, sizeof bt);
    bt.present = t.present;
    if (!t.present) return;
    bt.fast = t.fast;
    bt.r0 = t.r0;
    bt.max_depth = t.max_depth;
    bt.nslots = t.geom.nslots;
    bt.nbuckets = t.geom.nbuckets;
    bt.salt = t.geom.salt;
    bt.seed_bits = t.geom.seed_bits;
    bt.spill_slots = t.geom.spill ? spill_slots_of(t.geom.nslots) : 0u;
    bt.spill_buckets = t.geom.spill ? spill_buckets_of(t.geom.nbuckets) : 0u;
    bt.n_nodes = t.n_nodes;
    bt.n_patterns = uint32_t(n_patterns);
    bt.rec_off = w.add(t.records.data(), t.records.size());
    bt.seeds_off = w.add(t.seeds.data(), t.seeds.size());
    bt.node_off = w.add(t.slot_node.data(), t.slot_node.size() * 4);
    bt.pid_off = w.add(t.slot_pid.data(), t.slot_pid.size() * 4);
    bt.pool_off = w.add(t.pool.data(), t.pool.size() * 4);
    bt.has_overflow = t.has_overflow;
    if (t.has_overflow) bt.ovf_off = w.add(t.slot_ovf.data(), t.slot_ovf.size() * 8);
}


TagWeightMap collect_tag_weights(const PatternSet& ps, size_t n_tokens, size_t window) {
    TagWeightMap m(n_tokens, std::vector<std::unordered_map<uint32_t, std::vector<int32_t>>>(window + 1));
    for (size_t pid = 0; pid < ps.tags.size(); ++pid)
        for (const auto& kv : ps.tags[pid]) m[kv.first.first][kv.first.second][uint32_t(pid)] = kv.second;
    return m;
}

}  // namespace

// Predictor::new (reference predictor.rs:450-508)
HostPredictor build_host_predictor(const Model& m, bool predict_tags) {
    HostPredictor hp;
    HostPredictor* p = &hp;
    p->predict_tags = predict_tags;

    std::vector<const std::vector<TagNgramEntry>*> tag_char, tag_type;
    if (predict_tags) {
        for (size_t i = 0; i < m.tag_models.size(); ++i) {
            const auto& t = m.tag_models[i];
            p->n_tags = std::max(p->n_tags, t.tags.size());
            TagPredictorHost tp{t.tags, t.bias};
            if (tp.bias.size() < 8) tp.bias.resize(8, 0);
            p->token_ids[t.token] = uint32_t(i);  // "token does not duplicate in the model": last insert wins
            p->tag_preds.push_back(std::move(tp));
            tag_char.push_back(&t.char_ngrams);
            tag_type.push_back(&t.type_ngrams);
        }
    }

    // variant selection: CharScorer::new (char_scorer.rs:92-124), TypeScorer::new (type_scorer.rs:104-143)
    const bool has_char = !((m.char_ngrams.empty() && m.dict.empty()) || m.char_window == 0);
    const bool has_type = !(m.type_ngrams.empty() || m.type_window == 0);
    const bool tags = !tag_char.empty();
    int type_variant = 0;  // 0 none, 1 Boundary (automaton), 2 BoundaryCache, 3 BoundaryTag
    if (has_type) type_variant = tags ? 3 : (m.type_window <= 3 ? 2 : 1);
    const int char_variant = has_char ? (tags ? 2 : 1) : 0;

    PatternSet cps, tps;
    NodeTable ctab, ttab;
    std::vector<int32_t> tcache;
    std::vector<uint32_t> tstate3;
    // seed bytes the tile kernel keeps in shared memory (kernels.cu kSeedCap); VPT_SEED_BUDGET overrides it so that
    // tests can drive small models through the fat-bucket and dense 16-bit-seed table layouts
    uint32_t kSeedBudget = 37632;
    if (const char* e = getenv("VPT_SEED_BUDGET")) {
        const long v = atol(e);
        if (v > 0 && v < 37632) kSeedBudget = uint32_t(v);
    }
    // Type scorer.  The boundary scores of the automaton variants equal the cached table's whenever the window is
    // <= 3 (sum of all boundary n-gram occurrences either way), so tag predictors with short type patterns use the
    // table for scores and a 512-entry direct table for the pattern-id states; only windows > 3 or long tag type
    // n-grams need the type node table on the device.
    bool type_table_on_device = false;
    if (type_variant == 2) tcache = build_type_cache(m.type_ngrams, m.type_window);
    else if (type_variant != 0) {
        tps = build_patterns(m.type_ngrams, nullptr, m.type_window, tag_type, false);
        bool light = false;
        // (exact only when every boundary weight vector lies inside the 2W window: the table indexes weights by
        //  window position, the automaton variant adds whatever the row holds)
        bool in_window = true;
        for (const auto& d : m.type_ngrams)
            in_window = in_window && d.ngram.size() <= size_t(2 * m.type_window) &&
                        d.weights.size() + d.ngram.size() <= size_t(2 * m.type_window) + 1;
        if (type_variant == 3 && m.type_window <= 3 && in_window && build_type_state3(tps, tstate3)) {
            try {
                tcache = build_type_cache(m.type_ngrams, m.type_window);
                light = true;
            } catch (const Error&) {  // duplicate boundary n-grams: the merger adds them, the cache builder rejects them
                tstate3.clear();
            }
        }
        if (!light) {
            ttab = build_node_table(tps, true, kSeedBudget);
            type_table_on_device = true;
        }
    }
    // a general-format type table forces the general kernels, which need general char records
    const bool need_general = type_table_on_device;
    if (has_char) {
        cps = build_patterns(m.char_ngrams, &m.dict, m.char_window, tag_char, true);
        ctab = build_node_table(cps, need_general, kSeedBudget);
    }
    if (tags) {
        if (has_char) { p->char_tag_weight = collect_tag_weights(cps, m.tag_models.size(), m.char_window); p->char_suffix_link = cps.suffix_link; p->char_tags = true; }
        if (type_variant == 3) { p->type_tag_weight = collect_tag_weights(tps, m.tag_models.size(), m.type_window); p->type_suffix_link = tps.suffix_link; p->type_tags = true; }
    }

    BlobWriter w;
    BlobHeader h{};
    w.buf.resize(sizeof(BlobHeader));
    memcpy(h.magic, kBlobMagic, 8);
    h.bias = m.bias;
    h.char_window = m.char_window;
    h.type_window = m.type_window;
    h.type_cache_window = tcache.empty() ? 0 : m.type_window;
    h.emit_states = tags ? 1 : 0;
    h.char_variant = char_variant;
    h.type_variant = type_variant;
    h.max_char_pattern_len = int32_t(cps.max_len);
    write_table(w, ctab, cps.raw.size(), h.ct);
    write_table(w, ttab, tps.raw.size(), h.tt);
    if (!tstate3.empty()) h.type_state3_off = w.add(tstate3.data(), tstate3.size() * 4);
    if (!tcache.empty()) {
        h.type_cache_off = w.add(tcache.data(), tcache.size() * 4);
        std::vector<int32_t> ta, tb;
        if (build_type_split(m.type_ngrams, m.type_window, ta, tb)) {
            h.type_a_off = w.add(ta.data(), ta.size() * 4);
            h.type_b_off = w.add(tb.data(), tb.size() * 4);
        }
    }
    w.buf.resize(align_up(w.buf.size(), 256));
    h.total_bytes = w.buf.size();
    memcpy(w.buf.data(), &h, sizeof h);
    p->hdr = h;
    p->blob.swap(w.buf);
    return hp;
}


}  // namespace vpt
