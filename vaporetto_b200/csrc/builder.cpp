#include "builder.hpp"

#include <algorithm>
#include <cstring>
#include <map>
#include <numeric>

#include "common.hpp"

namespace vpt {

namespace {

// ---- aligned weight rows --------------------------------------------------------------------------
// A positional weight is a dense run of weights starting at relative offset `off`
// (reference PositionalWeight, predictor.rs:138-141).  Adding two rows aligns them on the smaller
// offset and zero-fills (predictor.rs:149-165).
struct PosWeight {
    int off = 0;
    std::vector<int32_t> w;
};

void accumulate(PosWeight& dst, const PosWeight& src) {
    const int lo = std::min(dst.off, src.off);
    const int hi = std::max(dst.off + int(dst.w.size()), src.off + int(src.w.size()));
    std::vector<int32_t> out(size_t(hi - lo), 0);
    for (size_t k = 0; k < dst.w.size(); ++k) out[size_t(dst.off - lo) + k] = dst.w[k];
    for (size_t k = 0; k < src.w.size(); ++k) {
        int32_t& y = out[size_t(src.off - lo) + k];
        y = wrapping_add(y, src.w[k]);
    }
    dst.off = lo;
    dst.w.swap(out);
}

struct Entry {
    bool has_weight = false;
    PosWeight weight;
    // (token_id, rel_position) -> tag weights; kept ordered for determinism
    std::map<std::pair<uint32_t, uint8_t>, std::vector<int32_t>> tag;
};

// PositionalWeightWithTag += (predictor.rs:242-262)
void accumulate(Entry& dst, const Entry& src) {
    if (src.has_weight) {
        if (dst.has_weight) accumulate(dst.weight, src.weight);
        else { dst.weight = src.weight; dst.has_weight = true; }
    }
    for (const auto& kv : src.tag) {
        auto it = dst.tag.find(kv.first);
        if (it == dst.tag.end()) {
            dst.tag.emplace(kv.first, kv.second);
        } else {
            const size_t n = std::min(it->second.size(), kv.second.size());
            for (size_t k = 0; k < n; ++k) it->second[k] = wrapping_add(it->second[k], kv.second[k]);
        }
    }
}

std::vector<uint32_t> to_symbols(const std::string& s, bool utf8) {
    if (utf8) return utf8_to_codepoints(s);
    std::vector<uint32_t> v(s.size());
    for (size_t i = 0; i < s.size(); ++i) v[i] = uint8_t(s[i]);
    return v;
}

size_t symbol_count(const std::string& s, bool utf8) {
    if (!utf8) return s.size();
    size_t n = 0;
    for (unsigned char c : s) n += (c & 0xC0) != 0x80;
    return n;
}

}  // namespace

PatternSet build_patterns(const std::vector<NgramEntry>& ngrams, const std::vector<DictEntry>* dict, uint8_t window,
                          const std::vector<const std::vector<TagNgramEntry>*>& tag_ngrams, bool utf8) {
    // 1. union of all weights given to the same pattern string, in the reference's insertion order
    //    (n-grams, dictionary words, tag n-grams: char_scorer/boundary_tag_scorer.rs:68-96).
    std::map<std::string, Entry> table;  // ordered by bytes == pattern id order (BTreeMap<String,_>)
    auto add = [&](const std::string& key, const Entry& e) {
        if (key.empty()) throw Error(kInvalidModel, "InvalidModelError: failed to build the automaton");
        auto it = table.find(key);
        if (it == table.end()) table.emplace(key, e);
        else accumulate(it->second, e);
    };
    for (const auto& d : ngrams) {
        Entry e;
        e.has_weight = true;
        e.weight.off = -int(window);
        e.weight.w = d.weights;
        add(d.ngram, e);
    }
    if (dict) {
        for (const auto& d : *dict) {
            const size_t len = symbol_count(d.word, true);
            if (len > 32767)  // i16::try_from(word_len) (char_scorer/boundary_scorer.rs:67-72)
                throw Error(kInvalidModel,
                            "InvalidModelError: words must be shorter than or equal to 32767 characters");
            Entry e;
            e.has_weight = true;
            e.weight.off = -int(len);
            e.weight.w = d.weights;
            add(d.word, e);
        }
    }
    for (size_t t = 0; t < tag_ngrams.size(); ++t) {
        for (const auto& d : *tag_ngrams[t]) {
            for (const auto& tw : d.weights) {
                if (tw.rel_position > window)  // reference indexes tag_weight[token][rel] (len window+1): panic
                    throw Error(kInvalidModel, "InvalidModelError: tag rel_position exceeds the window size");
                Entry e;
                e.tag[{uint32_t(t), tw.rel_position}] = tw.weights;
                add(d.ngram, e);
            }
        }
    }

    PatternSet ps;
    ps.utf8 = utf8;
    ps.tag_variant = !tag_ngrams.empty();
    const size_t n = table.size();
    ps.raw.reserve(n);
    std::vector<Entry*> own;
    own.reserve(n);
    std::unordered_map<std::string, uint32_t> index;
    index.reserve(n * 2);
    for (auto& kv : table) {
        index.emplace(kv.first, uint32_t(ps.raw.size()));
        ps.raw.push_back(kv.first);
        own.push_back(&kv.second);
    }
    ps.syms.resize(n);
    for (size_t i = 0; i < n; ++i) {
        ps.syms[i] = to_symbols(ps.raw[i], utf8);
        ps.max_len = std::max(ps.max_len, ps.syms[i].size());
    }

    // 2. suffix sums: merged(p) = own(p) + merged(longest proper suffix of p that is a pattern)
    //    == own(p) + sum of own(q) over all proper-suffix patterns q  (char_scorer.rs:50-78).
    //    Processing patterns by increasing byte length guarantees the suffix is final.
    std::vector<uint32_t> order(n);
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(),
                     [&](uint32_t a, uint32_t b) { return ps.raw[a].size() < ps.raw[b].size(); });
    //    Tag weights are NOT materialised along the suffix chain (a frequent unigram tag n-gram would be copied
    //    into every longer pattern): each pattern keeps its own entries plus a link to its longest proper
    //    suffix pattern, and vpt_fill_tags evaluates the reference's merge (predictor.rs:242-262) lazily.
    ps.suffix_link.assign(n, kNoPattern);
    for (uint32_t p : order) {
        const std::string& s = ps.raw[p];
        for (size_t j = 1; j < s.size(); ++j) {
            if (utf8 && (uint8_t(s[j]) & 0xC0) == 0x80) continue;
            auto it = index.find(s.substr(j));
            if (it != index.end()) {
                Entry& dst = *own[p];
                const Entry& src = *own[it->second];
                if (src.has_weight) {
                    if (dst.has_weight) accumulate(dst.weight, src.weight);
                    else { dst.weight = src.weight; dst.has_weight = true; }
                }
                ps.suffix_link[p] = it->second;
                break;
            }
        }
    }

    // 3. export, trimming zero weights at both ends (adding zero is the identity)
    ps.rows.resize(n);
    ps.tags.resize(n);
    for (size_t i = 0; i < n; ++i) {
        const Entry& e = *own[i];
        Row& r = ps.rows[i];
        if (e.has_weight) {
            size_t lo = 0, hi = e.weight.w.size();
            while (lo < hi && e.weight.w[lo] == 0) ++lo;
            while (hi > lo && e.weight.w[hi - 1] == 0) --hi;
            r.present = true;
            r.off = e.weight.off + int(lo);
            r.w.assign(e.weight.w.begin() + long(lo), e.weight.w.begin() + long(hi));
        }
        for (const auto& kv : e.tag) ps.tags[i].push_back({kv.first, kv.second});
    }
    return ps;
}

std::vector<int32_t> build_type_cache(const std::vector<NgramEntry>& type_ngrams, uint8_t window) {
    const size_t seq = size_t(window) * 2;
    {   // DoubleArrayAhoCorasick::new rejects empty and duplicate patterns
        std::map<std::string, int> seen;
        for (const auto& d : type_ngrams)
            if (d.ngram.empty() || !seen.emplace(d.ngram, 1).second)
                throw Error(kInvalidModel, "InvalidModelError: invalid character type n-grams");
    }
    std::vector<int32_t> table(size_t(1) << (3 * seq), 0);
    // For each n-gram occurrence position inside the 2W-symbol window, add its weight to every window
    // whose remaining symbols range over 0..6 (7 never occurs: seqid_to_seq, boundary_scorer_cache.rs:83-93).
    std::vector<uint32_t> digits(seq);
    for (const auto& d : type_ngrams) {
        const size_t L = d.ngram.size();
        if (L > seq) continue;
        bool ok = true;
        for (unsigned char c : d.ngram) ok = ok && c <= 6;
        if (!ok) continue;
        for (size_t end = L; end <= seq; ++end) {
            const size_t widx = seq - end;  // weights[sequence_size - m.end()] (boundary_scorer_cache.rs:42-46)
            if (widx >= d.weights.size()) continue;
            const int32_t wv = d.weights[widx];
            if (wv == 0) continue;
            // fixed digits
            uint64_t fixed = 0;
            for (size_t k = 0; k < L; ++k) fixed |= uint64_t(uint8_t(d.ngram[k])) << (3 * (seq - 1 - (end - L + k)));
            std::vector<size_t> free_pos;
            for (size_t p = 0; p < seq; ++p)
                if (p < end - L || p >= end) free_pos.push_back(p);
            const size_t nf = free_pos.size();
            std::vector<uint32_t> ctr(nf, 0);
            for (;;) {
                uint64_t id = fixed;
                for (size_t k = 0; k < nf; ++k) id |= uint64_t(ctr[k]) << (3 * (seq - 1 - free_pos[k]));
                table[size_t(id)] = wrapping_add(table[size_t(id)], wv);
                size_t k = 0;
                while (k < nf && ++ctr[k] == 7) ctr[k++] = 0;
                if (k == nf) break;
            }
        }
    }
    return table;
}

bool build_type_split(const std::vector<NgramEntry>& type_ngrams, uint8_t window, std::vector<int32_t>& ta,
                      std::vector<int32_t>& tb) {
    if (window != 3) return false;
    for (const auto& d : type_ngrams)
        if (d.ngram.size() > 3) return false;
    const size_t seq = 6, sub = 4;
    ta.assign(size_t(1) << (3 * sub), 0);
    tb.assign(size_t(1) << (3 * sub), 0);
    for (const auto& d : type_ngrams) {
        const size_t L = d.ngram.size();
        bool ok = L > 0;
        for (unsigned char c : d.ngram) ok = ok && c <= 6;
        if (!ok) continue;
        for (size_t end = L; end <= seq; ++end) {  // occurrence covers window positions [end-L, end)
            const size_t widx = seq - end;
            if (widx >= d.weights.size() || d.weights[widx] == 0) continue;
            const int32_t wv = d.weights[widx];
            const bool in_a = end <= sub;                  // entirely inside positions 0..3
            const size_t shift = in_a ? 0 : 2;             // B covers positions 2..5
            std::vector<int32_t>& tab = in_a ? ta : tb;
            const size_t start = end - L - shift;          // position inside the 4-type sub-window
            for (size_t id = 0; id < tab.size(); ++id) {
                bool match = true, valid = true;
                for (size_t p = 0; p < sub; ++p) {
                    const uint32_t dgt = uint32_t(id >> (3 * (sub - 1 - p))) & 7u;
                    if (dgt == 7) { valid = false; break; }
                    if (p >= start && p < start + L && dgt != uint8_t(d.ngram[p - start])) { match = false; break; }
                }
                if (valid && match) tab[id] = wrapping_add(tab[id], wv);
            }
        }
    }
    return true;
}

bool build_type_state3(const PatternSet& tps, std::vector<uint32_t>& table) {
    if (tps.max_len > 3) return false;
    table.assign(512, kNoPattern);
    std::unordered_map<std::string, uint32_t> index;
    for (size_t i = 0; i < tps.raw.size(); ++i) index.emplace(tps.raw[i], uint32_t(i));
    for (uint32_t code = 0; code < 512; ++code) {
        const uint8_t t1 = uint8_t(code >> 6), t2 = uint8_t((code >> 3) & 7), t3 = uint8_t(code & 7);
        if (t3 == 0) continue;
        // longest suffix of (t1 t2 t3) that is a pattern; a zero type ends the context (sentence start)
        std::string s3{char(t1), char(t2), char(t3)}, s2{char(t2), char(t3)}, s1{char(t3)};
        uint32_t pid = kNoPattern;
        if (t1 != 0 && t2 != 0 && index.count(s3)) pid = index[s3];
        else if (t2 != 0 && index.count(s2)) pid = index[s2];
        else if (index.count(s1)) pid = index[s1];
        table[code] = pid;
    }
    return true;
}

uint32_t table_slot(const TableGeom& g, const uint8_t* seeds, uint64_t key) {
    uint32_t ha, hb;
    key_hashes(key, hash_consts(g.salt), ha, hb);
    const uint32_t bk = bucket_of(ha, g.nbuckets);
    const uint32_t seed = g.seed_bits == 16 ? uint32_t(seeds[2 * size_t(bk)]) | (uint32_t(seeds[2 * size_t(bk) + 1]) << 8) : seeds[bk];
    // (an 8-bit kSpillSeed only occurs in a table with a spill table, whose geometry follows from g: keys.hpp)
    if (g.seed_bits != 8 || seed != kSpillSeed) return slot_of_seeds<false>(ha, hb, seed, 0u, g.nslots, 0u, 0u);
    const uint32_t spill_seed = seeds[spill_bucket_of(hb, g.nbuckets, spill_buckets_of(g.nbuckets))];
    return slot_of_seeds<true>(ha, hb, seed, spill_seed, g.nslots, spill_slots_of(g.nslots), spill_mul(g.salt));
}

namespace {

struct TrieNode {
    uint32_t parent;
    uint32_t sym;
    uint32_t depth;
    uint32_t pat = kNoPattern;   // pattern ending exactly here
    uint32_t best = kNoPattern;  // longest pattern that is a suffix of the node string
    bool has_ext = false;
    uint32_t c1 = 0, c2 = 0, c3 = 0;  // shallow key symbols (depth <= 3)
};

// Hash-and-displace: gives every bucket of keys the first seed in [0, n_seeds) for which slot(key, seed) sends all
// its keys to distinct free slots (kSpillSeed is not a placing 8-bit seed).  Buckets are placed largest first.  Returns
// false when a bucket cannot be placed, unless `spilled` is given: then such a bucket keeps kSpillSeed and its keys
// are appended to `spilled`.
template <class SlotF>
bool place_buckets(const std::vector<std::vector<uint32_t>>& buckets, uint32_t n_seeds, SlotF slot, std::vector<uint8_t>& used,
                   std::vector<uint32_t>& seed_of_bucket, std::vector<uint32_t>& slot_of_key, std::vector<uint32_t>* spilled) {
    std::vector<uint32_t> order(buckets.size());
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(),
                     [&](uint32_t a, uint32_t b) { return buckets[a].size() > buckets[b].size(); });
    seed_of_bucket.assign(buckets.size(), 0);
    std::vector<uint32_t> tmp;
    for (uint32_t b : order) {
        const auto& ks = buckets[b];
        if (ks.empty()) break;
        bool placed = false;
        for (uint32_t seed = 0; seed < n_seeds && !placed; ++seed) {
            if (n_seeds == 256 && seed == kSpillSeed) continue;
            tmp.clear();
            bool ok = true;
            for (uint32_t ki : ks) {
                const uint32_t s = slot(ki, seed);
                if (used[s]) { ok = false; break; }
                for (uint32_t s2 : tmp) if (s2 == s) { ok = false; break; }
                if (!ok) break;
                tmp.push_back(s);
            }
            if (ok) {
                for (size_t k = 0; k < ks.size(); ++k) { used[tmp[k]] = 1; slot_of_key[ks[k]] = tmp[k]; }
                seed_of_bucket[b] = seed;
                placed = true;
            }
        }
        if (placed) continue;
        if (!spilled) return false;
        seed_of_bucket[b] = kSpillSeed;
        spilled->insert(spilled->end(), ks.begin(), ks.end());
    }
    return true;
}

// Perfect hash of `keys` with the geometry g (its nslots / nbuckets / salt / seed_bits).  With g.spill (8-bit seeds
// only), the buckets no seed places go to the spill table (keys.hpp: spill_slots_of ...); g.spill is cleared when none
// has to.
bool place_keys(const std::vector<uint64_t>& keys, TableGeom& g, std::vector<uint8_t>& seeds,
                std::vector<uint32_t>& slot_of_key) {
    const size_t n = keys.size();
    std::vector<uint32_t> ha(n), hb(n);
    std::vector<std::vector<uint32_t>> buckets(g.nbuckets);
    const HashK hk = hash_consts(g.salt);
    for (size_t i = 0; i < n; ++i) {
        key_hashes(keys[i], hk, ha[i], hb[i]);
        buckets[bucket_of(ha[i], g.nbuckets)].push_back(uint32_t(i));
    }
    {   // two keys with the same pair of hashes can never be separated by a seed: re-salt
        std::vector<uint64_t> pairs(n);
        for (size_t i = 0; i < n; ++i) pairs[i] = (uint64_t(ha[i]) << 32) | hb[i];
        std::sort(pairs.begin(), pairs.end());
        if (std::adjacent_find(pairs.begin(), pairs.end()) != pairs.end()) return false;
    }
    std::vector<uint8_t> used(g.nslots, 0);
    std::vector<uint32_t> seed_of_bucket, spilled;
    slot_of_key.assign(n, 0);
    const auto primary = [&](uint32_t ki, uint32_t seed) { return slot_of_seeds<false>(ha[ki], hb[ki], seed, 0, g.nslots, 0, 0); };
    if (!place_buckets(buckets, g.seed_bits == 16 ? 65536u : 256u, primary, used, seed_of_bucket, slot_of_key,
                       g.spill ? &spilled : nullptr))
        return false;
    g.spill = !spilled.empty();
    std::vector<uint32_t> spill_seeds;
    if (g.spill) {
        const uint32_t nsb = spill_buckets_of(g.nbuckets), nss = spill_slots_of(g.nslots), mul = spill_mul(g.salt);
        std::vector<std::vector<uint32_t>> sb(nsb);
        for (uint32_t ki : spilled) sb[spill_bucket_of(hb[ki], 0, nsb)].push_back(ki);
        std::vector<uint8_t> sused(nss, 0);
        const auto spill = [&](uint32_t ki, uint32_t seed) {
            return slot_of_seeds<true>(ha[ki], hb[ki], kSpillSeed, seed, g.nslots, nss, mul) - g.nslots;
        };
        std::vector<uint32_t> sk(slot_of_key);
        if (!place_buckets(sb, 256u, spill, sused, spill_seeds, sk, nullptr)) return false;
        for (uint32_t ki : spilled) slot_of_key[ki] = sk[ki] + g.nslots;
    }
    const size_t seed_bytes = g.seed_bits == 16 ? 2 : 1;
    seeds.assign(size_t(g.nbuckets) * seed_bytes + spill_seeds.size(), 0);
    for (size_t b = 0; b < g.nbuckets; ++b) {
        seeds[seed_bytes * b] = uint8_t(seed_of_bucket[b]);
        if (seed_bytes == 2) seeds[2 * b + 1] = uint8_t(seed_of_bucket[b] >> 8);
    }
    for (size_t b = 0; b < spill_seeds.size(); ++b) seeds[g.nbuckets + b] = uint8_t(spill_seeds[b]);
    return true;
}

}  // namespace

NodeTable build_node_table(const PatternSet& ps, bool force_general, uint32_t bucket_cap) {
    NodeTable t;
    if (ps.raw.empty()) return t;
    t.present = true;

    // 1. trie of reversed patterns: a node at depth d is a d-symbol string that is a suffix of some pattern
    std::vector<TrieNode> nodes(1);
    nodes[0] = TrieNode{0, 0, 0};
    std::unordered_map<uint64_t, uint32_t> child;  // (parent << 21 | sym) -> node
    child.reserve(ps.raw.size() * 3);
    for (size_t p = 0; p < ps.syms.size(); ++p) {
        const auto& s = ps.syms[p];
        uint32_t cur = 0;
        for (size_t d = 1; d <= s.size(); ++d) {
            const uint32_t sym = s[s.size() - d];
            if (sym == 0 || sym > 0x10FFFF) { cur = kNoPattern; break; }  // can never match text
            const uint64_t ck = (uint64_t(cur) << 21) | sym;
            auto it = child.find(ck);
            if (it == child.end()) {
                if (nodes.size() >= (1u << 31)) throw Error(kInvalidModel, "InvalidModelError: too many patterns");
                TrieNode nd{cur, sym, uint32_t(d)};
                const TrieNode& par = nodes[cur];
                if (d == 1) { nd.c3 = sym; }
                else if (d == 2) { nd.c3 = par.c3; nd.c2 = sym; }
                else if (d == 3) { nd.c3 = par.c3; nd.c2 = par.c2; nd.c1 = sym; }
                nodes[cur].has_ext = true;
                it = child.emplace(ck, uint32_t(nodes.size())).first;
                nodes.push_back(nd);
            }
            cur = it->second;
        }
        if (cur != kNoPattern && cur != 0) nodes[cur].pat = uint32_t(p);
    }
    for (size_t i = 1; i < nodes.size(); ++i) {
        nodes[i].best = nodes[i].pat != kNoPattern ? nodes[i].pat : nodes[nodes[i].parent].best;
        t.max_depth = std::max(t.max_depth, nodes[i].depth);
    }
    const size_t n = nodes.size() - 1;
    t.n_nodes = uint32_t(nodes.size());
    if (n == 0) { t.present = false; return t; }

    // 2. extent of all rows; inline format if every row fits one window of kInlineWidth positions
    bool any = false;
    for (const auto& r : ps.rows) {
        if (!r.present || r.w.empty()) continue;
        const int lo = r.off, hi = r.off + int(r.w.size());
        if (!any) { t.rel_min = lo; t.rel_max = hi; any = true; }
        else { t.rel_min = std::min(t.rel_min, lo); t.rel_max = std::max(t.rel_max, hi); }
    }
    // Inline format: the window is placed on the rows of the patterns of at most 3 symbols (n-grams, short words),
    // which must all fit; rows of longer patterns (dictionary words) may stick out: their records live at depth >= 4,
    // where the key has room for an overflow flag, and the outside part goes to the overflow pool.
    bool any_short = false;
    int smin = 0, smax = 0;
    for (size_t p = 0; p < ps.rows.size(); ++p) {
        const Row& r = ps.rows[p];
        if (!r.present || r.w.empty() || ps.syms[p].size() > 3) continue;
        const int lo = r.off, hi = r.off + int(r.w.size());
        if (!any_short) { smin = lo; smax = hi; any_short = true; }
        else { smin = std::min(smin, lo); smax = std::max(smax, hi); }
    }
    t.fast = !force_general && (!any_short || smax - smin <= kInlineWidth);
    t.r0 = any_short ? smin : (any ? std::max(t.rel_min, t.rel_max - kInlineWidth) : 0);
    if (t.r0 < -24 || t.r0 > 18) t.fast = false;  // shuffle gather reaches at most one warp left/right
    if (t.fast && any && (t.rel_min < -32000 || t.rel_max > 32000)) t.fast = false;  // overflow offsets are 16-bit
    t.has_overflow = t.fast && any && (t.rel_min < t.r0 || t.rel_max > t.r0 + kInlineWidth);

    // 3. keys and perfect hash
    std::vector<uint64_t> keys(n);
    for (size_t i = 1; i < nodes.size(); ++i) {
        const TrieNode& nd = nodes[i];
        keys[i - 1] = nd.depth <= 3 ? shallow_key(nd.c1, nd.c2, nd.c3) : deep_key(nd.parent, nd.sym);
    }
    std::vector<uint32_t> slot_of_key;
    bool ok = false;
    // load factor 0.6 and 8 keys per bucket on average: 256 seeds per bucket are enough in practice and
    // keep the seed array at one byte per 8 nodes (it is staged in shared memory by the tile kernel);
    // on failure retry with another salt and a sparser table, then with smaller buckets.
    static const double kAlpha[] = {0.60, 0.50, 0.42, 0.35, 0.30, 0.30, 0.25, 0.25, 0.20, 0.15};
    static const double kLambda[] = {8.0, 8.0, 8.0, 8.0, 8.0, 6.0, 6.0, 4.0, 4.0, 3.0};
    // Inline-format tables whose seeds fit the shared-memory budget are built dense: load 0.75 in the primary slots,
    // and the buckets no seed places there go to a small sparse spill table whose seeds share the budget (keys.hpp).
    // A probe is still one seed pair and one record load; the records take about a third less L2 than a sparse
    // table's, and L2 is what the probes are served from (DESIGN.md §4).
    if (t.fast && bucket_cap) {
        // (9 keys per primary bucket leave room in the budget for the spill seeds; config 2: 15 % of the keys spill)
        static const double kDenseLambda[] = {9.0, 9.0, 9.5};
        for (int attempt = 0; attempt < 3 && !ok; ++attempt) {
            t.geom.nslots = uint32_t(std::max<double>(16.0, double(n) / 0.75 + 1.0));
            t.geom.nbuckets = uint32_t(std::max<double>(1.0, double(n) / kDenseLambda[attempt] + 1.0));
            t.geom.salt = 0x3c6ef372fe94f82bULL * uint64_t(attempt + 1);
            t.geom.spill = true;
            if (t.geom.nbuckets + spill_buckets_of(t.geom.nbuckets) <= bucket_cap) ok = place_keys(keys, t.geom, t.seeds, slot_of_key);
        }
        if (!ok) t.geom.spill = false;
    }
    // Tables slightly too large for the kernel's shared seed buffer first try fatter buckets (<= 12 keys) on a
    // sparse table so that the seeds still fit.
    if (!ok && bucket_cap && double(n) / 8.0 + 1.0 > double(bucket_cap) && double(n) / 12.0 < double(bucket_cap)) {
        for (int attempt = 0; attempt < 2 && !ok; ++attempt) {
            t.geom.nslots = uint32_t(double(n) / (attempt ? 0.25 : 0.33) + 1.0);
            t.geom.nbuckets = bucket_cap;
            t.geom.salt = 0x7f4a7c159e3779b9ULL * uint64_t(attempt + 1);
            ok = place_keys(keys, t.geom, t.seeds, slot_of_key);
        }
    }
    // Tables far beyond the shared-memory seed budget are built dense instead (16-bit seeds, load factor 0.85):
    // what matters for them is staying resident in L2.
    if (!ok && bucket_cap && double(n) / 12.0 >= double(bucket_cap)) {
        static const double kDenseAlpha[] = {0.85, 0.80, 0.70};
        for (int attempt = 0; attempt < 3 && !ok; ++attempt) {
            t.geom.seed_bits = 16;
            t.geom.nslots = uint32_t(double(n) / kDenseAlpha[attempt] + 1.0);
            t.geom.nbuckets = uint32_t(double(n) / 5.0 + 1.0);
            t.geom.salt = 0x2545f4914f6cdd1dULL * uint64_t(attempt + 1);
            ok = place_keys(keys, t.geom, t.seeds, slot_of_key);
        }
        if (!ok) t.geom.seed_bits = 8;
    }
    for (int attempt = 0; attempt < 10 && !ok; ++attempt) {
        t.geom.nslots = uint32_t(std::max<double>(16.0, double(n) / kAlpha[attempt] + 1.0));
        t.geom.nbuckets = uint32_t(std::max<double>(1.0, double(n) / kLambda[attempt] + 1.0));
        t.geom.salt = 0x5bd1e9955bd1e995ULL * uint64_t(attempt + 1);
        ok = place_keys(keys, t.geom, t.seeds, slot_of_key);
    }
    if (!ok) throw Error(kInternal, "internal error: perfect hash construction failed");

    // 4. records
    const size_t total_slots = size_t(t.geom.nslots) + (t.geom.spill ? spill_slots_of(t.geom.nslots) : 0u);
    t.records.assign(total_slots * 32, 0);
    t.slot_node.assign(total_slots, 0);
    t.slot_pid.assign(total_slots, kNoPattern);
    std::vector<uint32_t> ovf_ptr;
    if (t.has_overflow) {
        t.slot_ovf.assign(total_slots, 0);
        ovf_ptr.assign(ps.rows.size(), kNoPattern);
        for (const auto& r : ps.rows)
            if (r.w.size() > 65535) throw Error(kInvalidModel, "InvalidModelError: weight row too long");
    }
    std::vector<uint32_t> row_ptr;
    if (!t.fast) {
        row_ptr.assign(ps.rows.size(), kNoPattern);
        for (size_t p = 0; p < ps.rows.size(); ++p) {
            const Row& r = ps.rows[p];
            if (!r.present || r.w.empty()) continue;
            row_ptr[p] = uint32_t(t.pool.size());
            t.pool.insert(t.pool.end(), r.w.begin(), r.w.end());
        }
        if (t.pool.empty()) t.pool.push_back(0);
    }
    // child masks of the 2-symbol nodes (keys.hpp: kChildMaskField)
    std::vector<uint32_t> child_mask(nodes.size(), 0);
    for (size_t i = 1; i < nodes.size(); ++i)
        if (nodes[i].depth == 3) child_mask[nodes[i].parent] |= 1u << child_bit(nodes[i].c1);
    for (size_t i = 1; i < nodes.size(); ++i) {
        const TrieNode& nd = nodes[i];
        const uint32_t slot = slot_of_key[i - 1];
        const uint64_t key = keys[i - 1] | (nd.has_ext ? kExtFlag : 0) | (nd.depth == 2 ? uint64_t(child_mask[i]) << 42 : 0);
        t.slot_node[slot] = uint32_t(i);
        t.slot_pid[slot] = nd.best;
        uint8_t* dst = t.records.data() + size_t(slot) * 32;
        if (t.fast) {
            FastRecord rec{};
            rec.key = key;
            if (nd.best != kNoPattern) {
                const Row& r = ps.rows[nd.best];
                bool outside = false;
                for (size_t k = 0; r.present && k < r.w.size(); ++k) {
                    const int rel = r.off + int(k) - t.r0;
                    if (rel >= 0 && rel < kInlineWidth) rec.w[rel] = r.w[k];
                    else if (r.w[k] != 0) outside = true;
                }
                if (outside) {
                    // only reachable for depth >= 4 (the window covers every pattern of <= 3 symbols)
                    if (nd.depth <= 3) throw Error(kInternal, "internal error: overflow row on a shallow node");
                    if (ovf_ptr[nd.best] == kNoPattern) {
                        ovf_ptr[nd.best] = uint32_t(t.pool.size());
                        for (size_t k = 0; k < r.w.size(); ++k) {
                            const int rel = r.off + int(k) - t.r0;
                            t.pool.push_back((rel >= 0 && rel < kInlineWidth) ? 0 : r.w[k]);
                        }
                    }
                    rec.key |= kOvfFlag;
                    t.slot_ovf[slot] = uint64_t(ovf_ptr[nd.best]) | (uint64_t(uint16_t(int16_t(r.off))) << 32) |
                                       (uint64_t(uint16_t(r.w.size())) << 48);
                }
            }
            memcpy(dst, &rec, 32);
        } else {
            GeneralRecord rec{};
            rec.key = key;
            rec.pid = nd.best;
            rec.row_ptr = kNoPattern;
            rec.node_id = uint32_t(i);
            if (nd.best != kNoPattern && row_ptr[nd.best] != kNoPattern) {
                rec.row_ptr = row_ptr[nd.best];
                rec.off = ps.rows[nd.best].off;
                rec.len = uint32_t(ps.rows[nd.best].w.size());
            }
            memcpy(dst, &rec, 32);
        }
    }
    return t;
}

}  // namespace vpt
