// Host-side construction of the flat tag-prediction tables (tags.hpp) from a HostPredictor.
#include <algorithm>
#include <cstring>
#include <string>

#include "common.hpp"
#include "tags.hpp"

namespace vpt {

namespace {

uint32_t pow2_at_least(size_t n) {
    uint32_t c = 16;
    while (c < n) c <<= 1;
    return c;
}

// suffix-chain depth of every pattern (1 = no suffix pattern): along a chain the depth falls by one per link
std::vector<uint32_t> chain_depths(const std::vector<uint32_t>& link) {
    std::vector<uint32_t> depth(link.size(), 0);
    std::vector<uint32_t> path;
    for (uint32_t p = 0; p < link.size(); ++p) {
        if (depth[p]) continue;
        path.clear();
        uint32_t q = p;
        while (q != kNoPattern && q < link.size() && depth[q] == 0 && path.size() <= link.size()) { path.push_back(q); q = link[q]; }
        uint32_t d = (q != kNoPattern && q < link.size()) ? depth[q] : 0;
        for (size_t i = path.size(); i-- > 0;) depth[path[i]] = ++d;
    }
    return depth;
}

std::vector<TagChain> chain_table(const std::vector<uint32_t>& link) {
    std::vector<TagChain> t(link.size());
    for (uint32_t p = 0; p < link.size(); ++p) {
        uint32_t q = p;
        for (int k = 0; k < 4; ++k) {
            q = (q != kNoPattern && q < link.size()) ? link[q] : kNoPattern;
            t[p].next[k] = q;
        }
    }
    return t;
}

// the entries of token `tid` of one scorer, sorted by (rel, chain depth descending)
void append_keys(const TagWeightMap& tw, size_t tid, const std::vector<uint32_t>& depth, std::vector<TagKey>& keys,
                 std::vector<int32_t>& pool, uint32_t& rels) {
    if (tid >= tw.size()) return;
    const size_t first = keys.size();
    rels = std::max<uint32_t>(rels, uint32_t(tw[tid].size()));
    for (size_t rel = 0; rel < tw[tid].size(); ++rel)
        for (const auto& kv : tw[tid][rel]) {
            TagKey k;
            k.pid = kv.first;
            k.off = uint32_t(pool.size());
            k.len = uint32_t(kv.second.size());
            k.rel = uint32_t(rel);
            pool.insert(pool.end(), kv.second.begin(), kv.second.end());
            keys.push_back(k);
        }
    std::sort(keys.begin() + first, keys.end(), [&](const TagKey& a, const TagKey& b) {
        if (a.rel != b.rel) return a.rel < b.rel;
        const uint32_t da = a.pid < depth.size() ? depth[a.pid] : 0, db = b.pid < depth.size() ? depth[b.pid] : 0;
        if (da != db) return da > db;
        return a.pid < b.pid;
    });
}

}  // namespace

TagTablesHost build_tag_tables(const HostPredictor& hp) {
    TagTablesHost t;
    t.n_tags = uint32_t(hp.n_tags);
    t.n_tokens = uint32_t(hp.tag_preds.size());
    if (!hp.predict_tags || hp.n_tags == 0 || hp.n_tags > size_t(kTagMaxSlots) || hp.tag_preds.size() >= (1u << 24)) return t;
    t.pool.push_back(0);  // offset 0 is never a real vector (keeps "off" non-zero for debugging)
    // token info + bias
    t.tok_info.resize(hp.tag_preds.size());
    for (size_t i = 0; i < hp.tag_preds.size(); ++i) {
        const TagPredictorHost& tp = hp.tag_preds[i];
        TagTokenInfo& ti = t.tok_info[i];
        memset(&ti, 0, sizeof ti);
        ti.usable = tp.bias.size() <= size_t(kTagMaxScores) && tp.tags.size() <= size_t(kTagMaxSlots);
        ti.bias_off = uint32_t(t.pool.size());
        ti.bias_len = uint16_t(std::min<size_t>(tp.bias.size(), 65535));
        ti.n_slots = uint8_t(std::min<size_t>(tp.tags.size(), size_t(kTagMaxSlots)));
        for (size_t k = 0; k < size_t(kTagMaxSlots); ++k) {
            const size_t nc = k < tp.tags.size() ? tp.tags[k].size() : 0;
            ti.cand[k] = uint8_t(std::min<size_t>(nc, 255));
            if (nc >= 255) ti.usable = 0;
        }
        t.pool.insert(t.pool.end(), tp.bias.begin(), tp.bias.end());
    }
    // tag strings, escaped
    for (size_t i = 0; i < hp.tag_preds.size(); ++i) {
        const TagPredictorHost& tp = hp.tag_preds[i];
        t.ts_slot.push_back(uint32_t(t.ts_cand.size()));
        uint32_t suffix = 0;
        for (size_t k = 0; k < tp.tags.size(); ++k) {
            t.ts_cand.push_back(uint32_t(t.ts_ref.size() / 2));
            uint32_t longest = 0;
            for (const std::string& tag : tp.tags[k]) {
                const uint32_t off = uint32_t(t.ts_bytes.size());
                for (unsigned char c : tag) {
                    if (c == ' ' || c == '\\' || c == '/') t.ts_bytes.push_back('\\');
                    t.ts_bytes.push_back(c);
                }
                const uint32_t len = uint32_t(t.ts_bytes.size()) - off;
                t.ts_ref.push_back(off);
                t.ts_ref.push_back(len);
                longest = std::max(longest, len);
            }
            suffix += 1 + longest;
        }
        t.max_suffix = std::max(t.max_suffix, suffix);
    }
    t.ts_slot.push_back(uint32_t(t.ts_cand.size()));
    t.ts_cand.push_back(uint32_t(t.ts_ref.size() / 2));
    t.ts_ref.push_back(0); t.ts_ref.push_back(0);
    t.ts_bytes.resize(t.ts_bytes.size() + 16, 0);
    // token table (the map already holds "last insert wins" for duplicate tokens)
    const uint32_t cap = pow2_at_least(2 * hp.token_ids.size() + 16);
    t.tok_mask = cap - 1;
    t.tok_tab.assign(cap, TagTokenEntry{0, 0, 0, 0, 0});
    for (const auto& kv : hp.token_ids) {
        uint64_t h = kTagHashInit;
        for (unsigned char c : kv.first) h = tag_hash_step(h, c);
        h = tag_hash_finish(h);
        uint32_t s = uint32_t(h >> 20) & t.tok_mask;
        while (t.tok_tab[s].hash != 0) s = (s + 1) & t.tok_mask;
        t.tok_tab[s].hash = h;
        t.tok_tab[s].tid = kv.second;
        t.tok_tab[s].str_off = uint32_t(t.tok_bytes.size());
        t.tok_tab[s].len = uint32_t(kv.first.size());
        t.tok_bytes.insert(t.tok_bytes.end(), kv.first.begin(), kv.first.end());
        t.max_token_bytes = std::max<uint32_t>(t.max_token_bytes, uint32_t(kv.first.size()));
    }
    t.tok_bytes.resize(t.tok_bytes.size() + 16, 0);
    t.c_link = hp.char_suffix_link;
    t.t_link = hp.type_suffix_link;
    // key lists: per token, the char scorer's own (pattern, rel) vectors, then the type scorer's
    const std::vector<uint32_t> c_depth = chain_depths(t.c_link), t_depth = chain_depths(t.t_link);
    for (size_t i = 0; i < hp.tag_preds.size(); ++i) {
        TagTokenInfo& ti = t.tok_info[i];
        ti.key_off = uint32_t(t.keys.size());
        size_t before = t.keys.size();
        if (hp.char_tags) append_keys(hp.char_tag_weight, i, c_depth, t.keys, t.pool, t.char_rels);
        const size_t nc = t.keys.size() - before;
        before = t.keys.size();
        if (hp.type_tags) append_keys(hp.type_tag_weight, i, t_depth, t.keys, t.pool, t.type_rels);
        const size_t ntk = t.keys.size() - before;
        // per-rel counts (the lists are sorted by rel): rel 0 .. 3 in bytes, the rest (wider windows) as one count
        size_t ccnt[5] = {0, 0, 0, 0, 0}, tcnt[5] = {0, 0, 0, 0, 0};
        for (size_t j = 0; j < nc; ++j) ++ccnt[std::min<uint32_t>(t.keys[ti.key_off + j].rel, 4)];
        for (size_t j = 0; j < ntk; ++j) ++tcnt[std::min<uint32_t>(t.keys[ti.key_off + nc + j].rel, 4)];
        for (int r = 0; r < 4; ++r) {
            if (ccnt[r] > 255 || tcnt[r] > 255) ti.usable = 0;
            ti.ckeys[r] = uint8_t(std::min<size_t>(ccnt[r], 255));
            ti.tkeys[r] = uint8_t(std::min<size_t>(tcnt[r], 255));
        }
        if (ccnt[4] > 65535 || tcnt[4] > 65535) ti.usable = 0;
        ti.c_rest = uint16_t(std::min<size_t>(ccnt[4], 65535));
        ti.t_rest = uint16_t(std::min<size_t>(tcnt[4], 65535));
    }
    if (t.keys.empty()) t.keys.push_back(TagKey{kNoPattern, 0, 0, 0});
    t.c_chain = chain_table(t.c_link);
    t.t_chain = chain_table(t.t_link);
    if (t.c_link.empty()) { t.c_link.push_back(kNoPattern); t.c_chain.push_back(TagChain{{kNoPattern, kNoPattern, kNoPattern, kNoPattern}}); }
    if (t.t_link.empty()) { t.t_link.push_back(kNoPattern); t.t_chain.push_back(TagChain{{kNoPattern, kNoPattern, kNoPattern, kNoPattern}}); }
    t.usable = t.keys.size() < (1ull << 32) && t.pool.size() < (1ull << 32);
    t.all_tokens_usable = std::all_of(t.tok_info.begin(), t.tok_info.end(), [](const TagTokenInfo& ti) { return ti.usable != 0; });
    return t;
}

}  // namespace vpt
