// Host-side construction of the PatternMatchTagger rule table (tag_rules.hpp) from the arrays of vpt_tag_rules_new.
#include <algorithm>
#include <string>
#include <unordered_map>

#include "common.hpp"
#include "tag_rules.hpp"

namespace vpt {

namespace {

// str::from_utf8's rules: no overlong forms, no surrogates, nothing above U+10FFFF
bool valid_utf8(const uint8_t* s, uint64_t n) {
    for (uint64_t i = 0; i < n;) {
        const uint32_t b = s[i];
        if (b < 0x80) { ++i; continue; }
        uint32_t len, lo = 0x80, hi = 0xBF;
        if (b >= 0xC2 && b <= 0xDF) len = 2;
        else if (b >= 0xE0 && b <= 0xEF) { len = 3; if (b == 0xE0) lo = 0xA0; if (b == 0xED) hi = 0x9F; }
        else if (b >= 0xF0 && b <= 0xF4) { len = 4; if (b == 0xF0) lo = 0x90; if (b == 0xF4) hi = 0x8F; }
        else return false;
        if (n - i < len || s[i + 1] < lo || s[i + 1] > hi) return false;
        for (uint32_t k = 2; k < len; ++k)
            if (s[i + k] < 0x80 || s[i + k] > 0xBF) return false;
        i += len;
    }
    return true;
}

Error bad_rule(uint64_t i, const std::string& what) {
    return Error(kInvalidArgument, "InvalidArgumentError: rules: rule " + std::to_string(i) + ": " + what);
}

}  // namespace

TagRulesHost build_tag_rules(uint64_t n_rules, const uint8_t* surfaces, const uint64_t* surface_offsets,
                             const uint64_t* slot_offsets, const uint32_t* slots, const uint8_t* tags, uint64_t tags_len,
                             uint32_t n_tags) {
    if (!surface_offsets || !slot_offsets)
        throw Error(kInvalidArgument, "InvalidArgumentError: rules: surface_offsets and slot_offsets must not be NULL");
    if (n_rules >= (1u << 30)) throw Error(kInvalidArgument, "InvalidArgumentError: rules: too many rules");
    if (surface_offsets[n_rules] && !surfaces)
        throw Error(kInvalidArgument, "InvalidArgumentError: rules: surfaces must not be NULL");
    if (slot_offsets[n_rules] && !slots) throw Error(kInvalidArgument, "InvalidArgumentError: rules: slots must not be NULL");
    if (tags_len && !tags) throw Error(kInvalidArgument, "InvalidArgumentError: rules: tags must not be NULL");
    TagRulesHost t;
    t.n_rules = uint32_t(n_rules);
    uint32_t cap = 16;
    while (cap < 2 * n_rules + 16) cap <<= 1;
    t.mask = cap - 1;
    t.tab.assign(cap, TagTokenEntry{0, 0, 0, 0, 0});
    t.slot_first.push_back(0);
    std::unordered_map<std::string, uint64_t> seen;
    seen.reserve(size_t(n_rules));
    for (uint64_t i = 0; i < n_rules; ++i) {
        const uint64_t s0 = surface_offsets[i], s1 = surface_offsets[i + 1];
        if (s1 < s0) throw bad_rule(i, "surface_offsets must not decrease");
        if (s1 - s0 >= (1u << 28)) throw bad_rule(i, "surface longer than 256 MiB");
        if (!valid_utf8(surfaces + s0, s1 - s0)) throw bad_rule(i, "surface is not valid UTF-8");
        std::string key(reinterpret_cast<const char*>(surfaces) + s0, size_t(s1 - s0));
        if (!seen.emplace(key, i).second) throw bad_rule(i, "duplicate surface (also rule " + std::to_string(seen[key]) + ")");
        const uint64_t q0 = slot_offsets[i], q1 = slot_offsets[i + 1];
        if (q1 < q0) throw bad_rule(i, "slot_offsets must not decrease");
        uint32_t suffix = 0;
        for (uint64_t k = q0; k < q1; ++k) {
            const uint32_t off = slots[2 * k], len = slots[2 * k + 1];
            if (off != kRuleNone) {
                if (uint64_t(off) + len > tags_len) throw bad_rule(i, "tag outside the tag bytes");
                if (!valid_utf8(tags + off, len)) throw bad_rule(i, "tag is not valid UTF-8");
            }
            if (k - q0 >= n_tags) continue;  // slots beyond the predictor's n_tags are never read
            const uint32_t eoff = uint32_t(t.tag_bytes.size());
            if (off != kRuleNone)
                for (uint32_t j = 0; j < len; ++j) {
                    const uint8_t c = tags[off + j];
                    if (c == ' ' || c == '\\' || c == '/') t.tag_bytes.push_back('\\');
                    t.tag_bytes.push_back(c);
                }
            const uint32_t elen = uint32_t(t.tag_bytes.size()) - eoff;
            t.slot_ref.push_back(off == kRuleNone ? kRuleNone : eoff);
            t.slot_ref.push_back(off == kRuleNone ? 0 : elen);
            suffix += 1 + elen;
            if (t.tag_bytes.size() >= kRuleNone) throw bad_rule(i, "the tags take more than 4 GiB");
        }
        t.slot_first.push_back(uint32_t(t.slot_ref.size() / 2));
        t.suffix.push_back(suffix);
        if (key.empty()) continue;  // (never matches: a token has at least one character)
        uint64_t h = kTagHashInit;
        for (unsigned char c : key) h = tag_hash_step(h, c);
        h = tag_hash_finish(h);
        uint32_t s = uint32_t(h >> 20) & t.mask;
        while (t.tab[s].hash != 0) s = (s + 1) & t.mask;
        t.tab[s] = TagTokenEntry{h, uint32_t(i), uint32_t(t.surf.size()), uint32_t(key.size()), 0};
        t.surf.insert(t.surf.end(), key.begin(), key.end());
        if (t.surf.size() >= kRuleNone) throw bad_rule(i, "the surfaces take more than 4 GiB");
        t.max_bytes = std::max<uint32_t>(t.max_bytes, uint32_t(key.size()));
    }
    // (padding: the kernels never read past a key, the copies to the device need no empty vector)
    t.surf.resize(t.surf.size() + 16, 0);
    t.tag_bytes.resize(t.tag_bytes.size() + 16, 0);
    t.slot_ref.push_back(kRuleNone);
    t.slot_ref.push_back(0);
    t.suffix.push_back(0);
    return t;
}

}  // namespace vpt
