// TEST INFRASTRUCTURE: the host side of the PatternMatchTagger rules (vaporetto_b200/csrc/tag_rules.cpp: the table
// builder) and the per-thread code the kernels run (tag_rules.hpp: rule_lookup, merged_suffix_len / _write), compiled
// for the CPU so tests/test_tag_rules_cpu.py can compare them with Python and with the oracle.  Never linked into
// libvaporetto_b200.so.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../vaporetto_b200/csrc/common.hpp"
#include "../../vaporetto_b200/csrc/tag_rules.hpp"

using namespace vpt;

namespace {
struct Rules {
    TagRulesHost h;
    DevTagRules d;
};
}  // namespace

extern "C" {

// the builder's table (nullptr and the message in err on an error)
void* tr_new(uint64_t n_rules, const uint8_t* surfaces, const uint64_t* surface_offsets, const uint64_t* slot_offsets,
             const uint32_t* slots, const uint8_t* tags, uint64_t tags_len, uint32_t n_tags, char* err, size_t err_cap) {
    try {
        Rules* r = new Rules();
        r->h = build_tag_rules(n_rules, surfaces, surface_offsets, slot_offsets, slots, tags, tags_len, n_tags);
        r->d.tab = r->h.tab.data();
        r->d.surf = r->h.surf.data();
        r->d.slot_first = r->h.slot_first.data();
        r->d.slot_ref = reinterpret_cast<const uint2*>(r->h.slot_ref.data());
        r->d.tag_bytes = r->h.tag_bytes.data();
        r->d.suffix = r->h.suffix.data();
        r->d.mask = r->h.mask;
        r->d.max_bytes = r->h.max_bytes;
        return r;
    } catch (const Error& e) {
        snprintf(err, err_cap, "%d %s", e.code, e.what());
        return nullptr;
    }
}

void tr_free(void* r) { delete static_cast<Rules*>(r); }

uint32_t tr_capacity(const void* r) { return static_cast<const Rules*>(r)->h.mask + 1; }

int32_t tr_find(const void* r, const uint8_t* bytes, uint32_t len, int norm) {
    return rule_lookup(static_cast<const Rules*>(r)->d, bytes, len, norm);
}

// The "/tag/.." suffix the writer gives a token `bytes` whose model tags are model_ref[2k] (offset into model_bytes,
// or UINT32_MAX for no candidate), model_ref[2k + 1] (length); model_ref == nullptr: the token has no tag model.
// Returns the suffix length (the length pass), -1 when the write pass wrote a different number of bytes.
long tr_suffix(const void* rp, uint32_t n_tags, const uint8_t* bytes, uint32_t len, int norm, const uint32_t* model_ref,
               const uint8_t* model_bytes, uint8_t* out, size_t cap) {
    const Rules* r = static_cast<const Rules*>(rp);
    // the model's tag tables for one token id with one (escaped) candidate per slot
    std::vector<uint32_t> ts_slot{0}, ts_cand, ts_ref;
    std::vector<uint8_t> ts_bytes, cands(n_tags, 255);
    for (uint32_t k = 0; k < n_tags; ++k) {
        ts_cand.push_back(k);
        const uint32_t off = uint32_t(ts_bytes.size());
        if (model_ref && model_ref[2 * k] != kRuleNone) {
            cands[k] = 0;
            for (uint32_t j = 0; j < model_ref[2 * k + 1]; ++j) {
                const uint8_t c = model_bytes[model_ref[2 * k] + j];
                if (c == ' ' || c == '\\' || c == '/') ts_bytes.push_back('\\');
                ts_bytes.push_back(c);
            }
        }
        ts_ref.push_back(off);
        ts_ref.push_back(uint32_t(ts_bytes.size()) - off);
    }
    ts_bytes.push_back(0);
    const int32_t tid = model_ref ? 0 : -1;
    const int32_t rid = rule_lookup(r->d, bytes, len, norm);
    const uint2* ref = reinterpret_cast<const uint2*>(ts_ref.data());
    const uint32_t n = merged_suffix_len(n_tags, tid, cands.data(), ts_slot.data(), ts_cand.data(), ref, rid, r->d);
    if (n > cap) return long(n);
    std::vector<uint8_t> buf(n + 64, 0xEE);
    merged_suffix_write(n_tags, tid, cands.data(), ts_slot.data(), ts_cand.data(), ref, ts_bytes.data(), rid, r->d, buf.data());
    for (size_t i = n; i < buf.size(); ++i)
        if (buf[i] != 0xEE) return -1;
    memcpy(out, buf.data(), n);
    return long(n);
}

}  // extern "C"
