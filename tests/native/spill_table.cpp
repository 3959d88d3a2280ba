// TEST INFRASTRUCTURE: the char node table the product's host builder (vaporetto_b200/csrc/predictor_build.cpp) makes
// for a model, read back through the product's own probe rule (builder.cpp: table_slot), for tests/test_spill_table.py.
// Not part of the product; never linked into libvaporetto_b200.so.
#include <cstdint>
#include <cstring>

#include "../../vaporetto_b200/csrc/common.hpp"
#include "../../vaporetto_b200/csrc/predictor_build.hpp"

using namespace vpt;

extern "C" {

// out = {nodes, seed_bits, nslots, nbuckets, spill_slots, spill_buckets, records in spill slots}, and the symbols
// (c1, c2, c3; 0 = absent) of up to `cap` nodes of at most 3 symbols whose records sit in spill slots, found by
// probing for them.  Returns how many such nodes were written, or -(status).
long spill_char_table(const uint8_t* model, size_t model_len, uint64_t* out, uint32_t* syms, size_t cap) {
    try {
        size_t consumed = 0;
        Model m = Model::read(model, model_len, &consumed);
        HostPredictor hp = build_host_predictor(m, false);
        const BlobTable& t = hp.hdr.ct;
        const uint8_t* base = hp.blob.data();
        TableGeom g;
        g.nslots = t.nslots;
        g.nbuckets = t.nbuckets;
        g.salt = t.salt;
        g.seed_bits = t.seed_bits;
        auto key_at = [&](uint32_t slot) {
            uint64_t k;
            memcpy(&k, base + t.rec_off + size_t(slot) * 32, 8);
            return k;
        };
        uint64_t spilled = 0;
        size_t found = 0;
        for (uint32_t s = t.nslots; s < t.nslots + t.spill_slots; ++s) {
            const uint64_t key = key_at(s);
            if (key == 0) continue;
            ++spilled;
            if ((key >> 42 & 0x1FFFFFu) >= kDeepMarker) continue;  // (parent node, symbol) key of a deeper node
            const uint32_t c3 = uint32_t(key) & 0x1FFFFFu, c2 = uint32_t(key >> 21) & 0x1FFFFFu, c1 = uint32_t(key >> 42) & 0x1FFFFFu;
            const uint32_t cand[3][3] = {{c1, c2, c3}, {0, c2, c3}, {0, 0, c3}};
            for (const auto& c : cand) {
                // (the key of a 2-symbol record carries its child mask in the c1 field: match it the way the kernels do)
                const uint64_t want = shallow_key(c[0], c[1], c[2]);
                const uint64_t mask = c[0] ? kExtFlag : (kExtFlag | kChildMaskField);
                if (found < cap && table_slot(g, base + t.seeds_off, want) == s && (key & ~mask) == want) {
                    memcpy(syms + 3 * found++, c, sizeof c);
                    break;
                }
            }
        }
        const uint64_t v[7] = {t.n_nodes - 1u, t.seed_bits, t.nslots, t.nbuckets, t.spill_slots, t.spill_buckets, spilled};
        memcpy(out, v, sizeof v);
        return long(found);
    } catch (const Error& e) {
        return -long(e.code);
    }
}

}
