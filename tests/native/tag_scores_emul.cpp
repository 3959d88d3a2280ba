// TEST INFRASTRUCTURE: the tag kernels' own score code (csrc/tags_token.hpp: tag_score_count, which k_tok_lookup writes
// per record, and tag_score_token<true>, which k_tok_score runs) compiled for the host and run over the flat tag tables
// tags_build.cpp makes, one token record at a time as the per-token path walks them.  Linked with host_emul.cpp (its
// emul_predict gives the pattern-id states).  Not part of the product.
#include <cstdint>
#include <string>
#include <vector>

#include "../../vaporetto_b200/csrc/common.hpp"
#include "../../vaporetto_b200/csrc/predictor_build.hpp"
#include "../../vaporetto_b200/csrc/tags.hpp"
#include "../../vaporetto_b200/csrc/tags_token.hpp"

using namespace vpt;

namespace {
std::string g_error;
}

extern "C" {

// Token records of one sentence with final boundaries (n_chars - 1 bytes, 1 = boundary) and its pattern-id states:
// ids_out[r] = the token id the kernels report (-1: unknown, beyond the device limits or malformed), and the score
// vectors of the records with an id >= 0 concatenated in scores_out (score_cap entries; *n_scores = the total).  Returns
// the number of records, or -(status).  Checks that the count k_tok_lookup writes agrees with what k_tok_score stores.
long emul_tag_scores(const uint8_t* model, size_t model_len, const uint8_t* utf8, size_t nbytes, const uint8_t* boundaries,
                     const uint32_t* cstates, const uint32_t* tstates, int norm, int32_t* ids_out, int32_t* scores_out,
                     int32_t* unserved, size_t score_cap, uint64_t* n_scores) {
    try {
        size_t consumed = 0;
        Model m = Model::read(model, model_len, &consumed);
        HostPredictor hp = build_host_predictor(m, true);
        const TagTablesHost t = build_tag_tables(hp);
        if (!t.usable) throw Error(kInternal, "tag tables not usable");
        DevTags d;  // the same fields capi.cpp fills, pointing at the host tables
        d.tok_tab = t.tok_tab.data();
        d.tok_bytes = t.tok_bytes.data();
        d.tok_info = t.tok_info.data();
        d.pool = t.pool.data();
        d.keys = t.keys.data();
        d.c_chain = t.c_chain.data();
        d.t_chain = t.t_chain.data();
        d.c_link = t.c_link.data();
        d.t_link = t.t_link.data();
        d.tok_mask = t.tok_mask;
        d.n_tags = t.n_tags;
        d.char_rels = hp.char_tags ? t.char_rels : 0;
        d.type_rels = hp.type_tags ? t.type_rels : 0;
        d.max_token_bytes = t.max_token_bytes;
        d.n_char_patterns = uint32_t(hp.char_suffix_link.size());
        d.n_type_patterns = uint32_t(hp.type_suffix_link.size());
        std::vector<uint32_t> start;
        for (size_t i = 0; i < nbytes; ++i) if ((utf8[i] & 0xC0) != 0x80) start.push_back(uint32_t(i));
        const size_t n = start.size();
        start.push_back(uint32_t(nbytes));
        uint32_t uns = 0;
        uint64_t total = 0;
        long rec = 0;
        size_t tok_start = 0;
        for (size_t i = 0; i < n; ++i) {
            if (!(i + 1 == n || boundaries[i] == 1)) continue;
            int32_t tok = -1;
            uint32_t tid = 0;
            const uint8_t* bytes = utf8 + start[tok_start];
            const uint32_t len = start[i + 1] - start[tok_start];
            tok_start = i + 1;
            // k_tok_lookup
            uint32_t count = 0;
            if (token_lookup(d, bytes, len, norm, tid)) {
                if (d.tok_info[tid].usable) count = tag_score_count(d.tok_info[tid], d.n_tags);
                // k_tok_score, the record's vector at the running offset
                int32_t cand[kTagMaxSlots];
                int32_t vec[kTagMaxScores];
                tok = tag_score_token<true>(d, tid, d.char_rels ? cstates : nullptr, d.type_rels ? tstates : nullptr,
                                            uint32_t(i), uint32_t(n), cand, &uns, vec);
                if ((tok >= 0) != (count > 0 || d.tok_info[tid].bias_len == 0))
                    throw Error(kInternal, "the score count disagrees with the token id");
                if (tok >= 0) {
                    for (uint32_t k = 0; k < count; ++k)
                        if (total + k < score_cap) scores_out[total + k] = vec[k];
                    total += count;
                }
            }
            ids_out[rec++] = tok;
        }
        if (unserved) *unserved = int32_t(uns);
        *n_scores = total;
        return rec;
    } catch (const Error& e) {
        g_error = e.what();
        return -long(e.code);
    }
}

const char* emul_tag_scores_error() { return g_error.c_str(); }

}
