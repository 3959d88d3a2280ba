// CPU oracle of the tag candidate scores of vpt_predict_batch_compact_tag_scores and vpt_token_spans_tag_scores: the
// `raw_scores` the oracle's Predictor::fill_tags computes (the `scores` the reference's predict_tags stores with
// store_tag_scores, predictor.rs:599-601 / :632-634), laid out per token record.  The oracle is compiled in unchanged
// through spans_oracle.cpp.  Test infrastructure only: tests/vpt_testlib/tag_scores_oracle.py builds and loads it.
#include "spans_oracle.cpp"

namespace ora_scores {

// Appends the records of one tagged sentence: every token (boundaries == 1 split) in text order, its token id and, when
// the id is >= 0, the score vector of its last character.
static void append_records(const ora::Sentence& s, const vector<int32_t>& tt, const vector<vector<int32_t>>& raw,
                           vector<int32_t>& ids, vector<int32_t>& scores) {
    const size_t n = s.len();
    for (size_t i = 0; i < n; ++i) {
        if (i + 1 < n && s.boundaries[i] != 1) continue;
        ids.push_back(tt[i]);
        if (tt[i] >= 0) scores.insert(scores.end(), raw[i].begin(), raw[i].end());
    }
}

static int copy_out(const vector<int32_t>& ids, const vector<int32_t>& scores, int32_t* ids_out, size_t id_cap,
                    int32_t* scores_out, size_t score_cap, uint64_t* n_records, uint64_t* n_scores) {
    *n_records = ids.size();
    *n_scores = scores.size();
    if (ids.size() > id_cap || scores.size() > score_cap) return 2;
    std::copy(ids.begin(), ids.end(), ids_out);
    std::copy(scores.begin(), scores.end(), scores_out);
    return 0;
}

}  // namespace ora_scores

extern "C" {

// The compact chain: every sentence of the batch predicted and tagged on its raw text; empty, NUL and invalid UTF-8
// sentences have no tokens.  Returns 0, or 2 with the totals set when a capacity is too small.
int ora_compact_tag_scores(const void* p, const char* utf8, const uint64_t* offsets, size_t n_sent, int32_t* ids_out,
                           size_t id_cap, int32_t* scores_out, size_t score_cap, uint64_t* n_records, uint64_t* n_scores) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    vector<int32_t> ids, scores, tt, ti;
    vector<vector<int32_t>> raw;
    Sentence s;
    for (size_t d = 0; d < n_sent; ++d) {
        const string text(utf8 + offsets[d], size_t(offsets[d + 1] - offsets[d]));
        if (text.empty() || !valid_utf8(text) || text.find('\0') != string::npos) continue;
        s.parse_raw(text.data(), text.size());
        pr->predict(s);
        pr->fill_tags(s, tt, ti, &raw);
        ora_scores::append_records(s, tt, raw, ids, scores);
    }
    return ora_scores::copy_out(ids, scores, ids_out, id_cap, scores_out, score_cap, n_records, n_scores);
    ORA_CATCH(idret)
}

// The spans chain (ora_token_spans): pre-filter unless no_norm, predict, line-break split, the wsconst post-filters,
// then the tags and scores of that sentence.  Returns as ora_compact_tag_scores.
int ora_spans_tag_scores(const void* p, const char* utf8, const uint64_t* offsets, size_t n_docs, int no_norm,
                         uint32_t wsconst_types, int32_t* ids_out, size_t id_cap, int32_t* scores_out, size_t score_cap,
                         uint64_t* n_records, uint64_t* n_scores) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    vector<int32_t> ids, scores, tt, ti;
    vector<vector<int32_t>> raw;
    Sentence s, s_orig;
    for (size_t d = 0; d < n_docs; ++d) {
        const string text(utf8 + offsets[d], size_t(offsets[d + 1] - offsets[d]));
        if (text.empty() || !valid_utf8(text) || text.find('\0') != string::npos) continue;
        s_orig.parse_raw(text.data(), text.size());
        Sentence* sp = &s_orig;
        if (!no_norm) {
            string pre;
            for (uint32_t c : s_orig.chars) append_utf8(pre, kytea_fullwidth_cp(c));
            s.parse_raw(pre.data(), pre.size());
            sp = &s;
        }
        pr->predict(*sp);
        ora_spans::split_linebreaks(*sp);
        for (uint8_t ty = 1; ty <= 6; ++ty) if (wsconst_types & (1u << ty)) wsconst_filter(*sp, ty);
        if (wsconst_types & 0x80u) grapheme_filter(*sp);
        pr->fill_tags(*sp, tt, ti, &raw);
        ora_scores::append_records(*sp, tt, raw, ids, scores);
    }
    return ora_scores::copy_out(ids, scores, ids_out, id_cap, scores_out, score_cap, n_records, n_scores);
    ORA_CATCH(idret)
}

}  // extern "C"
