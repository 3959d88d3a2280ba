// CPU oracle of vpt_token_spans: vaporetto_tantivy's token_stream (vaporetto_tantivy/src/lib.rs:157-199) restated over
// the oracle's Sentence / Predictor (oracle/vaporetto_oracle.cpp, compiled into this library unchanged) with its own
// restatement of SplitLinebreaksFilter (vaporetto_rules/src/sentence_filters/split_linebreaks.rs:9-37) and of
// `boundary_pos` (lib.rs:179-188).  Test infrastructure only: tests/vpt_testlib/spans_oracle.py builds and loads it.
#include "../../oracle/vaporetto_oracle.cpp"

namespace ora_spans {

// SplitLinebreaksFilter::filter: for every pair of neighbouring characters (prev_c, c) at boundary i, a '\r' or '\n' on
// either side makes the boundary WordBoundary
static void split_linebreaks(ora::Sentence& s) {
    for (size_t i = 0; i + 1 < s.chars.size(); ++i) {
        const uint32_t prev_c = s.chars[i], c = s.chars[i + 1];
        if (prev_c == '\r' || prev_c == '\n' || c == '\r' || c == '\n') s.boundaries[i] = 1;
    }
}

}  // namespace ora_spans

extern "C" {

// token_stream for every document of a batch: pre-filter (unless no_norm), predict, split_linebreaks, the wsconst
// post-filters (bit t: KyteaWsConstFilter for type t; bit 7: ConcatGraphemeClustersFilter), with fill_tags the tags of
// the filtered sentence, then boundary_pos on the original text.  Outputs as vpt_token_spans; status 1 / 2 / 3 for an
// empty / NUL / invalid UTF-8 document (invalid UTF-8 first).  Returns 0, or 2 with *total set when `cap` is too small.
int ora_token_spans(const void* p, const char* utf8, const uint64_t* offsets, size_t n_docs, int no_norm,
                    uint32_t wsconst_types, int fill_tags, uint32_t* n_tokens, uint8_t* status, uint32_t* ends,
                    int32_t* tok_ids, uint8_t* tok_cands, size_t cap, uint64_t* total) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    const size_t nt = pr->n_tags;
    uint64_t t = 0;
    Sentence s, s_orig;
    vector<int32_t> tt, ti;
    for (size_t d = 0; d < n_docs; ++d) {
        const char* doc = utf8 + offsets[d];
        const size_t len = size_t(offsets[d + 1] - offsets[d]);
        n_tokens[d] = 0;
        const string text(doc, len);
        if (!valid_utf8(text)) { status[d] = 3; continue; }
        if (text.find('\0') != string::npos) { status[d] = 2; continue; }
        if (len == 0) { status[d] = 1; continue; }
        status[d] = 0;
        s_orig.parse_raw(doc, len);
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
        if (fill_tags) pr->fill_tags(*sp, tt, ti, nullptr);
        // boundary_pos: the byte position (in the original text) of every character after a WordBoundary, then the length
        vector<uint32_t> pos;
        for (size_t i = 0; i < sp->boundaries.size(); ++i)
            if (sp->boundaries[i] == 1) pos.push_back(s_orig.char_to_str_pos[i + 1]);
        pos.push_back(uint32_t(len));
        size_t last = 0;  // index of the token's last character
        for (size_t r = 0; r < pos.size(); ++r) {
            if (t + r < cap) {
                ends[t + r] = pos[r];
                last = r + 1 < pos.size() ? s_orig.str_to_char_pos[pos[r]] - 1 : s_orig.len() - 1;
                if (fill_tags) {
                    tok_ids[t + r] = tt[last];
                    for (size_t k = 0; k < nt; ++k) {
                        const int32_t ci = ti[last * nt + k];
                        tok_cands[(t + r) * nt + k] = tt[last] >= 0 && ci >= 0 ? uint8_t(ci) : uint8_t(255);
                    }
                }
            }
        }
        n_tokens[d] = uint32_t(pos.size());
        t += pos.size();
    }
    *total = t;
    return t > cap ? 2 : 0;
    ORA_CATCH(idret)
}

}  // extern "C"
