// CPU oracle of vpt_tokenize_dev: the tokenized text of every document of a batch, restated over the oracle's Sentence /
// Predictor (oracle/vaporetto_oracle.cpp, compiled into this library unchanged).  Per document: Sentence::from_raw of the
// whole document ('\r' and '\n' are ordinary characters), KyteaFullwidthFilter (unless no_norm), predict, the wsconst
// post-filters, fill_tags, then write_tokenized_text of the original document with the predicted boundaries and tags.
// PatternMatchTagger is applied on top by tests/vpt_testlib/tokenize_doc_oracle.py.  Test infrastructure only.
#include "../../oracle/vaporetto_oracle.cpp"

extern "C" {

// Writes the documents' strings back to back into buf (capacity cap) and their offsets into out_offsets [n_docs + 1];
// status 1 / 2 / 3 for an empty / NUL / invalid UTF-8 document (invalid UTF-8 first), whose string is empty.  Returns 0,
// or 2 when `cap` is too small (the offsets are then complete, nothing is written past cap).
int ora_tokenize_docs(const void* p, const char* utf8, const uint64_t* offsets, size_t n_docs, int no_norm,
                      uint32_t wsconst_types, int predict_tags, uint64_t* out_offsets, uint8_t* status, char* buf,
                      size_t cap) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    Sentence s, s_orig;
    vector<int32_t> tt, ti;
    uint64_t at = 0;
    out_offsets[0] = 0;
    for (size_t d = 0; d < n_docs; ++d) {
        const char* doc = utf8 + offsets[d];
        const size_t len = size_t(offsets[d + 1] - offsets[d]);
        const string text(doc, len);
        string out;
        if (!valid_utf8(text)) status[d] = 3;
        else if (text.find('\0') != string::npos) status[d] = 2;
        else if (len == 0) status[d] = 1;
        else {
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
            for (uint8_t ty = 1; ty <= 6; ++ty) if (wsconst_types & (1u << ty)) wsconst_filter(*sp, ty);
            if (wsconst_types & 0x80u) grapheme_filter(*sp);
            if (predict_tags) pr->fill_tags(*sp, tt, ti, nullptr);
            if (sp != &s_orig) s_orig.boundaries = sp->boundaries;
            out = write_tokenized(*pr, s_orig, predict_tags ? &tt : nullptr, predict_tags ? &ti : nullptr);
        }
        if (at + out.size() <= cap) memcpy(buf + at, out.data(), out.size());
        at += out.size();
        out_offsets[d + 1] = at;
    }
    return at > cap ? 2 : 0;
    ORA_CATCH(idret)
}

}  // extern "C"
