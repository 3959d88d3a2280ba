// CPU oracle of vpt_reannotate_lines: the chain the C header defines, composed from the restatements of
// partial_oracle.cpp (parse_partial_annotation, which keeps every character's tag fields) and annotate_oracle.cpp
// (write_partial_annotation_text, TokenIterator, the rules blob), over the oracle's Sentence / Predictor
// (oracle/vaporetto_oracle.cpp, compiled into this library unchanged).  Test infrastructure only:
// tests/vpt_testlib/reannotate_oracle.py builds and loads it.
//
// Both restatements include the oracle; #import includes it once and marks it once-only, so their own includes of it
// are skipped (a GCC extension: the oracle has no include guard of its own).
#import "../../oracle/vaporetto_oracle.cpp"
#include "partial_oracle.cpp"
#include "annotate_oracle.cpp"

extern "C" {

// The chain of vpt_reannotate_lines over a buffer (lines split as ora_tokenize_lines splits them); `rules_blob` as in
// ora_annotate_lines.  Returns 0, 2 (InvalidArgument) or 5 (IOError) with the message in ora_last_error() and the bad
// line in *err_line (as ora_partial_lines), or 99 when the output exceeds cap (*out_len holds its size); `buf` receives
// the output of the lines before an error.
int ora_reannotate_lines(const void* p, const char* utf8, size_t nbytes, int no_norm, uint32_t wsconst_types,
                         int predict_tags, int32_t margin, int keep_tags, const uint8_t* rules_blob, char* buf,
                         size_t cap, uint64_t* out_len, uint64_t* n_lines, uint64_t* err_line) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    const ora_ann::Rules rules = ora_ann::read_rules(rules_blob);
    string out;
    uint64_t nl = 0;
    size_t lo = 0;
    Sentence s, s_orig;
    vector<int32_t> tt, ti;
    int rc = 0;
    while (lo < nbytes) {
        const void* q = memchr(utf8 + lo, '\n', nbytes - lo);
        size_t end = q ? size_t(static_cast<const char*>(q) - utf8) : nbytes;
        const size_t next = q ? end + 1 : nbytes;
        if (q && end > lo && utf8[end - 1] == '\r') --end;
        const string line(utf8 + lo, end - lo);
        if (!valid_utf8(line)) {
            g_err = "stream did not contain valid UTF-8 (line " + std::to_string(nl) + ")";
            rc = 5;
            break;
        }
        if (!line.empty()) {
            const ora_part::Parsed pa = ora_part::parse(line);
            if (pa.err) {
                g_err = ora_part::message(pa) + " (line " + std::to_string(nl) + ")";
                rc = 2;
                break;
            }
            s_orig.parse_raw(pa.text.data(), pa.text.size());
            Sentence* sp = &s_orig;
            if (!no_norm) {
                string pre;
                for (uint32_t c : s_orig.chars) append_utf8(pre, kytea_fullwidth_cp(c));
                s.parse_raw(pre.data(), pre.size());
                sp = &s;
            }
            pr->predict(*sp);
            for (size_t i = 0; i < sp->boundaries.size(); ++i) {
                const int32_t sc = sp->boundary_scores[sp->score_padding + i];
                if (-margin < sc && sc < margin) sp->boundaries[i] = 2;
            }
            for (uint8_t t = 1; t <= 6; ++t) if (wsconst_types & (1u << t)) wsconst_filter(*sp, t);
            if (wsconst_types & 0x80u) grapheme_filter(*sp);
            for (size_t i = 0; i < pa.given.size(); ++i)
                if (pa.given[i] != 2) sp->boundaries[i] = pa.given[i];
            ora_ann::Tags tags(sp->len());
            const bool with_tags = predict_tags && pr->n_tags;
            if (with_tags) {
                // as ora_annotate_lines: fill_tags, then PatternMatchTagger over iter_tokens
                pr->fill_tags(*sp, tt, ti, nullptr);
                vector<const TagPredictor*> tps(pr->tag_predictor.size(), nullptr);
                for (auto& kv : pr->tag_predictor) tps[kv.second.first] = &kv.second.second;
                tags.assign(sp->len(), vector<std::optional<string>>(pr->n_tags));
                for (size_t i = 0; i < sp->len(); ++i)
                    for (size_t k = 0; k < pr->n_tags; ++k)
                        if (ti[i * pr->n_tags + k] >= 0) tags[i][k] = tps[size_t(tt[i])]->tags[k][size_t(ti[i * pr->n_tags + k])];
                for (const auto& [st, en] : ora_ann::iter_tokens(sp->boundaries)) {
                    const string surf = sp->text.substr(sp->char_to_str_pos[st], sp->char_to_str_pos[en] - sp->char_to_str_pos[st]);
                    const auto it = rules.r.find(surf);
                    if (it == rules.r.end()) continue;
                    auto& ts = tags[en - 1];
                    for (size_t k = 0; k < ts.size() && k < it->second.size(); ++k)
                        if (!ts[k]) ts[k] = it->second[k];
                }
            }
            // keep_tags: a character with a non-empty input field gets exactly its input fields ("" is None)
            bool kept = false;
            if (keep_tags) {
                for (size_t i = 0; i < pa.tags.size(); ++i) {
                    bool any = false;
                    for (const string& f : pa.tags[i]) any |= !f.empty();
                    if (!any) continue;
                    tags[i].clear();
                    for (const string& f : pa.tags[i]) tags[i].push_back(f.empty() ? std::nullopt : std::optional<string>(f));
                    kept = true;
                }
            }
            out += ora_ann::write_partial(s_orig.text, s_orig.char_to_str_pos, sp->boundaries,
                                          with_tags || kept ? &tags : nullptr);
        }
        out.push_back('\n');
        ++nl;
        lo = next;
    }
    *n_lines = nl;
    *err_line = nl;
    *out_len = out.size();
    if (out.size() > cap) return 99;
    memcpy(buf, out.data(), out.size());
    return rc;
    ORA_CATCH(idret)
}

}  // extern "C"
