// CPU oracle of the predict CLI's score dumps (vpt_line_stream_new_scores): the loop of predict/src/main.rs:125-181 with
// print_scores (main.rs:66-75) and print_tag_scores (main.rs:77-93), over the oracle's Sentence / Predictor
// (oracle/vaporetto_oracle.cpp, compiled into this library unchanged).  Test infrastructure only:
// tests/vpt_testlib/dump_oracle.py builds and loads it.
#include "../../oracle/vaporetto_oracle.cpp"

namespace ora_dump {

// print_scores: "{i}:{prev_c}{c} {score}\n" for every boundary of the predicted sentence, then "\n"
static void print_scores(const ora::Sentence& s, string& out) {
    for (size_t i = 0; i + 1 < s.chars.size(); ++i) {
        out += std::to_string(i) + ":";
        append_utf8(out, s.chars[i]);
        append_utf8(out, s.chars[i + 1]);
        out += " " + std::to_string(s.boundary_scores[s.score_padding + i]) + "\n";
    }
    out += "\n";
}

// print_tag_scores with Token::tag_candidates (sentence.rs:1219-1250): for every token its surface, then per slot of its
// tag model "\t" and the (tag, score) pairs; raw[i] is the score vector fill_tags kept at the token's last character.
// A token whose slots need more scores than its vector has is printed bare (the reference panics on scores[i]).
static void print_tag_scores(const ora::Predictor& p, const ora::Sentence& s, const vector<int32_t>& tt,
                             const vector<vector<int32_t>>& raw, string& out) {
    const size_t n = s.chars.size();
    size_t start = 0;
    for (size_t i = 0; i < n; ++i) {
        if (i + 1 < n && s.boundaries[i] != 1) continue;
        const string surface = s.text.substr(s.char_to_str_pos[start], s.char_to_str_pos[i + 1] - s.char_to_str_pos[start]);
        out += surface;
        if (tt[i] >= 0) {
            const auto& tags = p.tag_predictor.at(surface).second.tags;
            size_t need = 0;
            for (const auto& c : tags) if (c.size() >= 2) need += c.size();
            if (need <= raw[i].size()) {
                size_t k = 0;
                for (const auto& cands : tags) {
                    out += "\t";
                    for (size_t j = 0; j < cands.size(); ++j) {
                        if (j) out += ",";
                        out += cands[j] + ":" + std::to_string(cands.size() == 1 ? 0 : raw[i][k + j]);
                    }
                    if (cands.size() >= 2) k += cands.size();
                }
            }
        }
        out += "\n";
        start = i + 1;
    }
    out += "\n";
}

}  // namespace ora_dump

extern "C" {

// The predict CLI over a buffer of lines (BufRead::lines as ora_tokenize_lines reads them) with --scores (`scores`)
// and --tag-scores (`tag_scores`, needs `predict_tags`).  `token_lines` (nullable) replaces the token line of line k by
// the k-th '\n'-terminated line of that buffer (a test composes tag rules this way; they change the token line only).
// Returns the output size, or -(1000000 + needed) when `cap` is too small.
long ora_dump_lines(const void* p, const char* utf8, size_t nbytes, int no_norm, uint32_t wsconst_types, int predict_tags,
                    int scores, int tag_scores, const char* token_lines, size_t token_lines_len, char* buf, size_t cap,
                    uint64_t* n_lines) {
    auto neg = [](int c) { return -long(c); };
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    string out;
    uint64_t nl = 0;
    size_t lo = 0, tl = 0;
    Sentence s, s_orig;
    vector<int32_t> tt, ti;
    vector<vector<int32_t>> raw;
    while (lo < nbytes) {
        const void* q = memchr(utf8 + lo, '\n', nbytes - lo);
        size_t end = q ? size_t(static_cast<const char*>(q) - utf8) : nbytes;
        const size_t next = q ? end + 1 : nbytes;
        if (q && end > lo && utf8[end - 1] == '\r') --end;
        ++nl;
        bool ok = true;
        try { s_orig.parse_raw(utf8 + lo, end - lo); } catch (const Error&) { ok = false; }
        Sentence* sp = &s_orig;  // the sentence that was predicted
        string line;
        if (ok) {
            if (!no_norm) {
                string pre;
                for (uint32_t c : s_orig.chars) append_utf8(pre, kytea_fullwidth_cp(c));
                s.parse_raw(pre.data(), pre.size());
                sp = &s;
            }
            pr->predict(*sp);
            for (uint8_t t = 1; t <= 6; ++t) if (wsconst_types & (1u << t)) wsconst_filter(*sp, t);
            if (wsconst_types & 0x80u) grapheme_filter(*sp);
            if (predict_tags) pr->fill_tags(*sp, tt, ti, &raw);
            if (!no_norm) s_orig.boundaries = s.boundaries;
            line = write_tokenized(*pr, s_orig, predict_tags ? &tt : nullptr, predict_tags ? &ti : nullptr);
        }
        if (token_lines) {
            const void* e = memchr(token_lines + tl, '\n', token_lines_len - tl);
            if (!e) throw Error(INVALID_ARGUMENT, "token_lines: fewer lines than the input");
            const size_t te = size_t(static_cast<const char*>(e) - token_lines);
            line.assign(token_lines + tl, te - tl);
            tl = te + 1;
        }
        // main.rs:136-141 (--no-norm: the scores before the line's '\n') and 155-175 (after it)
        if (ok) {
            out += line;
            if (no_norm) {
                if (scores) ora_dump::print_scores(*sp, out);
                out += "\n";
            } else {
                out += "\n";
                if (scores) ora_dump::print_scores(*sp, out);
            }
        } else {
            out += "\n";
        }
        if (tag_scores) {
            // The reference prints the default sentence's token " " with the candidates of entry 0 of the last tagged
            // line's tag_scores, which Sentence::set_default leaves in place (sentence.rs:140-158, 1234), and panics if
            // no line was tagged before.  The device prints the token alone; so does this restatement.
            if (ok) ora_dump::print_tag_scores(*pr, *sp, tt, raw, out);
            else out += " \n\n";
        }
        lo = next;
    }
    if (n_lines) *n_lines = nl;
    if (out.size() > cap) return -long(1000000 + out.size());
    memcpy(buf, out.data(), out.size());
    return long(out.size());
    ORA_CATCH(neg)
}

}  // extern "C"
