// CPU oracle of vpt_annotate_lines: a restatement of `Sentence::write_partial_annotation_text` (reference
// sentence.rs:907-944), of `TokenIterator` (sentence.rs:1273-1299) for PatternMatchTagger, and of the chain the C header
// defines (predict, the margin, the wsconst post-filters, fill_tags, the rules, the writer), over the oracle's Sentence /
// Predictor (oracle/vaporetto_oracle.cpp, compiled into this library unchanged).  Test infrastructure only:
// tests/vpt_testlib/annotate_oracle.py builds and loads it.
#include <map>
#include <optional>

#include "../../oracle/vaporetto_oracle.cpp"

namespace ora_ann {

using Tags = vector<vector<std::optional<string>>>;  // per character: its tag slots

// write_partial_annotation_text, branch for branch: the first character, then per character its marker and itself,
// and behind every character its tags up to the last Some (unescaped)
static string write_partial(const string& text, const vector<uint32_t>& char_pos, const vector<uint8_t>& bnd,
                            const Tags* tags) {
    string buf;
    const size_t n = char_pos.size() - 1;
    for (size_t i = 0; i < n; ++i) {
        if (i > 0) buf.push_back(bnd[i - 1] == 0 ? '-' : bnd[i - 1] == 1 ? '|' : ' ');
        buf += text.substr(char_pos[i], char_pos[i + 1] - char_pos[i]);
        if (!tags) continue;
        const auto& ts = (*tags)[i];
        size_t end = 0;
        for (size_t k = 0; k < ts.size(); ++k) if (ts[k]) end = k + 1;
        for (size_t k = 0; k < end; ++k) {
            buf.push_back('/');
            if (ts[k]) buf += *ts[k];
        }
    }
    return buf;
}

// TokenIterator::next over boundaries with Unknown: the tokens [start, end) it yields (tokens holding or next to an
// Unknown boundary are skipped)
static vector<std::pair<size_t, size_t>> iter_tokens(const vector<uint8_t>& bnd) {
    vector<std::pair<size_t, size_t>> out;
    size_t start = 0;
    bool skip = false;
    for (size_t i = 0; i < bnd.size(); ++i) {
        if (bnd[i] == 1) {
            if (!skip) out.emplace_back(start, i + 1);
            skip = false;
            start = i + 1;
        } else if (bnd[i] == 2) {
            skip = true;
        }
    }
    if (!skip) out.emplace_back(start, bnd.size() + 1);
    return out;
}

struct Rules {
    std::map<string, vector<std::optional<string>>> r;
};

// blob: u32 n, then per entry u32 length + bytes and u32 n_slots + per slot i32 length (-1: None) + bytes
static const uint8_t* get_u32(const uint8_t* p, uint32_t& v) { memcpy(&v, p, 4); return p + 4; }
static vector<std::optional<string>> read_slots(const uint8_t*& p) {
    uint32_t ns;
    p = get_u32(p, ns);
    vector<std::optional<string>> out;
    for (uint32_t k = 0; k < ns; ++k) {
        uint32_t l;
        p = get_u32(p, l);
        if (int32_t(l) < 0) { out.emplace_back(); continue; }
        out.emplace_back(string(reinterpret_cast<const char*>(p), l));
        p += l;
    }
    return out;
}
static Rules read_rules(const uint8_t* p) {
    Rules rs;
    if (!p) return rs;
    uint32_t n;
    p = get_u32(p, n);
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t l;
        p = get_u32(p, l);
        string surf(reinterpret_cast<const char*>(p), l);
        p += l;
        rs.r[surf] = read_slots(p);
    }
    return rs;
}

}  // namespace ora_ann

extern "C" {

// write_partial_annotation_text of a sentence given as its text, its boundaries (n_chars - 1 values 0 / 1 / 2) and,
// when tags_blob is not NULL, the tag slots of every character (per character: u32 n_slots, then per slot i32 length
// (-1: None) + bytes).  Returns the length, or -(length) when it exceeds cap.
long ora_write_partial_annotation(const char* text, size_t n, const uint8_t* bnd, const uint8_t* tags_blob, char* buf,
                                  size_t cap) {
    Sentence s;
    s.parse_raw(text, n);
    ora_ann::Tags tags;
    if (tags_blob) {
        const uint8_t* p = tags_blob;
        for (size_t i = 0; i < s.len(); ++i) tags.push_back(ora_ann::read_slots(p));
    }
    const string out = ora_ann::write_partial(s.text, s.char_to_str_pos, vector<uint8_t>(bnd, bnd + s.len() - 1),
                                              tags_blob ? &tags : nullptr);
    if (out.size() > cap) return -long(out.size());
    memcpy(buf, out.data(), out.size());
    return long(out.size());
}

// The chain of vpt_annotate_lines over a buffer (lines split as ora_tokenize_lines splits them); `rules_blob` (nullable,
// with predict_tags): PatternMatchTagger's rules (u32 n, then per rule u32 length + surface and its slots as in
// ora_write_partial_annotation), keyed by the KyteaFullwidthFilter image of a token unless no_norm.  Returns 0, or 99
// when the output exceeds cap (*out_len holds its size).
int ora_annotate_lines(const void* p, const char* utf8, size_t nbytes, int no_norm, uint32_t wsconst_types,
                       int predict_tags, int32_t margin, const uint8_t* rules_blob, char* buf, size_t cap,
                       uint64_t* out_len, uint64_t* n_lines) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
    const ora_ann::Rules rules = ora_ann::read_rules(rules_blob);
    string out;
    uint64_t nl = 0;
    size_t lo = 0;
    Sentence s, s_orig;
    vector<int32_t> tt, ti;
    while (lo < nbytes) {
        const void* q = memchr(utf8 + lo, '\n', nbytes - lo);
        size_t end = q ? size_t(static_cast<const char*>(q) - utf8) : nbytes;
        const size_t next = q ? end + 1 : nbytes;
        if (q && end > lo && utf8[end - 1] == '\r') --end;
        bool ok = true;
        try {
            s_orig.parse_raw(utf8 + lo, end - lo);  // update_raw: empty, NUL and invalid UTF-8 lines are rejected
        } catch (const Error&) {
            ok = false;
        }
        if (ok) {
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
            ora_ann::Tags tags;
            const bool with_tags = predict_tags && pr->n_tags;
            if (with_tags) {
                pr->fill_tags(*sp, tt, ti, nullptr);
                vector<const TagPredictor*> tps(pr->tag_predictor.size(), nullptr);
                for (auto& kv : pr->tag_predictor) tps[kv.second.first] = &kv.second.second;
                tags.assign(sp->len(), vector<std::optional<string>>(pr->n_tags));
                for (size_t i = 0; i < sp->len(); ++i)
                    for (size_t k = 0; k < pr->n_tags; ++k)
                        if (ti[i * pr->n_tags + k] >= 0) tags[i][k] = tps[size_t(tt[i])]->tags[k][size_t(ti[i * pr->n_tags + k])];
                // PatternMatchTagger::filter (pattern_match_tagger.rs:21-41) over iter_tokens
                for (const auto& [st, en] : ora_ann::iter_tokens(sp->boundaries)) {
                    const string surf = sp->text.substr(sp->char_to_str_pos[st], sp->char_to_str_pos[en] - sp->char_to_str_pos[st]);
                    const auto it = rules.r.find(surf);
                    if (it == rules.r.end()) continue;
                    auto& ts = tags[en - 1];
                    for (size_t k = 0; k < ts.size() && k < it->second.size(); ++k)
                        if (!ts[k]) ts[k] = it->second[k];
                }
            }
            out += ora_ann::write_partial(s_orig.text, s_orig.char_to_str_pos, sp->boundaries, with_tags ? &tags : nullptr);
        }
        out.push_back('\n');
        ++nl;
        lo = next;
    }
    *n_lines = nl;
    *out_len = out.size();
    if (out.size() > cap) return 99;
    memcpy(buf, out.data(), out.size());
    return 0;
    ORA_CATCH(idret)
}

}  // extern "C"
