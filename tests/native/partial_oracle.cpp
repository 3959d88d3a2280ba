// CPU oracle of vpt_tokenize_partial_lines: a restatement of `Sentence::parse_partial_annotation` (reference
// sentence.rs:516-631) and of the chain the C header defines (parse, predict the raw text, the wsconst post-filters, the
// caller's markers over the boundaries, fill_tags, write_tokenized_text), over the oracle's Sentence / Predictor
// (oracle/vaporetto_oracle.cpp, compiled into this library unchanged).  Test infrastructure only:
// tests/vpt_testlib/partial_oracle.py builds and loads it; tests/native/partial_parse_test.cpp includes it.
#include "../../oracle/vaporetto_oracle.cpp"

namespace ora_part {

// The result of parse_partial_annotation on one line, with where its error is (the byte position of the character
// the loop stopped at; the line's length for "invalid annotation").
struct Parsed {
    string text;                     // as_raw_text()
    vector<uint32_t> char_pos;       // byte position of every character of `text` in the line
    vector<uint8_t> given;           // [chars - 1]: 0 NotWordBoundary, 1 WordBoundary, 2 Unknown
    vector<vector<string>> tags;     // per character: the tag fields that follow it (n_tags wide after padding; "" None)
    size_t n_tags = 0;
    int err = 0;                     // 0, or 1 empty, 2 NUL, 3 invalid boundary character, 4 invalid annotation
    size_t err_pos = 0;
    string err_char;                 // kind 3: the character
};

static const char* reason(int err) {
    switch (err) {
        case 1: return "must contain at least one character";
        case 2: return "must not contain NULL";
        case 3: return "contains an invalid boundary character: ";
        default: return "invalid annotation";
    }
}

static string message(const Parsed& p) {
    string m = string("InvalidArgumentError: partial_annotation_text: ") + reason(p.err);
    if (p.err == 3) m += "'" + p.err_char + "'";
    return m;
}

// parse_partial_annotation's loop over the characters of a valid UTF-8 line, branch for branch
static Parsed parse(const string& line) {
    Parsed r;
    if (line.empty()) { r.err = 1; return r; }
    bool escape = false, is_char = true, have_tag = false;
    string tag_str;
    size_t pos = 0;
    while (pos < line.size()) {
        const uint8_t b = uint8_t(line[pos]);
        const size_t l = b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4;
        const string c = line.substr(pos, l);
        const size_t at = pos;
        pos += l;
        if (is_char) {
            if (c[0] == '\0') { r.err = 2; r.err_pos = at; return r; }
            r.text += c;
            r.char_pos.push_back(uint32_t(at));
            r.tags.emplace_back();
            is_char = false;
            continue;
        }
        auto push_tag = [&] {
            if (have_tag) r.tags.back().push_back(tag_str);
            have_tag = false;
            tag_str.clear();
        };
        if (!escape && c == "\\") {
            escape = true;
        } else if (!escape && (c == " " || c == "-" || c == "|")) {
            push_tag();
            r.given.push_back(c == " " ? 2 : c == "-" ? 0 : 1);
            is_char = true;
        } else if (!escape && c == "/") {
            push_tag();
            have_tag = true;
        } else {
            escape = false;
            if (have_tag) tag_str += c;
            else { r.err = 3; r.err_pos = at; r.err_char = c; return r; }
        }
    }
    if (is_char) { r.err = 4; r.err_pos = line.size(); return r; }
    if (have_tag) r.tags.back().push_back(tag_str);
    for (const auto& t : r.tags) r.n_tags = std::max(r.n_tags, t.size());
    for (auto& t : r.tags) t.resize(r.n_tags);
    return r;
}

// write_tokenized_text (sentence.rs:850-886) of the parsed sentence itself, with its own tags (a token's tags are those
// of its last character; tokens next to an Unknown boundary are skipped)
static string write_parsed(const Parsed& p) {
    string buf;
    auto esc = [&](const string& t) {
        for (char c : t) { if (c == ' ' || c == '\\' || c == '/') buf.push_back('\\'); buf.push_back(c); }
    };
    const size_t n = p.char_pos.size();
    vector<size_t> off(n + 1);
    for (size_t i = 0, o = 0; i < n; ++i) {
        off[i] = o;
        const uint8_t b = uint8_t(p.text[o]);
        o += b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4;
        off[i + 1] = o;
    }
    auto emit = [&](size_t st, size_t en) {
        if (!buf.empty()) buf.push_back(' ');
        esc(p.text.substr(off[st], off[en] - off[st]));
        const auto& ts = p.tags[en - 1];
        int last = -1;
        for (size_t k = 0; k < ts.size(); ++k) if (!ts[k].empty()) last = int(k);
        for (int k = 0; k <= last; ++k) { buf.push_back('/'); esc(ts[size_t(k)]); }
    };
    size_t start = 0;
    bool skip = false;
    for (size_t i = 0; i + 1 < n; ++i) {
        if (p.given[i] == 1) {
            if (!skip) emit(start, i + 1);
            skip = false;
            start = i + 1;
        } else if (p.given[i] == 2) skip = true;
    }
    if (!skip) emit(start, n);
    return buf;
}

}  // namespace ora_part

extern "C" {

// parse_partial_annotation of one line: returns 0 with the raw text in `text` (*text_len), the markers in `given`
// (*n_given), or the error kind (1..4) with its byte position in *err_pos; ora_last_error() holds the message.
int ora_partial_parse(const char* line, size_t n, char* text, size_t* text_len, uint8_t* given, size_t* n_given,
                      size_t* err_pos) {
    const ora_part::Parsed p = ora_part::parse(string(line, n));
    *err_pos = p.err_pos;
    if (p.err) { g_err = ora_part::message(p); return p.err; }
    memcpy(text, p.text.data(), p.text.size());
    *text_len = p.text.size();
    memcpy(given, p.given.data(), p.given.size());
    *n_given = p.given.size();
    return 0;
}

// from_partial_annotation + write_tokenized_text of one line; returns the size, or -(error kind)
long ora_partial_write(const char* line, size_t n, char* buf, size_t cap) {
    const ora_part::Parsed p = ora_part::parse(string(line, n));
    if (p.err) { g_err = ora_part::message(p); return -long(p.err); }
    const string out = ora_part::write_parsed(p);
    if (out.size() > cap) return -1000000 - long(out.size());
    memcpy(buf, out.data(), out.size());
    return long(out.size());
}

// The chain of vpt_tokenize_partial_lines over a buffer (lines split as ora_tokenize_lines splits them).  Returns 0, 2
// (InvalidArgument) or 5 (IOError) with the message in ora_last_error() and the bad line in *err_line; `buf` receives
// the output of the lines before it (*out_len bytes), *n_lines the number of lines read.
int ora_partial_lines(const void* p, const char* utf8, size_t nbytes, int no_norm, uint32_t wsconst_types,
                      int predict_tags, char* buf, size_t cap, uint64_t* out_len, uint64_t* n_lines, uint64_t* err_line) {
    ORA_TRY
    auto* pr = static_cast<const Predictor*>(p);
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
            for (uint8_t t = 1; t <= 6; ++t) if (wsconst_types & (1u << t)) wsconst_filter(*sp, t);
            if (wsconst_types & 0x80u) grapheme_filter(*sp);
            for (size_t i = 0; i < pa.given.size(); ++i)
                if (pa.given[i] != 2) sp->boundaries[i] = pa.given[i];
            if (predict_tags) pr->fill_tags(*sp, tt, ti, nullptr);
            s_orig.boundaries = sp->boundaries;
            out += write_tokenized(*pr, s_orig, predict_tags ? &tt : nullptr, predict_tags ? &ti : nullptr);
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
