// Host test of the input tag regions of k_part_tags (partial.cu, partial_parse.hpp's pa_tag_class / PaTagRun): every
// string of up to `max_len` symbols from partial_parse_test.cpp's alphabet {a, é, あ, 𠮷, ' ', '-', '|', '/', '\', NUL}
// goes through the walk the way the kernel drives it -- the line at an offset inside 4-byte words, each lane's state from
// the words before it composed onto the carried state, each lane's own walk from nothing, the walks of the lanes before
// it and of the earlier steps combined by max, a region written at every marker after a character and at the line's
// end -- and every region, unescaped, is compared with what the reference writer writes for the character's tag fields
// as the restatement of parse_partial_annotation in partial_oracle.cpp parses them ('/' + tag up to the last non-empty
// one).  Malformed lines are walked too: their regions must stay inside their characters.  The offset and the words per
// step change from string to string, so the carries are cut at every place a string offers.
#include "partial_oracle.cpp"

#include "../../vaporetto_b200/csrc/partial_parse.hpp"

namespace {

struct Region {
    uint32_t first = 0, len = 0;
    bool written = false;
};

// k_part_tags's walk over one line at byte offset `off` of a word-aligned buffer, `words` 4-byte words per step; returns
// false when it writes outside the line's characters (or twice to one)
bool device_regions(const vector<uint8_t>& buf, uint32_t b0, uint32_t b1, int words, vector<Region>& out) {
    uint32_t carry_state = vpt::kPaChar, chars = 0;
    vpt::PaTagRun carry;
    bool ok = true;
    auto put = [&](uint32_t k, const vpt::PaTagRun& r) {
        if (k >= out.size() || out[k].written) { ok = false; return; }
        out[k].written = true;
        out[k].len = vpt::pa_tag_region(r, out[k].first);
        out[k].first += b0;
    };
    const int lanes = words;
    for (uint32_t w0 = 0; w0 < b1; w0 += 4u * uint32_t(lanes)) {
        const size_t nl = size_t(lanes);
        vector<uint32_t> lo(nl, 0), in80(nl, 0), s0(nl, 0), st80(nl, 0);
        vector<vpt::PaTagRun> own(nl);
        uint32_t prefix = vpt::kPaIdentity;
        for (int w = 0; w < lanes; ++w) {
            const uint32_t addr = w0 + 4u * uint32_t(w);
            if (addr < b1) {
                memcpy(&lo[size_t(w)], buf.data() + addr, 4);
                for (uint32_t j = 0; j < 4; ++j)
                    if (addr + j >= b0 && addr + j < b1) in80[size_t(w)] |= 0x80u << (8 * j);
            }
            s0[size_t(w)] = vpt::pa_apply(prefix, carry_state);
            uint32_t s = s0[size_t(w)];
            for (int j = 0; j < 4; ++j) {
                if (!(in80[size_t(w)] & (0x80u << (8 * j)))) continue;
                const uint32_t b = (lo[size_t(w)] >> (8 * j)) & 0xFFu;
                const vpt::PaByte pb = vpt::pa_byte(s, b);
                if (pb.start) st80[size_t(w)] |= 0x80u << (8 * j);
                vpt::pa_tag_step(own[size_t(w)], pb.start, vpt::pa_tag_class(s, b), addr + uint32_t(j) - b0);
                s = pb.next;
            }
            prefix = vpt::pa_compose(prefix, vpt::pa_word_map(lo[size_t(w)], in80[size_t(w)]));
        }
        vpt::PaTagRun lanes_before = carry;  // carry, then the lanes before this one
        uint32_t k = chars;
        for (int w = 0; w < lanes; ++w) {
            const uint32_t addr = w0 + 4u * uint32_t(w);
            vpt::PaTagRun run = lanes_before;
            uint32_t s = s0[size_t(w)];
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (!(in80[size_t(w)] & bit)) continue;
                const uint32_t b = (lo[size_t(w)] >> (8 * j)) & 0xFFu;
                const uint32_t cls = vpt::pa_tag_class(s, b);
                if (st80[size_t(w)] & bit) ++k;
                vpt::pa_tag_step(run, (st80[size_t(w)] & bit) != 0, cls, addr + uint32_t(j) - b0);
                if (cls == vpt::kPaTagClose) {
                    if (k == 0) ok = false;
                    else put(k - 1, run);
                }
                s = vpt::pa_apply(vpt::pa_byte_map(b), s);
            }
            vpt::pa_tag_max(lanes_before, own[size_t(w)]);
        }
        carry_state = vpt::pa_apply(prefix, carry_state);
        chars = k;
        carry = lanes_before;
    }
    if (chars > 0 && carry_state != vpt::kPaChar && carry_state != vpt::kPaErr) put(chars - 1, carry);
    return ok;
}

// the bytes a region writes: its input bytes without the escaping '\' (k_pa_rewrite's unescaped_copy)
string unescape(const vector<uint8_t>& buf, const Region& r) {
    string o;
    for (uint32_t j = 0; j < r.len; ++j) {
        uint8_t c = buf[r.first + j];
        if (c == 0x5C) c = buf[r.first + ++j];
        o.push_back(char(c));
    }
    return o;
}

// write_partial_annotation_text's tags of one parsed character: '/' + tag for every field up to the last non-empty one
string reference_tags(const vector<string>& fields) {
    size_t end = 0;
    for (size_t k = 0; k < fields.size(); ++k)
        if (!fields[k].empty()) end = k + 1;
    string o;
    for (size_t k = 0; k < end; ++k) o += "/" + fields[k];
    return o;
}

const char* const kSymbols[10] = {"a", "\xC3\xA9", "\xE3\x81\x82", "\xF0\xA0\xAE\xB7", " ", "-", "|", "/", "\\", ""};

string show(const string& s) {
    string o;
    char t[8];
    for (unsigned char c : s) {
        if (c >= 0x20 && c < 0x7F) o.push_back(char(c));
        else { snprintf(t, sizeof t, "\\x%02X", c); o += t; }
    }
    return o;
}

}  // namespace

extern "C" {

// every string of 1 .. max_len symbols; returns the number checked, or -1 with the first disagreement in `msg`
long rt_check_all(int max_len, char* msg, size_t cap) {
    long checked = 0;
    vector<int> idx;
    for (int len = 1; len <= max_len; ++len) {
        idx.assign(size_t(len), 0);
        for (;;) {
            string line;
            for (int k : idx) {
                if (k == 9) line.push_back('\0');
                else line += kSymbols[k];
            }
            const int off = int(checked % 4), words = 1 + int((checked / 4) % 8);
            vector<uint8_t> buf(size_t(off) + line.size() + 8, 0x41);
            memcpy(buf.data() + off, line.data(), line.size());
            const ora_part::Parsed want = ora_part::parse(line);
            // at most one character per byte: a malformed line's walk may not write past the characters it counted
            vector<Region> got(want.err ? line.size() : want.char_pos.size());
            string why;
            if (!device_regions(buf, uint32_t(off), uint32_t(off + line.size()), words, got)) why = "write outside";
            else if (!want.err) {
                for (size_t i = 0; i < got.size() && why.empty(); ++i) {
                    if (!got[i].written) why = "no region for character " + std::to_string(i);
                    else if (unescape(buf, got[i]) != reference_tags(want.tags[i]))
                        why = "character " + std::to_string(i) + ": got \"" + show(unescape(buf, got[i])) + "\" want \"" +
                              show(reference_tags(want.tags[i])) + "\"";
                }
            }
            if (!why.empty()) {
                snprintf(msg, cap, "%s: line \"%s\" (offset %d, %d words per step)", why.c_str(), show(line).c_str(), off,
                         words);
                return -1;
            }
            ++checked;
            int k = len - 1;
            while (k >= 0 && ++idx[size_t(k)] == 10) idx[size_t(k--)] = 0;
            if (k < 0) break;
        }
    }
    return checked;
}

}  // extern "C"
