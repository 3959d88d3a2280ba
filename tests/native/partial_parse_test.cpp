// Host test of partial_parse.hpp, the byte automaton of k_part_parse (partial.cu): every string of up to `max_len`
// symbols from {a, é, あ, 𠮷, ' ', '-', '|', '/', '\', NUL} goes through the automaton the way the kernel drives it -- the
// line at an offset inside 4-byte words, each word's move composed from its bytes, the moves of the words before it in
// the step composed onto the carried state, the bytes walked from there, and the state carried across steps -- and the
// raw text, the marker before every character and the first error are compared with the restatement of
// parse_partial_annotation in partial_oracle.cpp.  The offset and the words per step change from string to string, so
// the carry is cut at every place a string offers.
#include "partial_oracle.cpp"

#include "../../vaporetto_b200/csrc/partial_parse.hpp"

namespace {

struct DeviceResult {
    string text;
    vector<uint8_t> given;  // [chars + 1], 0xEE where no marker was written
    uint32_t err_kind = 0;
    size_t err_pos = 0;
};

// k_part_parse's walk over one line at byte offset `off` of a word-aligned buffer, `words` 4-byte words per step
DeviceResult device_parse(const string& line, int off, int words) {
    DeviceResult r;
    vector<uint8_t> buf(size_t(off) + line.size() + 8, 0x41);
    memcpy(buf.data() + off, line.data(), line.size());
    const uint32_t b0 = uint32_t(off), b1 = uint32_t(off + line.size());
    r.given.assign(line.size() + 2, 0xEE);
    uint32_t carry = vpt::kPaChar;
    size_t chars = 0;
    bool have_err = false;
    for (uint32_t w0 = 0; w0 < b1; w0 += 4u * uint32_t(words)) {
        uint32_t prefix = vpt::kPaIdentity;  // the moves of the words before this one in the step
        for (int w = 0; w < words; ++w) {
            const uint32_t addr = w0 + 4u * uint32_t(w);
            if (addr >= b1) break;
            uint32_t x = 0, in80 = 0;
            memcpy(&x, buf.data() + addr, 4);
            for (uint32_t j = 0; j < 4; ++j)
                if (addr + j >= b0 && addr + j < b1) in80 |= 0x80u << (8 * j);
            uint32_t s = vpt::pa_apply(prefix, carry);
            for (int j = 0; j < 4; ++j) {
                if (!(in80 & (0x80u << (8 * j)))) continue;
                const vpt::PaByte pb = vpt::pa_byte(s, (x >> (8 * j)) & 0xFFu);
                s = pb.next;
                if (pb.start) ++chars;
                if (pb.surf) r.text.push_back(char((x >> (8 * j)) & 0xFFu));
                if (pb.code != 0xFFu) r.given[chars] = uint8_t(pb.code);
                if (pb.err && !have_err) {
                    have_err = true;
                    r.err_kind = pb.err;
                    r.err_pos = addr + uint32_t(j) - b0;
                }
            }
            prefix = vpt::pa_compose(prefix, vpt::pa_word_map(x, in80));
        }
        carry = vpt::pa_apply(prefix, carry);
    }
    if (!have_err && carry == vpt::kPaChar) {
        r.err_kind = vpt::kPartEnd;
        r.err_pos = line.size();
    }
    r.given.resize(chars + 1);
    return r;
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
long pp_check_all(int max_len, char* msg, size_t cap) {
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
            const ora_part::Parsed want = ora_part::parse(line);
            const DeviceResult got = device_parse(line, off, words);
            string why;
            if (uint32_t(want.err) != got.err_kind) why = "error kind";
            else if (want.err && want.err_pos != got.err_pos) why = "error position";
            else if (!want.err) {
                if (want.text != got.text) why = "raw text";
                else if (got.given.size() != want.given.size() + 2) why = "characters";
                else
                    for (size_t i = 0; i < want.given.size(); ++i)
                        if (got.given[i + 1] != want.given[i]) why = "marker " + std::to_string(i);
            }
            if (!why.empty()) {
                snprintf(msg, cap, "%s: line \"%s\" (offset %d, %d words per step): want kind %d at %zu, got %u at %zu",
                         why.c_str(), show(line).c_str(), off, words, want.err, want.err_pos, got.err_kind, got.err_pos);
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
