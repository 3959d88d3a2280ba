// Host check of the window arithmetic of the token-span kernels (vaporetto_b200/csrc/spans.hpp).  The warp loops of
// k_split_linebreaks and k_token_ends are run lane by lane over the same helpers (a warp's inclusive scan is a prefix
// sum) and compared with a byte-by-byte restatement of SplitLinebreaksFilter (split_linebreaks.rs:9-37) and of
// `boundary_pos` (vaporetto_tantivy/src/lib.rs:179-188), on random documents of 1- to 4-byte characters with '\r',
// '\n' and "\r\n" at every start alignment: window edges (documents of 127, 128 and 129 bytes and characters that
// straddle a window), line breaks at the start and the end, runs of line breaks, one-character documents and tokens
// spanning several windows.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../vaporetto_b200/csrc/spans.hpp"

using namespace vpt;

namespace {

int g_fail = 0;
#define CHECK(c, ...)                                                      \
    do {                                                                   \
        if (!(c)) {                                                        \
            if (g_fail++ < 10) { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } \
        }                                                                  \
    } while (0)

// one character, UTF-8
void put(std::string& s, uint32_t c) {
    if (c < 0x80) s += char(c);
    else if (c < 0x800) { s += char(0xC0 | (c >> 6)); s += char(0x80 | (c & 0x3F)); }
    else if (c < 0x10000) { s += char(0xE0 | (c >> 12)); s += char(0x80 | ((c >> 6) & 0x3F)); s += char(0x80 | (c & 0x3F)); }
    else { s += char(0xF0 | (c >> 18)); s += char(0x80 | ((c >> 12) & 0x3F)); s += char(0x80 | ((c >> 6) & 0x3F)); s += char(0x80 | (c & 0x3F)); }
}

uint32_t random_char(std::mt19937& rng, int lb_percent) {
    const int r = int(rng() % 100);
    if (r < lb_percent) return (rng() & 1) ? '\n' : '\r';
    switch (rng() % 4) {
        case 0: return 0x20 + rng() % 0x5F;                 // ASCII
        case 1: return 0x80 + rng() % (0x800 - 0x80);       // 2 bytes
        case 2: return 0x3041 + rng() % 0x6000;             // 3 bytes (kana, kanji)
        default: return 0x1F300 + rng() % 0x300;            // 4 bytes (emoji)
    }
}

// byte-by-byte restatements
std::vector<uint32_t> char_starts(const std::string& d) {
    std::vector<uint32_t> st;
    for (uint32_t i = 0; i < d.size(); ++i)
        if ((uint8_t(d[i]) & 0xC0) != 0x80) st.push_back(i);
    return st;
}
void split_linebreaks_ref(const std::string& d, const std::vector<uint32_t>& st, std::vector<uint8_t>& b) {
    for (size_t i = 0; i + 1 < st.size(); ++i) {
        const char p = d[st[i]], c = d[st[i + 1]];
        if (p == '\r' || p == '\n' || c == '\r' || c == '\n') b[i] = 1;
    }
}
std::vector<uint32_t> boundary_pos_ref(const std::string& d, const std::vector<uint32_t>& st, const std::vector<uint8_t>& b) {
    std::vector<uint32_t> pos;
    for (size_t i = 0; i < b.size(); ++i)
        if (b[i] == 1) pos.push_back(st[i + 1]);
    pos.push_back(uint32_t(d.size()));
    return pos;
}

// the kernels' warp loops, lane by lane: `buf` holds the document at byte b0 (0..3) of a 4-byte aligned buffer
struct Doc {
    std::vector<uint8_t> buf;
    uint32_t b0, b1;
    uint32_t word(uint32_t addr) const { uint32_t w; memcpy(&w, buf.data() + addr, 4); return w; }
};
Doc place(const std::string& d, uint32_t align) {
    Doc x;
    x.b0 = align;
    x.b1 = align + uint32_t(d.size());
    x.buf.assign(((x.b1 + 3) & ~3u) + 8, 0xEE);  // bytes past the end are junk the masks must ignore
    memcpy(x.buf.data() + align, d.data(), d.size());
    for (uint32_t i = 0; i < align; ++i) x.buf[i] = 0x0A;  // so are the bytes before the start
    return x;
}
void split_linebreaks_warp(const Doc& x, uint32_t n, std::vector<uint8_t>& bnd) {
    uint32_t chars = 0;
    for (uint32_t w0 = 0; w0 < x.b1; w0 += 128) {
        uint32_t incl = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) {
            const uint32_t addr = w0 + 4 * lane;
            uint32_t w = 0, in80 = 0;
            if (addr < x.b1) { w = x.word(addr); in80 = span_inside80(addr, x.b0, x.b1); }
            const uint32_t st80 = span_starts80(w, in80);
            const uint32_t nst = span_popc(st80);
            incl += nst;
            const uint32_t lb80 = span_linebreaks80(w, in80);
            if (lb80) span_set_linebreaks(st80, lb80, chars + incl - nst, n, bnd.data());
        }
        chars += incl;
    }
}
std::vector<uint32_t> token_ends_warp(const Doc& x, uint32_t n, const std::vector<uint8_t>& bnd) {
    std::vector<uint32_t> ends(x.b1 - x.b0 + 1, 0xFFFFFFFFu);
    uint32_t chars = 0, rank = 0;
    for (uint32_t w0 = 0; w0 < x.b1; w0 += 128) {
        uint32_t incl = 0, tincl = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) {
            const uint32_t addr = w0 + 4 * lane;
            uint32_t w = 0, in80 = 0;
            if (addr < x.b1) { w = x.word(addr); in80 = span_inside80(addr, x.b0, x.b1); }
            const uint32_t st80 = span_starts80(w, in80);
            const uint32_t nst = span_popc(st80);
            incl += nst;
            const uint32_t ts80 = st80 ? span_token_starts80(st80, chars + incl - nst, bnd.data()) : 0u;
            const uint32_t nts = span_popc(ts80);
            tincl += nts;
            if (ts80) span_store_ends(ts80, addr, x.b0, ends.data() + rank + tincl - nts);
        }
        chars += incl;
        rank += tincl;
    }
    if (n) ends[rank] = x.b1 - x.b0;
    ends.resize(n ? rank + 1 : 0);
    return ends;
}

void check_doc(const std::string& d, std::mt19937& rng, const char* what) {
    const std::vector<uint32_t> st = char_starts(d);
    const uint32_t n = uint32_t(st.size());
    for (uint32_t align = 0; align < 4; ++align) {
        const Doc x = place(d, align);
        // predicted boundaries: random, then the line-break split
        std::vector<uint8_t> pred(n ? n - 1 : 0);
        const uint32_t dens = rng() % 4;  // 0: none .. 3: many (long tokens at 0)
        for (auto& b : pred) b = dens && rng() % (1u << (4 - dens)) == 0;
        std::vector<uint8_t> want = pred, got = pred;
        split_linebreaks_ref(d, st, want);
        if (n >= 2) split_linebreaks_warp(x, n, got);
        CHECK(want == got, "%s: split_linebreaks differs (%zu bytes, align %u)", what, d.size(), align);
        // the post-filters may clear any boundary the split did not set: random clears
        for (size_t i = 0; i < want.size(); ++i)
            if (rng() % 8 == 0) want[i] = got[i] = 0;
        const std::vector<uint32_t> pos = boundary_pos_ref(d, st, want);
        const std::vector<uint32_t> ends = token_ends_warp(x, n, got);
        CHECK(pos == ends, "%s: token ends differ (%zu bytes, align %u, %zu vs %zu tokens)", what, d.size(), align,
              pos.size(), ends.size());
    }
}

std::string random_doc(std::mt19937& rng, size_t min_bytes, int lb_percent) {
    std::string d;
    while (d.size() < min_bytes) put(d, random_char(rng, lb_percent));
    return d;
}

}  // namespace

int main() {
    std::mt19937 rng(20261015);
    size_t docs = 0;
    // window edges: 127, 128 and 129 bytes of every character width, line breaks on the edge
    for (size_t len : {127u, 128u, 129u}) {
        for (uint32_t c : {0x61u, 0xE9u, 0x3042u, 0x1F600u}) {
            std::string d;
            while (d.size() < len) put(d, d.size() % 7 == 6 ? '\n' : c);
            for (int v = 0; v < 4; ++v, ++docs) {
                std::string e = d;
                if (v == 1 && e.size() > 2) { e[len > 128 ? 127 : e.size() - 1] = '\r'; }
                if (v == 2) e = "\r\n" + e + "\r\n";
                if (v == 3) e = "\n" + e;
                check_doc(e, rng, "edge");
            }
        }
        for (int k = 0; k < 200; ++k, ++docs) {
            std::string d = random_doc(rng, len - 4, 20);
            while (d.size() < len) d += 'x';
            check_doc(d.substr(0, len), rng, "edge-random");
        }
    }
    // a character straddling the window edge at every offset
    for (uint32_t pre = 120; pre < 132; ++pre)
        for (uint32_t c : {0xE9u, 0x3042u, 0x1F600u}) {
            std::string d(pre, 'a');
            put(d, c);
            d += "\n\r\nb";
            check_doc(d, rng, "straddle");
            ++docs;
        }
    // one-character documents and line breaks alone, runs of line breaks
    for (const char* s : {"a", "\n", "\r", "\r\n", "\n\n\n\n", "\r\r", "\n\r", "あ", "🤌", "é", "\n\nあ\r\r\nい\n\n"}) {
        check_doc(s, rng, "short");
        ++docs;
    }
    for (int k = 0; k < 300; ++k, ++docs) {
        std::string d;
        const int runs = 1 + int(rng() % 6);
        for (int r = 0; r < runs; ++r) {
            d += random_doc(rng, rng() % 300, 0);
            for (uint32_t q = rng() % 200; q; --q) d += (rng() & 1) ? '\n' : '\r';
        }
        check_doc(d, rng, "runs");
    }
    // random documents up to a few windows, and long tokens over several windows
    for (int k = 0; k < 3000; ++k, ++docs) check_doc(random_doc(rng, 1 + rng() % 700, int(rng() % 30)), rng, "random");
    for (int k = 0; k < 50; ++k, ++docs) check_doc(random_doc(rng, 2000 + rng() % 8000, 0), rng, "long");
    if (g_fail) {
        printf("spans FAILED: %d mismatches\n", g_fail);
        return 1;
    }
    printf("spans ok: %zu documents x 4 alignments\n", docs);
    return 0;
}
