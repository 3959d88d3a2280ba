// TEST INFRASTRUCTURE: the chunk cutting of the line stream (vaporetto_b200/csrc/line_feed.hpp) on the host, over random
// byte strings (mixed "\n", "\r\n", "\r", multi-byte UTF-8, long lines) x random feed splits (empty and 1-byte feeds
// included) x chunk sizes from 64 B to 1 MiB x random flush points.  Prints "line feed ok" and exits 0 when every check
// holds.  Not part of the product.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../vaporetto_b200/csrc/line_feed.hpp"

using namespace vpt;

namespace {

int failures = 0;
#define CHECK(c, ...)                                                    \
    do {                                                                 \
        if (!(c)) {                                                      \
            if (++failures <= 20) {                                      \
                fprintf(stderr, "FAIL %s:%d: %s: ", __FILE__, __LINE__, #c); \
                fprintf(stderr, __VA_ARGS__);                            \
                fprintf(stderr, "\n");                                   \
            }                                                            \
        }                                                                \
    } while (0)

struct TooLong : std::runtime_error {
    TooLong() : std::runtime_error("too long") {}
};

struct Chunk {
    std::string bytes;
    size_t nominal;  // nominal size of the chunk when it was cut
};

struct Host {
    std::vector<Chunk> chunks;
    const LineFeed<Host>* feed = nullptr;
    size_t live = 0;  // buffers handed out and not yet taken back
    FeedBuf fresh(size_t min_cap) {
        FeedBuf b;
        b.cap = min_cap;
        b.data = static_cast<uint8_t*>(malloc(min_cap));
        ++live;
        return b;
    }
    void grow(FeedBuf& b, size_t min_cap) {
        const size_t cap = std::max(min_cap, 2 * b.cap);
        b.data = static_cast<uint8_t*>(realloc(b.data, cap));
        b.cap = cap;
    }
    void emit(FeedBuf& b) {
        CHECK(b.size > 0 && b.size <= b.cap, "chunk of %zu bytes in a buffer of %zu", b.size, b.cap);
        // the feed counts the chunk before it is emitted: its nominal size is the previous index's
        chunks.push_back({std::string(reinterpret_cast<const char*>(b.data), b.size), feed->nominal_at(feed->n_chunks() - 1)});
        free(b.data);
        --live;
        b = FeedBuf();
    }
    void too_long() { throw TooLong(); }
};

std::string random_input(std::mt19937_64& rng, size_t target, size_t long_len) {
    static const char* pieces[] = {"\n", "\r\n", "\r", "a", "b", " ", "\xe3\x81\x82", "\xc3\xa9", "\xf0\xa0\x80\x80",
                                   "\xe7\x81\xab\xe6\x98\x9f", "\xff", "\r\r\n", "\n\n"};
    std::string s;
    while (s.size() < target) {
        const unsigned r = unsigned(rng() % 1000);
        if (r < 8) {
            // a long line (longer than most chunk sizes)
            const size_t n = 1 + rng() % long_len;
            for (size_t i = 0; i < n; ++i) s += "\xe3\x81\x82"[i % 3];
        } else {
            s += pieces[rng() % (sizeof(pieces) / sizeof(pieces[0]))];
        }
    }
    if (rng() % 2) s.resize(rng() % (s.size() + 1));  // cut anywhere: inside a character, between '\r' and '\n'
    return s;
}

// the longest line (with its '\n'; an unterminated last line as it is)
size_t longest_line(const std::string& s) {
    size_t best = 0, lo = 0;
    for (size_t i = 0; i < s.size(); ++i)
        if (s[i] == '\n') { best = std::max(best, i + 1 - lo); lo = i + 1; }
    return std::max(best, s.size() - lo);
}

void run_case(std::mt19937_64& rng, const std::string& in, size_t big, size_t max_chunk, int flush_mode) {
    Host h;
    LineFeed<Host> f(h, big, max_chunk);
    h.feed = &f;
    const bool expect_too_long = longest_line(in) > max_chunk;
    bool threw = false;
    std::vector<size_t> flushed_at;  // chunks emitted when each flush returned
    try {
        size_t pos = 0;
        while (pos < in.size()) {
            size_t n;
            switch (rng() % 6) {
                case 0: n = 0; break;
                case 1: n = 1; break;
                case 2: n = rng() % 8; break;
                default: n = rng() % (3 * big + 1); break;
            }
            n = std::min(n, in.size() - pos);
            f.feed(reinterpret_cast<const uint8_t*>(in.data()) + pos, n);
            pos += n;
            if (flush_mode && rng() % (flush_mode == 1 ? 3 : 20) == 0) {
                f.flush();
                // no complete line is held after a flush
                CHECK(!f.held() || !memchr(f.held_data(), '\n', f.held()), "a complete line held after flush");
                flushed_at.push_back(h.chunks.size());
            }
            // a nominal chunk or more is held only while it is one open line
            CHECK(f.held() < f.nominal() || !memchr(f.held_data(), '\n', f.held()), "a full chunk held");
        }
        f.finish();
    } catch (const TooLong&) {
        threw = true;
    }
    FeedBuf rest = f.release();
    if (rest.data) { free(rest.data); --h.live; }
    CHECK(threw == expect_too_long, "too_long %d, expected %d (longest line %zu, limit %zu)", int(threw),
          int(expect_too_long), longest_line(in), max_chunk);
    if (threw) return;
    CHECK(h.live == 0, "%zu buffers not taken back", h.live);
    std::string cat;
    for (size_t i = 0; i < h.chunks.size(); ++i) {
        const Chunk& c = h.chunks[i];
        cat += c.bytes;
        CHECK(!c.bytes.empty(), "empty chunk");
        if (i + 1 < h.chunks.size()) CHECK(c.bytes.back() == '\n', "chunk %zu of %zu does not end in a newline", i, h.chunks.size());
        if (c.bytes.size() > c.nominal) {
            const size_t first_nl = c.bytes.find('\n');
            CHECK(first_nl == std::string::npos || first_nl + 1 == c.bytes.size(),
                  "chunk of %zu bytes over its nominal %zu holds several lines", c.bytes.size(), c.nominal);
        }
        CHECK(c.bytes.size() <= max_chunk, "chunk of %zu over the limit", c.bytes.size());
    }
    CHECK(cat == in, "chunks do not concatenate to the input (%zu vs %zu bytes)", cat.size(), in.size());
    if (in.empty()) CHECK(h.chunks.empty(), "chunks from no input");
}

}  // namespace

int main() {
    // the up-ramp of ramp_schedule (capi.cpp): big / 8 doubling while below big
    CHECK((feed_ramp(64) == std::vector<size_t>{8, 16, 32}), "ramp of 64");
    CHECK((feed_ramp(100) == std::vector<size_t>{12, 24, 48, 96}), "ramp of 100");
    CHECK((feed_ramp(16 << 20) == std::vector<size_t>{2 << 20, 4 << 20, 8 << 20}), "ramp of 16 MiB");
    std::mt19937_64 rng(12345);
    const size_t bigs[] = {64, 100, 1000, 4096, 65536, 1 << 20};
    size_t cases = 0;
    for (int it = 0; it < 4000; ++it) {
        const size_t big = bigs[rng() % 6];
        const size_t target = it % 50 == 0 ? 0 : 1 + rng() % std::min<size_t>(8 * big, it % 10 == 0 ? (3 << 20) : 40000);
        const size_t long_len = std::min<size_t>(3 * big, 200000);
        const std::string in = random_input(rng, target, long_len);
        // the limit: the library's 1 GiB (never reached here), or one a long line exceeds now and then
        const size_t max_chunk = rng() % 4 ? (size_t(1) << 30) : std::max(big, long_len / 2);
        run_case(rng, in, big, max_chunk, int(rng() % 3));
        ++cases;
    }
    // the edge cases by name: empty input, only newlines, a trailing '\r', an unterminated line, a 1-byte chunk size
    for (const char* s : {"", "\n", "\n\n\n", "a\r", "a\r\n", "abc", "\r", "\xe3\x81"})
        for (size_t big : {size_t(1), size_t(2), size_t(64)})
            for (int fm = 0; fm < 3; ++fm) { run_case(rng, s, big, size_t(1) << 30, fm); ++cases; }
    if (failures) {
        fprintf(stderr, "%d failures\n", failures);
        return 1;
    }
    printf("line feed ok: %zu cases\n", cases);
    return 0;
}
