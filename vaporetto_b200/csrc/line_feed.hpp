// Cuts a byte stream, fed in pieces of any size, into chunks of complete lines: the host side of the line stream
// (vpt_line_stream_*, capi.cpp).  Host-only (no CUDA), so the cutting rules are tested with g++ alone
// (tests/native/line_feed_test.cpp).
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

namespace vpt {

// A staging buffer: `size` bytes held, room for `cap`.
struct FeedBuf {
    uint8_t* data = nullptr;
    size_t size = 0, cap = 0;
};

// Nominal sizes of a stream's first chunks: the up-ramp of ramp_schedule (capi.cpp), big / 8 doubling while below `big`;
// every later chunk is `big`.  A stream does not know where it ends, so there is no ramp down.
inline std::vector<size_t> feed_ramp(size_t big) {
    std::vector<size_t> up;
    for (size_t v = std::max<size_t>(big / 8, 1); v < big; v *= 2) up.push_back(v);
    return up;
}

// The cutting rules.  `Host` supplies the buffers and takes the chunks:
//   FeedBuf fresh(size_t min_cap)          an empty buffer with room for at least min_cap bytes
//   void grow(FeedBuf& b, size_t min_cap)  more room for b, keeping its bytes
//   void emit(FeedBuf& b)                  a chunk: the host takes the buffer over (b is left empty)
//   void too_long()                        a chunk would exceed `max_chunk` bytes (a line over the limit); throws
// Every chunk is non-empty and is a run of complete lines ending in '\n'; only the chunk finish() emits may end without
// one.  A chunk exceeds its nominal size only when it is a single line.  A cut is made when the open chunk reaches its
// nominal size (after the last '\n' within it) and at flush() (after the last '\n' held), so the bytes moved to the
// next buffer are less than one chunk.  Invariant: while the open buffer holds a nominal chunk or more, it holds no
// '\n' (a line longer than a chunk, still open).
template <class Host>
class LineFeed {
public:
    LineFeed(Host& h, size_t big, size_t max_chunk) : h_(h), ramp_(feed_ramp(big)), big_(big), max_(max_chunk) {}

    void feed(const uint8_t* p, size_t n) {
        while (n) {
            const size_t nom = nominal();
            if (open_.size < nom) {
                const size_t take = std::min(n, nom - open_.size);
                append(p, take);
                p += take;
                n -= take;
                if (open_.size < nom) return;
                const void* q = memrchr(open_.data, '\n', open_.size);
                if (q) { cut(size_t(static_cast<const uint8_t*>(q) - open_.data) + 1); continue; }
            }
            // a line longer than the chunk: it is taken whole, up to its '\n'
            const void* q = memchr(p, '\n', n);
            const size_t take = q ? size_t(static_cast<const uint8_t*>(q) - p) + 1 : n;
            if (open_.size + take > max_) h_.too_long();
            append(p, take);
            p += take;
            n -= take;
            if (q) cut(open_.size);
        }
    }

    // emits every complete line held
    void flush() {
        if (!open_.size) return;
        const void* q = memrchr(open_.data, '\n', open_.size);
        if (q) cut(size_t(static_cast<const uint8_t*>(q) - open_.data) + 1);
    }

    // emits everything held, an unterminated last line included
    void finish() {
        if (open_.size) cut(open_.size);
    }

    size_t held() const { return open_.size; }
    const uint8_t* held_data() const { return open_.data; }
    size_t n_chunks() const { return k_; }
    size_t nominal() const { return nominal_at(k_); }
    size_t nominal_at(size_t k) const { return k < ramp_.size() ? ramp_[k] : big_; }
    // the open buffer, handed back to the caller (for freeing)
    FeedBuf release() { FeedBuf b = open_; open_ = FeedBuf(); return b; }

private:
    void append(const uint8_t* p, size_t n) {
        if (!n) return;
        if (!open_.data) open_ = h_.fresh(std::max(nominal(), n));
        if (open_.size + n > open_.cap) h_.grow(open_, open_.size + n);
        memcpy(open_.data + open_.size, p, n);
        open_.size += n;
    }

    // emits open_[0, at) and keeps the tail in a fresh buffer
    void cut(size_t at) {
        if (at > max_) h_.too_long();
        const size_t tail = open_.size - at;
        FeedBuf next;
        if (tail) {
            next = h_.fresh(std::max(nominal_at(k_ + 1), tail));  // the tail's buffer holds the next chunk
            memcpy(next.data, open_.data + at, tail);
            next.size = tail;
        }
        FeedBuf chunk = open_;
        chunk.size = at;
        open_ = next;
        ++k_;
        h_.emit(chunk);
    }

    Host& h_;
    std::vector<size_t> ramp_;
    size_t big_, max_;
    size_t k_ = 0;  // chunks emitted
    FeedBuf open_;
};

}  // namespace vpt
