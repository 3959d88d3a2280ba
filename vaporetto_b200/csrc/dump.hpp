// The predict CLI's score dumps for one line (print_scores / print_tag_scores, predict/src/main.rs:66-93, in the loop of
// main.rs:125-181): the per-line code of the dump kernels (dump.cu).  It has no warp operations, so it also compiles
// for the host: tests/native/dump_test.cpp checks the digit counts and UTF-8 lengths below against snprintf and the
// oracle's encoder.
//
// One function, dump_line, walks a line's output and hands every piece to a sink.  The size pass gives it a sink that
// only adds lengths (dec_len, utf8_len); the write pass one that stores the bytes.  Both passes run the same walk, so a
// line's bytes always fill exactly the room the size pass gave it.
//
// Output of line i, after the token line's bytes (its '\n' excluded):
//   default      "\n" + score block + tag block
//   --no-norm    score block + "\n" + tag block     (main.rs:136-141: the scores are written before the line's '\n')
// Score block (dumps & kDumpScores, valid lines only): "{i}:{c_i}{c_i+1} {score_i}\n" for every boundary, then "\n";
// the characters are those of the predicted sentence (the full-width image unless --no-norm).
// Tag block (dumps & kDumpTagScores, every line): per token of the predicted sentence its surface (the image, not
// escaped), then per tag slot of its tag model "\t" + "tag:score" pairs joined by ',' (a one-candidate slot gives
// "tag:0"), then "\n"; one more "\n" after the last token.
//
// Deviations from the reference, each where the reference panics or prints stale data:
//   1. A rejected line (empty, NUL, invalid UTF-8) gives the tag block " \n\n".  The reference prints the default
//      sentence's token " " with the candidates of entry 0 of the last tagged line's tag scores, which set_default does
//      not clear (sentence.rs:140-158, 1234), and panics if no line before it was tagged.
//   2. --tag-scores without tag prediction, or with a model without tag slots, is refused when the stream is created;
//      the reference panics in tag_candidates (sentence.rs:1230-1233).
//   3. A token whose slots list more candidates than its score vector has (record id -1 of the tag-scores path) gives
//      its surface alone; the reference panics on scores[i] (sentence.rs:1242).
#pragma once
#include <cstdint>

#include "tag_rules.hpp"
#include "tags.hpp"
#include "textnorm.hpp"

#if defined(__CUDA_ARCH__)
#define VPT_DUMP_LDG(p) __ldg(p)
#else
#define VPT_DUMP_LDG(p) (*(p))
#endif

namespace vpt {

constexpr uint32_t kDumpScores = 1;     // VPT_DUMP_SCORES
constexpr uint32_t kDumpTagScores = 2;  // VPT_DUMP_TAG_SCORES

// decimal digits of v (Rust's Display form of an unsigned integer)
VPT_HD uint32_t dec_len_u64(uint64_t v) {
    uint32_t n = 1;
    while (v >= 10) { v /= 10; ++n; }
    return n;
}
// bytes of an i32 in Rust's Display form: a '-' for negative values (INT32_MIN included: its magnitude fits in u32)
VPT_HD uint32_t dec_len(int32_t v) {
    return v < 0 ? 1u + dec_len_u64(uint64_t(0) - uint64_t(int64_t(v))) : dec_len_u64(uint64_t(v));
}
// UTF-8 bytes of a code point
VPT_HD uint32_t utf8_len(uint32_t c) { return c < 0x80u ? 1u : c < 0x800u ? 2u : c < 0x10000u ? 3u : 4u; }

// The lines of a chunk and what the dumps read (all device pointers on the device).
struct DumpArgs {
    uint64_t n_sent = 0;
    uint32_t dumps = 0;                     // kDumpScores | kDumpTagScores
    int norm = 0;                           // the predicted sentence is the full-width image (no --no-norm)
    const uint8_t* text = nullptr;          // the chunk's lines
    const uint64_t* offsets = nullptr;      // [n_sent + 1]
    const uint8_t* trims = nullptr;         // [n_sent] terminator bytes
    const int32_t* status = nullptr;        // [n_sent] 0: the line was predicted
    const uint32_t* n_chars = nullptr;      // [n_sent]
    const uint64_t* bound_offsets = nullptr;  // [n_sent + 1] first boundary (score) of a line
    const uint8_t* boundaries = nullptr;    // after the post-filters
    const int32_t* scores = nullptr;        // boundary scores (kDumpScores)
    // with tags: the token records of the tag prediction (the token lines' "/tag" suffixes), the rule ids with rules
    const uint64_t* tok_base = nullptr;     // [n_sent + 1]; nullptr: no tags
    const int32_t* tok_ids = nullptr;
    const uint8_t* tok_cands = nullptr;
    uint32_t n_tags = 0;
    const int32_t* tok_rule = nullptr;      // nullptr: no rules
    DevTagRules rules;
    // kDumpTagScores: the tokens' places and their score vectors (TagScoreArgs)
    const uint4* tok_desc = nullptr;
    const uint32_t* rec_off = nullptr;     // offset of a record's vector inside its block of kScoreScanBlock records
    const uint64_t* score_blk = nullptr;   // the blocks' offsets
    const int32_t* tag_scores = nullptr;
    const TagTokenInfo* tok_info = nullptr;
    const uint32_t* ts_slot = nullptr;      // the escaped tag strings of the tag tables (DevTags)
    const uint32_t* ts_cand = nullptr;
    const uint2* ts_ref = nullptr;
    const uint8_t* ts_bytes = nullptr;
    // the token lines k_tok_write wrote, each '\n'-terminated (a tag string may hold a '\n' too)
    const uint8_t* tok_lines = nullptr;
    // size pass, per line: its token line's bytes (token_line_len) and its dump bytes (dump_line), each with its
    // exclusive prefix inside its block of kDumpBlock lines; then the block prefixes and the chunk's totals
    uint64_t* tl_len = nullptr;             // [n_sent]
    uint64_t* tl_off = nullptr;             // [n_sent]
    uint64_t* size = nullptr;               // [n_sent]
    uint64_t* blk = nullptr;                // [2 x (n_sent / kDumpBlock + 2)]: (dump, token line) per block
    uint64_t* total_host = nullptr;         // pinned host words: the chunk's dump bytes, its token line bytes
    uint8_t* out = nullptr;                 // line i at its token line's offset - i + its dump prefix
};
constexpr int kDumpBlock = 256;  // lines per block of the size pass and its scan

// next code point of valid UTF-8 at p (advanced)
VPT_HD uint32_t dump_next_cp(const uint8_t*& p) {
    const uint32_t b0 = VPT_DUMP_LDG(p);
    const uint32_t l = b0 < 0x80u ? 1u : b0 < 0xE0u ? 2u : b0 < 0xF0u ? 3u : 4u;
    uint32_t c = l == 1 ? b0 : b0 & (0x3Fu >> (l - 1));
    for (uint32_t k = 1; k < l; ++k) c = (c << 6) | (VPT_DUMP_LDG(p + k) & 0x3Fu);
    p += l;
    return c;
}

// Bytes k_tok_write / k_tok_write_tags wrote for line l (lines.cu), '\n' included: a rejected line is "\n"; a predicted
// one is its text with a '\\' before every ' ', '/' and '\\', a ' ' per word boundary, every token's "/tag" suffix
// (merged_suffix_len, the writers' own rule) and the '\n'.  The token lines cannot be found by their '\n's: a tag string
// may hold one.  The host checks the chunk's sum against the writer's total.
VPT_HD uint64_t token_line_len(const DumpArgs& a, uint64_t l) {
    if (a.status[l] != 0) return 1;
    const uint64_t lo = a.offsets[l], hi = a.offsets[l + 1] - a.trims[l];
    uint64_t n = hi - lo + 1;
    for (uint64_t p = lo; p < hi; ++p) {
        const uint32_t b = VPT_DUMP_LDG(a.text + p);
        n += (b == 0x20u) | (b == 0x2Fu) | (b == 0x5Cu);
    }
    const uint8_t* bnd = a.boundaries + a.bound_offsets[l];
    for (uint32_t i = 0; i + 1 < a.n_chars[l]; ++i) n += VPT_DUMP_LDG(bnd + i) == 1;
    if (a.tok_base)
        for (uint64_t r = a.tok_base[l]; r < a.tok_base[l + 1]; ++r)
            n += merged_suffix_len(a.n_tags, a.tok_ids[r], a.tok_cands + r * a.n_tags, a.ts_slot, a.ts_cand, a.ts_ref,
                                   a.tok_rule ? a.tok_rule[r] : -1, a.rules);
    return n;
}

// Sink of the size pass: lengths only.
struct DumpCount {
    uint64_t n = 0;
    VPT_HD void byte(uint32_t) { n += 1; }
    VPT_HD void cp(uint32_t c) { n += utf8_len(c); }
    VPT_HD void u64(uint64_t v) { n += dec_len_u64(v); }
    VPT_HD void i32(int32_t v) { n += dec_len(v); }
};

// Sink of the write pass: the bytes.
struct DumpWrite {
    uint8_t* p;
    VPT_HD void byte(uint32_t b) { *p++ = uint8_t(b); }
    VPT_HD void cp(uint32_t c) {
        if (c < 0x80u) { byte(c); }
        else if (c < 0x800u) { byte(0xC0u | (c >> 6)); byte(0x80u | (c & 0x3Fu)); }
        else if (c < 0x10000u) { byte(0xE0u | (c >> 12)); byte(0x80u | ((c >> 6) & 0x3Fu)); byte(0x80u | (c & 0x3Fu)); }
        else { byte(0xF0u | (c >> 18)); byte(0x80u | ((c >> 12) & 0x3Fu)); byte(0x80u | ((c >> 6) & 0x3Fu)); byte(0x80u | (c & 0x3Fu)); }
    }
    VPT_HD void u64(uint64_t v) {
        const uint32_t n = dec_len_u64(v);
        for (uint32_t k = n; k-- > 0;) { p[k] = uint8_t('0' + v % 10); v /= 10; }
        p += n;
    }
    VPT_HD void i32(int32_t v) {
        if (v < 0) byte('-');
        u64(v < 0 ? uint64_t(0) - uint64_t(int64_t(v)) : uint64_t(v));
    }
};

// The score block of a valid line of n characters at [p, ...): print_scores (main.rs:66-75).
template <typename S>
VPT_HD void dump_scores(const uint8_t* p, uint32_t n, int norm, const int32_t* scores, S& s) {
    if (n) {
        uint32_t prev = dump_next_cp(p);
        if (norm) prev = kytea_fullwidth(prev);
        for (uint32_t i = 0; i + 1 < n; ++i) {
            uint32_t c = dump_next_cp(p);
            if (norm) c = kytea_fullwidth(c);
            s.u64(i);
            s.byte(':');
            s.cp(prev);
            s.cp(c);
            s.byte(' ');
            s.i32(VPT_DUMP_LDG(scores + i));
            s.byte('\n');
            prev = c;
        }
    }
    s.byte('\n');
}

// One token of the tag block: print_tag_scores' body (main.rs:78-90) for the token of record r.
template <typename S>
VPT_HD void dump_token(const DumpArgs& a, uint64_t r, S& s) {
    const uint4 d = a.tok_desc[r];
    const uint8_t* p = a.text + ((uint64_t(d.y & 0xFFFFu) << 32) | d.x);
    const uint8_t* e = p + d.w;
    while (p < e) {
        const uint32_t c = dump_next_cp(p);
        s.cp(a.norm ? kytea_fullwidth(c) : c);
    }
    const int32_t tid = a.tok_ids[r];
    if (tid >= 0) {
        const TagTokenInfo& ti = a.tok_info[tid];
        const int32_t* sc = a.tag_scores + a.score_blk[r / kScoreScanBlock] + a.rec_off[r];
        const uint32_t slot0 = VPT_DUMP_LDG(a.ts_slot + tid);
        uint32_t i = 0;  // next score of the vector
        for (uint32_t k = 0; k < ti.n_slots; ++k) {
            const uint32_t nc = ti.cand[k];
            const uint32_t ref0 = VPT_DUMP_LDG(a.ts_cand + slot0 + k);
            s.byte('\t');
            for (uint32_t c = 0; c < nc; ++c) {
                if (c) s.byte(',');
                // the tag tables hold the escaped strings (write_tokenized_text): a '\\' escapes the byte after it
                const uint2 ref = VPT_DUMP_LDG(a.ts_ref + ref0 + c);
                for (uint32_t b = 0; b < ref.y; ++b) {
                    uint32_t x = VPT_DUMP_LDG(a.ts_bytes + ref.x + b);
                    if (x == '\\') x = VPT_DUMP_LDG(a.ts_bytes + ref.x + ++b);
                    s.byte(x);
                }
                s.byte(':');
                s.i32(nc == 1 ? 0 : VPT_DUMP_LDG(sc + i + c));
            }
            if (nc >= 2) i += nc;
        }
    }
    s.byte('\n');
}

// The dump bytes of line `l` (everything behind its token line's surface and tags), in the order of the mode.
template <typename S>
VPT_HD void dump_line(const DumpArgs& a, uint64_t l, S& s) {
    const bool valid = a.status[l] == 0;
    const auto scores = [&] {
        if (valid && (a.dumps & kDumpScores))
            dump_scores(a.text + a.offsets[l], a.n_chars[l], a.norm, a.scores + a.bound_offsets[l], s);
    };
    if (a.norm) { s.byte('\n'); scores(); }
    else { scores(); s.byte('\n'); }
    if (a.dumps & kDumpTagScores) {
        if (!valid) { s.byte(' '); s.byte('\n'); }  // deviation 1 (see the header)
        for (uint64_t r = a.tok_base[l]; r < a.tok_base[l + 1]; ++r) dump_token(a, r, s);
        s.byte('\n');
    }
}

cudaError_t launch_dump_size(const DumpArgs& a, cudaStream_t stream);   // size + scan: a.tl_len, a.tl_off, a.size, a.blk,
                                                                        // a.total_host[0..1]
cudaError_t launch_dump_write(const DumpArgs& a, cudaStream_t stream);  // the chunk's output at a.out

}  // namespace vpt
