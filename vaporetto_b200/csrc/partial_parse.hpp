// The character loop of `Sentence::parse_partial_annotation` (reference sentence.rs:516-631) as a byte automaton, for
// k_part_parse (partial.cu).  Plain arithmetic: tests/native/partial_parse_test.cpp runs it on the host against a
// restatement of the reference loop, with the state carried across cuts as the kernel carries it across lanes and steps.
//
// The loop alternates a character position and a marker position.  In marker position '\' sets a pending escape, an
// unescaped ' ', '-' or '|' ends the marker (Unknown, NotWordBoundary, WordBoundary), an unescaped '/' opens a tag field,
// and every other character -- escaped or not -- belongs to the open tag field, or is an invalid boundary character
// when no field is open.  A NUL in character position is an error; the line must end in marker position.  States:
//
//   kPaChar     expecting a character               kPaTag      inside a tag field
//   kPaMark     marker position, no field open      kPaTagEsc   inside a tag field, '\' pending
//   kPaMarkEsc  marker position, '\' pending        kPaErr      after an error
//
// Over bytes: a lead byte moves the state as its character does; a continuation byte leaves it alone.  kPaMark is only
// entered by the lead byte of a character read in character position and left by the next lead byte, so a continuation
// byte met in kPaMark belongs to that character.  A byte's move is a map of the six states (3 bits each, in a u32);
// the maps of consecutive bytes compose associatively, which is what a warp scan needs.
#pragma once
#include <cstdint>

#include "common.hpp"

namespace vpt {

enum PartState : uint32_t { kPaChar = 0, kPaMark = 1, kPaMarkEsc = 2, kPaTag = 3, kPaTagEsc = 4, kPaErr = 5 };

// error kinds of a line, in the low 3 bits of its key (position in the line + 1) << 3 | kind (as the gold keys of
// evaluate.cu: the smallest key of a chunk is the first error of its lowest bad line)
enum PartError : uint32_t {
    kPartUtf8 = 1,      // not valid UTF-8 (BufRead::lines fails before the line is parsed); position 0
    kPartNul = 2,       // "must not contain NULL": a NUL in character position
    kPartBoundary = 3,  // "contains an invalid boundary character: '<c>'": <c> is the character at the position
    kPartEnd = 4,       // "invalid annotation": the line ends in character position
};

// given-boundary codes: the values of CharacterBoundary (NotWordBoundary, WordBoundary, Unknown)
constexpr uint8_t kPaNot = 0, kPaWord = 1, kPaUnknown = 2;

constexpr uint32_t kPaIdentity = 0u | 1u << 3 | 2u << 6 | 3u << 9 | 4u << 12 | 5u << 15;

VPT_HD uint32_t pa_apply(uint32_t map, uint32_t s) { return (map >> (3u * s)) & 7u; }

// the map of `first` then `second`
VPT_HD uint32_t pa_compose(uint32_t first, uint32_t second) {
    uint32_t m = 0;
    for (uint32_t s = 0; s < 6; ++s) m |= pa_apply(second, pa_apply(first, s)) << (3u * s);
    return m;
}

VPT_HD bool pa_marker(uint32_t b) { return b == 0x20u || b == 0x2Du || b == 0x7Cu; }

// the move of one byte
VPT_HD uint32_t pa_byte_map(uint32_t b) {
    if ((b & 0xC0u) == 0x80u) return kPaIdentity;
    const uint32_t c = b == 0 ? kPaErr : kPaMark;
    const uint32_t m = b == 0x5Cu ? kPaMarkEsc : pa_marker(b) ? kPaChar : b == 0x2Fu ? kPaTag : kPaErr;
    const uint32_t t = b == 0x5Cu ? kPaTagEsc : pa_marker(b) ? kPaChar : kPaTag;
    return c | m << 3 | kPaErr << 6 | t << 9 | kPaTag << 12 | kPaErr << 15;
}

// the move of the bytes of `x` (low byte first) whose bit 7 is set in `in80`; the others are skipped
VPT_HD uint32_t pa_word_map(uint32_t x, uint32_t in80) {
    uint32_t m = kPaIdentity;
    for (int j = 0; j < 4; ++j)
        if (in80 & (0x80u << (8 * j))) m = pa_compose(m, pa_byte_map((x >> (8 * j)) & 0xFFu));
    return m;
}

// What one byte is, read in state `s`
struct PaByte {
    uint32_t next;  // the state after it
    bool surf;      // a byte of the raw text (a character read in character position)
    bool start;     // the lead byte of such a character
    uint32_t code;  // a marker: its code (kPaNot / kPaWord / kPaUnknown); else 0xFF
    uint32_t err;   // the error it raises (kPartNul / kPartBoundary), else 0
};

VPT_HD PaByte pa_byte(uint32_t s, uint32_t b) {
    PaByte r;
    r.next = pa_apply(pa_byte_map(b), s);
    const bool cont = (b & 0xC0u) == 0x80u;
    r.start = !cont && s == kPaChar && b != 0;
    r.surf = r.start || (cont && s == kPaMark);
    r.code = !cont && (s == kPaMark || s == kPaTag) && pa_marker(b) ? (b == 0x7Cu ? kPaWord : b == 0x2Du ? kPaNot : kPaUnknown)
                                                                      : 0xFFu;
    r.err = s != kPaErr && r.next == kPaErr ? (s == kPaChar ? kPartNul : kPartBoundary) : 0u;
    return r;
}

// ---- input tags (k_part_tags, vpt_reannotate_lines) ----------------------------------------------------------------
//
// A character's input tags are written back as the reference writes a parsed sentence's tags (sentence.rs:907-944):
// '/' + tag for every field up to the last non-empty one, unescaped.  In bytes that is its tag region -- from the '/'
// that opens it to the marker that ends it, or to the line's end -- with every escaping '\' dropped, up to and including
// the last content byte.  What a byte is to that region, read in state `s` (a continuation byte is read in the state
// its lead byte left, so it follows its lead byte):
enum PaTagClass : uint32_t {
    kPaTagNone = 0,     // not part of a tag region
    kPaTagOpen = 1,     // the '/' that opens the region (read in kPaMark): written
    kPaTagSep = 2,      // a later '/' separator: written
    kPaTagDrop = 3,     // an escaping '\': dropped
    kPaTagContent = 4,  // tag content, escaped or not: written
    kPaTagClose = 5,    // the marker after the character (with or without a region)
};

VPT_HD uint32_t pa_tag_class(uint32_t s, uint32_t b) {
    if (s == kPaTagEsc) return kPaTagContent;
    if (s == kPaMark) return b == 0x2Fu ? kPaTagOpen : pa_marker(b) ? kPaTagClose : kPaTagNone;
    if (s != kPaTag) return kPaTagNone;
    return b == 0x2Fu ? kPaTagSep : b == 0x5Cu ? kPaTagDrop : pa_marker(b) ? kPaTagClose : kPaTagContent;
}

// Where the walk over a line is: the last character start, region open and content byte before it (position + 1 in
// the line; 0: none).  Positions only grow, so the walk over bytes [a, c) is the elementwise max of its walks over
// [a, b) and [b, c): lanes and steps combine by max.
struct PaTagRun {
    uint32_t start = 0, open = 0, content = 0;
};

VPT_HD void pa_tag_step(PaTagRun& r, bool start, uint32_t cls, uint32_t pos) {
    if (start) r.start = pos + 1;
    if (cls == kPaTagOpen) r.open = pos + 1;
    if (cls == kPaTagContent) r.content = pos + 1;
}

VPT_HD void pa_tag_max(PaTagRun& r, const PaTagRun& o) {
    r.start = r.start > o.start ? r.start : o.start;
    r.open = r.open > o.open ? r.open : o.open;
    r.content = r.content > o.content ? r.content : o.content;
}

// The written region of the current character: its first byte in the line and its length up to and including its last
// content byte; length 0 when the character opened no region or its region holds no content (its fields are all empty)
VPT_HD uint32_t pa_tag_region(const PaTagRun& r, uint32_t& first) {
    first = r.open ? r.open - 1 : 0;
    return r.open > r.start && r.content > r.open ? r.content - r.open + 1 : 0u;
}

}  // namespace vpt
