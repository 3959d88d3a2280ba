// Device-side view of a predictor (pointers into the flat model blob in HBM) and the launch API
// between the C ABI (capi.cpp) and the kernels (kernels.cu).
#pragma once
#include <cstdint>

#include <cuda_runtime.h>

#include "keys.hpp"

namespace vpt {

struct DevTable {
    const void* records = nullptr;     // nslots x 32 B (FastRecord or GeneralRecord)
    const uint8_t* seeds = nullptr;    // nbuckets
    const uint32_t* slot_node = nullptr;
    const uint32_t* slot_pid = nullptr;
    const int32_t* pool = nullptr;     // general rows / overflow rows
    const uint64_t* slot_ovf = nullptr; // fast tables with overflow rows: ptr | off16 << 32 | len16 << 48
    uint64_t salt = 0;
    HashK hk{};                        // hash multipliers derived from the salt (keys.hpp)
    uint32_t nslots = 0;
    uint32_t nbuckets = 0;
    uint32_t spill_slots = 0;          // spill table (keys.hpp: slot_of_seeds); its seeds follow the nbuckets ones
    uint32_t spill_buckets = 0;
    uint32_t spill_mul = 0;
    int32_t r0 = 0;
    uint32_t max_depth = 0;
    int32_t present = 0;
    int32_t fast = 0;
    int32_t seed16 = 0;                // seeds are 16-bit (dense tables; never staged in shared memory)
    int32_t has_overflow = 0;          // fast table whose deep records may carry kOvfFlag
};

struct DevModel {
    DevTable ct;                         // char + dictionary patterns
    DevTable tt;                         // type patterns (automaton variant only)
    const int32_t* type_cache = nullptr; // 8^(2W) table (cache variant only)
    int32_t type_cache_window = 0;       // 0 = no cache table
    const int32_t* type_a = nullptr;     // split tables for window 3 (T = A[t0..t3] + B[t2..t5]), or null
    const int32_t* type_b = nullptr;
    const uint32_t* type_state3 = nullptr;  // tag variant: pattern id by (t[-2] t[-1] t[0]) code, or null
    int32_t bias = 0;
    int32_t char_window = 0;
    int32_t type_window = 0;
    int32_t emit_states = 0;             // tag variant: pattern-id states are meaningful
    int32_t kytea_norm = 0;              // per call: score KyteaFullwidthFilter(text) (textnorm.hpp) instead of text
};

// Per-batch device buffers (all device pointers).
struct BatchArgs {
    const uint8_t* text = nullptr;        // concatenated UTF-8, 16-byte aligned, readable up to a multiple of 16
    const uint64_t* offsets = nullptr;    // [n_sent + 1] byte offsets into text
    const uint8_t* trims = nullptr;       // nullable [n_sent]: separator bytes at the end of [offsets[i], offsets[i+1])
                                          // that are not part of sentence i (line terminators, see lines.cu)
    uint64_t n_sent = 0;
    // scratch written by the count pass
    uint32_t* n_chars = nullptr;          // [n_sent]
    int32_t* status = nullptr;            // [n_sent] 0 ok, 1 empty, 2 NUL, 3 invalid UTF-8
    uint32_t* local_bound = nullptr;      // [n_sent] boundary offset inside its 64-sentence group
    uint32_t* local_char = nullptr;       // [n_sent] char offset inside its group
    uint64_t* group_bound = nullptr;      // [n_groups + 1]
    uint64_t* group_char = nullptr;       // [n_groups + 1]
    uint32_t* ticket = nullptr;           // work counter of the persistent tile kernel (zeroed by the scan)
    bool prezeroed = false;               // k_fused: group_bound / group_char / ticket are already zero (no memset node)
    bool self_clean = false;              // k_fused, single-CTA launches only: zero them again before the kernel ends
    uint64_t* totals_host = nullptr;      // nullable: pinned host memory [2]; the scan also stores the batch's boundary
                                          // and character totals there (no D2H copy queued behind bulk copies)
    // outputs
    int32_t* scores = nullptr;            // [sum(max(chars_i - 1, 0))] (nullable: boundaries only)
    uint8_t* boundaries = nullptr;        // same length
    uint64_t* bound_offsets = nullptr;    // [n_sent + 1]; values are chunk-local offsets + bound_base
    uint64_t bound_base = 0;              // added to the bound_offsets / char_offsets written out
    uint64_t char_base = 0;
    uint64_t* char_offsets = nullptr;     // [n_sent + 1] (nullable)
    uint32_t* char_states = nullptr;      // [sum(chars_i)] (nullable)
    uint32_t* type_states = nullptr;      // [sum(chars_i)] (nullable)
};

constexpr int kGroup = 64;  // sentences per count-pass block

// Launch helpers; all asynchronous on `stream`.  Return cudaError_t of the launch.
cudaError_t launch_count(const BatchArgs& a, cudaStream_t stream);  // count + scan
cudaError_t launch_count_only(const BatchArgs& a, cudaStream_t stream);
cudaError_t launch_scan_only(const BatchArgs& a, cudaStream_t stream);
cudaError_t launch_score(const DevModel& m, const BatchArgs& a, cudaStream_t stream);
// fused.cu: validation, counts, output offsets (decoupled look-back) and scoring of a batch in one launch, for the
// inline-row model shapes fused_ok() accepts; needs neither launch_count nor the count pass's scratch arrays
// (group_bound / group_char / ticket are used as look-back descriptors and cleared by a memset node)
bool fused_ok(const DevModel& m);
cudaError_t launch_fused(const DevModel& m, const BatchArgs& a, cudaStream_t stream);
// count (+ scan) + score, or the fused launch when the model qualifies
cudaError_t launch_batch(const DevModel& m, const BatchArgs& a, cudaStream_t stream);
// number of kernel launches issued by launch_batch for this model
int launches_per_batch(const DevModel& m);
// true when launch_score accepts BatchArgs::scores == nullptr (boundaries only) for this model
bool scores_optional(const DevModel& m);

// ---- lines.cu: device-side line splitting and tokenised output -------------------------------------
constexpr int kSplitBlockBytes = 8192;  // bytes of text per CTA of the line splitter

struct SplitArgs {
    const uint8_t* text = nullptr;   // 16-byte aligned, readable up to a multiple of 16
    uint64_t n_bytes = 0;
    uint32_t* blk = nullptr;         // [n_blocks] newline count per block (scratch)
    uint64_t* blk_base = nullptr;    // [n_blocks] lines before each block (scratch)
    uint64_t* n_lines = nullptr;     // device scalar: number of lines
    uint64_t* n_lines_host = nullptr;  // nullable: pinned host memory, receives the same number
    uint64_t* offsets = nullptr;     // [n_lines + 1] out: line starts (+ n_bytes)
    uint8_t* trims = nullptr;        // [n_lines] out: terminator bytes of each line (0, 1 or 2)
};
cudaError_t launch_split_count(const SplitArgs& s, cudaStream_t stream);  // fills *n_lines (and the scratch)
cudaError_t launch_split_write(const SplitArgs& s, cudaStream_t stream);  // fills offsets / trims

struct TokArgs {
    const uint8_t* text = nullptr;          // as BatchArgs (4-byte aligned is enough)
    const uint64_t* offsets = nullptr;
    const uint8_t* trims = nullptr;         // nullable
    uint64_t n_sent = 0;
    const int32_t* status = nullptr;        // from the count pass
    const uint32_t* n_chars = nullptr;
    const uint8_t* boundaries = nullptr;    // 4-byte aligned; from the scoring pass
    const uint64_t* bound_offsets = nullptr;  // index of a sentence's first boundary in `boundaries`
    uint64_t* tok_state = nullptr;          // [n_groups] scratch: look-back state of every 64-sentence group
    uint32_t* ticket = nullptr;             // scratch: group ticket (the 8 bytes after tok_state)
    uint64_t* total = nullptr;              // device scalar out: total output bytes
    uint64_t* total_host = nullptr;         // nullable: pinned host memory, receives the same number
    uint8_t* out = nullptr;                 // tokenised lines, each terminated by '\n'
    // tags (vpt_tokenize_lines_tags): the per-token records of the tag prediction and the model's tag strings; a token's
    // "/tag" suffixes are written behind its surface (Sentence::write_tokenized_text, sentence.rs:850-886)
    const uint64_t* tok_base = nullptr;     // [n_sent + 1] index of a sentence's first token record; nullptr = no tags
    const int32_t* tok_ids = nullptr;       // [n_tokens] token id or -1
    const uint8_t* tok_cands = nullptr;     // [n_tokens * n_tags] chosen candidate per slot, 255 = none
    uint32_t n_tags = 0;
    const uint32_t* ts_slot = nullptr;      // [n_token_ids] first slot entry of a token id
    const uint32_t* ts_cand = nullptr;      // [sum of slots] first string reference of a slot
    const uint2* ts_ref = nullptr;          // [sum of candidates] (offset, length) of the escaped tag string
    const uint8_t* ts_bytes = nullptr;
};
// zeroes tok_state[0 .. n_groups] (ticket included), then one pass: lengths, offsets (look-back), output bytes
cudaError_t launch_tokenize(const TokArgs& t, cudaStream_t stream);
// The column output of vpt_tokenize_dev (launch_tokenize_column, tag_rules.hpp): one string per sentence without '\n' at
// TokArgs::out, a rejected sentence writes none; TokArgs::total points at offsets[n_sent]
struct ColOut {
    uint64_t* offsets = nullptr;  // [n_sent + 1] out: offsets[s] = output offset of sentence s, the total last
    uint64_t capacity = 0;        // bytes at TokArgs::out: sentence s is written iff offsets[s + 1] <= capacity
    uint8_t* status = nullptr;    // [n_sent] out: TokArgs::status as bytes (VPT_SENT_*)
};
// KyteaWsConstFilter for the character types in `mask` (bit t = CharacterType t): clears boundaries between two
// characters of such a type; uses text / offsets / trims / status / n_chars / bound_offsets of `t`
cudaError_t launch_wsconst(const TokArgs& t, uint8_t* boundaries, uint32_t mask, bool norm, cudaStream_t stream);
cudaError_t launch_grapheme(const TokArgs& t, uint8_t* boundaries, bool norm, cudaStream_t stream);

// ---- evaluate.cu: gold corpus parsing (Sentence::from_tokenized) and the evaluate metrics ---------------------------
// error kinds of a gold line, in the low 3 bits of its error key (position in the line + 1) << 3 | kind; a chunk's
// key is line << 34 | line key, so the smallest key is the first error of the lowest bad line
constexpr uint64_t kGoldNoError = ~0ull;
enum GoldError : uint32_t {
    kGoldUtf8 = 1,       // not valid UTF-8 (BufRead::lines fails before the line is parsed)
    kGoldEmpty = 2,      // "must contain at least one character" (a lone '\')
    kGoldStartWs = 3,    // "must not start with a whitespace"
    kGoldDoubleWs = 4,   // "must not contain consecutive whitespaces"
    kGoldSlash = 5,      // "a slash must follow a character"
    kGoldNul = 6,        // "must not contain NULL"
    kGoldEndWs = 7,      // "must not end with a whitespace"
};
// how the system's tags compare with the gold tags (evaluate/src/main.rs:110-120 with predictor.rs:553)
enum EvalTagMode : int32_t {
    kTagsAlwaysEqual = 0,  // --no-norm without tag prediction: the sentence keeps the gold tags
    kTagsGoldEmpty = 1,    // normalised, no tag prediction: empty system tags, equal where the line has no tag field
    kTagsCompare = 2,      // tag prediction with n_tags > 0: equal where the gold width is n_tags and every slot matches
};
constexpr int kEvalTotals = 8;  // tp tn fp fn n_sys n_ref n_cor n_sentences

struct EvalArgs {
    // the chunk's lines (SplitArgs outputs)
    const uint8_t* text = nullptr;          // readable up to a multiple of 4 past the end
    const uint64_t* offsets = nullptr;      // [n_sent + 1]
    const uint8_t* trims = nullptr;         // [n_sent]
    uint64_t n_sent = 0;
    // k_gold_parse outputs
    uint8_t* surface = nullptr;             // raw sentence text of every line, concatenated
    uint64_t* surf_offsets = nullptr;       // [n_sent + 1] into surface
    uint64_t* char_offsets = nullptr;       // [n_sent + 1] first character of every line
    uint8_t* gold_bnd = nullptr;            // [characters] 1: a word boundary is before the character
    uint32_t* tag_pos = nullptr;            // nullable [characters]: at a token's last character, the position in text of
                                            // its first tag '/'; else ~0
    uint32_t* width = nullptr;              // [n_sent] gold tag width (the sentence's n_tags)
    uint64_t* state = nullptr;              // [n_groups] look-back scratch
    uint32_t* ticket = nullptr;             // the 8 bytes after state
    uint64_t* err = nullptr;                // device scalar: smallest error key (set to kGoldNoError before the launch)
    // k_eval inputs: the system's sentences (scored on `surface`) and tag records
    const int32_t* status = nullptr;
    const uint32_t* n_chars = nullptr;
    const uint8_t* boundaries = nullptr;    // after the post-filters
    const uint64_t* bound_offsets = nullptr;
    int32_t tag_mode = kTagsAlwaysEqual;
    uint32_t n_tags = 0;                    // kTagsCompare: the model's n_tags; records and strings as in TokArgs
    const uint64_t* tok_base = nullptr;
    const int32_t* tok_ids = nullptr;
    const uint8_t* tok_cands = nullptr;
    const uint32_t* ts_slot = nullptr;
    const uint32_t* ts_cand = nullptr;
    const uint2* ts_ref = nullptr;
    const uint8_t* ts_bytes = nullptr;
    // k_eval outputs
    uint32_t* line_counts = nullptr;        // nullable [n_sent * 7]: tp tn fp fn n_sys n_ref n_cor of every line
    uint64_t* totals = nullptr;             // [kEvalTotals], added to
};
// zeroes state[0 .. n_groups] (ticket included), then parses the lines
cudaError_t launch_gold_parse(const EvalArgs& e, cudaStream_t stream);
cudaError_t launch_eval(const EvalArgs& e, cudaStream_t stream);

// ---- partial.cu: partially annotated lines (Sentence::from_partial_annotation, partial_parse.hpp) --------------------
struct PartArgs {
    // the chunk's lines (SplitArgs outputs)
    const uint8_t* text = nullptr;          // readable up to a multiple of 4 past the end
    const uint64_t* offsets = nullptr;      // [n_sent + 1]
    const uint8_t* trims = nullptr;         // [n_sent]
    uint64_t n_sent = 0;
    // k_part_parse outputs
    uint8_t* surface = nullptr;             // raw sentence text of every line, concatenated
    uint64_t* surf_offsets = nullptr;       // [n_sent + 1] into surface
    uint64_t* char_offsets = nullptr;       // [n_sent + 1] first character of every line
    uint8_t* given = nullptr;               // [characters + 1] the marker before character k of a line (k >= 1) at
                                            // char_offsets[line] + k: kPaNot / kPaWord / kPaUnknown
    uint64_t* state = nullptr;              // [n_groups] look-back scratch
    uint32_t* ticket = nullptr;             // the 8 bytes after state
    uint64_t* err = nullptr;                // device scalar: smallest error key line << 34 | (position + 1) << 3 | kind
                                            // (set to kGoldNoError before the launch)
    // k_part_apply inputs: the sentences scored on `surface`, after the post-filters
    const int32_t* status = nullptr;
    const uint32_t* n_chars = nullptr;
    const uint64_t* bound_offsets = nullptr;
    uint8_t* boundaries = nullptr;
};
// zeroes state[0 .. n_groups] (ticket included), then parses the lines
cudaError_t launch_part_parse(const PartArgs& e, cudaStream_t stream);
// every given '|' / '-' over the boundary it marks
cudaError_t launch_part_apply(const PartArgs& e, cudaStream_t stream);

// k_part_tags: the input tags of every character (vpt_reannotate_lines), as the byte range of the chunk's input that
// holds them (partial_parse.hpp, pa_tag_region)
struct PartTagArgs {
    const uint8_t* text = nullptr;          // the chunk's input, as PartArgs; kept on the device until the writer ran
    const uint64_t* offsets = nullptr;      // [n_sent + 1]
    const uint8_t* trims = nullptr;         // [n_sent]
    uint64_t n_sent = 0;
    const uint64_t* char_offsets = nullptr; // [n_sent + 1] from k_part_parse
    uint2* regions = nullptr;               // [characters] out, at char_offsets[line] + k: {first byte in `text`, bytes
                                            // up to and including the last content byte}; y == 0: no input tags
};
cudaError_t launch_part_tags(const PartTagArgs& e, cudaStream_t stream);

// ---- annotate.cu: partially annotated output (Sentence::write_partial_annotation_text, vpt_annotate_lines) ------------
struct AnnArgs {
    int32_t margin = 0;                     // boundaries with -margin < score < margin become Unknown (0: none)
    // the scored sentences (BatchArgs outputs)
    uint64_t n_sent = 0;
    const int32_t* status = nullptr;
    const uint32_t* n_chars = nullptr;
    const uint64_t* bound_offsets = nullptr;
    const int32_t* scores = nullptr;        // with margin > 0
    uint8_t* boundaries = nullptr;
    uint8_t* marks = nullptr;               // [boundaries] out: '-', '|' or ' ' per boundary
    // k_pa_untag: the tag records (launch_tag_records)
    const uint64_t* tok_base = nullptr;
    int32_t* tok_ids = nullptr;
    int32_t* tok_rule = nullptr;            // nullable: the rule id of every record
};
// boundary byte 2 (Unknown) for the scores inside the margin; nothing when margin == 0
cudaError_t launch_pa_margin(const AnnArgs& a, cudaStream_t stream);
// the marker of every boundary into marks, and the predicted boundary (score > 0) back into every Unknown one
cudaError_t launch_pa_marks(const AnnArgs& a, cudaStream_t stream);
// tok_ids (and tok_rule) = -1 for every token record next to or across a ' ' marker; nothing when margin == 0
cudaError_t launch_pa_untag(const AnnArgs& a, cudaStream_t stream);
struct TagRuleArgs;
// launch_tokenize_rules in the partial-annotation format: the markers from `marks`, the tags of TokArgs (tok_base
// non-null) and of the rules (ra.tok_rule non-null) unescaped; zeroes tok_state[0 .. n_groups] (ticket included)
cudaError_t launch_pa_write(const TokArgs& t, const TagRuleArgs& ra, const uint8_t* marks, cudaStream_t stream);
// launch_pa_write with the caller's input tags (vpt_reannotate_lines): every character whose region (PartTagArgs, at
// regions[char_offsets[line] + k]) is not empty gets the bytes of `input` it names, unescaped, after it, in place of
// the suffix of the token it ends
cudaError_t launch_pa_rewrite(const TokArgs& t, const TagRuleArgs& ra, const uint8_t* marks, const uint8_t* input,
                              const uint2* regions, const uint64_t* char_offsets, cudaStream_t stream);

// ---- spans.cu: documents -> token byte spans (vaporetto_tantivy's token_stream, vpt_token_spans) --------------------
struct SpanArgs {
    const uint8_t* text = nullptr;          // as BatchArgs (offsets absolute; readable up to a multiple of 4 past the end)
    const uint64_t* offsets = nullptr;      // [n_sent + 1]
    uint64_t n_sent = 0;
    const int32_t* status = nullptr;        // from the count pass
    const uint32_t* n_chars = nullptr;
    uint8_t* boundaries = nullptr;          // from the scoring pass; 4-byte aligned, readable up to a multiple of 4
    const uint64_t* bound_offsets = nullptr;  // chunk-local
    // launch_span_count outputs
    uint8_t* status8 = nullptr;             // [n_sent]
    uint32_t* n_tokens = nullptr;           // [n_sent] boundaries set + 1 for a scored document, else 0
    uint64_t* tok_base = nullptr;           // [n_sent + 1] exclusive prefix of n_tokens, the total behind it
    uint32_t* tok_local = nullptr;          // [n_sent] scratch: prefix inside a block of kSpanDocs documents
    uint64_t* tok_blk = nullptr;            // [n_sent / kSpanDocs + 2] scratch: block totals, then their prefix
    uint64_t* tok_total_host = nullptr;     // nullable: pinned host word that receives the total
    // launch_token_ends output
    uint32_t* token_ends = nullptr;         // [total] token r of document s ends at token_ends[tok_base[s] + r]
};
constexpr int kSpanDocs = 256;  // documents per block of launch_span_count
// SplitLinebreaksFilter: the boundary on either side of every '\r' / '\n' becomes 1
cudaError_t launch_split_linebreaks(const SpanArgs& a, cudaStream_t stream);
// tokens per document (status8, n_tokens) and their prefix (tok_base)
cudaError_t launch_span_count(const SpanArgs& a, cudaStream_t stream);
// the byte offset of every token's exclusive end, relative to its document
cudaError_t launch_token_ends(const SpanArgs& a, cudaStream_t stream);

// ---- doc_offsets.cu: the caller's device offsets of vpt_token_spans_dev (doc_offsets.hpp) ----------------------------
struct DocArgs {
    const void* offsets = nullptr;  // [n_docs + 1] int64 (wide) or int32, as the caller passed them
    int32_t wide = 0;
    uint64_t n_docs = 0;
    uint64_t n_bytes = 0;
    uint32_t shift = 0;             // the text's address mod 16
    uint64_t* out = nullptr;        // [n_docs + 1] rebased offsets into the text rounded down to 16 bytes
    uint8_t* bad = nullptr;         // [n_docs] 1: the document is out of range (VPT_SENT_BAD_RANGE)
    uint64_t* blk = nullptr;        // [doc_offsets_blocks(n_docs)] scratch
};
uint64_t doc_offsets_blocks(uint64_t n_docs);
// out and bad from the caller's offsets
cudaError_t launch_doc_offsets(const DocArgs& a, cudaStream_t stream);
// status[d] = VPT_SENT_BAD_RANGE for every flagged document (after the scoring pass, before launch_split_linebreaks)
cudaError_t launch_doc_status(const DocArgs& a, int32_t* status, cudaStream_t stream);

}  // namespace vpt
