// vaporetto_b200.hpp — header-only C++ mirror of the reference's Rust API over the C ABI (vaporetto_b200.h).
//
// Same names, argument meaning and error behaviour as the crate (vaporetto/src/lib.rs:82-91):
//   vaporetto::Model      model.rs:58   (read / read_slice / to_vec; read_kytea = KyteaModel::read + try_from,
//                                         kytea_model.rs:423-550)
//   vaporetto::Predictor  predictor.rs:434   (new(model, predict_tags), predict(&mut Sentence);
//                                             tokenize_lines = the `predict` CLI loop, predict/src/main.rs:126-181)
//   vaporetto::Sentence   sentence.rs:85   (from_raw, update_raw, as_raw_text, char_types, boundaries,
//                                           boundaries_mut, boundary_scores, fill_tags, tags, n_tags,
//                                           iter_tokens, write_tokenized_text)
//   vaporetto::CharacterBoundary / CharacterType   sentence.rs:9-29,70-82
//   vaporetto::VaporettoError   errors.rs:15-38 (thrown as a C++ exception; `Result<_, VaporettoError>`)
//   vaporetto::LineStream   (this library's own) tokenize_lines / evaluate_lines / tokenize_partial_lines / annotate_lines / reannotate_lines on input fed
//                           in pieces, output to a sink
// Where the reference panics (fill_tags on a predictor created with predict_tags = false, predictor.rs:547-551)
// this mirror throws VaporettoError(InvalidArgument).
#pragma once
#include <algorithm>
#include <cstdint>
#include <exception>
#include <functional>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "vaporetto_b200.h"

namespace vaporetto {

enum class CharacterBoundary : uint8_t { NotWordBoundary = 0, WordBoundary = 1, Unknown = 2 };
enum class CharacterType : uint8_t { Digit = 1, Roman = 2, Hiragana = 3, Katakana = 4, Kanji = 5, Other = 6 };

class VaporettoError : public std::runtime_error {
public:
    VaporettoError(int code, const std::string& msg) : std::runtime_error(msg), code_(code) {}
    int code() const { return code_; }  // vpt_status
private:
    int code_;
};

namespace detail {
inline void check(int rc) {
    if (rc != VPT_OK) throw VaporettoError(rc, vpt_last_error());
}
}  // namespace detail

class Predictor;

/// `vaporetto::Model` — an on-disk model image (raw, un-zstd'd bytes).
class Model {
public:
    /// `Model::read_slice(&[u8]) -> Result<(Model, &[u8])>`: returns the model and the number of bytes consumed.
    static std::pair<Model, size_t> read_slice(const uint8_t* data, size_t len) {
        vpt_model* h = nullptr;
        size_t used = 0;
        detail::check(vpt_model_read(data, len, &h, &used));
        return {Model(h), used};
    }
    /// `Model::read(R: Read)`: the whole buffer is the model.
    static Model read(const std::vector<uint8_t>& bytes) { return read_slice(bytes.data(), bytes.size()).first; }

    /// `Model::read(&mut zstd::Decoder::new(file)?)` (predict/src/main.rs:110-111): a *.model.zst image (or a raw one).
    static Model read_zstd(const std::vector<uint8_t>& bytes) {
        vpt_model* h = nullptr;
        detail::check(vpt_model_read_zstd(bytes.data(), bytes.size(), &h));
        return Model(h);
    }
    /// `KyteaModel::read` + `Model::try_from(KyteaModel)` (kytea_model.rs:423-550): converts a KyTea binary model.
    static Model read_kytea(const std::vector<uint8_t>& bytes) {
        vpt_model* h = nullptr;
        detail::check(vpt_model_read_kytea(bytes.data(), bytes.size(), &h));
        return Model(h);
    }
    /// `Model::to_vec` (model.rs:99-104): the model file image.
    std::vector<uint8_t> to_vec() const {
        uint8_t* p = nullptr;
        uint64_t n = 0;
        detail::check(vpt_model_to_vec(h_, &p, &n));
        std::vector<uint8_t> out(p, p + n);
        vpt_blob_free(p);
        return out;
    }

    Model(Model&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Model& operator=(Model&& o) noexcept { std::swap(h_, o.h_); return *this; }
    Model(const Model&) = delete;
    ~Model() { if (h_) vpt_model_free(h_); }

private:
    friend class Predictor;
    explicit Model(vpt_model* h) : h_(h) {}
    vpt_model* release() { vpt_model* h = h_; h_ = nullptr; return h; }
    vpt_model* h_;
};

class Sentence;

/// `vaporetto::Token` (sentence.rs:1195-1258)
struct Token {
    const Sentence* sentence;
    size_t start_, end_;
    std::string surface() const;
    size_t start() const { return start_; }
    size_t end() const { return end_; }
    std::vector<std::optional<std::string>> tags() const;
};

class TagRules;
namespace detail {
inline const vpt_tag_rules* rules_handle(const TagRules* r);
}

/// `vaporetto::Predictor` resident on one CUDA device.
class Predictor {
public:
    /// `Predictor::new(model: Model, predict_tags: bool) -> Result<Predictor>` — consumes the model.
    /// `device`: CUDA ordinal; -1 = host-only handle (tags / helpers only, scoring fails: no CPU fallback).
    Predictor(Model&& model, bool predict_tags, int device = 0) {
        detail::check(vpt_predictor_new(model.release(), predict_tags ? 1 : 0, device, &h_));
        detail::check(vpt_predictor_get_info(h_, &info_));
    }
    Predictor(Predictor&& o) noexcept : h_(o.h_), info_(o.info_) { o.h_ = nullptr; }
    Predictor(const Predictor&) = delete;
    ~Predictor() { if (h_) vpt_predictor_free(h_); }

    /// `Predictor::predict(&self, &mut Sentence)` (predictor.rs:518-543).
    inline void predict(Sentence& s) const;

    /// The loop of the reference's `predict` CLI over a buffer of raw lines (predict/src/main.rs:126-181;
    /// `vpt_tokenize_lines`): line splitting, the KyteaFullwidthFilter pre-filter (unless `no_norm`), prediction and
    /// `write_tokenized_text` + '\n' all run on the device.  Returns the output text.
    /// `predict_tags`: the CLI's --predict-tags (`vpt_tokenize_lines_tags`: fill_tags + tags in the output text).
    /// `tag_rules`: PatternMatchTagger after fill_tags (`vpt_tokenize_lines_tags_rules`; with predict_tags only).
    std::string tokenize_lines(const std::string& text, bool no_norm = false, uint32_t wsconst_types = 0,
                               bool predict_tags = false, const TagRules* tag_rules = nullptr) const {
        size_t n_lines = 0;
        for (char c : text) n_lines += c == '\n';
        std::string out((predict_tags ? 19 : 3) * text.size() + n_lines + 1, '\0');
        uint64_t n_out = 0, nl = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const int rc = predict_tags
                ? vpt_tokenize_lines_tags_rules(h_, detail::rules_handle(tag_rules), reinterpret_cast<const uint8_t*>(text.data()), text.size(), no_norm ? 1 : 0,
                                                wsconst_types, reinterpret_cast<uint8_t*>(&out[0]), out.size(), &n_out, &nl)
                : vpt_tokenize_lines(h_, reinterpret_cast<const uint8_t*>(text.data()), text.size(), no_norm ? 1 : 0,
                                     wsconst_types, reinterpret_cast<uint8_t*>(&out[0]), out.size(), &n_out, &nl);
            if (rc != 0 && attempt == 0 && n_out > out.size()) { out.assign(size_t(n_out) + 1, '\0'); continue; }  // long tag strings
            detail::check(rc);
            break;
        }
        out.resize(size_t(n_out));
        return out;
    }

    /// tokenize_lines for partially annotated lines (`vpt_tokenize_partial_lines`, Sentence::from_partial_annotation's
    /// format): the model predicts the raw text, the post-filters run, then every '|' / '-' of a line overrides the
    /// boundary it marks; tags (and `tag_rules`) follow with `predict_tags`.  A malformed line throws, naming it.
    std::string tokenize_partial_lines(const std::string& text, bool no_norm = false, uint32_t wsconst_types = 0,
                                       bool predict_tags = false, const TagRules* tag_rules = nullptr) const {
        size_t n_lines = 0;
        for (char c : text) n_lines += c == '\n';
        std::string out((predict_tags ? 19 : 3) * text.size() + n_lines + 1, '\0');
        uint64_t n_out = 0, nl = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const int rc = vpt_tokenize_partial_lines(h_, detail::rules_handle(tag_rules), reinterpret_cast<const uint8_t*>(text.data()),
                                                      text.size(), no_norm ? 1 : 0, wsconst_types, predict_tags ? 1 : 0,
                                                      reinterpret_cast<uint8_t*>(&out[0]), out.size(), &n_out, &nl);
            if (rc != 0 && attempt == 0 && n_out > out.size()) { out.assign(size_t(n_out) + 1, '\0'); continue; }  // long tag strings
            detail::check(rc);
            break;
        }
        out.resize(size_t(n_out));
        return out;
    }

    /// The predicted lines in the partial-annotation format (`vpt_annotate_lines`, Sentence::write_partial_annotation_text):
    /// the boundaries whose score lies strictly between -margin and margin stay Unknown (' '), and the tokens next to
    /// them get no tags.  Tags are written unescaped.
    std::string annotate_lines(const std::string& text, int32_t margin = 0, bool no_norm = false, uint32_t wsconst_types = 0,
                               bool predict_tags = false, const TagRules* tag_rules = nullptr) const {
        size_t n_lines = 0;
        for (char c : text) n_lines += c == '\n';
        std::string out((predict_tags ? 19 : 3) * text.size() + n_lines + 1, '\0');
        uint64_t n_out = 0, nl = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const int rc = vpt_annotate_lines(h_, detail::rules_handle(tag_rules), reinterpret_cast<const uint8_t*>(text.data()),
                                              text.size(), no_norm ? 1 : 0, wsconst_types, predict_tags ? 1 : 0, margin,
                                              reinterpret_cast<uint8_t*>(&out[0]), out.size(), &n_out, &nl);
            if (rc != 0 && attempt == 0 && n_out > out.size()) { out.assign(size_t(n_out) + 1, '\0'); continue; }  // long tag strings
            detail::check(rc);
            break;
        }
        out.resize(size_t(n_out));
        return out;
    }

    /// Partially annotated lines in, partially annotated lines out (`vpt_reannotate_lines`): the caller's '|' / '-' and,
    /// with `keep_tags`, the characters' input tags stay as written; the model decides the ' ' positions and leaves open
    /// those whose score lies strictly between -margin and margin.  A malformed line throws, naming it.
    std::string reannotate_lines(const std::string& text, int32_t margin = 0, bool keep_tags = true, bool no_norm = false,
                                 uint32_t wsconst_types = 0, bool predict_tags = false,
                                 const TagRules* tag_rules = nullptr) const {
        size_t n_lines = 0;
        for (char c : text) n_lines += c == '\n';
        std::string out((predict_tags ? 19 : 3) * text.size() + n_lines + 1, '\0');
        uint64_t n_out = 0, nl = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const int rc = vpt_reannotate_lines(h_, detail::rules_handle(tag_rules), reinterpret_cast<const uint8_t*>(text.data()),
                                                text.size(), no_norm ? 1 : 0, wsconst_types, predict_tags ? 1 : 0, margin,
                                                keep_tags ? 1 : 0, reinterpret_cast<uint8_t*>(&out[0]), out.size(), &n_out, &nl);
            if (rc != 0 && attempt == 0 && n_out > out.size()) { out.assign(size_t(n_out) + 1, '\0'); continue; }  // long tag strings
            detail::check(rc);
            break;
        }
        out.resize(size_t(n_out));
        return out;
    }

    /// The reference's `evaluate` command (evaluate/src/main.rs:69-195; `vpt_evaluate_lines`) over a gold corpus in
    /// the tokenized format: the counts of both metrics.  `line_counts` (optional) receives tp, tn, fp, fn, n_sys,
    /// n_ref, n_cor of every input line.
    vpt_eval_counts evaluate_lines(const std::string& text, bool no_norm = false, uint32_t wsconst_types = 0,
                                   bool predict_tags = false, std::vector<uint32_t>* line_counts = nullptr) const {
        vpt_eval_counts c{};
        uint64_t n_lines = 0;
        if (line_counts) {
            for (char ch : text) n_lines += ch == '\n';
            if (!text.empty() && text.back() != '\n') ++n_lines;
            line_counts->assign(size_t(n_lines) * 7, 0);
        }
        detail::check(vpt_evaluate_lines(h_, reinterpret_cast<const uint8_t*>(text.data()), text.size(), no_norm ? 1 : 0,
                                         wsconst_types, predict_tags ? 1 : 0, &c,
                                         line_counts ? line_counts->data() : nullptr, n_lines));
        return c;
    }

    /// Result of `predict_batch_compact`: see `vpt_predict_batch_compact` (include/vaporetto_b200.h).
    struct CompactResult {
        std::vector<uint32_t> boundary_bits;   // the batch's boundaries, one bit each
        std::vector<uint32_t> n_chars;         // per sentence
        std::vector<uint8_t> status;           // per sentence
        std::vector<uint32_t> n_tokens;        // per sentence
        std::vector<int32_t> token_ids;        // per token (tags requested)
        std::vector<uint8_t> token_cands;      // per token x n_tags, 255 = none
        std::vector<int32_t> tag_scores;       // score vectors of the tokens with id >= 0, record order (tag_scores requested)
        uint64_t n_boundaries = 0, n_unserved = 0;
        /// boundaries [first_bit, first_bit + n) as bytes (0 / 1)
        std::vector<uint8_t> boundaries(uint64_t first_bit, uint64_t n) const {
            std::vector<uint8_t> out(n);
            detail::check(vpt_unpack_boundaries(boundary_bits.data(), first_bit, n, out.data()));
            return out;
        }
    };
    /// predict (+ predict_tags when `tags`) for a batch of sentences given as concatenated UTF-8 + byte offsets, with
    /// compact results: one bit per boundary, one record per token; `tag_scores` (with `tags`): the tag candidate scores
    /// of the records too (`vpt_predict_batch_compact_tag_scores`).
    CompactResult predict_batch_compact(const std::string& text, const std::vector<uint64_t>& byte_offsets, bool tags = false,
                                        bool tag_scores = false) const {
        CompactResult r;
        const size_t n = byte_offsets.empty() ? 0 : byte_offsets.size() - 1;
        const size_t cap = text.size() + 1;
        r.boundary_bits.assign(cap / 32 + 2, 0);
        r.n_chars.assign(n, 0);
        r.status.assign(n, 0);
        r.n_tokens.assign(n, 0);
        const size_t nt = tags ? size_t(info_.n_tags) : 0;
        if (tags) { r.token_ids.assign(cap, -1); r.token_cands.assign(cap * (nt ? nt : 1), 255); }
        uint64_t ntok = 0, nsc = 0;
        if (tag_scores) r.tag_scores.assign(std::max<size_t>(cap * max_score_len(), 1), 0);
        if (n)
            detail::check(vpt_predict_batch_compact_tag_scores(
                h_, reinterpret_cast<const uint8_t*>(text.data()), byte_offsets.data(), n, r.boundary_bits.data(),
                r.boundary_bits.size(), r.n_chars.data(), r.status.data(), r.n_tokens.data(), tags ? r.token_ids.data() : nullptr,
                tags ? r.token_cands.data() : nullptr, tags ? cap : 0, &r.n_boundaries, &ntok, &r.n_unserved,
                tag_scores ? r.tag_scores.data() : nullptr, r.tag_scores.size(), &nsc));
        r.boundary_bits.resize(size_t((r.n_boundaries + 31) / 32));
        if (tags) { r.token_ids.resize(size_t(ntok)); r.token_cands.resize(size_t(ntok) * (nt ? nt : 1)); }
        r.tag_scores.resize(size_t(nsc));
        return r;
    }

    /// Result of `token_spans`: see `vpt_token_spans` (include/vaporetto_b200.h).
    struct SpansResult {
        std::vector<uint32_t> n_tokens;        // per document
        std::vector<uint8_t> status;           // per document, VPT_SENT_*
        std::vector<uint64_t> token_base;      // n_documents + 1: first token record of every document
        std::vector<uint32_t> token_ends;      // per token: exclusive end, in bytes from its document's start
        std::vector<int32_t> token_ids;        // per token (tags requested)
        std::vector<uint8_t> token_cands;      // per token x n_tags, 255 = none
        std::vector<int32_t> tag_scores;       // score vectors of the tokens with id >= 0, record order (tag_scores requested)
        /// [from, to) byte offsets of token r of document d
        std::pair<uint32_t, uint32_t> span(size_t d, size_t r) const {
            const size_t i = size_t(token_base[d]) + r;
            return {r ? token_ends[i - 1] : 0u, token_ends[i]};
        }
    };
    /// vaporetto_tantivy's `token_stream` (lib.rs:157-229; `vpt_token_spans`) for documents given as concatenated UTF-8 +
    /// byte offsets: the full-width pre-filter (unless `no_norm`), predict, the line-break split and the `wsconst_types`
    /// post-filters on the device; the token byte spans (+ tag records when `tags`) come back.
    SpansResult token_spans(const std::string& text, const std::vector<uint64_t>& byte_offsets, bool no_norm = false,
                            uint32_t wsconst_types = 0, bool tags = false, bool tag_scores = false) const {
        SpansResult r;
        const size_t n = byte_offsets.empty() ? 0 : byte_offsets.size() - 1;
        const size_t cap = text.size() + 1;  // a token has at least one byte
        r.n_tokens.assign(n, 0);
        r.status.assign(n, 0);
        r.token_ends.assign(cap, 0);
        const size_t nt = tags ? size_t(info_.n_tags) : 0;
        if (tags) { r.token_ids.assign(cap, -1); r.token_cands.assign(cap * (nt ? nt : 1), 255); }
        uint64_t ntok = 0, nsc = 0;
        if (tag_scores) r.tag_scores.assign(std::max<size_t>(cap * max_score_len(), 1), 0);
        if (n)
            detail::check(vpt_token_spans_tag_scores(h_, reinterpret_cast<const uint8_t*>(text.data()), byte_offsets.data(), n,
                                                     no_norm ? 1 : 0, wsconst_types, r.n_tokens.data(), r.status.data(),
                                                     r.token_ends.data(), tags ? r.token_ids.data() : nullptr,
                                                     tags ? r.token_cands.data() : nullptr, cap, &ntok,
                                                     tag_scores ? r.tag_scores.data() : nullptr, r.tag_scores.size(), &nsc));
        r.token_ends.resize(size_t(ntok));
        r.tag_scores.resize(size_t(nsc));
        if (tags) { r.token_ids.resize(size_t(ntok)); r.token_cands.resize(size_t(ntok) * nt); }
        r.token_base.assign(n + 1, 0);
        for (size_t d = 0; d < n; ++d) r.token_base[d + 1] = r.token_base[d] + r.n_tokens[d];
        return r;
    }

    /// Device buffers of `token_spans_dev` (see `vpt_token_spans_dev` for their sizes)
    struct DeviceSpans {
        uint64_t* token_offsets = nullptr;  // n_documents + 1
        uint32_t* n_tokens = nullptr;
        uint8_t* status = nullptr;
        uint32_t* token_ends = nullptr;
        int32_t* token_ids = nullptr;       // nullable: tags
        uint8_t* token_cands = nullptr;
        void* workspace = nullptr;          // token_spans_dev_workspace_size bytes
        uint64_t workspace_bytes = 0;
    };
    /// bytes of device scratch `token_spans_dev` needs (vpt_token_spans_dev_workspace_size)
    uint64_t token_spans_dev_workspace_size(size_t n_docs, uint64_t n_bytes, bool tags) const {
        return vpt_token_spans_dev_workspace_size(h_, n_docs, n_bytes, tags ? 1 : 0);
    }
    /// `token_spans` for documents already in device memory (`vpt_token_spans_dev`): `d_offsets` holds n_docs + 1 int32
    /// (offset_bytes 4) or int64 (8) offsets into `d_utf8`; all work is queued on `stream` (a cudaStream_t), nothing is
    /// synchronised or allocated, so the call can be captured in a CUDA graph.
    void token_spans_dev(const uint8_t* d_utf8, uint64_t n_bytes, const void* d_offsets, int offset_bytes, size_t n_docs,
                         const DeviceSpans& out, bool no_norm = false, uint32_t wsconst_types = 0,
                         void* stream = nullptr) const {
        detail::check(vpt_token_spans_dev(h_, d_utf8, n_bytes, d_offsets, offset_bytes, n_docs, no_norm ? 1 : 0, wsconst_types,
                                          out.token_offsets, out.n_tokens, out.status, out.token_ends, out.token_ids,
                                          out.token_cands, out.workspace, out.workspace_bytes, stream));
    }

    /// Device buffers of `tokenize_dev` (see `vpt_tokenize_dev` for their sizes)
    struct DeviceText {
        int64_t* offsets = nullptr;         // n_documents + 1
        uint8_t* chars = nullptr;           // capacity bytes; nullable when capacity == 0 (offsets only)
        uint64_t capacity = 0;
        uint8_t* status = nullptr;          // n_documents
        void* workspace = nullptr;          // tokenize_dev_workspace_size bytes
        uint64_t workspace_bytes = 0;
    };
    /// bytes of device scratch `tokenize_dev` needs (vpt_tokenize_dev_workspace_size)
    uint64_t tokenize_dev_workspace_size(size_t n_docs, uint64_t n_bytes, bool predict_tags = false,
                                         const TagRules* tag_rules = nullptr) const {
        return vpt_tokenize_dev_workspace_size(h_, detail::rules_handle(tag_rules), n_docs, n_bytes, predict_tags ? 1 : 0);
    }
    /// a capacity of `DeviceText::chars` with which every document is written (vpt_tokenize_dev_out_bound)
    uint64_t tokenize_dev_out_bound(size_t n_docs, uint64_t n_bytes, bool predict_tags = false,
                                    const TagRules* tag_rules = nullptr) const {
        return vpt_tokenize_dev_out_bound(h_, detail::rules_handle(tag_rules), n_docs, n_bytes, predict_tags ? 1 : 0);
    }
    /// `tokenize` for documents already in device memory (`vpt_tokenize_dev`): the tokenized text of every document as
    /// a device string column; `d_offsets` holds n_docs + 1 int32 (offset_bytes 4) or int64 (8) offsets into `d_utf8`.
    /// All work is queued on `stream` (a cudaStream_t), nothing is synchronised or allocated, so the call can be captured
    /// in a CUDA graph.  `tag_rules`: PatternMatchTagger after fill_tags (with predict_tags only).
    void tokenize_dev(const uint8_t* d_utf8, uint64_t n_bytes, const void* d_offsets, int offset_bytes, size_t n_docs,
                      const DeviceText& out, bool no_norm = false, uint32_t wsconst_types = 0, bool predict_tags = false,
                      const TagRules* tag_rules = nullptr, void* stream = nullptr) const {
        detail::check(vpt_tokenize_dev(h_, detail::rules_handle(tag_rules), d_utf8, n_bytes, d_offsets, offset_bytes, n_docs,
                                       no_norm ? 1 : 0, wsconst_types, predict_tags ? 1 : 0, out.offsets, out.chars,
                                       out.capacity, out.status, out.workspace, out.workspace_bytes, stream));
    }

    /// the longest tag score vector of the predictor's tokens (vpt_tag_score_len)
    size_t max_score_len() const {
        size_t m = 0;
        for (uint32_t t = 0, n = vpt_tag_n_tokens(h_); t < n; ++t) m = std::max<size_t>(m, vpt_tag_score_len(h_, t));
        return m;
    }

    const vpt_predictor_info& info() const { return info_; }
    const vpt_predictor* handle() const { return h_; }

private:
    vpt_predictor* h_ = nullptr;
    vpt_predictor_info info_{};
};

/// `vaporetto::Sentence` — the raw-text subset used around `predict` (annotation parsers are out of scope).
class Sentence {
public:
    /// `Sentence::from_raw(text) -> Result<Sentence>`: InvalidArgument for "" or a text containing U+0000.
    static Sentence from_raw(std::string text) {
        Sentence s;
        s.set(std::move(text));
        return s;
    }
    /// `Sentence::update_raw(&mut self, text) -> Result<()>`: on error the sentence becomes " " (sentence.rs:264-283).
    void update_raw(std::string text) {
        try {
            set(std::move(text));
        } catch (const VaporettoError&) {
            set(" ");
            throw;
        }
    }
    const std::string& as_raw_text() const { return text_; }
    const std::vector<uint8_t>& char_types() const { return types_; }
    const std::vector<uint8_t>& boundaries() const { return boundaries_; }       // CharacterBoundary values
    std::vector<uint8_t>& boundaries_mut() { return boundaries_; }
    const std::vector<int32_t>& boundary_scores() const { return scores_; }      // sentence.rs:1040-1046
    size_t n_tags() const { return tags_filled_ ? n_tags_ : 0; }
    const std::vector<std::optional<std::string>>& tags() const { return tags_; }

    /// `vaporetto_rules::sentence_filters::SplitLinebreaksFilter::filter(&mut sentence)` (split_linebreaks.rs:9-37).
    void split_linebreaks() {
        detail::check(vpt_split_linebreaks(reinterpret_cast<const uint8_t*>(text_.data()), text_.size(), boundaries_.data(),
                                           boundaries_.size()));
    }
    /// `vaporetto_rules::sentence_filters::ConcatGraphemeClustersFilter::filter(&mut sentence)`
    /// (concat_grapheme_clusters.rs:10-35).
    void concat_grapheme_clusters() {
        detail::check(vpt_concat_grapheme_clusters(reinterpret_cast<const uint8_t*>(text_.data()), text_.size(),
                                                   boundaries_.data(), boundaries_.size()));
    }

    /// `Sentence::fill_tags(&mut self)` (sentence.rs:1144) -> `Predictor::predict_tags` (predictor.rs:546-637).
    void fill_tags() {
        if (!predictor_) return;
        const size_t n = types_.size(), k = size_t(predictor_->info().n_tags);
        tag_token_.assign(n, -1);
        tag_cand_.assign(n * k + 1, -1);
        detail::check(vpt_fill_tags(predictor_->handle(), reinterpret_cast<const uint8_t*>(text_.data()), text_.size(),
                                    boundaries_.data(), char_states_.empty() ? nullptr : char_states_.data(),
                                    type_states_.empty() ? nullptr : type_states_.data(), tag_token_.data(),
                                    tag_cand_.data(), nullptr, 0));
        n_tags_ = k;
        tags_.assign(n * k, std::nullopt);
        for (size_t i = 0; i < n; ++i)
            for (size_t s = 0; s < k; ++s) {
                const int32_t c = tag_cand_[i * k + s];
                if (tag_token_[i] >= 0 && c >= 0)
                    tags_[i * k + s] = vpt_tag_string(predictor_->handle(), uint32_t(tag_token_[i]), uint32_t(s), uint32_t(c));
            }
        tags_filled_ = true;
    }

    /// `Sentence::iter_tokens` (TokenIterator, sentence.rs:1273-1299): tokens next to Unknown boundaries are skipped.
    std::vector<Token> iter_tokens() const {
        std::vector<Token> out;
        size_t start = 0;
        bool skip = false;
        for (size_t i = 0; i < boundaries_.size(); ++i) {
            if (boundaries_[i] == uint8_t(CharacterBoundary::WordBoundary)) {
                if (!skip) out.push_back(Token{this, start, i + 1});
                skip = false;
                start = i + 1;
            } else if (boundaries_[i] == uint8_t(CharacterBoundary::Unknown)) {
                skip = true;
            }
        }
        if (!skip) out.push_back(Token{this, start, types_.size()});
        return out;
    }

    /// `Sentence::write_tokenized_text(&self, buf: &mut String)` (sentence.rs:850-886).
    void write_tokenized_text(std::string& buf) const {
        // the C call reports the full length even when it had to truncate: size the buffer from a first guess and
        // retry once with the exact length (tag strings come from the model file and can be arbitrarily long)
        uint64_t need = 0;
        std::vector<char> tmp(2 * text_.size() + 64);
        for (int attempt = 0; attempt < 2; ++attempt) {
            detail::check(vpt_write_tokenized_text(predictor_ ? predictor_->handle() : nullptr,
                                                   reinterpret_cast<const uint8_t*>(text_.data()), text_.size(),
                                                   boundaries_.data(), tags_filled_ ? tag_token_.data() : nullptr,
                                                   tags_filled_ ? tag_cand_.data() : nullptr, tmp.data(), tmp.size(), &need));
            if (need < tmp.size()) break;
            tmp.resize(size_t(need) + 1);
        }
        if (need >= tmp.size()) throw std::runtime_error("write_tokenized_text: length changed between calls");
        buf.assign(tmp.data(), size_t(need));
    }

    /// `Sentence::write_partial_annotation_text(&self, buf: &mut String)` (sentence.rs:907-944): tags unescaped.
    void write_partial_annotation_text(std::string& buf) const {
        uint64_t need = 0;
        std::vector<char> tmp(2 * text_.size() + 64);
        for (int attempt = 0; attempt < 2; ++attempt) {
            detail::check(vpt_write_partial_annotation_text(predictor_ ? predictor_->handle() : nullptr,
                                                            reinterpret_cast<const uint8_t*>(text_.data()), text_.size(),
                                                            boundaries_.data(), tags_filled_ ? tag_token_.data() : nullptr,
                                                            tags_filled_ ? tag_cand_.data() : nullptr, tmp.data(),
                                                            tmp.size(), &need));
            if (need < tmp.size()) break;
            tmp.resize(size_t(need) + 1);
        }
        if (need >= tmp.size()) throw std::runtime_error("write_partial_annotation_text: length changed between calls");
        buf.assign(tmp.data(), size_t(need));
    }

private:
    friend class Predictor;
    friend struct Token;
    void set(std::string text) {
        std::vector<uint8_t> types(text.size() + 1);
        uint64_t n = 0;
        detail::check(vpt_char_types(reinterpret_cast<const uint8_t*>(text.data()), text.size(), types.data(), types.size(), &n));
        types.resize(size_t(n));
        text_ = std::move(text);
        types_ = std::move(types);
        pos_.clear();
        for (size_t i = 0; i < text_.size(); ++i)
            if ((uint8_t(text_[i]) & 0xC0) != 0x80) pos_.push_back(i);
        pos_.push_back(text_.size());
        boundaries_.assign(types_.size() - 1, uint8_t(CharacterBoundary::Unknown));
        scores_.clear();
        char_states_.clear();
        type_states_.clear();
        predictor_ = nullptr;
        tags_.clear();
        tags_filled_ = false;
    }
    std::string text_;
    std::vector<uint8_t> types_, boundaries_;
    std::vector<int32_t> scores_;
    std::vector<uint32_t> char_states_, type_states_;
    std::vector<size_t> pos_;
    const Predictor* predictor_ = nullptr;
    std::vector<int32_t> tag_token_, tag_cand_;
    std::vector<std::optional<std::string>> tags_;
    size_t n_tags_ = 0;
    bool tags_filled_ = false;
};

/// `vaporetto_rules::sentence_filters::PatternMatchTagger::new(rules)` for the tagged line path (`vpt_tag_rules_new`):
/// surface -> one entry per tag slot (std::nullopt leaves the slot alone).  Fills the tag slots the model left None;
/// unless no_norm, tokens are matched by their KyteaFullwidthFilter image and keys are not normalised.  Bound to the
/// predictor, which must outlive it; it must outlive every call and stream that uses it.
class TagRules {
public:
    TagRules(const Predictor& predictor, const std::vector<std::pair<std::string, std::vector<std::optional<std::string>>>>& rules) {
        std::string surf, tags;
        std::vector<uint64_t> soff{0}, qoff{0};
        std::vector<uint32_t> slots;
        for (const auto& r : rules) {
            surf += r.first;
            soff.push_back(surf.size());
            for (const auto& t : r.second) {
                slots.push_back(t ? uint32_t(tags.size()) : UINT32_MAX);
                slots.push_back(t ? uint32_t(t->size()) : 0);
                if (t) tags += *t;
            }
            qoff.push_back(slots.size() / 2);
        }
        detail::check(vpt_tag_rules_new(predictor.handle(), rules.size(), reinterpret_cast<const uint8_t*>(surf.data()),
                                        soff.data(), qoff.data(), slots.data(), reinterpret_cast<const uint8_t*>(tags.data()),
                                        tags.size(), &h_));
    }
    TagRules(const TagRules&) = delete;
    TagRules& operator=(const TagRules&) = delete;
    ~TagRules() { vpt_tag_rules_free(h_); }
    const vpt_tag_rules* handle() const { return h_; }

private:
    vpt_tag_rules* h_ = nullptr;
};

namespace detail {
inline const vpt_tag_rules* rules_handle(const TagRules* r) { return r ? r->handle() : nullptr; }
}

/// A line stream (`vpt_line_stream_*`): Predictor::tokenize_lines or evaluate_lines on input fed in pieces of any size,
/// split at any byte, with host memory bounded by the pipeline rather than by the input.  The output goes to `sink` in
/// input order as chunks complete, on the thread that calls feed / flush / finish; an exception thrown by the sink
/// aborts the stream and is rethrown from that call.  After any error every call throws it again.
class LineStream {
public:
    using Sink = std::function<void(const uint8_t* bytes, size_t n)>;
    struct PartialLines {};  ///< selects the stream of Predictor::tokenize_partial_lines
    /// The stream of Predictor::tokenize_partial_lines (`vpt_line_stream_new_partial`).
    LineStream(const Predictor& predictor, PartialLines, Sink sink, bool no_norm = false, uint32_t wsconst_types = 0,
               bool predict_tags = false, const TagRules* tag_rules = nullptr)
        : sink_(std::move(sink)) {
        detail::check(vpt_line_stream_new_partial(predictor.handle(), detail::rules_handle(tag_rules), no_norm ? 1 : 0,
                                                  wsconst_types, predict_tags ? 1 : 0,
                                                  sink_ ? &LineStream::write : nullptr, this, &h_));
    }
    /// The stream of Predictor::annotate_lines (`vpt_line_stream_new_annotate`).
    struct AnnotateLines {
        int32_t margin = 0;
    };
    LineStream(const Predictor& predictor, AnnotateLines a, Sink sink, bool no_norm = false, uint32_t wsconst_types = 0,
               bool predict_tags = false, const TagRules* tag_rules = nullptr)
        : sink_(std::move(sink)) {
        detail::check(vpt_line_stream_new_annotate(predictor.handle(), detail::rules_handle(tag_rules), no_norm ? 1 : 0,
                                                   wsconst_types, predict_tags ? 1 : 0, a.margin,
                                                   sink_ ? &LineStream::write : nullptr, this, &h_));
    }
    /// The stream of Predictor::reannotate_lines (`vpt_line_stream_new_reannotate`).
    struct ReannotateLines {
        int32_t margin = 0;
        bool keep_tags = true;
    };
    LineStream(const Predictor& predictor, ReannotateLines a, Sink sink, bool no_norm = false, uint32_t wsconst_types = 0,
               bool predict_tags = false, const TagRules* tag_rules = nullptr)
        : sink_(std::move(sink)) {
        detail::check(vpt_line_stream_new_reannotate(predictor.handle(), detail::rules_handle(tag_rules), no_norm ? 1 : 0,
                                                     wsconst_types, predict_tags ? 1 : 0, a.margin, a.keep_tags ? 1 : 0,
                                                     sink_ ? &LineStream::write : nullptr, this, &h_));
    }
    /// kind: VPT_STREAM_TOKENIZE (`sink` receives the tokenised lines) or VPT_STREAM_EVALUATE (`sink` may be empty).
    /// tag_rules: as in Predictor::tokenize_lines.  dumps: VPT_DUMP_SCORES | VPT_DUMP_TAG_SCORES, the predict CLI's
    /// --scores / --tag-scores behind every token line (VPT_STREAM_TOKENIZE only; vpt_line_stream_new_scores).
    LineStream(const Predictor& predictor, int kind, Sink sink, bool no_norm = false, uint32_t wsconst_types = 0,
               bool predict_tags = false, const TagRules* tag_rules = nullptr, uint32_t dumps = 0)
        : sink_(std::move(sink)) {
        if (dumps && kind != VPT_STREAM_TOKENIZE)
            throw VaporettoError(VPT_INVALID_ARGUMENT, "InvalidArgumentError: dumps: VPT_STREAM_TOKENIZE only");
        if (dumps)
            detail::check(vpt_line_stream_new_scores(predictor.handle(), detail::rules_handle(tag_rules), no_norm ? 1 : 0,
                                                     wsconst_types, predict_tags ? 1 : 0, dumps,
                                                     sink_ ? &LineStream::write : nullptr, this, &h_));
        else
            detail::check(vpt_line_stream_new_rules(predictor.handle(), detail::rules_handle(tag_rules), kind, no_norm ? 1 : 0,
                                                    wsconst_types, predict_tags ? 1 : 0, sink_ ? &LineStream::write : nullptr,
                                                    this, &h_));
    }
    LineStream(const LineStream&) = delete;
    LineStream& operator=(const LineStream&) = delete;
    ~LineStream() { vpt_line_stream_free(h_); }

    /// copies the bytes into the stream; delivers the output of the oldest chunk when four are in flight
    void feed(const void* bytes, size_t n) { check(vpt_line_stream_feed(h_, static_cast<const uint8_t*>(bytes), n)); }
    void feed(const std::string& bytes) { feed(bytes.data(), bytes.size()); }
    /// delivers the output of every complete line fed so far
    void flush() { check(vpt_line_stream_flush(h_)); }
    /// delivers the rest; returns the number of input lines, `counts` (evaluate) receives the totals
    uint64_t finish(vpt_eval_counts* counts = nullptr) {
        uint64_t n = 0;
        check(vpt_line_stream_finish(h_, &n, counts));
        return n;
    }

private:
    static int write(void* ctx, const uint8_t* bytes, size_t n) {
        LineStream* self = static_cast<LineStream*>(ctx);
        try {
            self->sink_(bytes, n);
            return 0;
        } catch (...) {
            self->error_ = std::current_exception();
            return 1;
        }
    }
    void check(int rc) {
        if (error_) std::rethrow_exception(std::exchange(error_, nullptr));
        detail::check(rc);
    }
    Sink sink_;
    std::exception_ptr error_;
    vpt_line_stream* h_ = nullptr;
};

inline void Predictor::predict(Sentence& s) const {
    const size_t n = s.types_.size();
    s.scores_.assign(n > 1 ? n - 1 : 1, 0);
    s.boundaries_.assign(n > 1 ? n - 1 : 1, 0);
    const bool states = info_.char_scorer == 2 || info_.type_scorer == 3;
    if (states) {
        s.char_states_.assign(n, VPT_NO_PATTERN);
        s.type_states_.assign(n, VPT_NO_PATTERN);
    }
    uint64_t nch = 0;
    detail::check(vpt_predict(h_, reinterpret_cast<const uint8_t*>(s.text_.data()), s.text_.size(), s.scores_.data(),
                              s.boundaries_.data(), s.scores_.size(), states ? s.char_states_.data() : nullptr,
                              states ? s.type_states_.data() : nullptr, n, &nch));
    s.scores_.resize(n - 1);
    s.boundaries_.resize(n - 1);
    s.predictor_ = this;
    s.tags_.clear();
    s.tags_filled_ = false;
}

inline std::string Token::surface() const {
    return sentence->text_.substr(sentence->pos_[start_], sentence->pos_[end_] - sentence->pos_[start_]);
}
inline std::vector<std::optional<std::string>> Token::tags() const {
    const size_t k = sentence->n_tags();
    return {sentence->tags_.begin() + long((end_ - 1) * k), sentence->tags_.begin() + long(end_ * k)};
}

}  // namespace vaporetto
