/* vaporetto_b200 — C ABI of the CUDA `Predictor::predict` path.
 *
 * The reference (daac-tools/vaporetto, crate `vaporetto` 0.6.5) has no FFI layer: its surface is the
 * Rust API `Model` / `Predictor` / `Sentence` (vaporetto/src/lib.rs:82-91).  Every entry point below
 * names the Rust item it stands in for (paths relative to the reference's vaporetto/src/).  A Rust shim
 * that keeps the crate API and forwards to these symbols is sketched in INTEGRATION.md.
 *
 * Conventions
 *  - every function returns a vpt_status (0 = ok); the message of the last failure on the calling thread
 *    is available from vpt_last_error() (mirrors `VaporettoError`'s Display, errors.rs:41-56).
 *  - no panics/aborts cross the ABI; CUDA failures are reported as VPT_CUDA_ERROR.
 *  - a predictor is immutable after creation and may be shared by many host threads
 *    (`Predictor: Send + Sync`, shared as Arc<Predictor> in vaporetto_tantivy/src/lib.rs:62-67);
 *    each call uses its own CUDA stream and staging buffers.
 *  - there is no CPU fallback: without a usable CUDA device every compute entry point fails.
 */
#ifndef VAPORETTO_B200_H
#define VAPORETTO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef enum vpt_status {
    VPT_OK = 0,
    VPT_INVALID_MODEL = 1,    /* VaporettoError::InvalidModel    (errors.rs:16) */
    VPT_INVALID_ARGUMENT = 2, /* VaporettoError::InvalidArgument (errors.rs:19) */
    VPT_INVALID_SENTENCE = 3, /* VaporettoError::InvalidSentence (errors.rs:22) */
    VPT_DECODE_ERROR = 4,     /* VaporettoError::DecodeError     (errors.rs:34) */
    VPT_IO_ERROR = 5,         /* VaporettoError::IOError         (errors.rs:28) */
    VPT_CUDA_ERROR = 16,
    VPT_UNSUPPORTED = 17,
    VPT_INTERNAL = 18
} vpt_status;

/* per-sentence status written by the batch entry points (what `Sentence::from_raw` / `update_raw`
 * would have rejected, sentence.rs:174-189, plus malformed UTF-8 which a Rust &str cannot hold) */
enum {
    VPT_SENT_OK = 0,
    VPT_SENT_EMPTY = 1,        /* "text: must contain at least one character" */
    VPT_SENT_NUL = 2,          /* "text: must not contain NULL" */
    VPT_SENT_BAD_UTF8 = 3,
    VPT_SENT_BAD_RANGE = 4     /* vpt_token_spans_dev only: the document's offsets are not a range in the batch */
};

#define VPT_NO_PATTERN 0xFFFFFFFFu /* u32::MAX in char_pma_states / type_pma_states (boundary_tag_scorer.rs:122-123) */

typedef struct vpt_model vpt_model;
typedef struct vpt_predictor vpt_predictor;

/* Message of the last error raised on this thread ("" if none). */
const char* vpt_last_error(void);

/* ---- Model --------------------------------------------------------------------------------------- */

/* `Model::read_slice(&[u8]) -> Result<(Model, &[u8])>` (model.rs:127-134) and `Model::read` (model.rs:142-153).
 * `data` is the raw (already un-zstd'd) model image; `*consumed` (nullable) receives the bytes used. */
int vpt_model_read(const uint8_t* data, size_t len, vpt_model** out, size_t* consumed);

/* The model loading of the reference's `predict` command (predict/src/main.rs:110-111:
 * `Model::read(&mut zstd::Decoder::new(File::open(path)?)?)`): `data` is the content of a *.model.zst file.  The zstd
 * frames are decoded inside the library (libzstd.so.1, opened at run time; IOError when it is absent); an image that
 * does not start with a zstd magic number is read as a raw model, as `vpt_model_read` does. */
int vpt_model_read_zstd(const uint8_t* data, size_t len, vpt_model** out);

/* `KyteaModel::read` + `Model::try_from(KyteaModel)` (kytea_model.rs:423-450, :453-550; the reference's
 * `convert_kytea_model` tool): a KyTea binary model becomes a vaporetto model — the word-segmentation linear model's
 * character / type n-gram weights (i16 -> i32, truncated to the window), bias, and the dictionary words with their
 * left / inside / right weights by word-length bucket; KyTea's tag models are not converted (as in the reference). */
int vpt_model_read_kytea(const uint8_t* data, size_t len, vpt_model** model_out);

/* `Model::dictionary` (model.rs:155-158) / `WordWeightRecord::get_word, get_weights, get_comment` (dict_model.rs:53-66):
 * record `index` of the model's word dictionary; the pointers stay valid until the model is freed or its dictionary
 * replaced. */
uint64_t vpt_model_dictionary_len(const vpt_model* model);
int vpt_model_dictionary_get(const vpt_model* model, uint64_t index, const char** word, const int32_t** weights,
                             uint64_t* n_weights, const char** comment);

/* `Model::replace_dictionary` (model.rs:160-163) with the check of `WordWeightRecord::new` (dict_model.rs:39-50):
 * every record needs chars(word) + 1 weights, else VPT_INVALID_ARGUMENT and the model is unchanged.  `comments` (and
 * its elements) may be NULL.  With vpt_model_to_vec this is the reference's `manipulate_model` tool. */
int vpt_model_replace_dictionary(vpt_model* model, const char* const* words, const int32_t* const* weights,
                                 const uint64_t* n_weights, const char* const* comments, uint64_t n_records);

/* `Model::to_vec` / `Model::write` (model.rs:99-120): the model file image (magic + bincode standard encoding);
 * byte-identical to what the reference writes for the same model.  Release the buffer with vpt_blob_free. */
int vpt_model_to_vec(const vpt_model* model, uint8_t** bytes_out, uint64_t* len_out);
void vpt_model_free(vpt_model* model);

/* ---- Predictor ----------------------------------------------------------------------------------- */

/* `Predictor::new(model: Model, predict_tags: bool) -> Result<Predictor>` (predictor.rs:450-508).
 * Consumes `model` (it is freed, success or failure), builds the merged weight rows and the flat device
 * tables, and uploads them to CUDA device `device`.  device = -1 creates a host-only handle (tag prediction and
 * Sentence helpers work, every scoring entry point fails with VPT_CUDA_ERROR — there is no CPU scoring path). */
int vpt_predictor_new(vpt_model* model, int predict_tags, int device, vpt_predictor** out);
void vpt_predictor_free(vpt_predictor* predictor);

typedef struct vpt_predictor_info {
    int32_t device;
    int32_t predict_tags;       /* created with predict_tags = true */
    int32_t n_tags;             /* Sentence::n_tags after fill_tags (predictor.rs:553) */
    int32_t char_scorer;        /* 0 none, 1 Boundary, 2 BoundaryTag       (char_scorer.rs:84-89) */
    int32_t type_scorer;        /* 0 none, 1 Boundary, 2 BoundaryCache, 3 BoundaryTag (type_scorer.rs:92-101) */
    int32_t fast_path;          /* 1: k_score_fast (all rows inline), 0: k_score_general */
    int32_t bias;
    int32_t char_window, type_window;
    uint32_t n_char_patterns, n_type_patterns;
    uint32_t n_char_nodes, n_type_nodes;
    uint32_t max_char_pattern_len;
    uint64_t blob_bytes;        /* size of the device-resident model */
    int32_t kernel_launches_per_batch;
} vpt_predictor_info;
int vpt_predictor_get_info(const vpt_predictor* predictor, vpt_predictor_info* out);

/* The scoring kernel a batch of this predictor runs, the template variant of it and its tile geometry.  with_states != 0:
 * a batch that asks for pattern-id states (char_states_out / type_states_out).  Works on host-only handles too. */
typedef struct vpt_kernel_plan {
    int32_t kernel;             /* 1 k_fused, 2 k_tile_fast, 3 k_score_fast, 4 k_score_general */
    int32_t seeds_smem;         /* k_fused, k_tile_fast: perfect-hash seed bytes staged in shared memory */
    int32_t common_shape;       /* k_fused: char window 3 + type window 3 with split tables */
    int32_t deep;               /* k_fused: 0 patterns <= 3 chars, 1 longer ones, 2 also rows outside the inline window */
    int32_t states;             /* k_fused: pattern-id states are written */
    int32_t r0_fixed;           /* k_tile_fast: inline window start -3 compiled in */
    int32_t general;            /* k_tile_fast: general rows */
    int32_t split3;             /* k_tile_fast: type window 3 with split tables */
    int32_t overflow;           /* k_tile_fast: long dictionary rows */
    int32_t text_cap;           /* bytes of text a tile stages (0: no tiles, one warp per sentence) */
    int32_t slot_cap;           /* character + separator slots per tile */
    int32_t gap;                /* separator slots in front of every sentence of a tile */
    int32_t lag;                /* k_fused: slots between a boundary's slot and the slot that finishes it */
    int32_t sub_blocks;         /* independent 256-thread sub-blocks per CTA */
    int32_t group;              /* sentences per group */
} vpt_kernel_plan;
int vpt_predictor_kernel_plan(const vpt_predictor* predictor, int with_states, vpt_kernel_plan* out);

/* Flat device model: serialise on one rank, broadcast as bytes (NCCL), rebuild on the others.
 * (Replaces `Predictor::serialize_to_vec` / `deserialize_from_slice_unchecked`, predictor.rs:640-664, whose
 * daachorse-private layout is not reproducible; the blob format is this library's own.)
 * Predictors made from a blob score boundaries; tag prediction needs vpt_predictor_new. */
/* Host-only build of the flat model (no CUDA device needed): what vpt_predictor_new uploads.  Consumes `model`.
 * The returned buffer is released with vpt_blob_free. */
int vpt_blob_build(vpt_model* model, int predict_tags, uint8_t** blob_out, uint64_t* len_out);
void vpt_blob_free(uint8_t* blob);
uint64_t vpt_predictor_blob_size(const vpt_predictor* predictor);
int vpt_predictor_blob_export(const vpt_predictor* predictor, void* dst, uint64_t capacity);
int vpt_predictor_from_blob(const void* blob, uint64_t len, int device, vpt_predictor** out);

/* ---- predict ------------------------------------------------------------------------------------- */

/* Batched `Predictor::predict(&self, &mut Sentence)` (predictor.rs:518-543) over HOST buffers.
 *
 * Sentence i is utf8[byte_offsets[i] .. byte_offsets[i+1]) (raw text, as given to `Sentence::from_raw`).
 * With n_i = number of characters of sentence i, its boundaries occupy
 *   scores_out / boundaries_out [ bound_offsets_out[i] .. bound_offsets_out[i] + max(n_i - 1, 0) )
 * (`Sentence::boundary_scores()`, sentence.rs:1040-1046; `Sentence::boundaries()` as 0 = NotWordBoundary,
 * 1 = WordBoundary, sentence.rs:70-82) and, when requested, its pattern states occupy
 *   char_states_out / type_states_out [ char_offsets_out[i] .. + n_i )
 * (`char_pma_states` / `type_pma_states`, sentence.rs:92-93; only meaningful for a predictor created with
 * predict_tags = true on a model that has tag models).
 * Rejected sentences (status_out[i] != 0) keep their slots, filled with zeros / VPT_NO_PATTERN.
 *
 * out_capacity / states_capacity are the element capacities of the output arrays; if too small the call
 * fails with VPT_INVALID_ARGUMENT and the required sizes are in *n_boundaries_out / *n_chars_out.
 * scores_out, char_states_out, type_states_out, char_offsets_out, status_out may be NULL (without scores_out the
 * inline-row kernel skips the score stores and only boundaries cross PCIe).
 * For full PCIe bandwidth pass page-locked (pinned) host buffers.  The batch flows through an internal pipeline
 * (copy-in + kernels and copy-out on separate streams, four chunks in flight, chunk sizes ramping up from 1/8 of
 * env VPT_CHUNK_SENTENCES, default 262144); VPT_TRACE=1 prints its per-chunk timeline to stderr. */
int vpt_predict_batch(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                      int32_t* scores_out, uint8_t* boundaries_out, size_t out_capacity, uint64_t* bound_offsets_out,
                      int32_t* status_out, uint32_t* char_states_out, uint32_t* type_states_out,
                      size_t states_capacity, uint64_t* char_offsets_out, uint64_t* n_boundaries_out,
                      uint64_t* n_chars_out);

/* Same over DEVICE buffers, asynchronous on `cuda_stream` (a cudaStream_t; NULL = default stream).
 * d_utf8 must be 16-byte aligned and its allocation readable up to the next multiple of 16 bytes.
 * d_workspace: vpt_workspace_size(n_sent) bytes of scratch.  d_scores/d_boundaries must hold the batch's
 * total boundary count (an upper bound is total_bytes - 1); d_bound_offsets [n_sent+1];
 * d_status [n_sent]; d_char_states / d_type_states / d_char_offsets nullable. */
uint64_t vpt_workspace_size(size_t n_sent);

/* PCI bus id ("0000:1b:00.0") of CUDA device `device` as this process sees it (CUDA_VISIBLE_DEVICES applied): what a
 * launcher needs to bind a rank to the GPU's NUMA node (/sys/bus/pci/devices/<id>/numa_node).  buf: >= 16 bytes. */
int vpt_device_pci_bus_id(int device, char* buf, size_t capacity);
int vpt_predict_batch_dev(const vpt_predictor* predictor, const uint8_t* d_utf8, const uint64_t* d_byte_offsets,
                          size_t n_sent, void* d_workspace, uint64_t workspace_bytes, int32_t* d_scores,
                          uint8_t* d_boundaries, uint64_t* d_bound_offsets, int32_t* d_status,
                          uint32_t* d_char_states, uint32_t* d_type_states, uint64_t* d_char_offsets,
                          void* cuda_stream);

/* vpt_predict_batch_dev with CUDA events recorded on `cuda_stream` around each stage; synchronises the stream
 * and returns the device time of each stage in milliseconds: stage_ms[0] = k_count, [1] = k_scan_groups,
 * [2] = k_score_*  (bench.py's roofline leg times the dominant kernel with this). */
int vpt_predict_batch_dev_profiled(const vpt_predictor* predictor, const uint8_t* d_utf8,
                                   const uint64_t* d_byte_offsets, size_t n_sent, void* d_workspace,
                                   uint64_t workspace_bytes, int32_t* d_scores, uint8_t* d_boundaries,
                                   uint64_t* d_bound_offsets, int32_t* d_status, uint32_t* d_char_states,
                                   uint32_t* d_type_states, uint64_t* d_char_offsets, void* cuda_stream,
                                   float* stage_ms);

/* Single-sentence `Predictor::predict` (batch of one).  Returns VPT_INVALID_ARGUMENT with the reference's
 * message for an empty text or a text containing U+0000 (sentence.rs:174-189).  *n_chars_out receives n;
 * scores_out/boundaries_out need n-1 entries (capacity in elements), states n entries (nullable).
 * Sentences of up to 2 KiB on an inline-row model take a path without copy calls: the text goes into a pinned block the
 * kernel reads over PCIe, the results are stored into the same block: one launch + one synchronisation per call, which
 * costs more than a CPU needs to score such a sentence (batch the sentences: vpt_predict_batch / vpt_tokenize_lines). */
int vpt_predict(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes, int32_t* scores_out,
                uint8_t* boundaries_out, size_t out_capacity, uint32_t* char_states_out, uint32_t* type_states_out,
                size_t states_capacity, uint64_t* n_chars_out);

/* ---- tags on the device (`Predictor::predict_tags`, predictor.rs:546-637, for a whole batch) ------------------------
 * After vpt_predict_batch_dev with state outputs: for every character position i (indexed like the states, by
 * d_char_offsets) that ends a token known to the tag model, d_tag_token[i] = token id (else -1) and
 * d_tag_cand[i * n_tags + k] = index of the chosen candidate of tag slot k (else -1): the arrays vpt_fill_tags writes for
 * one sentence.  Token lookup (exact, by bytes), the weight vectors keyed by (pattern id, token, rel position) with the
 * reference's suffix merge (PositionalWeightWithTag +=, predictor.rs:242-262) and the per-slot arg-max (first strict
 * maximum, predictor.rs:286-304) run in one kernel, k_tags; tokens of any length are served.  *d_unserved (nullable,
 * zero it first) counts tokens whose own tag model exceeds the limits of the device tables (more than 64 scores or 8 tag
 * slots; none of the reference's models): their entries are -1 and vpt_fill_tags serves them.  Returns VPT_UNSUPPORTED when the whole model is beyond
 * the limits, VPT_INVALID_ARGUMENT for a predictor created with predict_tags = false (the reference panics).
 * d_utf8 must be 16-byte aligned and its allocation readable up to the next multiple of 16 bytes, as for
 * vpt_predict_batch_dev.  d_boundaries holds 0 / 1 per pair of adjacent characters, as vpt_predict_batch_dev writes
 * them; a caller may set its own 0 / 1 boundaries there to have the tags of that segmentation predicted. */
int vpt_predict_tags_batch_dev(const vpt_predictor* predictor, const uint8_t* d_utf8, const uint64_t* d_byte_offsets,
                               size_t n_sent, const int32_t* d_status, const uint8_t* d_boundaries,
                               const uint64_t* d_bound_offsets, const uint64_t* d_char_offsets,
                               const uint32_t* d_char_states, const uint32_t* d_type_states, int32_t* d_tag_token,
                               int32_t* d_tag_cand, uint32_t* d_unserved, void* cuda_stream);

/* Host-buffer form: predict + predict_tags for a batch; the pattern-id states never leave the device.  Outputs as
 * vpt_predict_batch (scores_out nullable) plus tag_token_out [chars], tag_cand_out [chars * n_tags] and
 * char_offsets_out [n_sent + 1]; chars_capacity in characters. */
int vpt_predict_batch_tags(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                           int32_t* scores_out, uint8_t* boundaries_out, size_t out_capacity, uint64_t* bound_offsets_out,
                           int32_t* status_out, int32_t* tag_token_out, int32_t* tag_cand_out, size_t chars_capacity,
                           uint64_t* char_offsets_out, uint64_t* n_boundaries_out, uint64_t* n_chars_out,
                           uint64_t* n_unserved_out);

/* ---- tags (host side; `Sentence::fill_tags` -> `Predictor::predict_tags`, predictor.rs:546-637) ------ */

/* For one sentence with final boundaries (0 not / 1 boundary / 2 unknown, sentence.rs:70-82) and the
 * states produced by predict: for every character position i that ends a token known to the tag model,
 * tag_token_out[i] = token id (else -1) and tag_cand_out[i*n_tags + k] = index of the chosen candidate of
 * tag slot k (else -1).  tag_scores_out (nullable, n_chars * score_stride) receives the raw score vectors
 * (`Predictor::store_tag_scores`, predictor.rs:512).  Fails with VPT_INVALID_ARGUMENT
 * ("this predictor is created with predict_tags = false") where the reference panics (predictor.rs:547-551). */
int vpt_fill_tags(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes, const uint8_t* boundaries,
                  const uint32_t* char_states, const uint32_t* type_states, int32_t* tag_token_out,
                  int32_t* tag_cand_out, int32_t* tag_scores_out, size_t score_stride);
/* tag string of (token id, slot, candidate); NULL if out of range. Valid for the predictor's lifetime. */
const char* vpt_tag_string(const vpt_predictor* predictor, uint32_t token_id, uint32_t slot, uint32_t cand);
/* number of candidates of a slot (0 if out of range) and the score-vector length of a token */
uint32_t vpt_tag_n_candidates(const vpt_predictor* predictor, uint32_t token_id, uint32_t slot);
uint32_t vpt_tag_score_len(const vpt_predictor* predictor, uint32_t token_id);
uint32_t vpt_tag_n_tokens(const vpt_predictor* predictor);
/* number of tag slots of a token's own model (0 if out of range): `Token::tag_candidates` (sentence.rs:1219-1250) has one
 * list per slot, empty slots included, which vpt_tag_n_candidates cannot tell from slots that do not exist */
uint32_t vpt_tag_n_slots(const vpt_predictor* predictor, uint32_t token_id);

/* predict (+ fill_tags) of a batch with COMPACT results, for callers that want the segmentation and the tags rather
 * than the score strip: what crosses PCIe is one bit per boundary and one small record per token.
 *   boundary_bits_out  the boundaries of all sentences as one bit stream (bit k of the stream = bit k % 32 of word
 *                      k / 32; 1 = WordBoundary): sentence s owns the bits [B_s, B_s + max(n_chars_out[s], 1) - 1)
 *                      with B_s = the sum over the earlier sentences (CharacterBoundary values of
 *                      `Sentence::boundaries()`, sentence.rs:1016-1046; vpt_unpack_boundaries gives the byte form);
 *   n_chars_out[s]     characters of the sentence (a rejected sentence, status_out[s] >= 2, keeps its count and owns
 *                      zero bits; an empty one has 0); status_out[s] as in vpt_predict_batch;
 *   n_tokens_out[s]    (nullable unless tags are requested) tokens of the sentence = boundaries set + 1;
 *   token_ids_out / token_cands_out (both NULL: no tag prediction; needs predict_tags = true otherwise): token r of
 *                      sentence s in text order is record T_s + r (T_s = the sum of n_tokens_out over the earlier
 *                      sentences): the token id for vpt_tag_string (-1: the token has no tag model) and, per tag slot,
 *                      the chosen candidate as one byte (255: none) -- `Predictor::predict_tags`, predictor.rs:546-637,
 *                      the same choice vpt_predict_batch_tags reports per character.
 * The totals come back in *n_boundaries_out / *n_tokens_total_out; *n_unserved_out counts tokens whose own tag model
 * exceeds the device limits (0 for the reference's models; vpt_fill_tags serves those; the length of a token never
 * matters).  Too small capacities return
 * InvalidArgument with the totals set. */
int vpt_predict_batch_compact(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets,
                              size_t n_sent, uint32_t* boundary_bits_out, size_t bits_capacity_words,
                              uint32_t* n_chars_out, uint8_t* status_out, uint32_t* n_tokens_out, int32_t* token_ids_out,
                              uint8_t* token_cands_out, size_t token_capacity, uint64_t* n_boundaries_out,
                              uint64_t* n_tokens_total_out, uint64_t* n_unserved_out);
/* Tag candidate scores (`Predictor::store_tag_scores(true)`, predictor.rs:511-514, as `Token::tag_candidates`,
 * sentence.rs:1219-1250, reads them) of the batch, next to the token records of vpt_predict_batch_compact.  The other
 * arguments and results are those of vpt_predict_batch_compact; tags are required (token_ids_out), and a predictor made
 * with predict_tags = 0 gets its message.  With tag_scores_out == NULL the call IS vpt_predict_batch_compact.
 *  - Which records.  A record gets scores exactly when its token_ids_out entry is >= 0.  Unknown tokens, tokens beyond the
 *    device limits (counted in *n_unserved_out; vpt_fill_tags serves them with scores) and tokens whose model is
 *    malformed (more candidates than scores: vpt_fill_tags reports InvalidModel) have id -1 and no scores.
 *  - What.  The token's whole score vector, vpt_tag_score_len(token id) entries: its bias plus the char and type scorers'
 *    tag weights, added with i32 wrap-around -- the `scores` predict_tags stores.  The candidate chosen for a slot with
 *    two or more candidates is the first strict maximum of that slot's part of the vector (the parts follow each other in
 *    slot order; slots with fewer than two candidates own no part).
 *  - Layout.  The vectors of all records are concatenated in record order, with no gaps and no per-record offsets: the
 *    vector of record r starts at the sum of vpt_tag_score_len(token_ids_out[q]) over the earlier records q with an id
 *    >= 0.  The same input gives the same bytes.
 *  - Capacity.  score_capacity is the number of int32 entries tag_scores_out holds; *n_scores_total_out receives the
 *    total.  If it is too small the call returns VPT_INVALID_ARGUMENT with *n_scores_total_out set to the number needed.
 *    An upper bound is token_capacity x the largest vpt_tag_score_len over the predictor's tokens. */
int vpt_predict_batch_compact_tag_scores(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets,
                                         size_t n_sent, uint32_t* boundary_bits_out, size_t bits_capacity_words,
                                         uint32_t* n_chars_out, uint8_t* status_out, uint32_t* n_tokens_out,
                                         int32_t* token_ids_out, uint8_t* token_cands_out, size_t token_capacity,
                                         uint64_t* n_boundaries_out, uint64_t* n_tokens_total_out, uint64_t* n_unserved_out,
                                         int32_t* tag_scores_out, size_t score_capacity, uint64_t* n_scores_total_out);
/* bits [first_bit, first_bit + n) of a boundary bit stream as bytes (0 / 1) */
int vpt_unpack_boundaries(const uint32_t* boundary_bits, uint64_t first_bit, uint64_t n, uint8_t* boundaries_out);

/* ---- Sentence helpers (host side) ----------------------------------------------------------------- */

/* `CharacterType::get_type` per character (sentence.rs:50-67) / `Sentence::char_types()` (sentence.rs:993).
 * Returns the reference's InvalidArgument errors for empty text / NUL.  *n_chars_out receives n. */
int vpt_char_types(const uint8_t* utf8, size_t n_bytes, uint8_t* types_out, size_t capacity, uint64_t* n_chars_out);

/* `SplitLinebreaksFilter::filter(&mut Sentence)` (vaporetto_rules/src/sentence_filters/split_linebreaks.rs:9-37) on the
 * host, for the Sentence API: the boundary on either side of every '\r' / '\n' becomes WordBoundary (1).  (The lines
 * path never sees these characters inside a sentence: it splits at them.) */
int vpt_split_linebreaks(const uint8_t* utf8, size_t n_bytes, uint8_t* boundaries, size_t n_boundaries);

/* `ConcatGraphemeClustersFilter::filter(&mut Sentence)` (vaporetto_rules/src/sentence_filters/
 * concat_grapheme_clusters.rs:10-35) on the host, for the Sentence API: `boundaries` (n_chars - 1 values, 0 / 1, as
 * vpt_predict returns them) loses every boundary inside an extended grapheme cluster of the text (UAX #29 as in
 * unicode-segmentation 1.12 `graphemes(true)`; the rule engine vpt_tokenize_lines runs on the device for
 * VPT_WSCONST_GRAPHEME). */
int vpt_concat_grapheme_clusters(const uint8_t* utf8, size_t n_bytes, uint8_t* boundaries, size_t n_boundaries);

/* `Sentence::write_tokenized_text` (sentence.rs:850-886): tokens joined by ' ', with '/tag' suffixes when
 * tag_token/tag_cand are given (NULL otherwise), escaping ' ', '\\', '/'.  Tokens adjacent to an Unknown
 * boundary are skipped.  Returns the byte length needed in *len_out; writes at most `capacity` bytes. */
int vpt_write_tokenized_text(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes,
                             const uint8_t* boundaries, const int32_t* tag_token, const int32_t* tag_cand,
                             char* buf, size_t capacity, uint64_t* len_out);

/* `Sentence::write_partial_annotation_text` (sentence.rs:907-944): the characters of the text with a marker between each
 * two ('-' NotWordBoundary, '|' WordBoundary, ' ' Unknown; `boundaries` holds n_chars - 1 values 0 / 1 / 2) and, behind
 * every character whose tag_cand row has a tag (tag_token/tag_cand as vpt_fill_tags writes them, NULL for none), '/' +
 * tag for each slot up to the last one that has a tag.  Nothing is escaped, as in the reference: a tag holding ' ', '-',
 * '|', '/' or '\' does not read back through from_partial_annotation.  Returns the byte length needed in *len_out;
 * writes at most `capacity` bytes, the last of them a NUL. */
int vpt_write_partial_annotation_text(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes,
                                      const uint8_t* boundaries, const int32_t* tag_token, const int32_t* tag_cand,
                                      char* buf, size_t capacity, uint64_t* len_out);

/* ---- Whole-buffer tokenisation: the reference CLI's loop on the device ----------------------------- */

/* The loop of the reference's `predict` CLI (predict/src/main.rs:126-181) over a whole buffer of raw file bytes:
 *   for line in stdin.lines():
 *       s = KyteaFullwidthFilter(line) unless --no-norm          (main.rs:98,154; vaporetto_rules kytea_fullwidth.rs)
 *       if s.update_raw(..).is_ok() { predict(s); copy the boundaries to the original line; write_tokenized_text }
 *       write "\n"
 * Lines are split ON THE DEVICE with `BufRead::lines` semantics ('\n' or "\r\n" terminated; the last line may
 * be unterminated; a trailing '\n' adds no empty line), scored by the same kernels as vpt_predict_batch (with the
 * full-width character map applied to the code points the kernels look up when no_norm == 0; the map is one
 * character to one character, so the boundaries apply to the original text), and the tokenised ORIGINAL text
 * (' ' between tokens; '\\' before ' ', '\\', '/': sentence.rs:850-886) is materialised on the device: the only
 * transfers are the input bytes in and the output bytes out.  Lines that update_raw rejects (empty, or
 * containing U+0000) produce an empty line as in the CLI; so do lines that are not valid UTF-8 (the CLI stops
 * with an I/O error on those).  Score printing (--scores, --tag-scores) is not part of this path; tags: below.
 * `no_norm`: the CLI flag of the same name (0 = apply KyteaFullwidthFilter, the CLI default).
 * `wsconst_types`: the CLI's `--wsconst D/R/H/T/K/O` options as a bit set, bit t for CharacterType t (VPT_WSCONST_*):
 * `KyteaWsConstFilter` (vaporetto_rules/src/sentence_filters/kytea_wsconst.rs:27-44) clears the boundary between two
 * characters of such a type after prediction (types of the filtered text when no_norm == 0, main.rs:157);
 * VPT_WSCONST_GRAPHEME is `--wsconst G`: `ConcatGraphemeClustersFilter` (sentence_filters/concat_grapheme_clusters.rs:
 * 10-35) clears the boundaries inside every extended grapheme cluster (UAX #29 as in unicode-segmentation 1.12).
 * `out` receives the output lines, each terminated by '\n' (at most 3 * n_bytes + n_lines bytes); *out_len
 * the number of bytes produced (also when `out_capacity` was too small, which returns InvalidArgument);
 * *n_lines the number of input lines.  Chunk size of the internal pipeline: env VPT_CHUNK_BYTES (16 MiB, with
 * smaller chunks at both ends); VPT_TRACE=1 prints the pipeline's per-chunk timeline to stderr.
 * For input that arrives in pieces or does not fit in memory (a pipe, a file read in pieces, an interactive session),
 * the line stream below (vpt_line_stream_*, VPT_STREAM_TOKENIZE) gives the same output in bounded memory. */
#define VPT_WSCONST_DIGIT (1u << 1)    /* --wsconst D */
#define VPT_WSCONST_ROMAN (1u << 2)    /* --wsconst R */
#define VPT_WSCONST_HIRAGANA (1u << 3) /* --wsconst H */
#define VPT_WSCONST_KATAKANA (1u << 4) /* --wsconst T */
#define VPT_WSCONST_KANJI (1u << 5)    /* --wsconst K */
#define VPT_WSCONST_OTHER (1u << 6)    /* --wsconst O */
#define VPT_WSCONST_GRAPHEME (1u << 7) /* --wsconst G: ConcatGraphemeClustersFilter */
int vpt_tokenize_lines(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes, int no_norm,
                       uint32_t wsconst_types, uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines);

/* The same loop with the CLI's `--predict-tags` (predict/src/main.rs:130-136,159-166): `fill_tags` on the sentence that
 * was predicted (after the post-filters), tags copied to the original line, `write_tokenized_text` with tags
 * (sentence.rs:850-886: every token is followed by '/' + tag for its tag slots up to the last one that has a tag, the
 * tag strings escaped like the surface).  Tag prediction (token lookup by the bytes of the pre-filtered token, tag
 * weights, arg-max) and the output with its tag strings run on the device; the predictor must have been created with
 * predict_tags = 1.  `out` needs room for the tags: at most 3 * n_bytes + n_lines + n_bytes * (longest tag suffix).
 * Returns VPT_UNSUPPORTED, before writing anything, when the tag model of any token exceeds the limits of the device
 * tables (see vpt_predict_tags_batch_dev): this path has no per-token fall-back to vpt_fill_tags.
 * The line stream (vpt_line_stream_*, VPT_STREAM_TOKENIZE with predict_tags) gives the same output in bounded memory. */
int vpt_tokenize_lines_tags(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes, int no_norm,
                            uint32_t wsconst_types, uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines);

/* The reference's `evaluate` command (evaluate/src/main.rs:69-195) over a buffer holding a gold corpus in the tokenized
 * format (`まぁ/名詞/マー 社長/名詞/シャチョー ...`, one sentence per line).  Lines are split as in vpt_tokenize_lines;
 * an empty line is skipped.  Every other line is parsed by `Sentence::from_tokenized` (sentence.rs:285-467) for the
 * gold boundaries and tags, predicted like the `predict` CLI (KyteaFullwidthFilter unless `no_norm`, the
 * `wsconst_types` post-filters, and with `predict_tags` fill_tags) and compared with the gold:
 *   - char metric (main.rs:121-147): tp, tn, fp, fn over all character boundaries;
 *   - word metric (main.rs:149-191, Nagata 1994): n_sys / n_ref are the system / gold tokens, n_cor the tokens both
 *     have at the same span with equal tags.  Tags compare as the reference's Vec<Option<String>>: with no_norm and no
 *     tag prediction the sentence keeps the gold tags (always equal); normalised without tag prediction it has none
 *     (equal only on lines without a tag field); with tag prediction and a model with k > 0 tag slots, a token is equal
 *     where its line has exactly k gold tag fields on some token and every slot matches (a predictor with k == 0 keeps
 *     the sentence's tags, predictor.rs:553).
 * Parsing, prediction and both metrics run on the device; only the totals (and the optional per-line counts) come back.
 * Errors stop the whole call, as they stop the CLI, and name the 0-based line (every line counts, empty ones too):
 * the lowest bad line's first violation, in the order the reference's character loop meets them, returns
 * VPT_INVALID_ARGUMENT "InvalidArgumentError: tokenized_text: <reason>"; a line that is not valid UTF-8 returns
 * VPT_IO_ERROR ("stream did not contain valid UTF-8").  Two documented differences: a line holding a lone '\' has no
 * character and is the "must contain at least one character" error (the reference divides by zero,
 * sentence.rs:450), and the counts are 64-bit (the reference's i32 counters wrap beyond 2^31).
 * `predict_tags` and `wsconst_types` are checked as in vpt_tokenize_lines_tags.  `line_counts` (nullable) receives
 * tp, tn, fp, fn, n_sys, n_ref, n_cor of every input line (zeros for empty lines), `line_capacity` rows of 7; a
 * buffer with fewer rows than lines returns VPT_INVALID_ARGUMENT after the totals are filled in.
 * The line stream (vpt_line_stream_*, VPT_STREAM_EVALUATE) gives the same totals on a corpus fed in pieces. */
typedef struct vpt_eval_counts {
    uint64_t n_lines, n_sentences;       /* input lines; non-empty lines evaluated */
    uint64_t tp, tn, fp, fn;             /* --metric char  (evaluate/src/main.rs:121-147) */
    uint64_t n_sys, n_ref, n_cor;        /* --metric word  (:149-191, Nagata 1994) */
} vpt_eval_counts;
int vpt_evaluate_lines(const vpt_predictor* predictor, const uint8_t* utf8, size_t n_bytes, int no_norm,
                       uint32_t wsconst_types, int predict_tags, vpt_eval_counts* out,
                       uint32_t* line_counts /* nullable, [n_lines * 7] */, uint64_t line_capacity);

/* ---- Line stream: the same loops fed in pieces, for input of any size -------------------------------------------------
 *
 * vpt_tokenize_lines, vpt_tokenize_lines_tags and vpt_evaluate_lines take one whole buffer, and their output buffer
 * grows with it.  A line stream runs the same loops on input fed in pieces of any size, split at any byte, as the
 * reference's CLIs read stdin line by line: the output is handed back in input order as chunks complete, and host
 * memory stays bounded by the pipeline depth times the chunk size, plus the longest line.
 *
 * Equivalence: for every way of cutting a buffer B into feeds, the stream gives what the whole-buffer call on B with
 * the same flags gives: the concatenation of the bytes passed to `write`, and *n_lines, equal the output and line
 * count of vpt_tokenize_lines (vpt_tokenize_lines_tags with predict_tags); the totals, and the error status and message
 * with its "(line N)", equal those of vpt_evaluate_lines.  Cuts inside a multi-byte character or between '\r' and
 * '\n', empty feeds, an unterminated last line and a trailing '\r' included: the stream cuts its input only after a
 * '\n', so every chunk is a run of complete lines.  (A line over 1 GiB is an error in both; the whole-buffer calls
 * report it before anything else, the stream when it reaches the line.)
 *
 * Flags are checked by vpt_line_stream_new with the statuses and messages of the whole-buffer calls (wsconst bits, tags
 * on a predictor without tags, a tag model beyond the device limits).
 *
 * Progress:
 *  - feed copies the bytes into pinned staging and returns; the caller may reuse its buffer at once.  A chunk is
 *    submitted once the open chunk reaches the chunk size (env VPT_CHUNK_BYTES, 16 MiB; the first chunks ramp up from
 *    1/8 of it) and holds a '\n'.  With four chunks in flight, feed waits for the oldest and delivers its output: this
 *    back-pressure bounds the memory.
 *  - flush submits every complete line held, waits for all chunks in flight and delivers their output; a partial
 *    last line stays held.
 *  - finish submits the rest, an unterminated last line included, and delivers everything.  *n_lines (nullable)
 *    receives the number of input lines; `counts` (nullable; VPT_STREAM_EVALUATE) the totals of vpt_evaluate_lines.
 *    There are no per-line counts on the stream.
 * Memory: one pinned input buffer per chunk in flight plus the open one, a pinned output buffer sized by the largest
 * chunk output met (tokenize), and the device scratch of four whole-buffer chunks; none of it grows with the total
 * input, only a line longer than a chunk grows the open buffer.
 * `write` (VPT_STREAM_TOKENIZE) is called in input order on the thread that called feed / flush / finish, never with
 * zero bytes; the bytes are valid only during the call.  A nonzero return aborts the stream with VPT_IO_ERROR ("write
 * callback failed").
 * Errors poison the stream: after any error (a bad gold line, invalid UTF-8 in evaluate, a line over 1 GiB, a CUDA
 * error, a failed `write`) every later call returns the same status and message, and `write` is not called again.
 * feed, flush or finish after finish return VPT_INVALID_ARGUMENT.
 * vpt_line_stream_free works at any point, finished or not: it waits for the stream's work on the device, calls
 * nothing back, and leaves the predictor usable.  A stream is used by one thread at a time; several streams on one
 * predictor (and whole-buffer calls) may run concurrently.  VPT_TRACE=1 prints the stream's per-chunk timeline. */
typedef struct vpt_line_stream vpt_line_stream;
typedef int (*vpt_stream_write_fn)(void* ctx, const uint8_t* bytes, size_t n);
#define VPT_STREAM_TOKENIZE 0 /* vpt_tokenize_lines / _tags output, through `write` */
#define VPT_STREAM_EVALUATE 1 /* vpt_evaluate_lines totals at finish; `write` unused (may be NULL) */
int vpt_line_stream_new(const vpt_predictor* predictor, int kind, int no_norm, uint32_t wsconst_types, int predict_tags,
                        vpt_stream_write_fn write, void* ctx, vpt_line_stream** out);
int vpt_line_stream_feed(vpt_line_stream* stream, const uint8_t* bytes, size_t n);
int vpt_line_stream_flush(vpt_line_stream* stream);
int vpt_line_stream_finish(vpt_line_stream* stream, uint64_t* n_lines, vpt_eval_counts* counts /* EVALUATE only */);
void vpt_line_stream_free(vpt_line_stream* stream);

/* ---- Tag rules: vaporetto_rules' PatternMatchTagger in the tagged line path --------------------------------------------
 *
 * `PatternMatchTagger::new(rules)` and `filter` (vaporetto_rules/src/sentence_filters/pattern_match_tagger.rs:21-41): a
 * table surface -> [Option<tag>] that supplies tags the model does not predict, typically for out-of-vocabulary words
 * (proper nouns, product names) from a user dictionary.  The filter runs on the sentence that was predicted, right after
 * fill_tags, as if the `predict` CLI's loop called it there (main.rs:130-136,157-159); the tags are then copied to the
 * original line as usual.  For every token, every tag slot j < n_tags that is still None after tag prediction becomes
 * rules[surface][j] when the surface is a key; a rule with fewer entries leaves the later slots None, entries beyond
 * n_tags are ignored, and predicted tags are never overwritten.  Some("") is a tag: it writes a '/' with nothing after
 * it and counts for the last slot written.  With n_tags == 0 (no tag models) the rules do nothing, and rejected lines
 * (invalid UTF-8, U+0000) still print an empty line.
 * Surface matching: unless no_norm, a token is matched by its KyteaFullwidthFilter image, because that is the sentence
 * the filter sees.  Rule keys are not normalised: a half-width key ("ABC") matches only with no_norm; give the
 * full-width key ("ＡＢＣ") for the default.
 *
 * Layout: rule i has the surface surfaces[surface_offsets[i] .. surface_offsets[i+1]) and the tag slots
 * slot_offsets[i] .. slot_offsets[i+1]; slot k is the pair slots[2k] (offset into `tags`, or UINT32_MAX for None),
 * slots[2k+1] (length; 0 is Some("")).  surface_offsets and slot_offsets have n_rules + 1 entries.  Everything is
 * copied: the caller's arrays may be freed on return.  Errors (VPT_INVALID_ARGUMENT, naming the rule): NULL arrays, an
 * offset that decreases or a tag outside `tags`, a surface or tag that is not valid UTF-8, a duplicate surface.  An
 * empty surface, or one containing U+0000, is accepted and never matches.
 * The rules are bound to `predictor` (its device and its n_tags: slots beyond it are dropped here) and must outlive
 * every call and line stream that uses them; they are read-only and may be shared by concurrent calls.  Rules on a
 * call without tag prediction, or with no rules at all, change nothing: the output is that of the call without rules. */
typedef struct vpt_tag_rules vpt_tag_rules;
int vpt_tag_rules_new(const vpt_predictor* predictor, uint64_t n_rules, const uint8_t* surfaces,
                      const uint64_t* surface_offsets, const uint64_t* slot_offsets, const uint32_t* slots,
                      const uint8_t* tags, uint64_t tags_len, vpt_tag_rules** out);
void vpt_tag_rules_free(vpt_tag_rules* rules);
/* The largest device output buffer, in bytes, that a chunk of a call with these rules has used (a diagnostic of the
 * output sizing: a chunk's buffer is sized by the rule suffixes its tokens actually matched, not by the longest rule).
 * On a stream with score dumps (vpt_line_stream_new_scores) it is the buffer of the token lines, which the rules size;
 * the dumps behind them are sized separately. */
uint64_t vpt_tag_rules_max_output(const vpt_tag_rules* rules);

/* vpt_tokenize_lines_tags with `rules` (nullable: NULL is vpt_tokenize_lines_tags).  Same arguments and errors; a rule's
 * tag can be long, so `out` needs room for the matched rule tags too, and *out_len reports the size needed. */
int vpt_tokenize_lines_tags_rules(const vpt_predictor* predictor, const vpt_tag_rules* rules, const uint8_t* utf8,
                                  size_t n_bytes, int no_norm, uint32_t wsconst_types, uint8_t* out, size_t out_capacity,
                                  uint64_t* out_len, uint64_t* n_lines);
/* vpt_line_stream_new with `rules` (nullable), applied as in vpt_tokenize_lines_tags_rules on a VPT_STREAM_TOKENIZE
 * stream with predict_tags; ignored otherwise. */
int vpt_line_stream_new_rules(const vpt_predictor* predictor, const vpt_tag_rules* rules, int kind, int no_norm,
                              uint32_t wsconst_types, int predict_tags, vpt_stream_write_fn write, void* ctx,
                              vpt_line_stream** out);

/* ---- Partially annotated lines: the caller's boundaries stay, the model decides the rest, then tags --------------------
 *
 * Every line is in the format of `Sentence::from_partial_annotation` (sentence.rs:516-631, the reference train CLI's
 * --part corpora): a character, then a marker, then a character, ...: '|' is a word boundary, '-' is not one, ' ' leaves
 * the boundary to the model; tag fields may follow a marker position after '/', and '\' escapes the next character of a
 * tag field.  Lines are split as in vpt_tokenize_lines.  For every line:
 *
 *   pa = Sentence::from_partial_annotation(line)       // given[i]: NotWordBoundary, WordBoundary or Unknown
 *   s  = Sentence::from_raw(pa.as_raw_text())          // KyteaFullwidthFilter of it unless no_norm
 *   predictor.predict(&mut s); the wsconst_types post-filters on s
 *   for every i with given[i] != Unknown: s.boundaries_mut()[i] = given[i]      // the caller's markers win, last
 *   with predict_tags: s.fill_tags(), then the PatternMatchTagger `rules` (nullable)
 *   boundaries and tags onto the raw text; write_tokenized_text; "\n"
 *
 * The output has the format and escaping of vpt_tokenize_lines_tags.  Definitions of this library, not of a reference
 * command:
 *   - the markers apply after the post-filters: a '|' between two Kanji stays with VPT_WSCONST_KANJI;
 *   - the tags in the input are parsed and checked as the reference parses them, and dropped: output tags are predicted
 *     tags and rule tags only (fill_tags resets a sentence's tags, predictor.rs:559-562);
 *   - an empty line gives an empty output line, so output lines stay aligned with input lines
 *     (`from_partial_annotation("")` is an error; the predict CLI likewise prints an empty line for a line it cannot read).
 * A malformed line stops the call, as a bad gold line stops vpt_evaluate_lines, and is named by its 0-based line: the
 * lowest bad line's first violation in the reference's character loop returns VPT_INVALID_ARGUMENT
 * "InvalidArgumentError: partial_annotation_text: <reason> (line N)" with the reference's reasons "must not contain
 * NULL" (a NUL in character position), "contains an invalid boundary character: '<c>'" and "invalid annotation" (the
 * line ends where a character is expected); a line that is not valid UTF-8 returns VPT_IO_ERROR ("stream did not
 * contain valid UTF-8 (line N)") before anything else on that line.  Output delivered before an error (the line stream's
 * `write` calls) is a prefix of the output that ends at a line end.
 * The parse, scoring, post-filters, markers, tags and writer run on the device.  Flags are checked as in
 * vpt_tokenize_lines_tags(_rules); `out`, `out_capacity`, *out_len and *n_lines as there (the output of a line is at most
 * that of its raw text in vpt_tokenize_lines_tags).
 * Not offered: a device-resident variant, keeping the input's tags, and score dumps (partially annotated output is
 * vpt_annotate_lines; partially annotated output that keeps the input's markers and tags is vpt_reannotate_lines). */
int vpt_tokenize_partial_lines(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */,
                               const uint8_t* utf8, size_t n_bytes, int no_norm, uint32_t wsconst_types, int predict_tags,
                               uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines);

/* A line stream of vpt_tokenize_partial_lines: the same output, errors and line count, on input fed in pieces, with
 * the progress, memory and error rules above (a malformed line poisons the stream after the output of the lines before
 * its chunk was written). */
int vpt_line_stream_new_partial(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */, int no_norm,
                                uint32_t wsconst_types, int predict_tags, vpt_stream_write_fn write, void* ctx,
                                vpt_line_stream** out);

/* ---- Partially annotated output: the boundaries the model is unsure of stay open ----------------------------------------
 *
 * The predicted lines in the format of `Sentence::write_partial_annotation_text` (sentence.rs:907-944), with every
 * boundary whose score lies strictly between -margin and margin left Unknown (' '), for an annotator to resolve before
 * the corpus goes to the reference's `train --part`.  Lines are split as in vpt_tokenize_lines.  For every line:
 *
 *   s = Sentence::from_raw(line)                        // KyteaFullwidthFilter of it unless no_norm
 *   predictor.predict(&mut s)
 *   for every boundary i with -margin < score[i] < margin:  s.boundaries_mut()[i] = Unknown      // score: i32
 *   the wsconst_types post-filters on s                 // they set NotWordBoundary, Unknown or not
 *   with predict_tags: s.fill_tags(), then the PatternMatchTagger `rules` (nullable)
 *   boundaries and tags onto the line; write_partial_annotation_text; "\n"
 *
 * So:
 *   - margin 0 leaves nothing Unknown: the output is vpt_tokenize_lines(_tags)'s segmentation in this format;
 *     a score of exactly +-margin is known, and margin 1 leaves only the scores 0 Unknown;
 *   - a boundary a post-filter cleared is '-' whatever its score;
 *   - fill_tags (predictor.rs:567-570) and the rules (iter_tokens, sentence.rs:1273-1299) skip every token next to or
 *     across an Unknown boundary: such tokens have no tags; every other token has the tags vpt_tokenize_lines_tags(_rules)
 *     gives it;
 *   - the characters and the tags are written unescaped, as the reference writes them: a tag that holds ' ', '-', '|',
 *     '/' or '\' (UniDic-style tags such as "名詞-普通名詞-一般") does not read back through from_partial_annotation;
 *   - a line update_raw rejects (empty, with a NUL, not valid UTF-8) gives an empty output line.
 * `margin` must not be negative (VPT_INVALID_ARGUMENT); 0x7FFFFFFF leaves every boundary Unknown that no post-filter
 * decides except those with the score INT32_MIN.  The scoring, margin, post-filters, tags, rules and writer run on the
 * device.  Flags are checked as in vpt_tokenize_partial_lines; `out`, `out_capacity`, *out_len and *n_lines as there
 * (the output of a line is at most that of its text in vpt_tokenize_lines_tags).
 * Not offered: a device-resident variant, score dumps, escaped tags (partially annotated input is
 * vpt_reannotate_lines). */
int vpt_annotate_lines(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */, const uint8_t* utf8,
                       size_t n_bytes, int no_norm, uint32_t wsconst_types, int predict_tags, int32_t margin, uint8_t* out,
                       size_t out_capacity, uint64_t* out_len, uint64_t* n_lines);

/* A line stream of vpt_annotate_lines: the same output and line count on input fed in pieces, with the progress, memory
 * and error rules of vpt_line_stream_new_rules. */
int vpt_line_stream_new_annotate(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */, int no_norm,
                                 uint32_t wsconst_types, int predict_tags, int32_t margin, vpt_stream_write_fn write,
                                 void* ctx, vpt_line_stream** out);

/* ---- Re-annotation: partially annotated lines in, partially annotated lines out ---------------------------------------
 *
 * The second round of the domain-adaptation loop: a corpus that an annotator has partly resolved (vpt_annotate_lines'
 * output with some ' ' turned into '|' or '-' and some tags fixed) goes through a retrained model.  Every decision in the
 * input stays as written; only the positions still undecided are predicted, and those the model is unsure of stay open.
 * Lines are split as in vpt_tokenize_lines.  For every line:
 *
 *   pa = Sentence::from_partial_annotation(line)      // given[i] in {Not, Word, Unknown}; input tag fields per character
 *   s  = Sentence::from_raw(pa.as_raw_text())          // KyteaFullwidthFilter of it unless no_norm
 *   predictor.predict(&mut s)
 *   for every i with -margin < score[i] < margin: s.boundaries[i] = Unknown          // i32 score, wrapped as the reference sums it
 *   the wsconst_types post-filters on s                                              // they set NotWordBoundary, Unknown or not
 *   for every i with given[i] != Unknown: s.boundaries[i] = given[i]                 // the caller's markers win, last
 *   with predict_tags: fill_tags, then the PatternMatchTagger rules                  // tokens next to or across an Unknown get none
 *   with keep_tags: every character that carries an input tag gets exactly its input tags   // replaces what the model or a rule put there
 *   write_partial_annotation_text over the raw text; "\n"
 *
 * Definitions of this library, not of a reference command:
 *   - markers: a given '|' / '-' is written as given, whatever the score or the post-filters say; a given ' ' is written
 *     as '|' / '-' when the model is sure, as '-' when a post-filter cleared it, and stays ' ' otherwise;
 *   - a character carries input tags when at least one of its tag fields is non-empty ("火/" and "火//" carry none, so
 *     the model's and the rules' tags may appear there);
 *   - a character's input tags are written as the reference writer writes a parsed sentence's tags: '/' + tag for every
 *     field up to the last non-empty one, unescaped (sentence.rs:907-944).  In bytes: the character's tag region, from
 *     the '/' that follows it to the marker that ends it (or the line's end), with every escaping '\' dropped, up to and
 *     including the last content byte.  As in vpt_annotate_lines, a tag that holds ' ', '-', '|', '/' or '\' does not
 *     read back;
 *   - input tags stay at their character even when it does not end a token, and even next to a ' ': the reference
 *     writer writes tags per character;
 *   - keep_tags == 0: the input tags are parsed, checked and dropped, as vpt_tokenize_partial_lines drops them (for a
 *     corpus whose first-round tags are the old model's guesses rather than an annotator's corrections);
 *   - an empty line gives an empty output line; a malformed line stops the call with exactly vpt_tokenize_partial_lines'
 *     errors and line numbers (UTF-8 first), and output delivered before the error ends at a line end;
 *   - `margin` must not be negative (VPT_INVALID_ARGUMENT); with margin 0 only the caller's ' ' positions change, and
 *     they become '|' or '-'.
 * The parse, input tag regions, scoring, margin, post-filters, markers, tags, rules and writer run on the device.  Flags
 * are checked as in vpt_tokenize_partial_lines; `out`, `out_capacity`, *out_len and *n_lines as there (the output of a
 * line is at most that of its raw text in vpt_tokenize_lines_tags plus its input bytes).
 * Not offered: a device-resident variant, score dumps, escaped tags, a scoring pass that skips given boundaries. */
int vpt_reannotate_lines(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */, const uint8_t* utf8,
                         size_t n_bytes, int no_norm, uint32_t wsconst_types, int predict_tags, int32_t margin,
                         int keep_tags, uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines);

/* A line stream of vpt_reannotate_lines: the same output, errors and line count on input fed in pieces, with the
 * progress, memory and error rules of vpt_line_stream_new_partial. */
int vpt_line_stream_new_reannotate(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */,
                                   int no_norm, uint32_t wsconst_types, int predict_tags, int32_t margin, int keep_tags,
                                   vpt_stream_write_fn write, void* ctx, vpt_line_stream** out);

/* ---- Score dumps: the predict CLI's --scores and --tag-scores (predict/src/main.rs:66-93, 125-181) ------------------
 *
 * A VPT_STREAM_TOKENIZE line stream (with `rules`, nullable, as vpt_line_stream_new_rules) whose output is, per input
 * line, the token line followed by the dumps the reference CLI prints for it:
 *   VPT_DUMP_SCORES      valid lines: "{i}:{c_i}{c_i+1} {score_i}\n" per boundary, then "\n".  The characters are those
 *                        of the predicted sentence (the KyteaFullwidthFilter image unless no_norm), the scores are
 *                        predict's, before the wsconst filters, as i32 (sums wrap).  With no_norm the block comes
 *                        before the line's '\n', as the CLI writes it (main.rs:136-141); otherwise after it.
 *   VPT_DUMP_TAG_SCORES  every line: per token of the predicted sentence its surface (not escaped), then per tag slot of
 *                        its tag model "\t" and the slot's "tag:score" pairs joined by ',' (one candidate: "tag:0"),
 *                        then "\n"; one more "\n" after the last token.  Tag rules change the token line only.
 * The output has no useful bound from the input (about 5x it with VPT_DUMP_SCORES), so there is no whole-buffer call.
 * Device memory: with VPT_DUMP_TAG_SCORES each of the four chunks in flight also holds 4 x VPT_CHUNK_BYTES x the
 * predictor's longest tag score vector bytes (512 MiB for 16 MiB chunks and 8-score vectors); see DESIGN §17.
 * dumps == 0 is vpt_line_stream_new_rules.  Errors: those of vpt_line_stream_new_rules, and InvalidArgument for other
 * `dumps` bits and for VPT_DUMP_TAG_SCORES without predict_tags or with a model without tag slots.
 * Deviations from the reference, each where it panics or prints stale data:
 *   1. A rejected line (empty, NUL, invalid UTF-8) gives the tag block " \n\n"; the reference prints the token " " with
 *      the candidates of a stale entry of the last tagged line (sentence.rs:140-158, 1234), or panics if there is none.
 *   2. VPT_DUMP_TAG_SCORES without tag prediction or tag slots is refused here; the reference panics at the first token.
 *   3. A token whose slots list more candidates than its score vector has prints its surface alone; the reference
 *      panics on scores[i]. */
#define VPT_DUMP_SCORES 1u
#define VPT_DUMP_TAG_SCORES 2u
int vpt_line_stream_new_scores(const vpt_predictor* predictor, const vpt_tag_rules* rules, int no_norm,
                               uint32_t wsconst_types, int predict_tags, uint32_t dumps, vpt_stream_write_fn write,
                               void* ctx, vpt_line_stream** out);

/* ---- Token spans: vaporetto_tantivy's token_stream for a batch of documents ---------------------------------------
 *
 * `VaporettoTokenizer::token_stream` (vaporetto_tantivy/src/lib.rs:157-229) on the device, for many documents: only text
 * goes in and only token byte offsets (and optional tag records) come out.
 *  - Documents.  Document d is utf8[byte_offsets[d] .. byte_offsets[d+1]).  It is one Sentence: '\r' and '\n' are ordinary
 *    characters in it (type Other), not line ends.
 *  - Filters.  The chain of token_stream, in this order:
 *      1. KyteaFullwidthFilter as the pre-filter, unless `no_norm` (the adapter always applies it; `no_norm` is there for
 *         parity with the CLI);
 *      2. predict;
 *      3. SplitLinebreaksFilter (vaporetto_rules/src/sentence_filters/split_linebreaks.rs:9-37), always: the boundary on
 *         either side of every '\r' / '\n' becomes WordBoundary;
 *      4. the `wsconst_types` post-filters (VPT_WSCONST_*, the bit set of vpt_tokenize_lines).
 *    The line-break split is the only filter that sets boundaries and the wsconst filters only clear them, so D/R/H/T/K/O/G
 *    commute with each other but not with it: "。\n" under O is one token, and so is "\r\n" under G.
 *  - Output.  Token r of document d is record T_d + r, T_d = the sum of n_tokens_out over the earlier documents.
 *    token_ends_out[T_d + r] is the byte offset, from the document's first byte, of the token's exclusive end; its start
 *    is the previous token's end (0 for the first).  The last end is the document's byte length: the tokens tile the
 *    document.  This is `boundary_pos` (lib.rs:179-188); a token's `position` is r and its `position_length` is
 *    n_tokens_out[d] (lib.rs:207-219).
 *  - Empty and rejected documents.  An empty document has 0 tokens and status VPT_SENT_EMPTY (the adapter returns no
 *    token for ""); a document with U+0000 or invalid UTF-8 has 0 tokens and status VPT_SENT_NUL / VPT_SENT_BAD_UTF8
 *    (the adapter panics on NUL: a documented difference).  status_out[d] as in vpt_predict_batch_compact.
 *  - Tags.  With token_ids_out (the predictor needs predict_tags = 1), token_ids_out / token_cands_out receive the
 *    records of vpt_predict_batch_compact, one per token: the token id (-1: no tag model) and per tag slot the chosen
 *    candidate as one byte (255: none).  They are predicted after the post-filters, on the pre-filtered token bytes when
 *    normalising, as vpt_tokenize_lines_tags predicts them; the flags are checked as there, with the same statuses and
 *    messages (a model with no tag slots gives -1 for every token).  The adapter itself predicts no tags.
 *  - Capacity and limits.  token_capacity is the number of records the token arrays hold; an upper bound is the total
 *    number of bytes.  If it is too small the call returns VPT_INVALID_ARGUMENT with *n_tokens_total_out set to the
 *    number needed.  A document over 1 GiB is VPT_INVALID_ARGUMENT before anything runs; n_docs == 0 is OK.
 * The documents flow through the pipeline of vpt_predict_batch_compact (four chunks in flight); a chunk closes at env
 * VPT_CHUNK_SENTENCES documents (262144) or at env VPT_CHUNK_BYTES of text (16 MiB), whichever comes first, both
 * ramping up over the first chunks, and a larger document is a chunk by itself.  VPT_TRACE=1 prints the per-chunk
 * timeline under the tag "spans". */
int vpt_token_spans(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_docs,
                    int no_norm, uint32_t wsconst_types,
                    uint32_t* n_tokens_out,      /* [n_docs] */
                    uint8_t* status_out,         /* [n_docs], VPT_SENT_* */
                    uint32_t* token_ends_out,    /* [token_capacity] */
                    int32_t* token_ids_out,      /* nullable: tag prediction, as vpt_predict_batch_compact */
                    uint8_t* token_cands_out,    /* nullable: [token_capacity * n_tags] */
                    size_t token_capacity, uint64_t* n_tokens_total_out);
/* vpt_token_spans with the tag candidate scores of every token record, under the contract of
 * vpt_predict_batch_compact_tag_scores: the scores are those of the sentence that was tagged, i.e. of the pre-filtered
 * text after the line-break and wsconst filters, where the tags come from.  A model with no tag slots gives id -1 for
 * every token and no scores.  With tag_scores_out == NULL the call IS vpt_token_spans. */
int vpt_token_spans_tag_scores(const vpt_predictor* predictor, const uint8_t* utf8, const uint64_t* byte_offsets,
                               size_t n_docs, int no_norm, uint32_t wsconst_types, uint32_t* n_tokens_out,
                               uint8_t* status_out, uint32_t* token_ends_out, int32_t* token_ids_out,
                               uint8_t* token_cands_out, size_t token_capacity, uint64_t* n_tokens_total_out,
                               int32_t* tag_scores_out, size_t score_capacity, uint64_t* n_scores_total_out);

/* ---- Token spans of documents already in device memory ---------------------------------------------------------------
 *
 * vpt_token_spans over DEVICE buffers, for text that already lives on the GPU (cuDF / Arrow string columns: a chars buffer
 * and int32 or int64 offsets; torch tensors).  The outputs are exactly those of vpt_token_spans for the same documents:
 * the filter chain, statuses, token ends relative to the document and tag records; d_token_offsets is the exclusive prefix
 * of the token counts, with the total behind it.
 *
 * Contract: the call never synchronises, allocates, creates events or streams, or writes host memory.  All its work is
 * queued on `cuda_stream` (a cudaStream_t; NULL = the legacy default stream) and it may be captured in a CUDA graph.  Every
 * output is sized by a bound the host knows (tokens <= characters <= bytes), never by a total read back.
 *
 *  - Documents.  Document d is d_utf8[o[d] .. o[d+1]) with o = d_offsets, int32 (offset_bytes = 4) or int64 (8), Arrow
 *    style: [n_docs + 1] entries, o[0] may be > 0.  d_utf8 may have any alignment; the documents lie in [0, n_bytes).  The
 *    kernels read the 16-byte blocks that hold [d_utf8, d_utf8 + n_bytes) and nothing else.
 *  - Offsets are checked on the device.  A document with o[d] < 0, o[d] > o[d+1], o[d+1] > n_bytes or more than 1 GiB, or
 *    that starts before an earlier offset of the array, gets status VPT_SENT_BAD_RANGE and 0 tokens; the others keep their
 *    exact range.
 *  - Outputs: d_token_offsets [n_docs + 1] (token r of document d is record d_token_offsets[d] + r; the last entry is the
 *    total), d_n_tokens and d_status [n_docs], d_token_ends [max(n_bytes, 1)]: its first d_token_offsets[n_docs] entries
 *    are written.  Tags (nullable, the predictor needs predict_tags): d_token_ids [n_bytes] and d_token_cands
 *    [n_bytes * n_tags], as in vpt_token_spans (a model without tag slots: ids -1).  Tag scores are not returned.
 *  - d_workspace: vpt_token_spans_dev_workspace_size(predictor, n_docs, n_bytes, tags) bytes of device scratch.
 *  - Checked on the host, before anything is queued: NULL pointers, offset_bytes, the workspace size, the flags (as
 *    vpt_token_spans), that every pointer is device memory of the predictor's device, and the batch limit: n_bytes and
 *    n_docs at most 2^32 - 16 (32-bit character and token indexes of the tag kernels).
 *  - n_docs == 0 writes d_token_offsets[0] = 0 and returns VPT_OK (the per-document outputs and the workspace may then be
 *    NULL). */
uint64_t vpt_token_spans_dev_workspace_size(const vpt_predictor* predictor, size_t n_docs, uint64_t n_bytes, int tags);
int vpt_token_spans_dev(const vpt_predictor* predictor,
                        const uint8_t* d_utf8, uint64_t n_bytes,
                        const void* d_offsets, int offset_bytes,
                        size_t n_docs, int no_norm, uint32_t wsconst_types,
                        uint64_t* d_token_offsets,
                        uint32_t* d_n_tokens, uint8_t* d_status,
                        uint32_t* d_token_ends,
                        int32_t* d_token_ids, uint8_t* d_token_cands,
                        void* d_workspace, uint64_t workspace_bytes, void* cuda_stream);

/* ---- Tokenized text of documents already in device memory -----------------------------------------------------------
 *
 * The predict CLI's tokenized text (Sentence::write_tokenized_text, sentence.rs:850-886) for documents that already live
 * on the GPU, written as a device string column: one string per document and int64 Arrow-style offsets.  Document d is
 * d_utf8[o[d] .. o[d+1]) with the offsets of vpt_token_spans_dev (int32 or int64, o[0] may be > 0, any text alignment).
 * Its string is write_tokenized_text of the original document after, in order: KyteaFullwidthFilter (unless no_norm),
 * predict, the wsconst post-filters (as vpt_tokenize_lines, VPT_WSCONST_GRAPHEME included), with predict_tags fill_tags
 * and, with `rules`, PatternMatchTagger keyed as vpt_tokenize_lines_tags_rules keys it.  '\r' and '\n' are ordinary
 * characters: there is no line splitting and no terminator, so a document without '\n', followed by "\n", is what
 * vpt_tokenize_lines writes for it as one line with the same flags.  A document that Sentence::from_raw rejects gets
 * d_status VPT_SENT_EMPTY / VPT_SENT_NUL / VPT_SENT_BAD_UTF8, one whose offsets are not a range VPT_SENT_BAD_RANGE
 * (as vpt_token_spans_dev), and an empty string; the others VPT_SENT_OK.
 *
 * Contract: the call never synchronises, allocates, creates events or streams, or writes host memory.  All its work is
 * queued on `cuda_stream` (a cudaStream_t; NULL = the legacy default stream) and it may be captured in a CUDA graph.
 *
 *  - Output.  d_out_offsets [n_docs + 1] is always written in full: [0] = 0 and [d+1] - [d] is the length of document d's
 *    string.  Document d's bytes go to d_out[d_out_offsets[d] ..] if and only if d_out_offsets[d+1] <= out_capacity;
 *    nothing else in d_out is touched.  out_capacity == 0 (d_out may then be NULL) is an offsets-only sizing pass.
 *  - vpt_tokenize_dev_out_bound is a bound the host knows: with out_capacity at least this, every document is written.
 *    It is 3 * n_bytes (surface bytes, at most one '\' per byte, at most one ' ' per character), plus with tags
 *    n_bytes * (the model's longest "/tag.." suffix + the rules' longest, computed once by vpt_tag_rules_new).
 *  - d_workspace: vpt_tokenize_dev_workspace_size(predictor, rules, n_docs, n_bytes, predict_tags) bytes of device
 *    scratch, 256-byte aligned inside.
 *  - Checked on the host, before anything is queued: NULL pointers, offset_bytes, the workspace size, the flags (as
 *    vpt_tokenize_lines_tags: VPT_UNSUPPORTED for a tag model beyond the device tables), that `rules` needs predict_tags
 *    and belongs to the predictor, that every pointer is device memory of the predictor's device, and the batch limit:
 *    n_bytes and n_docs at most 2^32 - 16, each document at most 1 GiB (a longer one is VPT_SENT_BAD_RANGE).
 *  - A predictor with predict_tags but no tag slots writes the untagged text, as vpt_tokenize_lines_tags.
 *  - n_docs == 0 writes d_out_offsets[0] = 0 and returns VPT_OK (d_status and the workspace may then be NULL). */
uint64_t vpt_tokenize_dev_workspace_size(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */,
                                         size_t n_docs, uint64_t n_bytes, int predict_tags);
uint64_t vpt_tokenize_dev_out_bound(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */,
                                    size_t n_docs, uint64_t n_bytes, int predict_tags);
int vpt_tokenize_dev(const vpt_predictor* predictor, const vpt_tag_rules* rules /* nullable */,
                     const uint8_t* d_utf8, uint64_t n_bytes, const void* d_offsets, int offset_bytes, size_t n_docs,
                     int no_norm, uint32_t wsconst_types, int predict_tags,
                     int64_t* d_out_offsets /* [n_docs + 1] */, uint8_t* d_out /* nullable if out_capacity == 0 */,
                     uint64_t out_capacity, uint8_t* d_status /* [n_docs] */,
                     void* d_workspace, uint64_t workspace_bytes, void* cuda_stream);

/* `KyteaFullwidthFilter` for one character (vaporetto_rules/src/string_filters/kytea_fullwidth.rs:13-118): the
 * same function the kernels apply (csrc/textnorm.hpp). */
uint32_t vpt_kytea_fullwidth(uint32_t code_point);

/* library build info, e.g. "vaporetto_b200 0.1.0 sm_90a" */
const char* vpt_version(void);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* VAPORETTO_B200_H */
