// C ABI (include/vaporetto_b200.h) — host side of the predictor: model parsing, table build, upload,
// batch staging, tag prediction and the Sentence helpers.  Compiled with nvcc (needs cuda_runtime.h).
#include "../../include/vaporetto_b200.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>

#include "builder.hpp"
#include "common.hpp"
#include "device_model.hpp"
#include "dump.hpp"
#include "kernel_plan.hpp"
#include "line_feed.hpp"
#include "model.hpp"
#include "partial_parse.hpp"
#include "predictor_build.hpp"
#include "grapheme.hpp"
#include "tag_rules.hpp"
#include "tags.hpp"
#include "zstd_loader.hpp"
#include "textnorm.hpp"

using namespace vpt;

struct vpt_model {
    Model m;
};

namespace {

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess)
        throw Error(kCudaError, std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}

// A grow-only device buffer of T, freed with its owner
template <class T>
class DevBuf {
public:
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p_) cudaFree(p_); }
    // At least `need` bytes, with an eighth and 256 bytes to spare when it grows.  The old buffer is freed before the
    // new one is allocated (the peak is the new size alone); a failed allocation leaves the buffer empty.
    T* ensure(size_t need) {
        if (need <= cap_) return p_;
        if (p_) cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
        const size_t want = align_up(need + need / 8 + 256, 256);
        cuda_check(cudaMalloc(&p_, want), "cudaMalloc(scratch)");
        cap_ = want;
        return p_;
    }
    T* get() const { return p_; }
    size_t capacity() const { return cap_; }  // bytes

private:
    T* p_ = nullptr;
    size_t cap_ = 0;
};

struct CudaFreeHost {
    void operator()(void* q) const { cudaFreeHost(q); }
};
struct CudaFree {
    void operator()(void* q) const { cudaFree(q); }
};

// The words a chunk's kernels and copies hand back to the host, in one pinned block per scratch
struct HostTotals {
    uint64_t bounds_chars[2];  // boundaries and characters of the count pass (BatchArgs::totals_host, written as a pair)
    uint64_t lines;            // lines of the split pass (SplitArgs::n_lines_host)
    uint64_t out_bytes;        // output bytes of a line chunk: the tokenized writer's, or dump_stage's with score dumps
    uint64_t tokens;           // tokens of the compact and span passes (tok_total_host)
    uint64_t tok_line_bytes;   // score dumps: the token line bytes the tokenized writer put in `stage`
    uint64_t rule_suffix;      // the matched rules' suffix bytes, copied from the front of `trule`
    uint64_t tag_scores;       // tag candidate scores of a chunk (TagScoreArgs::total_host)
    uint64_t dump[2];          // score dumps: dump bytes, token line bytes (DumpArgs::total_host, written as a pair)
    uint64_t eval[kEvalTotals + 1];  // evaluate: the chunk's totals, then the error key (also the partial parse's)
};

// Per-call scratch: two streams, grow-only device buffers and the pinned words the kernels write back.
struct Scratch {
    cudaStream_t stream = nullptr;      // copy-in + kernels
    cudaStream_t stream_out = nullptr;  // copy-out: a chunk's D2H never delays the next chunk's H2D on `stream`
    cudaEvent_t ev_kernels = nullptr;   // recorded on `stream` after a chunk's last kernel
    cudaEvent_t ev_out = nullptr;       // recorded on `stream_out` after a chunk's last D2H copy
    DevBuf<uint8_t> text;
    DevBuf<uint64_t> off;
    DevBuf<uint8_t> ws;                 // the scoring workspace, laid out by bind_workspace
    DevBuf<int32_t> status;
    DevBuf<uint64_t> boff;
    DevBuf<uint64_t> coff;
    DevBuf<int32_t> scores;
    DevBuf<uint8_t> bounds;
    DevBuf<uint32_t> cst;
    DevBuf<uint32_t> tst;
    // line splitting / tokenised output (vpt_tokenize_lines)
    DevBuf<uint8_t> trims;
    DevBuf<uint32_t> blk;
    DevBuf<uint64_t> blkbase;
    DevBuf<uint64_t> tokg;              // look-back state words, then a u32 ticket
    DevBuf<uint8_t> out;
    DevBuf<int32_t> tok;                // tag prediction outputs (vpt_predict_batch_tags)
    DevBuf<uint8_t> cand;               // u8 per token record; vpt_predict_batch_tags: i32 per character
    DevBuf<uint32_t> bits;              // compact outputs (vpt_predict_batch_compact)
    DevBuf<uint8_t> st8;
    DevBuf<uint32_t> ntok;
    DevBuf<uint64_t> tokbase;
    DevBuf<uint4> tokdesc;
    DevBuf<uint32_t> tokwork;           // work list of the per-token tag kernels (TagArgs::tok_work)
    DevBuf<uint32_t> toklocal;
    DevBuf<uint64_t> tokblk;
    DevBuf<uint32_t> ends;              // token byte ends (vpt_token_spans)
    DevBuf<unsigned long long> trule;   // tag rules: the matched suffix sum (8 bytes), then a rule id per token
    DevBuf<uint32_t> scoff;             // tag candidate scores (TagScoreArgs): per-record counts / offsets,
    DevBuf<uint64_t> scblk;             // block totals / prefix,
    DevBuf<int32_t> tagsc;              // the chunk's score vectors
    // score dumps of the lines path (dump.hpp): the token lines in front of their dumps, the per-line sizes
    DevBuf<uint8_t> stage;
    DevBuf<uint64_t> dsize;
    // gold corpus and metrics (vpt_evaluate_lines); the partial parse (vpt_tokenize_partial_lines) uses gtext, goff,
    // gcoff, gbnd (its marker codes) and evtot (its error key); vpt_annotate_lines keeps its output markers in gbnd,
    // vpt_reannotate_lines in pmark (gbnd holds the input's), and its input tag regions in ptag
    DevBuf<uint8_t> gtext;
    DevBuf<uint64_t> goff;
    DevBuf<uint64_t> gcoff;
    DevBuf<uint8_t> gbnd;
    DevBuf<uint32_t> gtag;
    DevBuf<uint32_t> gw;
    DevBuf<uint32_t> lc;
    DevBuf<uint64_t> evtot;
    DevBuf<uint8_t> pmark;
    DevBuf<uint2> ptag;
    std::unique_ptr<HostTotals, CudaFreeHost> totals;  // pinned, allocated with the scratch (ScratchLease)
    std::unique_ptr<uint32_t[], CudaFreeHost> h_side;  // pinned: first bit word of every chunk (vpt_predict_batch_compact)
    size_t side_words = 0;                             // words of h_side
    std::unique_ptr<uint8_t[], CudaFreeHost> h_io;     // pinned staging of the single-sentence call (vpt_predict), kSingleIoBytes
    std::unique_ptr<uint8_t[], CudaFree> d_io;         // its device twin
    ~Scratch() {
        if (ev_kernels) cudaEventDestroy(ev_kernels);
        if (ev_out) cudaEventDestroy(ev_out);
        if (stream_out) cudaStreamDestroy(stream_out);
        if (stream) cudaStreamDestroy(stream);
    }
};

}  // namespace

struct vpt_predictor : HostPredictor {
    int device = 0;
    bool from_blob = false;
    void* d_blob = nullptr;
    DevModel dm;
    // device-side tag prediction (tags.hpp): one allocation holding all tables; dt.tok_tab == nullptr when unavailable
    void* d_tags = nullptr;
    DevTags dt;
    bool tags_all_usable = false;  // every token's own model is within the device limits (TagTablesHost::all_tokens_usable)
    // scratch pool
    mutable std::mutex mu;
    mutable std::vector<std::unique_ptr<Scratch>> pool;
    // pinned staging buffers (pointer, bytes) of line streams that were freed, reused by later streams (under `mu`)
    mutable std::vector<std::pair<uint8_t*, size_t>> pinned_pool;

    ~vpt_predictor() {
        if (d_blob) {
            cudaSetDevice(device);
            pool.clear();
            for (auto& b : pinned_pool) cudaFreeHost(b.first);
            cudaFree(d_blob);
            if (d_tags) cudaFree(d_tags);
        }
    }
};

// PatternMatchTagger rules on the predictor's device (tag_rules.hpp): one allocation holding all tables
struct vpt_tag_rules {
    const vpt_predictor* p = nullptr;
    uint32_t n_rules = 0;
    void* d_mem = nullptr;
    DevTagRules dr;
    mutable std::atomic<uint64_t> max_out{0};  // largest device output buffer of a chunk with these rules
    uint32_t max_suffix = 0;                   // the longest TagRulesHost::suffix: bytes a rule adds behind one token
    ~vpt_tag_rules() {
        if (d_mem) {
            cudaSetDevice(p->device);
            cudaFree(d_mem);
        }
    }
};

namespace {

int fail(const Error& e) {
    set_last_error(e.what());
    return e.code;
}
int fail(const std::exception& e) {
    set_last_error(std::string("internal error: ") + e.what());
    return kInternal;
}

#define VPT_API_BEGIN try {
#define VPT_API_END \
    } catch (const Error& e) { return fail(e); } \
      catch (const std::exception& e) { return fail(e); }

DevTable dev_table(const BlobTable& bt, const uint8_t* base) {
    DevTable d;
    d.present = bt.present;
    if (!bt.present) return d;
    d.fast = bt.fast;
    d.r0 = bt.r0;
    d.max_depth = bt.max_depth;
    d.nslots = bt.nslots;
    d.nbuckets = bt.nbuckets;
    d.salt = bt.salt;
    d.hk = hash_consts(bt.salt);
    d.seed16 = bt.seed_bits == 16;
    d.spill_slots = bt.spill_slots;
    d.spill_buckets = bt.spill_buckets;
    d.spill_mul = spill_mul(bt.salt);
    d.has_overflow = bt.has_overflow;
    d.slot_ovf = bt.has_overflow ? reinterpret_cast<const uint64_t*>(base + bt.ovf_off) : nullptr;
    d.records = base + bt.rec_off;
    d.seeds = base + bt.seeds_off;
    d.slot_node = reinterpret_cast<const uint32_t*>(base + bt.node_off);
    d.slot_pid = reinterpret_cast<const uint32_t*>(base + bt.pid_off);
    d.pool = reinterpret_cast<const int32_t*>(base + bt.pool_off);
    return d;
}

// Every section a blob header points at must lie inside the blob, and the geometry must be what the kernels were
// built for: a truncated or corrupted blob is an InvalidModel error, not an out-of-bounds read on the device.
void validate_blob_header(const BlobHeader& h, const uint8_t* base, uint64_t len) {
    auto inside = [&](uint64_t off, uint64_t bytes) { return off >= sizeof(BlobHeader) && off <= len && bytes <= len - off; };
    auto bad = [](const char* what) { return Error(kInvalidModel, std::string("InvalidModelError: model blob: bad ") + what); };
    auto table = [&](const BlobTable& t, const char* name) {
        if (!t.present) return;
        if (t.nslots == 0 || t.nbuckets == 0 || (t.seed_bits != 8 && t.seed_bits != 16)) throw bad(name);
        // a spill table needs 8-bit seeds that k_fused stages in shared memory, where it reads the spill seeds
        if ((t.spill_slots || t.spill_buckets) &&
            (t.spill_slots != spill_slots_of(t.nslots) || t.spill_buckets != spill_buckets_of(t.nbuckets) || t.seed_bits != 8 ||
             uint64_t(t.nbuckets) + t.spill_buckets > uint64_t(fused_detail::kSeedCap)))
            throw bad(name);
        const uint64_t slots = uint64_t(t.nslots) + t.spill_slots;
        const uint64_t seed_bytes = uint64_t(t.nbuckets) * (t.seed_bits / 8) + t.spill_buckets;
        if (slots > 0xFFFFFFFFull || !inside(t.rec_off, slots * 32) || !inside(t.seeds_off, seed_bytes) ||
            !inside(t.node_off, slots * 4) || !inside(t.pid_off, slots * 4) || !inside(t.pool_off, 4))
            throw bad(name);
        if (t.has_overflow && !inside(t.ovf_off, slots * 8)) throw bad(name);
        // an 8-bit table without a spill table carries no spill seed (its probes would land behind the records)
        if (t.seed_bits == 8 && !t.spill_slots && memchr(base + t.seeds_off, int(kSpillSeed), t.nbuckets)) throw bad(name);
        if (t.r0 < -64 || t.r0 > 64) throw bad(name);
    };
    table(h.ct, "char table");
    table(h.tt, "type table");
    if (h.char_window < 0 || h.char_window > 255 || h.type_window < 0 || h.type_window > 255) throw bad("window");
    if (h.type_cache_window < 0 || h.type_cache_window > 3) throw bad("type table window");
    if (h.type_cache_window && !inside(h.type_cache_off, (uint64_t(4) << (6 * h.type_cache_window)))) throw bad("type table");
    if (h.type_a_off && (!inside(h.type_a_off, 4 * 4096) || !inside(h.type_b_off, 4 * 4096))) throw bad("split type tables");
    if (h.type_state3_off && !inside(h.type_state3_off, 4 * 512)) throw bad("type state table");
}

DevModel dev_model(const BlobHeader& h, const uint8_t* base);

void upload(vpt_predictor& p) {
    if (p.device == -1) return;  // host-only handle (tag prediction / Sentence helpers); cannot score
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        throw Error(kCudaError, std::string("no usable CUDA device (vaporetto_b200 has no CPU fallback): ") +
                                    cudaGetErrorString(e));
    if (p.device < 0 || p.device >= ndev) throw Error(kInvalidArgument, "InvalidArgumentError: device: out of range");
    cuda_check(cudaSetDevice(p.device), "cudaSetDevice");
    cuda_check(cudaMalloc(&p.d_blob, align_up(p.blob.size(), 256)), "cudaMalloc(model)");
    cuda_check(cudaMemcpy(p.d_blob, p.blob.data(), p.blob.size(), cudaMemcpyHostToDevice), "cudaMemcpy(model)");
    p.dm = dev_model(p.hdr, static_cast<const uint8_t*>(p.d_blob));
}

// The device view of a blob at `base` (the device copy, or the host copy when only the shape matters: kernel_plan)
DevModel dev_model(const BlobHeader& h, const uint8_t* base) {
    DevModel dm;
    dm.ct = dev_table(h.ct, base);
    dm.tt = dev_table(h.tt, base);
    dm.type_cache_window = h.type_cache_window;
    dm.type_cache = h.type_cache_window ? reinterpret_cast<const int32_t*>(base + h.type_cache_off) : nullptr;
    dm.type_a = h.type_a_off ? reinterpret_cast<const int32_t*>(base + h.type_a_off) : nullptr;
    dm.type_b = h.type_b_off ? reinterpret_cast<const int32_t*>(base + h.type_b_off) : nullptr;
    dm.type_state3 = h.type_state3_off ? reinterpret_cast<const uint32_t*>(base + h.type_state3_off) : nullptr;
    dm.bias = h.bias;
    dm.char_window = h.char_window;
    dm.type_window = h.type_window;
    dm.emit_states = h.emit_states;
    return dm;
}

// Tag tables of a tag predictor: built on the host (tags_build.cpp), one device allocation.
void upload_tags(vpt_predictor& p) {
    if (p.device == -1 || !p.predict_tags || p.n_tags == 0) return;
    const TagTablesHost t = build_tag_tables(p);
    if (!t.usable) return;
    struct Part { const void* src; size_t bytes; size_t off; };
    std::vector<Part> parts;
    size_t total = 0;
    auto add = [&](const void* src, size_t bytes) {
        parts.push_back({src, bytes, total});
        total = align_up(total + bytes, 256);
        return parts.size() - 1;
    };
    const size_t i_tok = add(t.tok_tab.data(), t.tok_tab.size() * sizeof(TagTokenEntry));
    const size_t i_bytes = add(t.tok_bytes.data(), t.tok_bytes.size());
    const size_t i_info = add(t.tok_info.data(), t.tok_info.size() * sizeof(TagTokenInfo));
    const size_t i_pool = add(t.pool.data(), t.pool.size() * 4);
    const size_t i_keys = add(t.keys.data(), t.keys.size() * sizeof(TagKey));
    const size_t i_tss = add(t.ts_slot.data(), t.ts_slot.size() * 4);
    const size_t i_tsc = add(t.ts_cand.data(), t.ts_cand.size() * 4);
    const size_t i_tsr = add(t.ts_ref.data(), t.ts_ref.size() * 4);
    const size_t i_tsb = add(t.ts_bytes.data(), t.ts_bytes.size());
    const size_t i_cc = add(t.c_chain.data(), t.c_chain.size() * sizeof(TagChain));
    const size_t i_tc = add(t.t_chain.data(), t.t_chain.size() * sizeof(TagChain));
    const size_t i_cl = add(t.c_link.data(), t.c_link.size() * 4);
    const size_t i_tl = add(t.t_link.data(), t.t_link.size() * 4);
    cuda_check(cudaSetDevice(p.device), "cudaSetDevice");
    cuda_check(cudaMalloc(&p.d_tags, total + 256), "cudaMalloc(tag tables)");
    uint8_t* base = static_cast<uint8_t*>(p.d_tags);
    for (const Part& q : parts)
        if (q.bytes) cuda_check(cudaMemcpy(base + q.off, q.src, q.bytes, cudaMemcpyHostToDevice), "cudaMemcpy(tag tables)");
    DevTags& d = p.dt;
    d.tok_tab = reinterpret_cast<const TagTokenEntry*>(base + parts[i_tok].off);
    d.tok_bytes = base + parts[i_bytes].off;
    d.tok_info = reinterpret_cast<const TagTokenInfo*>(base + parts[i_info].off);
    d.pool = reinterpret_cast<const int32_t*>(base + parts[i_pool].off);
    d.keys = reinterpret_cast<const TagKey*>(base + parts[i_keys].off);
    d.ts_slot = reinterpret_cast<const uint32_t*>(base + parts[i_tss].off);
    d.ts_cand = reinterpret_cast<const uint32_t*>(base + parts[i_tsc].off);
    d.ts_ref = reinterpret_cast<const uint2*>(base + parts[i_tsr].off);
    d.ts_bytes = base + parts[i_tsb].off;
    d.max_suffix = t.max_suffix;
    d.c_chain = reinterpret_cast<const TagChain*>(base + parts[i_cc].off);
    d.t_chain = reinterpret_cast<const TagChain*>(base + parts[i_tc].off);
    d.c_link = reinterpret_cast<const uint32_t*>(base + parts[i_cl].off);
    d.t_link = reinterpret_cast<const uint32_t*>(base + parts[i_tl].off);
    d.tok_mask = t.tok_mask;
    d.n_tags = t.n_tags;
    d.char_rels = p.char_tags ? t.char_rels : 0;
    d.type_rels = p.type_tags ? t.type_rels : 0;
    d.max_token_bytes = t.max_token_bytes;
    d.n_char_patterns = uint32_t(p.char_suffix_link.size());
    d.n_type_patterns = uint32_t(p.type_suffix_link.size());
    p.tags_all_usable = t.all_tokens_usable;
}

struct ScratchLease {
    const vpt_predictor& p;
    std::unique_ptr<Scratch> s;
    explicit ScratchLease(const vpt_predictor& pr) : p(pr) {
        {
            std::lock_guard<std::mutex> g(p.mu);
            if (!p.pool.empty()) { s = std::move(p.pool.back()); p.pool.pop_back(); }
        }
        if (!s) {
            s.reset(new Scratch());
            cuda_check(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking), "cudaStreamCreate");
            cuda_check(cudaStreamCreateWithFlags(&s->stream_out, cudaStreamNonBlocking), "cudaStreamCreate");
            cuda_check(cudaEventCreateWithFlags(&s->ev_kernels, cudaEventDisableTiming), "cudaEventCreate");
            cuda_check(cudaEventCreateWithFlags(&s->ev_out, cudaEventDisableTiming), "cudaEventCreate");
            HostTotals* h = nullptr;
            cuda_check(cudaMallocHost(reinterpret_cast<void**>(&h), sizeof(HostTotals)), "cudaMallocHost");
            s->totals.reset(h);
        }
    }
    ~ScratchLease() {
        // a lease can end on an exception path while copies into the caller's buffers or kernels are still queued:
        // drain both streams before the scratch becomes reusable and control returns to the caller
        if (s) {
            if (s->stream) cudaStreamSynchronize(s->stream);
            if (s->stream_out) cudaStreamSynchronize(s->stream_out);
        }
        std::lock_guard<std::mutex> g(p.mu);
        p.pool.push_back(std::move(s));
    }
};

struct WorkspaceLayout {
    size_t n_chars, local_bound, local_char, group_bound, group_char, ticket, total;
};
WorkspaceLayout workspace_layout(size_t n) {
    WorkspaceLayout l;
    // (the look-back descriptors of k_fused live in group_bound / group_char: its tiles hold at least 32 sentences)
    const size_t ng = (n + 31) / 32;
    size_t o = 0;
    l.n_chars = o; o = align_up(o + 4 * n, 256);
    l.local_bound = o; o = align_up(o + 4 * n, 256);
    l.local_char = o; o = align_up(o + 4 * n, 256);
    l.group_bound = o; o = align_up(o + 8 * (ng + 1), 256);
    l.group_char = o; o = align_up(o + 8 * (ng + 1), 256);
    l.ticket = o; o += 256;
    l.total = o + 256;
    return l;
}

void bind_workspace(BatchArgs& a, void* ws, size_t n) {
    const WorkspaceLayout l = workspace_layout(n);
    uint8_t* b = static_cast<uint8_t*>(ws);
    a.n_chars = reinterpret_cast<uint32_t*>(b + l.n_chars);
    a.local_bound = reinterpret_cast<uint32_t*>(b + l.local_bound);
    a.local_char = reinterpret_cast<uint32_t*>(b + l.local_char);
    a.group_bound = reinterpret_cast<uint64_t*>(b + l.group_bound);
    a.group_char = reinterpret_cast<uint64_t*>(b + l.group_char);
    a.ticket = reinterpret_cast<uint32_t*>(b + l.ticket);
}

// The fields of TagArgs that come from the scoring pass `a` (the pattern-id states only where the model's tags read them)
TagArgs tag_args(const DevTags& dt, const BatchArgs& a) {
    TagArgs t;
    t.text = a.text;
    t.offsets = a.offsets;
    t.trims = a.trims;
    t.n_sent = a.n_sent;
    t.status = a.status;
    t.boundaries = a.boundaries;
    t.bound_offsets = a.bound_offsets;
    t.char_offsets = a.char_offsets;
    t.char_states = dt.char_rels ? a.char_states : nullptr;
    t.type_states = dt.type_rels ? a.type_states : nullptr;
    return t;
}

// Ensures the per-token tag records of at most `m` tokens and binds them (tok_ids, tok_cands, tok_desc, tok_work,
// max_tokens) into `r`, a TagArgs or a SpanStage
template <class R>
void bind_token_records(const vpt_predictor& p, Scratch& s, R& r, uint64_t m) {
    r.tok_ids = s.tok.ensure(4 * m + 16);
    r.tok_cands = s.cand.ensure(m * std::max<size_t>(p.n_tags, 1) + 16);
    r.tok_desc = s.tokdesc.ensure(16 * m + 16);
    r.tok_work = s.tokwork.ensure(4 * m + 32);
    r.max_tokens = m;
}

// Ensures the token counts of `n` sentences, their prefix and its scratch and binds them (n_tokens, tok_base, tok_local,
// tok_blk) into `k`, a CompactArgs or a SpanStage; the prefix of both kernels runs in blocks of kSpanDocs sentences
template <class K>
void bind_token_counts(Scratch& s, K& k, size_t n) {
    k.n_tokens = s.ntok.ensure(4 * n + 16);
    k.tok_base = s.tokbase.ensure(8 * (n + 1) + 16);
    k.tok_local = s.toklocal.ensure(4 * n + 16);
    k.tok_blk = s.tokblk.ensure(8 * (n / kSpanDocs + 4));
}

// ---- host-side text helpers ------------------------------------------------------------------------

// Sentence::parse_raw checks (reference sentence.rs:160-196)
void check_raw_text(const uint8_t* s, size_t n) {
    if (!is_valid_utf8(s, n)) throw Error(kInvalidArgument, "InvalidArgumentError: text: must be valid UTF-8");
    if (memchr(s, 0, n) != nullptr) throw Error(kInvalidArgument, "InvalidArgumentError: text: must not contain NULL");
    if (n == 0) throw Error(kInvalidArgument, "InvalidArgumentError: text: must contain at least one character");
}

// CharacterType::get_type (reference sentence.rs:50-67)
uint8_t host_char_type(uint32_t c) {
    struct R { uint32_t lo, hi; uint8_t t; };
    static const R ranges[] = {
        {0x30, 0x39, 1}, {0xFF10, 0xFF19, 1},
        {0x41, 0x5A, 2}, {0x61, 0x7A, 2}, {0xFF21, 0xFF3A, 2}, {0xFF41, 0xFF5A, 2},
        {0x3040, 0x3096, 3},
        {0x30A0, 0x30FA, 4}, {0x30FC, 0x30FF, 4}, {0xFF66, 0xFF9F, 4},
        {0x3400, 0x4DBF, 5}, {0x4E00, 0x9FFF, 5}, {0xF900, 0xFAFF, 5}, {0x20000, 0x2A6DF, 5},
        {0x2A700, 0x2B73F, 5}, {0x2B740, 0x2B81F, 5}, {0x2B820, 0x2CEAF, 5}, {0x2F800, 0x2FA1F, 5},
    };
    for (const R& r : ranges) if (c >= r.lo && c <= r.hi) return r.t;
    return 6;
}

// byte offset of every character start, plus the end (char_to_str_pos, sentence.rs:100)
std::vector<uint32_t> char_starts(const uint8_t* s, size_t n) {
    std::vector<uint32_t> v;
    for (size_t i = 0; i < n; ++i) if ((s[i] & 0xC0) != 0x80) v.push_back(uint32_t(i));
    v.push_back(uint32_t(n));
    return v;
}

void add_truncated(const std::vector<int32_t>& w, std::vector<int32_t>& ys) {  // WeightVector::add_scores
    const size_t n = std::min(w.size(), ys.size());
    for (size_t i = 0; i < n; ++i) ys[i] = wrapping_add(ys[i], w[i]);
}

// Tag weight of pattern `pid` for one (token, rel) table, as the reference's build-time suffix merge would have
// produced it (PositionalWeightWithTag +=, predictor.rs:242-262, applied along the chain of suffix patterns,
// char_scorer.rs:50-78): a pattern's own vector plus the merged vector of its longest suffix pattern truncated
// to the own length; without an own vector, the suffix's merged vector unchanged.
bool merged_tag_weight(const std::unordered_map<uint32_t, std::vector<int32_t>>& table,
                       const std::vector<uint32_t>& suffix_link, uint32_t pid, std::vector<int32_t>& out) {
    // collect the chain entries (longest pattern first)
    std::vector<const std::vector<int32_t>*> chain;
    for (uint32_t q = pid; q != kNoPattern; q = suffix_link[q]) {
        auto it = table.find(q);
        if (it != table.end()) chain.push_back(&it->second);
    }
    const int n = int(chain.size());
    if (n == 0) return false;
    // evaluate from the shortest suffix outwards
    out = *chain[n - 1];
    for (int i = n - 2; i >= 0; --i) {
        std::vector<int32_t> cur = *chain[i];
        const size_t m = std::min(cur.size(), out.size());
        for (size_t k = 0; k < m; ++k) cur[k] = wrapping_add(cur[k], out[k]);
        out.swap(cur);
    }
    return true;
}

void add_tag_scores(const TagWeightMap& tw, const std::vector<uint32_t>& suffix_link, uint32_t token, size_t pos,
                    const uint32_t* states, size_t n, std::vector<int32_t>& scores) {  // boundary_tag_scorer.rs:154-174
    const auto& per_rel = tw[token];
    std::vector<int32_t> w;
    for (size_t r = 0; r < per_rel.size() && pos + r < n; ++r) {
        const uint32_t pid = states[pos + r];
        if (pid == kNoPattern || pid >= suffix_link.size() || per_rel[r].empty()) continue;
        if (merged_tag_weight(per_rel[r], suffix_link, pid, w)) add_truncated(w, scores);
    }
}

}  // namespace

extern "C" {

const char* vpt_last_error(void) { return last_error(); }
const char* vpt_version(void) { return "vaporetto_b200 0.1.0 sm_90a"; }

int vpt_model_read(const uint8_t* data, size_t len, vpt_model** out, size_t* consumed) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    std::unique_ptr<vpt_model> m(new vpt_model());
    m->m = Model::read(data, len, consumed);
    *out = m.release();
    return kOk;
    VPT_API_END
}

int vpt_model_read_zstd(const uint8_t* data, size_t len, vpt_model** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    if (len && !data) throw Error(kInvalidArgument, "InvalidArgumentError: data: must not be NULL");
    std::unique_ptr<vpt_model> m(new vpt_model());
    if (is_zstd_frame(data, len)) {
        const std::vector<uint8_t> raw = zstd_decode_all(data, len);
        m->m = Model::read(raw.data(), raw.size(), nullptr);
    } else {
        m->m = Model::read(data, len, nullptr);
    }
    *out = m.release();
    return kOk;
    VPT_API_END
}

int vpt_model_read_kytea(const uint8_t* data, size_t len, vpt_model** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    std::unique_ptr<vpt_model> m(new vpt_model());
    m->m = Model::from_kytea(data, len);
    *out = m.release();
    return kOk;
    VPT_API_END
}

int vpt_model_to_vec(const vpt_model* model, uint8_t** bytes_out, uint64_t* len_out) {
    VPT_API_BEGIN
    if (!model || !bytes_out || !len_out) throw Error(kInvalidArgument, "InvalidArgumentError: model/out: must not be NULL");
    *bytes_out = nullptr;
    const std::vector<uint8_t> v = model->m.to_vec();
    uint8_t* buf = static_cast<uint8_t*>(malloc(v.size() ? v.size() : 1));
    if (!buf) throw Error(kInternal, "internal error: out of memory");
    memcpy(buf, v.data(), v.size());
    *bytes_out = buf;
    *len_out = v.size();
    return kOk;
    VPT_API_END
}

uint64_t vpt_model_dictionary_len(const vpt_model* model) { return model ? model->m.dict.size() : 0; }

int vpt_model_dictionary_get(const vpt_model* model, uint64_t index, const char** word, const int32_t** weights,
                             uint64_t* n_weights, const char** comment) {
    VPT_API_BEGIN
    if (!model) throw Error(kInvalidArgument, "InvalidArgumentError: model: must not be NULL");
    if (index >= model->m.dict.size()) throw Error(kInvalidArgument, "InvalidArgumentError: index: out of range");
    const DictEntry& e = model->m.dict[index];
    if (word) *word = e.word.c_str();
    if (weights) *weights = e.weights.data();
    if (n_weights) *n_weights = e.weights.size();
    if (comment) *comment = e.comment.c_str();
    return kOk;
    VPT_API_END
}

int vpt_model_replace_dictionary(vpt_model* model, const char* const* words, const int32_t* const* weights,
                                 const uint64_t* n_weights, const char* const* comments, uint64_t n_records) {
    VPT_API_BEGIN
    if (!model) throw Error(kInvalidArgument, "InvalidArgumentError: model: must not be NULL");
    if (n_records && (!words || !weights || !n_weights))
        throw Error(kInvalidArgument, "InvalidArgumentError: words/weights/n_weights: must not be NULL");
    std::vector<DictEntry> dict;
    dict.reserve(n_records);
    for (uint64_t i = 0; i < n_records; ++i) {
        DictEntry e;
        e.word = words[i] ? words[i] : "";
        if (!is_valid_utf8(reinterpret_cast<const uint8_t*>(e.word.data()), e.word.size()))
            throw Error(kInvalidArgument, "InvalidArgumentError: word: must be valid UTF-8");
        // WordWeightRecord::new (dict_model.rs:39-50)
        if (n_weights[i] != utf8_to_codepoints(e.word).size() + 1)
            throw Error(kInvalidArgument, "InvalidArgumentError: weights: does not match the length of the `word`");
        if (n_weights[i] && !weights[i]) throw Error(kInvalidArgument, "InvalidArgumentError: weights: must not be NULL");
        e.weights.assign(weights[i], weights[i] + n_weights[i]);
        e.comment = (comments && comments[i]) ? comments[i] : "";
        dict.push_back(std::move(e));
    }
    model->m.dict = std::move(dict);
    return kOk;
    VPT_API_END
}

void vpt_model_free(vpt_model* model) { delete model; }

int vpt_predictor_new(vpt_model* model, int predict_tags, int device, vpt_predictor** out) {
    std::unique_ptr<vpt_model> owned(model);  // consumed like Predictor::new(model, ..)
    VPT_API_BEGIN
    if (!out || !model) throw Error(kInvalidArgument, "InvalidArgumentError: model/out: must not be NULL");
    *out = nullptr;
    std::unique_ptr<vpt_predictor> p(new vpt_predictor());
    static_cast<HostPredictor&>(*p) = build_host_predictor(owned->m, predict_tags != 0);
    p->device = device;
    upload(*p);
    upload_tags(*p);
    *out = p.release();
    return kOk;
    VPT_API_END
}

void vpt_predictor_free(vpt_predictor* predictor) { delete predictor; }

int vpt_predictor_get_info(const vpt_predictor* p, vpt_predictor_info* o) {
    VPT_API_BEGIN
    if (!p || !o) throw Error(kInvalidArgument, "InvalidArgumentError: predictor/out: must not be NULL");
    memset(o, 0, sizeof *o);
    o->device = p->device;
    o->predict_tags = p->predict_tags;
    o->n_tags = int32_t(p->n_tags);
    o->char_scorer = p->hdr.char_variant;
    o->type_scorer = p->hdr.type_variant;
    o->fast_path = (!p->hdr.ct.present || p->hdr.ct.fast) && !p->hdr.tt.present;
    o->bias = p->hdr.bias;
    o->char_window = p->hdr.char_window;
    o->type_window = p->hdr.type_window;
    o->n_char_patterns = p->hdr.ct.n_patterns;
    o->n_type_patterns = p->hdr.tt.n_patterns;
    o->n_char_nodes = p->hdr.ct.n_nodes;
    o->n_type_nodes = p->hdr.tt.n_nodes;
    o->max_char_pattern_len = uint32_t(p->hdr.max_char_pattern_len);
    o->blob_bytes = p->blob.size();
    o->kernel_launches_per_batch = launches_per_batch(p->dm);
    return kOk;
    VPT_API_END
}

int vpt_predictor_kernel_plan(const vpt_predictor* p, int with_states, vpt_kernel_plan* o) {
    VPT_API_BEGIN
    if (!p || !o) throw Error(kInvalidArgument, "InvalidArgumentError: predictor/out: must not be NULL");
    const KernelPlan pl = plan(p->d_blob ? p->dm : dev_model(p->hdr, p->blob.data()), with_states != 0);
    memset(o, 0, sizeof *o);
    o->kernel = pl.kernel;
    o->seeds_smem = pl.seeds_smem;
    o->common_shape = pl.common;
    o->deep = pl.deep;
    o->states = pl.states;
    o->r0_fixed = pl.r0_fixed;
    o->general = pl.general;
    o->split3 = pl.split3;
    o->overflow = pl.overflow;
    o->text_cap = pl.text_cap;
    o->slot_cap = pl.slot_cap;
    o->gap = pl.gap;
    o->lag = pl.lag;
    o->sub_blocks = pl.sub_blocks;
    o->group = pl.group;
    return kOk;
    VPT_API_END
}

int vpt_blob_build(vpt_model* model, int predict_tags, uint8_t** blob_out, uint64_t* len_out) {
    std::unique_ptr<vpt_model> owned(model);
    VPT_API_BEGIN
    if (!model || !blob_out || !len_out) throw Error(kInvalidArgument, "InvalidArgumentError: model/out: must not be NULL");
    *blob_out = nullptr;
    HostPredictor hp = build_host_predictor(owned->m, predict_tags != 0);
    uint8_t* buf = static_cast<uint8_t*>(malloc(hp.blob.size()));
    if (!buf) throw Error(kInternal, "internal error: out of memory");
    memcpy(buf, hp.blob.data(), hp.blob.size());
    *blob_out = buf;
    *len_out = hp.blob.size();
    return kOk;
    VPT_API_END
}

void vpt_blob_free(uint8_t* blob) { free(blob); }

uint64_t vpt_predictor_blob_size(const vpt_predictor* p) { return p ? p->blob.size() : 0; }

int vpt_predictor_blob_export(const vpt_predictor* p, void* dst, uint64_t capacity) {
    VPT_API_BEGIN
    if (!p || !dst) throw Error(kInvalidArgument, "InvalidArgumentError: predictor/dst: must not be NULL");
    if (capacity < p->blob.size()) throw Error(kInvalidArgument, "InvalidArgumentError: capacity: too small");
    memcpy(dst, p->blob.data(), p->blob.size());
    return kOk;
    VPT_API_END
}

int vpt_predictor_from_blob(const void* blob, uint64_t len, int device, vpt_predictor** out) {
    VPT_API_BEGIN
    if (!blob || !out) throw Error(kInvalidArgument, "InvalidArgumentError: blob/out: must not be NULL");
    *out = nullptr;
    BlobHeader h;
    if (len < sizeof h) throw Error(kInvalidModel, "InvalidModelError: blob too short");
    memcpy(&h, blob, sizeof h);
    if (memcmp(h.magic, kBlobMagic, 8) != 0 || h.total_bytes != len)
        throw Error(kInvalidModel, "InvalidModelError: not a vaporetto_b200 model blob");
    validate_blob_header(h, static_cast<const uint8_t*>(blob), len);
    std::unique_ptr<vpt_predictor> p(new vpt_predictor());
    p->device = device;
    p->from_blob = true;
    p->hdr = h;
    p->blob.assign(static_cast<const uint8_t*>(blob), static_cast<const uint8_t*>(blob) + len);
    upload(*p);
    *out = p.release();
    return kOk;
    VPT_API_END
}

uint64_t vpt_workspace_size(size_t n_sent) { return workspace_layout(n_sent).total; }

int vpt_device_pci_bus_id(int device, char* buf, size_t capacity) {
    VPT_API_BEGIN
    if (!buf || capacity < 16) throw Error(kInvalidArgument, "InvalidArgumentError: buf: needs at least 16 bytes");
    cuda_check(cudaDeviceGetPCIBusId(buf, int(capacity), device), "cudaDeviceGetPCIBusId");
    return kOk;
    VPT_API_END
}

static void require_device(const vpt_predictor* p) {
    if (!p) throw Error(kInvalidArgument, "InvalidArgumentError: predictor: must not be NULL");
    if (p->device < 0 || !p->d_blob)
        throw Error(kCudaError, "this predictor was created without a CUDA device (device = -1): it cannot score; "
                                "vaporetto_b200 has no CPU fallback");
}

static void run_batch_dev(const vpt_predictor* p, const uint8_t* d_utf8, const uint64_t* d_byte_offsets, size_t n_sent,
                          void* d_workspace, uint64_t workspace_bytes, int32_t* d_scores, uint8_t* d_boundaries,
                          uint64_t* d_bound_offsets, int32_t* d_status, uint32_t* d_char_states,
                          uint32_t* d_type_states, uint64_t* d_char_offsets, void* cuda_stream, float* stage_ms) {
    require_device(p);
    if (stage_ms) stage_ms[0] = stage_ms[1] = stage_ms[2] = 0.f;
    if (n_sent == 0) return;
    if (!d_utf8 || !d_byte_offsets || !d_workspace || !d_scores || !d_boundaries || !d_bound_offsets || !d_status)
        throw Error(kInvalidArgument, "InvalidArgumentError: device buffers: must not be NULL");
    if (workspace_bytes < workspace_layout(n_sent).total)
        throw Error(kInvalidArgument, "InvalidArgumentError: workspace: too small");
    if (reinterpret_cast<uintptr_t>(d_utf8) & 15)
        throw Error(kInvalidArgument, "InvalidArgumentError: d_utf8: must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    BatchArgs a;
    a.text = d_utf8;
    a.offsets = d_byte_offsets;
    a.n_sent = n_sent;
    bind_workspace(a, d_workspace, n_sent);
    a.status = d_status;
    a.scores = d_scores;
    a.boundaries = d_boundaries;
    a.bound_offsets = d_bound_offsets;
    a.char_offsets = d_char_offsets;
    a.char_states = d_char_states;
    a.type_states = d_type_states;
    if (!stage_ms) {
        cuda_check(launch_batch(p->dm, a, st), "launch(batch)");
        return;
    }
    cudaEvent_t ev[4];
    for (auto& e : ev) cuda_check(cudaEventCreate(&e), "cudaEventCreate");
    const bool fused = fused_ok(p->dm);  // one launch: the count and scan stages do not exist
    cuda_check(cudaEventRecord(ev[0], st), "record");
    if (!fused) cuda_check(launch_count_only(a, st), "launch(count)");
    cuda_check(cudaEventRecord(ev[1], st), "record");
    if (!fused) cuda_check(launch_scan_only(a, st), "launch(scan)");
    cuda_check(cudaEventRecord(ev[2], st), "record");
    cuda_check(launch_score(p->dm, a, st), "launch(score)");
    cuda_check(cudaEventRecord(ev[3], st), "record");
    cuda_check(cudaStreamSynchronize(st), "sync(profiled)");
    for (int i = 0; i < 3; ++i) cuda_check(cudaEventElapsedTime(&stage_ms[i], ev[i], ev[i + 1]), "elapsed");
    for (auto& e : ev) cudaEventDestroy(e);
}

int vpt_predict_batch_dev(const vpt_predictor* p, const uint8_t* d_utf8, const uint64_t* d_byte_offsets, size_t n_sent,
                          void* d_workspace, uint64_t workspace_bytes, int32_t* d_scores, uint8_t* d_boundaries,
                          uint64_t* d_bound_offsets, int32_t* d_status, uint32_t* d_char_states,
                          uint32_t* d_type_states, uint64_t* d_char_offsets, void* cuda_stream) {
    VPT_API_BEGIN
    run_batch_dev(p, d_utf8, d_byte_offsets, n_sent, d_workspace, workspace_bytes, d_scores, d_boundaries,
                  d_bound_offsets, d_status, d_char_states, d_type_states, d_char_offsets, cuda_stream, nullptr);
    return kOk;
    VPT_API_END
}

int vpt_predict_batch_dev_profiled(const vpt_predictor* p, const uint8_t* d_utf8, const uint64_t* d_byte_offsets,
                                   size_t n_sent, void* d_workspace, uint64_t workspace_bytes, int32_t* d_scores,
                                   uint8_t* d_boundaries, uint64_t* d_bound_offsets, int32_t* d_status,
                                   uint32_t* d_char_states, uint32_t* d_type_states, uint64_t* d_char_offsets,
                                   void* cuda_stream, float* stage_ms) {
    VPT_API_BEGIN
    if (!stage_ms) throw Error(kInvalidArgument, "InvalidArgumentError: stage_ms: must not be NULL");
    run_batch_dev(p, d_utf8, d_byte_offsets, n_sent, d_workspace, workspace_bytes, d_scores, d_boundaries,
                  d_bound_offsets, d_status, d_char_states, d_type_states, d_char_offsets, cuda_stream, stage_ms);
    return kOk;
    VPT_API_END
}

namespace {

// sentences per pipelined chunk of vpt_predict_batch (tuning knob: env VPT_CHUNK_SENTENCES)
size_t chunk_sentences() {
    static const size_t v = [] {
        const char* e = getenv("VPT_CHUNK_SENTENCES");
        const long long x = e ? atoll(e) : 0;
        return x >= 1024 ? size_t(x) : size_t(262144);
    }();
    return v;
}

// Chunk sizes of a copy/compute/copy pipeline over `total` units: small chunks first (the first copy-in and
// kernels are not overlapped with anything) growing by doubling to `big`, equal chunks of at most `big` in the
// middle, halving again to `small_down` at the end (the last copy-out is not overlapped either).
std::vector<size_t> ramp_schedule(size_t total, size_t big, size_t small_up, size_t small_down) {
    std::vector<size_t> up, down, out;
    size_t sum = 0;
    for (size_t v = std::max<size_t>(small_up, 1); v < big; v *= 2) { up.push_back(v); sum += v; }
    for (size_t v = std::max<size_t>(small_down, 1); v < big; v *= 2) { down.push_back(v); sum += v; }
    if (total <= sum + big) {
        // too small for the full ramps: equal chunks of about a quarter
        const size_t c = std::max<size_t>(std::min(big, (total + 3) / 4), std::min(small_up, big));
        for (size_t lo = 0; lo < total; lo += c) out.push_back(std::min(c, total - lo));
        return out;
    }
    const size_t middle = total - sum;
    const size_t nmid = (middle + big - 1) / big;
    out = up;
    for (size_t i = 0; i < nmid; ++i) out.push_back(middle / nmid + (i < middle % nmid ? 1 : 0));
    out.insert(out.end(), down.rbegin(), down.rend());
    return out;
}

// Pipeline chunks of vpt_predict_batch and vpt_predict_batch_compact as (first sentence, sentences): the ramp schedule
// over chunk_sentences()
std::vector<std::pair<size_t, size_t>> sentence_chunks(const uint64_t* byte_offsets, size_t n_sent) {
    const size_t cs = chunk_sentences();
    std::vector<std::pair<size_t, size_t>> out;
    size_t lo = 0;
    for (size_t sz : ramp_schedule(n_sent, cs, cs / 8, cs / 4)) {
        if (byte_offsets[lo + sz] < byte_offsets[lo])
            throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets: must be non-decreasing");
        out.emplace_back(lo, sz);
        lo += sz;
    }
    return out;
}

// Pipeline trace (env VPT_TRACE=1): per chunk, CUDA-event times of copy-in end, kernels start / end and copy-out
// end are printed to stderr when the call returns.
bool pipeline_trace() {
    const char* e = getenv("VPT_TRACE");
    return e && *e == '1';
}
struct TraceEvents {
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t sub[4] = {nullptr, nullptr, nullptr, nullptr};  // optional marks between the kernels of a chunk
    void mark_sub(int i, cudaStream_t st) {
        if (!sub[i]) cuda_check(cudaEventCreate(&sub[i]), "cudaEventCreate");
        cuda_check(cudaEventRecord(sub[i], st), "cudaEventRecord");
    }
    void mark(int i, cudaStream_t st) {
        if (!ev[i]) cuda_check(cudaEventCreate(&ev[i]), "cudaEventCreate");
        cuda_check(cudaEventRecord(ev[i], st), "cudaEventRecord");
    }
    void destroy() {
        for (cudaEvent_t& e : ev) if (e) { cudaEventDestroy(e); e = nullptr; }
        for (cudaEvent_t& e : sub) if (e) { cudaEventDestroy(e); e = nullptr; }
    }
    void print(const char* what, size_t c, unsigned long long units, const TraceEvents& first) const {
        float t[4] = {0, 0, 0, 0};
        for (int i = 0; i < 4; ++i)
            if (ev[i] && first.ev[0]) cudaEventElapsedTime(&t[i], first.ev[0], ev[i]);
        fprintf(stderr, "[vpt %s] chunk %zu (%llu): copy-in end %.3f  kernels %.3f..%.3f  copy-out end %.3f ms", what, c,
                units, t[0], t[1], t[2], t[3]);
        for (int i = 0; i < 4; ++i)
            if (sub[i] && first.ev[0]) {
                float x = 0;
                cudaEventElapsedTime(&x, first.ev[0], sub[i]);
                fprintf(stderr, "%s%.3f", i ? " " : "  marks ", x);
            }
        fprintf(stderr, "\n");
    }
};

constexpr size_t kRingDepth = 4;  // chunks in flight in the batch ring and the line ring

struct ChunkState {
    size_t s_lo = 0, n = 0;       // sentence range
    uint64_t byte_lo = 0, nbytes = 0;
    uint64_t nb = 0, nc = 0;      // boundaries and characters, from the count pass
    cudaEvent_t counted = nullptr, kernels = nullptr;
    bool issued = false;          // the chunk's kernels are queued
    TraceEvents tr;
    BatchArgs a;
};

// stage 1 of a chunk: H2D of text + offsets, count + scan, totals to pinned host memory
void chunk_count(Scratch& s, ChunkState& ch, const uint8_t* utf8, const uint64_t* byte_offsets) {
    cudaStream_t st = s.stream;
    const WorkspaceLayout wl = workspace_layout(ch.n);
    const size_t shift = size_t(ch.byte_lo & 15);
    BatchArgs& a = ch.a;
    a = BatchArgs();
    uint8_t* const text = s.text.ensure(shift + ch.nbytes + 64);
    uint64_t* const offsets = s.off.ensure(8 * (ch.n + 1));
    bind_workspace(a, s.ws.ensure(wl.total), ch.n);
    a.status = s.status.ensure(4 * ch.n);
    a.bound_offsets = s.boff.ensure(8 * (ch.n + 1));
    a.char_offsets = s.coff.ensure(8 * (ch.n + 1));
    if (ch.nbytes)
        cuda_check(cudaMemcpyAsync(text + shift, utf8 + ch.byte_lo, ch.nbytes, cudaMemcpyHostToDevice, st), "H2D(text)");
    cuda_check(cudaMemcpyAsync(offsets, byte_offsets + ch.s_lo, 8 * (ch.n + 1), cudaMemcpyHostToDevice, st), "H2D(offsets)");
    // the kernels overwrite buffers the previous chunk of this scratch may still be copying out
    cuda_check(cudaStreamWaitEvent(st, s.ev_out, 0), "cudaStreamWaitEvent");
    if (pipeline_trace()) ch.tr.mark(0, st);
    // offsets are absolute in the caller's buffer: bias the text pointer so that text[offset] is right
    a.text = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(text) + shift - uintptr_t(ch.byte_lo));
    a.offsets = offsets;
    a.n_sent = ch.n;
    // the totals come back through pinned host memory the scan kernel writes itself: an 8-byte D2H copy would
    // queue behind the bulk copy-out of earlier chunks on the copy engine
    a.totals_host = s.totals->bounds_chars;
    cuda_check(launch_count(a, st), "launch(count)");
    if (!ch.counted) cuda_check(cudaEventCreateWithFlags(&ch.counted, cudaEventDisableTiming), "cudaEventCreate");
    cuda_check(cudaEventRecord(ch.counted, st), "cudaEventRecord");
}

// ---- the batch ring: the chunk pipeline of vpt_predict_batch, vpt_predict_batch_compact* and vpt_token_spans* --------
//
// Every chunk of sentences (or documents) goes through chunk_count (copy-in, count pass), then its caller's `issue`
// (output bindings and kernels on the scratch's stream), then its caller's `copy_out` (D2H copies on stream_out).  Chunk c
// runs on lease c % kRingDepth, so the copy-in, kernels and copy-out of neighbouring chunks overlap; a chunk's kernels
// wait for the copy-out of its lease's previous chunk (ev_out, see chunk_count).  A call whose copy-out needs totals
// its kernels wrote (`wait_for_kernels`) copies each chunk out one step later, after a host wait for its kernels, and
// counts kRingDepth - 2 chunks ahead; otherwise a chunk is copied out in the step that issues it, and the count pass runs
// kRingDepth - 1 chunks ahead.
struct BatchRing {
    // returns false when it skipped the chunk (an output overflowed): no kernels, no copy-out
    using Issue = std::function<bool(size_t c, ChunkState& ch, Scratch& s)>;
    using CopyOut = std::function<void(size_t c, ChunkState& ch, Scratch& s, cudaStream_t stream_out)>;
    const char* const label;      // of the trace lines
    const char* const sync_what;  // of the final check of the kernels' streams
    std::vector<ChunkState> chunks;
    std::unique_ptr<ScratchLease> lease[kRingDepth];

    // `cuts`: (first sentence, sentences) of every chunk, in order
    BatchRing(const vpt_predictor& p, const char* what, const char* sync, const uint64_t* byte_offsets,
              const std::vector<std::pair<size_t, size_t>>& cuts)
        : label(what), sync_what(sync), chunks(cuts.size()) {
        for (size_t c = 0; c < cuts.size(); ++c) {
            ChunkState& ch = chunks[c];
            ch.s_lo = cuts[c].first;
            ch.n = cuts[c].second;
            ch.byte_lo = byte_offsets[ch.s_lo];
            ch.nbytes = byte_offsets[ch.s_lo + ch.n] - ch.byte_lo;
        }
        for (size_t i = 0; i < kRingDepth && i < chunks.size(); ++i) lease[i].reset(new ScratchLease(p));
    }

    ~BatchRing() {
        for (ChunkState& ch : chunks) {
            if (ch.counted) cudaEventDestroy(ch.counted);
            if (ch.kernels) cudaEventDestroy(ch.kernels);
            ch.tr.destroy();
        }
    }

    Scratch& scratch(size_t c) { return *lease[c % kRingDepth]->s; }

    // The whole batch through the ring.  The final synchronisation is checked: a failed copy-out is an error of the
    // call, not left to the leases' release.
    void run(const uint8_t* utf8, const uint64_t* byte_offsets, bool wait_for_kernels, const Issue& issue,
             const CopyOut& copy_out) {
        const size_t nchunks = chunks.size();
        const size_t ahead = wait_for_kernels ? kRingDepth - 2 : kRingDepth - 1;
        const size_t behind = wait_for_kernels ? 1 : 0;
        const bool trace = pipeline_trace();
        for (size_t c = 0; c < std::min(ahead, nchunks); ++c) chunk_count(scratch(c), chunks[c], utf8, byte_offsets);
        for (size_t step = 0; step < nchunks + 1; ++step) {
            if (step + ahead < nchunks) chunk_count(scratch(step + ahead), chunks[step + ahead], utf8, byte_offsets);
            if (step < nchunks) {
                ChunkState& ch = chunks[step];
                Scratch& s = scratch(step);
                cuda_check(cudaEventSynchronize(ch.counted), "sync(count)");
                ch.nb = s.totals->bounds_chars[0];
                ch.nc = s.totals->bounds_chars[1];
                ch.issued = issue(step, ch, s);
                if (ch.issued) {
                    if (trace) ch.tr.mark(2, s.stream);
                    if (!ch.kernels) cuda_check(cudaEventCreateWithFlags(&ch.kernels, cudaEventDisableTiming), "cudaEventCreate");
                    cuda_check(cudaEventRecord(ch.kernels, s.stream), "cudaEventRecord");
                }
            }
            if (step < behind || step - behind >= nchunks || !chunks[step - behind].issued) continue;
            const size_t c = step - behind;
            ChunkState& ch = chunks[c];
            Scratch& s = scratch(c);
            if (wait_for_kernels) cuda_check(cudaEventSynchronize(ch.kernels), "sync(kernels)");
            cuda_check(cudaStreamWaitEvent(s.stream_out, ch.kernels, 0), "cudaStreamWaitEvent");
            copy_out(c, ch, s, s.stream_out);
            cuda_check(cudaEventRecord(s.ev_out, s.stream_out), "cudaEventRecord");
            if (trace) ch.tr.mark(3, s.stream_out);
        }
        for (const std::unique_ptr<ScratchLease>& l : lease)
            if (l) {
                cuda_check(cudaStreamSynchronize(l->s->stream), sync_what);
                cuda_check(cudaStreamSynchronize(l->s->stream_out), "sync(copy-out)");
            }
        if (trace)
            for (size_t c = 0; c < nchunks; ++c) chunks[c].tr.print(label, c, chunks[c].n, chunks[0].tr);
    }
};

}  // namespace

int vpt_predict_batch(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                      int32_t* scores_out, uint8_t* boundaries_out, size_t out_capacity, uint64_t* bound_offsets_out,
                      int32_t* status_out, uint32_t* char_states_out, uint32_t* type_states_out,
                      size_t states_capacity, uint64_t* char_offsets_out, uint64_t* n_boundaries_out,
                      uint64_t* n_chars_out) {
    VPT_API_BEGIN
    require_device(p);
    if (n_boundaries_out) *n_boundaries_out = 0;
    if (n_chars_out) *n_chars_out = 0;
    if (!byte_offsets || !bound_offsets_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets/bound_offsets_out: must not be NULL");
    if (n_sent == 0) { bound_offsets_out[0] = 0; if (char_offsets_out) char_offsets_out[0] = 0; return kOk; }
    if (byte_offsets[n_sent] < byte_offsets[0])
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets: must be non-decreasing");
    if (byte_offsets[n_sent] > byte_offsets[0] && !utf8)
        throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");

    // The batch is cut into chunks that flow through the batch ring, so that the H2D copy of chunk c+2, the kernels of
    // chunk c+1 and the D2H copy of chunk c overlap.  Each chunk is an independent batch on the device; its output
    // offsets are rebased with the running totals (known on the host after its count pass).
    BatchRing ring(*p, "batch", "sync(score)", byte_offsets, sentence_chunks(byte_offsets, n_sent));
    const size_t nchunks = ring.chunks.size();
    const bool want_states = char_states_out || type_states_out;
    uint64_t nb_total = 0, nc_total = 0;
    bool overflow = false;
    auto issue = [&](size_t, ChunkState& ch, Scratch& s) {
        cudaStream_t st = s.stream;
        const uint64_t nb = ch.nb, nc = ch.nc;
        if (nb_total + nb > out_capacity || (nb && !boundaries_out) || (want_states && nc_total + nc > states_capacity))
            overflow = true;
        BatchArgs& a = ch.a;
        a.bound_base = nb_total;
        a.char_base = nc_total;
        nb_total += nb;
        nc_total += nc;
        if (overflow) return false;
        a.boundaries = s.bounds.ensure(nb + 4);
        a.scores = nullptr;  // boundaries only, when the caller wants no scores and the kernel can skip them
        if (scores_out || !scores_optional(p->dm)) a.scores = s.scores.ensure(4 * nb + 4);
        if (char_states_out) a.char_states = s.cst.ensure(4 * nc + 4);
        if (type_states_out) a.type_states = s.tst.ensure(4 * nc + 4);
        if (pipeline_trace()) ch.tr.mark(1, st);
        cuda_check(launch_score(p->dm, a, st), "launch(score)");
        return true;
    };
    auto copy_out = [&](size_t c, ChunkState& ch, Scratch& s, cudaStream_t so) {
        const uint64_t nb = ch.nb, nc = ch.nc, b0 = ch.a.bound_base, c0 = ch.a.char_base;
        if (nb) {
            if (scores_out) cuda_check(cudaMemcpyAsync(scores_out + b0, s.scores.get(), 4 * nb, cudaMemcpyDeviceToHost, so), "D2H(scores)");
            cuda_check(cudaMemcpyAsync(boundaries_out + b0, s.bounds.get(), nb, cudaMemcpyDeviceToHost, so), "D2H(boundaries)");
        }
        // the last element of a chunk's offsets is the first of the next chunk's: copy n (+1 for the last chunk)
        const size_t noff = ch.n + (c + 1 == nchunks ? 1 : 0);
        cuda_check(cudaMemcpyAsync(bound_offsets_out + ch.s_lo, s.boff.get(), 8 * noff, cudaMemcpyDeviceToHost, so), "D2H(offsets)");
        if (char_offsets_out)
            cuda_check(cudaMemcpyAsync(char_offsets_out + ch.s_lo, s.coff.get(), 8 * noff, cudaMemcpyDeviceToHost, so), "D2H(offsets)");
        if (status_out) cuda_check(cudaMemcpyAsync(status_out + ch.s_lo, s.status.get(), 4 * ch.n, cudaMemcpyDeviceToHost, so), "D2H(status)");
        if (nc && char_states_out) cuda_check(cudaMemcpyAsync(char_states_out + c0, s.cst.get(), 4 * nc, cudaMemcpyDeviceToHost, so), "D2H(states)");
        if (nc && type_states_out) cuda_check(cudaMemcpyAsync(type_states_out + c0, s.tst.get(), 4 * nc, cudaMemcpyDeviceToHost, so), "D2H(states)");
    };
    ring.run(utf8, byte_offsets, false, issue, copy_out);
    if (n_boundaries_out) *n_boundaries_out = nb_total;
    if (n_chars_out) *n_chars_out = nc_total;
    if (overflow) throw Error(kInvalidArgument, "InvalidArgumentError: out_capacity/states_capacity: too small for the batch");
    return kOk;
    VPT_API_END
}

namespace {

// bytes per pipelined chunk of vpt_tokenize_lines (tuning knob: env VPT_CHUNK_BYTES)
size_t chunk_bytes() {
    const char* e = getenv("VPT_CHUNK_BYTES");
    const long long x = e ? atoll(e) : 0;
    return x >= 64 ? size_t(x) : size_t(16) << 20;
}

constexpr uint64_t kMaxLineChunk = uint64_t(1) << 30;  // 32-bit group-local output offsets (3 bytes out per byte in)

struct LineChunk {
    uint64_t nbytes = 0;
    uint64_t n_lines = 0;
    cudaEvent_t split = nullptr, done = nullptr;
    TraceEvents tr;
    SplitArgs sp;
};

// What a line loop computes: the flags of vpt_tokenize_lines*, vpt_evaluate_lines or vpt_line_stream_new, checked
constexpr int kJobPartial = 2;  // vpt_tokenize_partial_lines / vpt_line_stream_new_partial (no public stream kind)
constexpr int kJobAnnotate = 3;  // vpt_annotate_lines / vpt_line_stream_new_annotate (no public stream kind)
constexpr int kJobReannotate = 4;  // vpt_reannotate_lines / vpt_line_stream_new_reannotate (no public stream kind)

struct LineJob {
    int kind;          // VPT_STREAM_TOKENIZE, VPT_STREAM_EVALUATE, kJobPartial, kJobAnnotate or kJobReannotate
    bool normalize;    // KyteaFullwidthFilter (no_norm == 0)
    uint32_t wsconst;  // post-filters (VPT_WSCONST_*)
    bool tags;         // tags predicted on the device
    int tag_mode;      // evaluate: how the system's tags compare with the gold's (kTags*)
    const vpt_tag_rules* rules = nullptr;  // PatternMatchTagger after fill_tags (tokenize with tags and rules only)
    uint32_t dumps = 0;    // tokenize: the predict CLI's --scores / --tag-scores (kDumpScores | kDumpTagScores, dump.hpp)
    int32_t margin = 0;    // (re)annotate: boundaries with -margin < score < margin are left Unknown
    bool keep_tags = false;  // reannotate: characters with input tags get them back
};

// stage 0 of a chunk: H2D of its `nbytes` at `bytes`, newline counts, the number of lines to pinned host memory
void lines_stage0(Scratch& s, LineChunk& ch, const uint8_t* bytes) {
    cudaStream_t st = s.stream;
    const size_t nblk = (ch.nbytes + kSplitBlockBytes - 1) / kSplitBlockBytes;
    SplitArgs& sp = ch.sp;
    sp = SplitArgs();
    uint8_t* const text = s.text.ensure(ch.nbytes + 64);
    sp.blk = s.blk.ensure(4 * nblk + 4);
    sp.blk_base = s.blkbase.ensure(8 * nblk + 16);
    cuda_check(cudaMemcpyAsync(text, bytes, ch.nbytes, cudaMemcpyHostToDevice, st), "H2D(text)");
    if (pipeline_trace()) ch.tr.mark(0, st);
    sp.text = text;
    sp.n_bytes = ch.nbytes;
    sp.n_lines = sp.blk_base + nblk;  // the element after the per-block bases
    sp.n_lines_host = &s.totals->lines;  // read back through pinned host memory written by the kernel (see chunk_count)
    cuda_check(launch_split_count(sp, st), "launch(split)");
    if (!ch.split) cuda_check(cudaEventCreateWithFlags(&ch.split, cudaEventDisableTiming), "cudaEventCreate");
    cuda_check(cudaEventRecord(ch.split, st), "cudaEventRecord");
}

size_t device_score_len_bound(const vpt_predictor* p);
TagScoreArgs bind_tag_scores(Scratch& s, uint64_t nc, size_t len_bound);

// Buffers of the per-token tag records behind a scoring pass (launch_tag_records)
struct TagRecords {
    uint8_t* status8 = nullptr;          // token counts and their prefix, as CompactArgs
    uint32_t* n_tokens = nullptr;
    uint64_t* tok_base = nullptr;
    uint32_t* tok_local = nullptr;
    uint64_t* tok_blk = nullptr;
    int32_t* tok_ids = nullptr;          // the records, as TagArgs
    uint8_t* tok_cands = nullptr;
    uint4* tok_desc = nullptr;
    uint32_t* tok_work = nullptr;
    uint64_t max_tokens = 0;
    const TagScoreArgs* scores = nullptr;  // nullable: store every record's score vector
    const vpt_tag_rules* rules = nullptr;  // nullable: PatternMatchTagger
    unsigned long long* rule_words = nullptr;  // with rules: the matched rules' suffix sum, then 4 bytes per token (+ 8)
};

// The tag part of the tokenized writers, after the post-filters (fill_tags sees the final boundaries,
// predict/src/main.rs:157-160): tokens per sentence and their prefix, the tag prediction into per-token records and, with
// rules, every record's rule id (ra).  Fills the tag fields of `t`.
void launch_tag_records(const vpt_predictor& p, const BatchArgs& a, bool normalize, const TagRecords& r, TokArgs& t,
                        TagRuleArgs* ra, cudaStream_t st) {
    CompactArgs k;
    k.n_sent = a.n_sent;
    k.status = a.status;
    k.n_chars = a.n_chars;
    k.boundaries = a.boundaries;
    k.bound_offsets = a.bound_offsets;
    k.n_bound = 0;  // no bit stream on this path
    k.status8 = r.status8;
    k.n_tokens = r.n_tokens;
    k.tok_base = r.tok_base;
    k.tok_local = r.tok_local;
    k.tok_blk = r.tok_blk;
    cuda_check(launch_compact(k, st), "launch(compact)");
    TagArgs g = tag_args(p.dt, a);
    g.tok_base = k.tok_base;
    g.tok_ids = r.tok_ids;
    g.tok_cands = r.tok_cands;
    g.tok_desc = r.tok_desc;
    g.tok_work = r.tok_work;
    g.max_tokens = r.max_tokens;
    g.norm = normalize ? 1 : 0;
    cuda_check(launch_tags(p.dt, g, st, r.scores), "launch(tags)");
    if (r.rules && ra) {
        // the rule id of every token, and the sum of the matched rules' suffix bounds in front of them
        ra->rules = r.rules->dr;
        ra->tok_rule = reinterpret_cast<int32_t*>(r.rule_words + 1);
        cuda_check(launch_rule_lookup(ra->rules, g, const_cast<int32_t*>(ra->tok_rule), r.rule_words, st), "launch(rules)");
    }
    t.tok_base = k.tok_base;
    t.tok_ids = g.tok_ids;
    t.tok_cands = g.tok_cands;
    t.n_tags = uint32_t(p.n_tags);
    t.ts_slot = p.dt.ts_slot;
    t.ts_cand = p.dt.ts_cand;
    t.ts_ref = p.dt.ts_ref;
    t.ts_bytes = p.dt.ts_bytes;
}

// Scores the sentences of `a` (text, offsets, trims, n_sent set; `nbytes` bounds their bytes), runs the --wsconst
// post-filters and, with `job.tags`, predicts the tags of every token into per-token records (the post-filters ran
// first: fill_tags sees the final boundaries, predict/src/main.rs:157-160).  Returns the sentences' TokArgs with the tag
// records; its output fields are left to the caller.  With the score dumps the boundary scores stay in `a.scores` and,
// for --tag-scores, every record's score vector is stored through `sc`.  With `part` (partially annotated lines), the
// caller's markers replace the boundaries they mark after the post-filters, before the tags.  With `ann` (partially
// annotated output, annotate.cu), the boundaries inside `ann->margin` become Unknown before the post-filters; after
// them every boundary's marker goes to `ann->marks` and the Unknown ones get their predicted value back; the tokens
// next to an Unknown boundary lose their tag records.
TokArgs predict_lines(const vpt_predictor& p, Scratch& s, LineChunk& ch, BatchArgs& a, uint64_t nbytes, const LineJob& job,
                      TagRuleArgs* ra = nullptr, TagScoreArgs* sc = nullptr, PartArgs* part = nullptr,
                      AnnArgs* ann = nullptr) {
    const bool normalize = job.normalize, tags = job.tags;
    cudaStream_t st = s.stream;
    const size_t n = size_t(a.n_sent);
    const WorkspaceLayout wl = workspace_layout(n);
    bind_workspace(a, s.ws.ensure(wl.total), n);
    a.status = s.status.ensure(4 * n);
    a.bound_offsets = s.boff.ensure(8 * (n + 1));
    a.boundaries = s.bounds.ensure(nbytes + 4);
    // the callers need the boundaries only (every character is at least one byte: the bytes bound the boundaries)
    a.scores = nullptr;
    DevModel dm = p.dm;
    dm.kytea_norm = normalize ? 1 : 0;
    if (!scores_optional(dm) || (job.dumps & kDumpScores) || (ann && ann->margin > 0))
        a.scores = s.scores.ensure(4 * nbytes + 4);
    if (tags) {
        // tag prediction needs the pattern-id states and the character offsets of the sentences
        a.char_states = s.cst.ensure(4 * nbytes + 16);
        a.type_states = s.tst.ensure(4 * nbytes + 16);
        a.char_offsets = s.coff.ensure(8 * (n + 1));
    }
    if (pipeline_trace()) ch.tr.mark_sub(0, st);  // after the line offsets
    if (!fused_ok(dm)) cuda_check(launch_count(a, st), "launch(count)");
    if (pipeline_trace()) ch.tr.mark_sub(1, st);  // after count + scan (none when the scoring launch is fused)
    cuda_check(launch_score(dm, a, st), "launch(score)");
    if (pipeline_trace()) ch.tr.mark_sub(2, st);  // after the scoring kernel
    TokArgs t;
    t.text = a.text;
    t.offsets = a.offsets;
    t.trims = a.trims;
    t.n_sent = n;
    t.status = a.status;
    t.n_chars = a.n_chars;
    t.boundaries = a.boundaries;
    t.bound_offsets = a.bound_offsets;
    if (ann) {
        ann->n_sent = n;
        ann->status = a.status;
        ann->n_chars = a.n_chars;
        ann->bound_offsets = a.bound_offsets;
        ann->scores = a.scores;
        ann->boundaries = a.boundaries;
        cuda_check(launch_pa_margin(*ann, st), "launch(margin)");
    }
    cuda_check(launch_wsconst(t, a.boundaries, job.wsconst, normalize, st), "launch(wsconst)");
    if (job.wsconst & 0x80u) cuda_check(launch_grapheme(t, a.boundaries, normalize, st), "launch(grapheme)");
    if (part) {
        part->status = a.status;
        part->n_chars = a.n_chars;
        part->bound_offsets = a.bound_offsets;
        part->boundaries = a.boundaries;
        cuda_check(launch_part_apply(*part, st), "launch(part apply)");
    }
    if (ann) cuda_check(launch_pa_marks(*ann, st), "launch(marks)");
    if (tags) {
        TagRecords r;
        r.status8 = s.st8.ensure(n + 16);
        bind_token_counts(s, r, n);
        bind_token_records(p, s, r, nbytes);
        if ((job.dumps & kDumpTagScores) && sc) {
            *sc = bind_tag_scores(s, nbytes, device_score_len_bound(&p));
            r.scores = sc;
        }
        if (job.rules && ra) {
            r.rules = job.rules;
            r.rule_words = s.trule.ensure(4 * nbytes + 16);
        }
        launch_tag_records(p, a, normalize, r, t, ra, st);
        if (ann) {
            ann->tok_base = t.tok_base;
            ann->tok_ids = const_cast<int32_t*>(t.tok_ids);
            ann->tok_rule = ra ? const_cast<int32_t*>(ra->tok_rule) : nullptr;
            cuda_check(launch_pa_untag(*ann, st), "launch(untag)");
        }
    }
    return t;
}

// The start of stage 1, for tokenize and evaluate alike: waits for the chunk's line count and, when it has lines, writes
// their offsets and trims.  Returns the line count; the chunk's `done` event exists on return.
size_t split_lines(Scratch& s, LineChunk& ch) {
    cudaStream_t st = s.stream;
    cuda_check(cudaEventSynchronize(ch.split), "sync(split)");
    const size_t n = size_t(s.totals->lines);
    ch.n_lines = n;
    if (!ch.done) cuda_check(cudaEventCreateWithFlags(&ch.done, cudaEventDisableTiming), "cudaEventCreate");
    if (n == 0) return 0;
    const size_t ng = (n + kGroup - 1) / kGroup;
    ch.sp.offsets = s.off.ensure(8 * (n + 1));
    ch.sp.trims = s.trims.ensure(n + 4);
    s.tokg.ensure(8 * (ng + 2));  // the look-back state words and ticket of the stage's parse and writer
    // the kernels of the stage overwrite outputs (out, lc) the previous chunk of this scratch may still be copying out
    cuda_check(cudaStreamWaitEvent(st, s.ev_out, 0), "cudaStreamWaitEvent");
    if (pipeline_trace()) ch.tr.mark(1, st);
    cuda_check(launch_split_write(ch.sp, st), "launch(split)");
    return n;
}

// The score dumps of a chunk (dump.hpp) behind its token lines, which `t` wrote to the staging buffer: every line's dump
// bytes and token line bytes with their prefixes and totals, one wait for the totals, then the output, sized exactly,
// with its size in `out_bytes`.  The token lines are placed by their computed sizes, not by their '\n's: a tag string
// (of the model or of a rule) may hold a '\n'.
void dump_stage(const vpt_predictor& p, Scratch& s, const TokArgs& t, const BatchArgs& a, const TagScoreArgs& sc,
                const TagRuleArgs& ra, const LineJob& job) {
    cudaStream_t st = s.stream;
    const size_t n = size_t(t.n_sent);
    DumpArgs d;
    d.n_sent = n;
    d.dumps = job.dumps;
    d.norm = job.normalize ? 1 : 0;
    d.text = t.text;
    d.offsets = t.offsets;
    d.trims = t.trims;
    d.status = t.status;
    d.n_chars = t.n_chars;
    d.bound_offsets = t.bound_offsets;
    d.boundaries = t.boundaries;
    d.scores = a.scores;
    if (t.tok_base) {
        d.tok_base = t.tok_base;
        d.tok_ids = t.tok_ids;
        d.tok_cands = t.tok_cands;
        d.n_tags = t.n_tags;
        d.ts_slot = t.ts_slot;
        d.ts_cand = t.ts_cand;
        d.ts_ref = t.ts_ref;
        d.ts_bytes = t.ts_bytes;
        d.tok_rule = ra.tok_rule;
        d.rules = ra.rules;
    }
    if (job.dumps & kDumpTagScores) {
        d.tok_desc = s.tokdesc.get();
        d.rec_off = sc.rec_off;
        d.score_blk = sc.blk;
        d.tag_scores = sc.scores;
        d.tok_info = p.dt.tok_info;
    }
    const size_t nblk = (n + kDumpBlock - 1) / kDumpBlock;
    d.size = s.dsize.ensure(8 * (3 * n + 2 * nblk + 4));
    d.tl_len = d.size + n;
    d.tl_off = d.tl_len + n;
    d.blk = d.tl_off + n;
    d.total_host = s.totals->dump;
    cuda_check(launch_dump_size(d, st), "launch(dump size)");
    cuda_check(cudaStreamSynchronize(st), "sync(dump size)");
    const uint64_t tok_bytes = s.totals->tok_line_bytes, dump_bytes = s.totals->dump[0];
    // token_line_len restates the writers' sizes: a disagreement would misplace every later line of the chunk
    if (s.totals->dump[1] != tok_bytes)
        throw Error(kInternal, "internal error: score dumps: token line sizes (" + std::to_string(s.totals->dump[1]) +
                                   ") disagree with the writer's (" + std::to_string(tok_bytes) + ")");
    d.out = s.out.ensure(tok_bytes + dump_bytes + 4);
    d.tok_lines = s.stage.get();
    cuda_check(launch_dump_write(d, st), "launch(dump)");
    s.totals->out_bytes = tok_bytes - n + dump_bytes;  // dump_line writes each token line's '\n' itself
}

// stage 1: line offsets, count + score, tokenised bytes; the output size to pinned host memory
void lines_stage1(const vpt_predictor& p, Scratch& s, LineChunk& ch, const LineJob& job) {
    cudaStream_t st = s.stream;
    const size_t n = split_lines(s, ch);
    s.totals->out_bytes = 0;
    if (n == 0) { cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord"); return; }
    const size_t ng = (n + kGroup - 1) / kGroup;
    // with the score dumps the token lines go to a staging buffer, and the dump writer puts them in front of their dumps
    DevBuf<uint8_t>& tok_buf = job.dumps ? s.stage : s.out;
    // surface bytes + at most one '\\' per byte + at most one ' ' per character + one '\n' per line
    // (with tags: every token -- at most one per byte -- may get the longest "/tag/.." suffix of the model; the
    // partial-annotation format has one marker per character and no escapes, so the same bound holds for it)
    const size_t out_need = 3 * ch.nbytes + n + 4 + (job.tags ? size_t(ch.nbytes) * p.dt.max_suffix : 0);
    tok_buf.ensure(out_need);
    const bool annotate = job.kind == kJobAnnotate;
    AnnArgs ann;
    if (annotate) {
        ann.margin = job.margin;
        ann.marks = s.gbnd.ensure(ch.nbytes + 4);
    }
    BatchArgs a;
    a.text = ch.sp.text;
    a.offsets = ch.sp.offsets;
    a.trims = ch.sp.trims;
    a.n_sent = n;
    TagRuleArgs ra;
    TagScoreArgs sc;
    TokArgs t = predict_lines(p, s, ch, a, ch.nbytes, job, &ra, &sc, nullptr, annotate ? &ann : nullptr);
    if (ra.tok_rule) {
        // A rule's tag may be long on a short surface, so the rules' share of the output is sized from the suffixes the
        // chunk's tokens actually matched: the host waits for the rule lookup and reads their sum.
        cuda_check(cudaMemcpyAsync(&s.totals->rule_suffix, s.trule.get(), 8, cudaMemcpyDeviceToHost, st), "D2H(rule suffixes)");
        cuda_check(cudaStreamSynchronize(st), "sync(rules)");
        tok_buf.ensure(out_need + size_t(s.totals->rule_suffix));
        uint64_t seen = job.rules->max_out.load();
        while (seen < tok_buf.capacity() && !job.rules->max_out.compare_exchange_weak(seen, tok_buf.capacity())) {}
    }
    t.tok_state = s.tokg.get();
    t.ticket = reinterpret_cast<uint32_t*>(t.tok_state + ng);
    t.total = t.tok_state + ng + 1;
    t.total_host = job.dumps ? &s.totals->tok_line_bytes : &s.totals->out_bytes;
    t.out = tok_buf.get();
    if (annotate) cuda_check(launch_pa_write(t, ra, ann.marks, st), "launch(annotate)");
    else cuda_check(launch_tokenize_rules(t, ra, st), "launch(tok)");
    if (job.dumps) dump_stage(p, s, t, a, sc, ra, job);
    if (pipeline_trace()) ch.tr.mark(2, st);
    cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord");
}

}  // namespace

uint32_t vpt_kytea_fullwidth(uint32_t code_point) { return kytea_fullwidth(code_point); }

namespace {
// The flags of the line loops (vpt_tokenize_lines*, vpt_evaluate_lines); returns whether tags are predicted on the device
bool check_lines_flags(const vpt_predictor* p, uint32_t wsconst_types, bool tags) {
    require_device(p);
    if (tags) {
        if (!p->predict_tags || p->from_blob)
            throw Error(kInvalidArgument, "InvalidArgumentError: this predictor is created with predict_tags = false");
        // (these paths have no per-token fall-back: a token the device cannot serve would be written without its tags)
        if (p->n_tags && (!p->dt.tok_tab || !p->tags_all_usable))
            throw Error(kUnsupported, "this tag model exceeds the limits of the device path (tags.hpp); use vpt_fill_tags");
        if (p->n_tags == 0) tags = false;  // predictor.rs:553-555: nothing to predict
    }
    if (wsconst_types & ~0xFEu)
        throw Error(kInvalidArgument, "InvalidArgumentError: wsconst_types: bits 1..6 (Digit .. Other) and 7 (grapheme clusters) only");
    return tags;
}

LineJob line_job(const vpt_predictor* p, int kind, int no_norm, uint32_t wsconst_types, bool predict_tags,
                 const vpt_tag_rules* rules = nullptr) {
    const bool tags = check_lines_flags(p, wsconst_types, predict_tags);
    // main.rs:110-120 with predictor.rs:553: the system keeps the gold tags (--no-norm) or has none, unless tags are
    // predicted with a model that has tag slots
    LineJob j{kind, no_norm == 0, wsconst_types, tags, tags ? kTagsCompare : no_norm ? kTagsAlwaysEqual : kTagsGoldEmpty};
    if (rules && rules->p != p)
        throw Error(kInvalidArgument, "InvalidArgumentError: rules: made for another predictor");
    // (rules act on predicted tags only: without them, or without any rule, the call is the one without rules)
    if (rules && tags && kind != VPT_STREAM_EVALUATE && rules->n_rules) j.rules = rules;
    return j;
}

// Cuts a buffer of lines into pipeline chunks that end after a '\n' (memrchr from the nominal cut; a line longer than a
// chunk extends it to the line's end); returns the end of every chunk
std::vector<size_t> line_chunks(const uint8_t* utf8, size_t n_bytes) {
    const size_t big = chunk_bytes();
    const std::vector<size_t> sizes = ramp_schedule(n_bytes, big, big / 8, big / 8);
    std::vector<size_t> ends;
    size_t cum = 0, k = 0;
    for (size_t lo = 0; lo < n_bytes;) {
        // every chunk ends at the next nominal cut of the schedule (a line that ran past cuts skips them)
        do { cum = k < sizes.size() ? cum + sizes[k++] : n_bytes; } while (cum <= lo);
        size_t hi = std::min(n_bytes, cum);
        if (hi < n_bytes) {
            const void* q = memrchr(utf8 + lo, 0x0A, hi - lo);
            if (q) hi = size_t(static_cast<const uint8_t*>(q) - utf8) + 1;
            else {
                const void* f = memchr(utf8 + hi, 0x0A, n_bytes - hi);
                hi = f ? size_t(static_cast<const uint8_t*>(f) - utf8) + 1 : n_bytes;
            }
        }
        if (hi - lo > kMaxLineChunk) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: a line is longer than 1 GiB");
        ends.push_back(hi);
        lo = hi;
    }
    return ends;
}

// stage 1 of an evaluate chunk: line offsets, the gold parse, count + score + post-filters (+ tags) on the raw
// sentences, the metrics; the chunk's totals and error key to pinned host memory, the per-line counts (if wanted) to
// `line_counts` from row `line_lo`
void eval_stage1(const vpt_predictor& p, Scratch& s, LineChunk& ch, const LineJob& job, uint32_t* line_counts,
                 uint64_t line_lo) {
    cudaStream_t st = s.stream;
    const size_t n = split_lines(s, ch);
    if (n == 0) {
        for (int i = 0; i < kEvalTotals; ++i) s.totals->eval[i] = 0;
        s.totals->eval[kEvalTotals] = kGoldNoError;
        cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord");
        return;
    }
    const size_t ng = (n + kGroup - 1) / kGroup;
    const size_t nb = ch.nbytes;  // bounds the surface bytes and characters of the chunk
    const int tag_mode = job.tag_mode;
    EvalArgs e;
    e.text = ch.sp.text;
    e.offsets = ch.sp.offsets;
    e.trims = ch.sp.trims;
    e.n_sent = n;
    e.surface = s.gtext.ensure(nb + 64);
    e.surf_offsets = s.goff.ensure(8 * (n + 1));
    e.char_offsets = s.gcoff.ensure(8 * (n + 1));
    e.gold_bnd = s.gbnd.ensure(nb + 4);
    e.width = s.gw.ensure(4 * n + 4);
    e.totals = s.evtot.ensure(8 * (kEvalTotals + 1));
    e.err = e.totals + kEvalTotals;
    e.tag_pos = tag_mode == kTagsCompare ? s.gtag.ensure(4 * nb + 4) : nullptr;
    e.line_counts = line_counts ? s.lc.ensure(28 * n + 4) : nullptr;
    e.state = s.tokg.get();
    e.ticket = reinterpret_cast<uint32_t*>(e.state + ng);
    cuda_check(cudaMemsetAsync(e.totals, 0, 8 * kEvalTotals, st), "cudaMemset");
    cuda_check(cudaMemsetAsync(e.err, 0xFF, 8, st), "cudaMemset");
    cuda_check(launch_gold_parse(e, st), "launch(gold)");
    BatchArgs a;
    a.text = e.surface;
    a.offsets = e.surf_offsets;
    a.n_sent = n;
    const TokArgs t = predict_lines(p, s, ch, a, nb, job);
    e.status = t.status;
    e.n_chars = t.n_chars;
    e.boundaries = t.boundaries;
    e.bound_offsets = t.bound_offsets;
    e.tag_mode = tag_mode;
    if (tag_mode == kTagsCompare) {
        e.n_tags = t.n_tags;
        e.tok_base = t.tok_base;
        e.tok_ids = t.tok_ids;
        e.tok_cands = t.tok_cands;
        e.ts_slot = t.ts_slot;
        e.ts_cand = t.ts_cand;
        e.ts_ref = t.ts_ref;
        e.ts_bytes = t.ts_bytes;
    }
    cuda_check(launch_eval(e, st), "launch(eval)");
    cuda_check(cudaMemcpyAsync(s.totals->eval, e.totals, 8 * (kEvalTotals + 1), cudaMemcpyDeviceToHost, st), "D2H(totals)");
    if (pipeline_trace()) ch.tr.mark(2, st);
    cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord");
    if (line_counts) {
        cuda_check(cudaEventRecord(s.ev_kernels, st), "cudaEventRecord");
        cuda_check(cudaStreamWaitEvent(s.stream_out, s.ev_kernels, 0), "cudaStreamWaitEvent");
        cuda_check(cudaMemcpyAsync(line_counts + 7 * line_lo, s.lc.get(), 28 * n, cudaMemcpyDeviceToHost, s.stream_out), "D2H(counts)");
        cuda_check(cudaEventRecord(s.ev_out, s.stream_out), "cudaEventRecord");
    }
}

// stage 1 of a chunk of partially annotated lines: line offsets, the parse (raw text, markers, error key), count +
// score + post-filters on the raw text, the caller's markers, tags, the tokenized writer over the raw text; the output
// size and the error key to pinned host memory.  kJobReannotate: the margin and the output markers as lines_stage1's
// annotate job, with the caller's markers applied after the post-filters, and the partial-annotation writer; with
// keep_tags the input tag region of every character (k_part_tags) goes to that writer.
void part_stage1(const vpt_predictor& p, Scratch& s, LineChunk& ch, const LineJob& job) {
    cudaStream_t st = s.stream;
    const size_t n = split_lines(s, ch);
    s.totals->out_bytes = 0;
    s.totals->eval[kEvalTotals] = kGoldNoError;
    if (n == 0) { cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord"); return; }
    const size_t ng = (n + kGroup - 1) / kGroup;
    const size_t nb = ch.nbytes;  // bounds the raw bytes, the characters and the markers of the chunk
    PartArgs e;
    e.surface = s.gtext.ensure(nb + 64);
    e.surf_offsets = s.goff.ensure(8 * (n + 1));
    e.char_offsets = s.gcoff.ensure(8 * (n + 1));
    e.given = s.gbnd.ensure(nb + 4);
    e.err = s.evtot.ensure(8 * (kEvalTotals + 1)) + kEvalTotals;
    // as lines_stage1: the raw bytes bound the output of the writer (with tags, the longest suffix per token).  The
    // reannotate writer's line is its raw text, a marker per character after the first, the written input tags and the
    // model's suffixes.  The written input tags of a character are at most the bytes of its tag region, and the raw text,
    // the markers and the tag regions are disjoint parts of the input line: all three together take at most the line's
    // input bytes, so the same bound holds.
    const size_t out_need = 3 * nb + n + 4 + (job.tags ? nb * p.dt.max_suffix : 0);
    const bool reannotate = job.kind == kJobReannotate;
    s.out.ensure(out_need);
    e.text = ch.sp.text;
    e.offsets = ch.sp.offsets;
    e.trims = ch.sp.trims;
    e.n_sent = n;
    e.state = s.tokg.get();
    e.ticket = reinterpret_cast<uint32_t*>(e.state + ng);
    cuda_check(cudaMemsetAsync(e.err, 0xFF, 8, st), "cudaMemset");
    cuda_check(launch_part_parse(e, st), "launch(part parse)");
    PartTagArgs pt;
    if (reannotate && job.keep_tags) {
        // every character of a line is followed by a marker or ends the line: at most (nb + 1) / 2 characters
        pt.regions = s.ptag.ensure(8 * ((nb + 1) / 2 + 2));
        pt.text = e.text;
        pt.offsets = e.offsets;
        pt.trims = e.trims;
        pt.n_sent = n;
        pt.char_offsets = e.char_offsets;
        cuda_check(launch_part_tags(pt, st), "launch(part tags)");
    }
    AnnArgs ann;
    if (reannotate) {
        ann.margin = job.margin;
        ann.marks = s.pmark.ensure(nb + 4);
    }
    BatchArgs a;
    a.text = e.surface;
    a.offsets = e.surf_offsets;
    a.n_sent = n;
    TagRuleArgs ra;
    TokArgs t = predict_lines(p, s, ch, a, nb, job, &ra, nullptr, &e, reannotate ? &ann : nullptr);
    if (ra.tok_rule) {
        // as lines_stage1: the rules' share of the output is sized from the suffixes the chunk's tokens matched
        cuda_check(cudaMemcpyAsync(&s.totals->rule_suffix, s.trule.get(), 8, cudaMemcpyDeviceToHost, st), "D2H(rule suffixes)");
        cuda_check(cudaStreamSynchronize(st), "sync(rules)");
        s.out.ensure(out_need + size_t(s.totals->rule_suffix));
        uint64_t seen = job.rules->max_out.load();
        while (seen < s.out.capacity() && !job.rules->max_out.compare_exchange_weak(seen, s.out.capacity())) {}
    }
    // the look-back words of the parse are free again: the writer's come from the same scratch (its launch zeroes them)
    t.tok_state = s.tokg.get();
    t.ticket = reinterpret_cast<uint32_t*>(t.tok_state + ng);
    t.total = t.tok_state + ng + 1;
    t.total_host = &s.totals->out_bytes;
    t.out = s.out.get();
    if (pt.regions) cuda_check(launch_pa_rewrite(t, ra, ann.marks, e.text, pt.regions, e.char_offsets, st), "launch(reannotate)");
    else if (reannotate) cuda_check(launch_pa_write(t, ra, ann.marks, st), "launch(annotate)");
    else cuda_check(launch_tokenize_rules(t, ra, st), "launch(tok)");
    cuda_check(cudaMemcpyAsync(&s.totals->eval[kEvalTotals], e.err, 8, cudaMemcpyDeviceToHost, st), "D2H(error key)");
    if (pipeline_trace()) ch.tr.mark(2, st);
    cuda_check(cudaEventRecord(ch.done, st), "cudaEventRecord");
}

// The error of a partially annotated line (partial_parse.hpp) from its key; `line` is the line's first byte in the
// chunk's input, which the host still holds
std::string part_error_text(uint32_t kind, const uint8_t* line, uint64_t pos) {
    switch (kind) {
        case kPartNul: return "must not contain NULL";
        case kPartBoundary: {
            // the character at the position (the line is valid UTF-8: its UTF-8 error would come first)
            const uint8_t b = line[pos];
            const size_t len = b < 0x80u ? 1 : b < 0xE0u ? 2 : b < 0xF0u ? 3 : 4;
            return "contains an invalid boundary character: '" + std::string(reinterpret_cast<const char*>(line + pos), len) + "'";
        }
        default: return "invalid annotation";
    }
}

const char* gold_error_text(uint32_t kind) {
    switch (kind) {
        case kGoldEmpty: return "must contain at least one character";
        case kGoldStartWs: return "must not start with a whitespace";
        case kGoldDoubleWs: return "must not contain consecutive whitespaces";
        case kGoldSlash: return "a slash must follow a character";
        case kGoldNul: return "must not contain NULL";
        default: return "must not end with a whitespace";
    }
}

// ---- the line ring: the chunk pipeline of vpt_tokenize_lines*, vpt_evaluate_lines and the line stream ----------------
//
// Every chunk of complete lines goes through lines_stage0 (copy-in, newline count), then lines_stage1 or eval_stage1
// (split, scoring, post-filters, tags, output or metrics), then its owner's copy-out.  Up to kRingDepth chunks are in
// flight, chunk c in slot c % kRingDepth on the slot's own ScratchLease, so the copy-in, kernels and copy-out of
// neighbouring chunks overlap: the two newest chunks are copied in and counted ahead of their kernels, and the next
// chunk's kernels are queued before the host waits for the oldest.  Chunks retire in order.  The ring knows neither where
// a chunk's bytes come from nor where tokenised bytes go: the whole-buffer calls submit cuts of the caller's buffer and
// copy into the caller's output, the stream submits its pinned staging buffers and hands its output to `write`.

struct LineRing {
    struct Slot {
        std::unique_ptr<ScratchLease> lease;
        LineChunk ch;
        bool stage1 = false;  // lines_stage1 / eval_stage1 / part_stage1 issued
        size_t index = 0;     // chunk number
        const uint8_t* input = nullptr;  // the chunk's bytes (untouched until it retires)
    };
    struct Traced {  // trace events of a chunk whose slot was reused before they were printed
        size_t index;
        uint64_t nbytes;
        TraceEvents tr;
    };
    const vpt_predictor& p;
    const LineJob job;
    const char* const label;  // of the trace lines
    const bool trace;
    Slot slots[kRingDepth];
    size_t n_chunks = 0, n_retired = 0;  // chunks [n_retired, n_chunks) are in flight
    uint64_t lines = 0, tot[kEvalTotals] = {};  // of the retired chunks
    // per-line counts of the whole-buffer evaluate call (none: nullptr); a chunk's rows go out only while the buffer has
    // room for all of them
    uint32_t* line_counts = nullptr;
    uint64_t line_capacity = 0, lines_issued = 0;
    bool counts_overflow = false;
    TraceEvents t0;  // trace origin: before the first chunk's copy-in
    std::vector<Traced> traced;

    LineRing(const vpt_predictor& pr, const LineJob& j, const char* what)
        : p(pr), job(j), label(what), trace(pipeline_trace()) {}

    ~LineRing() {
        // last slot first, so that slot 0's scratch is the next one leased: a later ring's slot 0 takes it again
        for (size_t i = kRingDepth; i-- > 0;) {
            Slot& sl = slots[i];
            sl.lease.reset();  // synchronises the lease's streams and hands its scratch back to the predictor
            if (sl.ch.split) cudaEventDestroy(sl.ch.split);
            if (sl.ch.done) cudaEventDestroy(sl.ch.done);
            sl.ch.tr.destroy();
        }
        for (Traced& t : traced) t.tr.destroy();
        t0.destroy();
    }

    Slot& slot(size_t chunk) { return slots[chunk % kRingDepth]; }
    bool full() const { return n_chunks - n_retired == kRingDepth; }

    // queues a chunk of `n` bytes of complete lines at `bytes`, which stay untouched until it retires; the ring must not
    // be full
    void submit(const uint8_t* bytes, size_t n) {
        Slot& sl = slot(n_chunks);  // chunks retire in order: this slot is free
        if (!sl.lease) sl.lease.reset(new ScratchLease(p));
        if (sl.ch.tr.ev[0]) {
            // the slot's last chunk is not printed yet, and its copy-out may still be running
            traced.push_back({sl.index, sl.ch.nbytes, sl.ch.tr});
            sl.ch.tr = TraceEvents();
        }
        sl.ch.nbytes = n;
        sl.ch.n_lines = 0;
        sl.stage1 = false;
        sl.input = bytes;
        sl.index = n_chunks++;
        Scratch& s = *sl.lease->s;
        if (trace && sl.index == 0) t0.mark(0, s.stream);
        lines_stage0(s, sl.ch, bytes);
        for (size_t c = n_retired; c + 2 < n_chunks; ++c)
            if (!slot(c).stage1) issue(slot(c));
    }

    void issue(Slot& sl) {
        Scratch& s = *sl.lease->s;
        if (job.kind == VPT_STREAM_TOKENIZE || job.kind == kJobAnnotate) {
            lines_stage1(p, s, sl.ch, job);
        } else if (job.kind == kJobPartial || job.kind == kJobReannotate) {
            part_stage1(p, s, sl.ch, job);
        } else {
            uint32_t* counts = nullptr;
            if (line_counts) {
                // the chunk's line count is known once its split pass is done
                cuda_check(cudaEventSynchronize(sl.ch.split), "sync(split)");
                if (lines_issued + s.totals->lines <= line_capacity) counts = line_counts;
                else counts_overflow = true;
            }
            eval_stage1(p, s, sl.ch, job, counts, lines_issued);
            lines_issued += sl.ch.n_lines;
        }
        sl.stage1 = true;
    }

    // Waits for the oldest chunk and takes it out of the ring: its lines are counted and, for evaluate, its error key is
    // checked and its totals are added.  Chunks retire in line order, so the first error met is the lowest bad line's.
    // The owner copies the chunk's output out of the returned slot before the next submit reuses it.
    Slot& retire() {
        // the next chunk's kernels are queued before the host waits for the oldest
        for (size_t c = n_retired; c < std::min(n_retired + 2, n_chunks); ++c)
            if (!slot(c).stage1) issue(slot(c));
        Slot& sl = slot(n_retired);
        Scratch& s = *sl.lease->s;
        cuda_check(cudaEventSynchronize(sl.ch.done), "sync(lines)");
        if (job.kind == VPT_STREAM_EVALUATE) {
            const uint64_t key = s.totals->eval[kEvalTotals];
            if (key != kGoldNoError) {
                const uint64_t line = lines + (key >> 34);
                const uint32_t kind = uint32_t(key & 7u);
                if (kind == kGoldUtf8)
                    throw Error(kIoError, "stream did not contain valid UTF-8 (line " + std::to_string(line) + ")");
                throw Error(kInvalidArgument, std::string("InvalidArgumentError: tokenized_text: ") + gold_error_text(kind) +
                                                  " (line " + std::to_string(line) + ")");
            }
            for (int i = 0; i < kEvalTotals; ++i) tot[i] += s.totals->eval[i];
        } else if (job.kind == kJobPartial || job.kind == kJobReannotate) {
            const uint64_t key = s.totals->eval[kEvalTotals];
            if (key != kGoldNoError) {
                const uint64_t l = key >> 34;
                const uint32_t kind = uint32_t(key & 7u);
                const std::string where = " (line " + std::to_string(lines + l) + ")";
                if (kind == kPartUtf8) throw Error(kIoError, "stream did not contain valid UTF-8" + where);
                // the line's first byte: after the l-th '\n' of the chunk
                const uint8_t* q = sl.input;
                for (uint64_t k = 0; k < l; ++k) q = static_cast<const uint8_t*>(memchr(q, 0x0A, sl.input + sl.ch.nbytes - q)) + 1;
                throw Error(kInvalidArgument, "InvalidArgumentError: partial_annotation_text: " +
                                                  part_error_text(kind, q, ((key >> 3) & 0x7FFFFFFFull) - 1) + where);
            }
        }
        lines += sl.ch.n_lines;
        ++n_retired;
        return sl;
    }

    void drain(const std::function<void(Slot&)>& deliver) {
        while (n_retired < n_chunks) deliver(retire());
    }

    // A whole buffer through the ring, in the chunks of line_chunks; `deliver` takes every retired slot.  The final
    // synchronisation is checked: a failed copy-out is an error of the call, not left to the leases' release.
    void run(const uint8_t* utf8, size_t n_bytes, const std::function<void(Slot&)>& deliver) {
        size_t lo = 0;
        for (const size_t hi : line_chunks(utf8, n_bytes)) {
            if (full()) deliver(retire());
            submit(utf8 + lo, hi - lo);
            lo = hi;
        }
        drain(deliver);
        for (Slot& sl : slots)
            if (sl.lease) {
                cuda_check(cudaStreamSynchronize(sl.lease->s->stream), "sync(lines)");
                cuda_check(cudaStreamSynchronize(sl.lease->s->stream_out), "sync(copy-out)");
            }
        if (!trace) return;
        for (const Traced& t : traced) t.tr.print(label, t.index, t.nbytes, t0);
        for (size_t k = 0; k < kRingDepth; ++k) {
            Slot& sl = slot(n_chunks + k);  // oldest first
            if (sl.ch.tr.ev[0]) print(sl);
        }
    }

    // prints the trace line of a retired chunk whose events are complete, and frees them
    void print(Slot& sl) {
        sl.ch.tr.print(label, sl.index, sl.ch.nbytes, t0);
        sl.ch.tr.destroy();
    }

    vpt_eval_counts counts() const {
        vpt_eval_counts c = vpt_eval_counts();
        c.n_lines = lines;
        c.tp = tot[0];
        c.tn = tot[1];
        c.fp = tot[2];
        c.fn = tot[3];
        c.n_sys = tot[4];
        c.n_ref = tot[5];
        c.n_cor = tot[6];
        c.n_sentences = tot[7];
        return c;
    }
};

int tokenize_lines_impl(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int no_norm, uint32_t wsconst_types, bool tags,
                        uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines_out,
                        const vpt_tag_rules* rules = nullptr, int kind = VPT_STREAM_TOKENIZE, int32_t margin = 0,
                        bool keep_tags = false) {
    VPT_API_BEGIN
    LineJob job = line_job(p, kind, no_norm, wsconst_types, tags, rules);
    job.margin = margin;
    job.keep_tags = keep_tags;
    if (out_len) *out_len = 0;
    if (n_lines_out) *n_lines_out = 0;
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    if (n_bytes == 0) return kOk;
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    LineRing ring(*p, job, kind == kJobPartial ? "partial" : kind == kJobAnnotate ? "annotate" : kind == kJobReannotate ? "reannotate" : "lines");
    uint64_t total = 0;  // counts on past an overflow: *out_len is the size needed
    bool overflow = false;
    ring.run(utf8, n_bytes, [&](LineRing::Slot& sl) {
        // the copy-out overlaps the next chunks' copy-in and kernels; the ring's final synchronisation waits for it
        Scratch& s = *sl.lease->s;
        const uint64_t nb = s.totals->out_bytes;
        if (total + nb > out_capacity || (nb && !out)) overflow = true;
        if (!overflow && nb) {
            cuda_check(cudaMemcpyAsync(out + total, s.out.get(), nb, cudaMemcpyDeviceToHost, s.stream_out), "D2H(text)");
            cuda_check(cudaEventRecord(s.ev_out, s.stream_out), "cudaEventRecord");
        }
        if (ring.trace) sl.ch.tr.mark(3, s.stream_out);
        total += nb;
    });
    if (out_len) *out_len = total;
    if (n_lines_out) *n_lines_out = ring.lines;
    if (overflow) throw Error(kInvalidArgument, "InvalidArgumentError: out_capacity: too small for the tokenized text");
    return kOk;
    VPT_API_END
}

}  // namespace

int vpt_tokenize_lines(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int no_norm, uint32_t wsconst_types,
                       uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines_out) {
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, false, out, out_capacity, out_len, n_lines_out);
}

int vpt_tokenize_lines_tags(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int no_norm, uint32_t wsconst_types,
                            uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines_out) {
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, true, out, out_capacity, out_len, n_lines_out);
}

int vpt_tag_rules_new(const vpt_predictor* p, uint64_t n_rules, const uint8_t* surfaces, const uint64_t* surface_offsets,
                      const uint64_t* slot_offsets, const uint32_t* slots, const uint8_t* tags, uint64_t tags_len,
                      vpt_tag_rules** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    if (!p) throw Error(kInvalidArgument, "InvalidArgumentError: predictor: must not be NULL");
    const TagRulesHost t = build_tag_rules(n_rules, surfaces, surface_offsets, slot_offsets, slots, tags, tags_len,
                                           uint32_t(p->n_tags));
    require_device(p);
    std::unique_ptr<vpt_tag_rules> r(new vpt_tag_rules());
    r->p = p;
    r->n_rules = t.n_rules;
    const size_t sizes[6] = {t.tab.size() * sizeof(TagTokenEntry), t.surf.size(), t.slot_first.size() * 4,
                             t.slot_ref.size() * 4, t.tag_bytes.size(), t.suffix.size() * 4};
    const void* srcs[6] = {t.tab.data(), t.surf.data(), t.slot_first.data(), t.slot_ref.data(), t.tag_bytes.data(),
                           t.suffix.data()};
    size_t offs[6], total = 0;
    for (int i = 0; i < 6; ++i) {
        offs[i] = total;
        total = align_up(total + sizes[i], 256);
    }
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    cuda_check(cudaMalloc(&r->d_mem, total), "cudaMalloc(tag rules)");
    uint8_t* base = static_cast<uint8_t*>(r->d_mem);
    for (int i = 0; i < 6; ++i)
        cuda_check(cudaMemcpy(base + offs[i], srcs[i], sizes[i], cudaMemcpyHostToDevice), "cudaMemcpy(tag rules)");
    DevTagRules& d = r->dr;
    d.tab = reinterpret_cast<const TagTokenEntry*>(base + offs[0]);
    d.surf = base + offs[1];
    d.slot_first = reinterpret_cast<const uint32_t*>(base + offs[2]);
    d.slot_ref = reinterpret_cast<const uint2*>(base + offs[3]);
    d.tag_bytes = base + offs[4];
    d.suffix = reinterpret_cast<const uint32_t*>(base + offs[5]);
    d.mask = t.mask;
    d.max_bytes = t.max_bytes;
    for (uint32_t x : t.suffix) r->max_suffix = std::max(r->max_suffix, x);
    *out = r.release();
    return kOk;
    VPT_API_END
}

void vpt_tag_rules_free(vpt_tag_rules* rules) { delete rules; }

uint64_t vpt_tag_rules_max_output(const vpt_tag_rules* rules) { return rules ? rules->max_out.load() : 0; }

int vpt_tokenize_lines_tags_rules(const vpt_predictor* p, const vpt_tag_rules* rules, const uint8_t* utf8, size_t n_bytes,
                                  int no_norm, uint32_t wsconst_types, uint8_t* out, size_t out_capacity, uint64_t* out_len,
                                  uint64_t* n_lines_out) {
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, true, out, out_capacity, out_len, n_lines_out, rules);
}

int vpt_tokenize_partial_lines(const vpt_predictor* p, const vpt_tag_rules* rules, const uint8_t* utf8, size_t n_bytes,
                               int no_norm, uint32_t wsconst_types, int predict_tags, uint8_t* out, size_t out_capacity,
                               uint64_t* out_len, uint64_t* n_lines_out) {
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, predict_tags != 0, out, out_capacity, out_len,
                               n_lines_out, rules, kJobPartial);
}

int vpt_annotate_lines(const vpt_predictor* p, const vpt_tag_rules* rules, const uint8_t* utf8, size_t n_bytes,
                       int no_norm, uint32_t wsconst_types, int predict_tags, int32_t margin, uint8_t* out,
                       size_t out_capacity, uint64_t* out_len, uint64_t* n_lines_out) {
    if (margin < 0) {
        if (out_len) *out_len = 0;
        if (n_lines_out) *n_lines_out = 0;
        return fail(Error(kInvalidArgument, "InvalidArgumentError: margin: must not be negative"));
    }
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, predict_tags != 0, out, out_capacity, out_len,
                               n_lines_out, rules, kJobAnnotate, margin);
}

int vpt_reannotate_lines(const vpt_predictor* p, const vpt_tag_rules* rules, const uint8_t* utf8, size_t n_bytes,
                         int no_norm, uint32_t wsconst_types, int predict_tags, int32_t margin, int keep_tags,
                         uint8_t* out, size_t out_capacity, uint64_t* out_len, uint64_t* n_lines_out) {
    if (margin < 0) {
        if (out_len) *out_len = 0;
        if (n_lines_out) *n_lines_out = 0;
        return fail(Error(kInvalidArgument, "InvalidArgumentError: margin: must not be negative"));
    }
    return tokenize_lines_impl(p, utf8, n_bytes, no_norm, wsconst_types, predict_tags != 0, out, out_capacity, out_len,
                               n_lines_out, rules, kJobReannotate, margin, keep_tags != 0);
}

int vpt_evaluate_lines(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int no_norm, uint32_t wsconst_types,
                       int predict_tags, vpt_eval_counts* out, uint32_t* line_counts, uint64_t line_capacity) {
    VPT_API_BEGIN
    const LineJob job = line_job(p, VPT_STREAM_EVALUATE, no_norm, wsconst_types, predict_tags != 0);
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = vpt_eval_counts();
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    if (n_bytes == 0) return kOk;
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    LineRing ring(*p, job, "evaluate");
    ring.line_counts = line_counts;
    ring.line_capacity = line_capacity;
    ring.run(utf8, n_bytes, [](LineRing::Slot&) {});
    *out = ring.counts();
    if (ring.counts_overflow) throw Error(kInvalidArgument, "InvalidArgumentError: line_capacity: too small for the lines");
    return kOk;
    VPT_API_END
}

// ---- line stream: the loops of vpt_tokenize_lines* and vpt_evaluate_lines, fed in pieces ----------------------------
//
// The stream cuts its input into chunks of complete lines in pinned staging buffers (line_feed.hpp) and submits them to
// a LineRing.  Invariants: a slot's pinned input buffer is not refilled before its chunk retires, which is after the
// chunk's `done` event (recorded after its H2D, on the same stream) has completed; the pinned output buffer is not reused
// before the `write` call that consumed it has returned (chunks retire one at a time, on the caller's thread).

struct vpt_line_stream {
    const vpt_predictor* p;
    const vpt_stream_write_fn write;
    void* const ctx;
    const size_t big;               // nominal chunk size (VPT_CHUNK_BYTES)
    std::unique_ptr<LineRing> ring;
    FeedBuf in[kRingDepth];         // the pinned input of the chunk in each slot of the ring
    std::vector<FeedBuf> spare;     // input buffers of retired chunks
    // every pinned buffer of the stream (pointer, bytes); the destructor hands them to the predictor's pool
    std::vector<std::pair<uint8_t*, size_t>> pinned;
    FeedBuf out;                    // pinned output staging (tokenize), sized by the largest chunk output seen
    LineFeed<vpt_line_stream> feed;
    int status = kOk;               // an earlier error: every later call returns it again with `message`
    std::string message;
    bool finished = false;

    vpt_line_stream(const vpt_predictor* pr, const LineJob& job, vpt_stream_write_fn w, void* c)
        : p(pr), write(w), ctx(c), big(chunk_bytes()), ring(new LineRing(*pr, job, "stream")), feed(*this, big, kMaxLineChunk) {}

    ~vpt_line_stream() {
        ring.reset();  // its leases synchronise their streams: no copy reads the pinned buffers any more
        // pinning memory costs more than a short stream's work: the buffers of chunk size are kept for later streams
        // (at most kRingDepth + 2 per concurrent stream), the others are freed
        std::lock_guard<std::mutex> g(p->mu);
        for (const auto& b : pinned) {
            if (b.second <= 2 * big + big / 2 && p->pinned_pool.size() < 4 * (kRingDepth + 2)) p->pinned_pool.push_back(b);
            else cudaFreeHost(b.first);
        }
    }

    // a pinned buffer of at least n bytes: from the predictor's pool, else a new one
    uint8_t* alloc(size_t& n) {
        {
            std::lock_guard<std::mutex> g(p->mu);
            auto& pool = p->pinned_pool;
            for (size_t i = 0; i < pool.size(); ++i)
                if (pool[i].second >= n && pool[i].second <= 2 * n) {
                    const auto b = pool[i];
                    pool.erase(pool.begin() + long(i));
                    pinned.push_back(b);
                    n = b.second;
                    return b.first;
                }
        }
        void* q = nullptr;
        cuda_check(cudaMallocHost(&q, n), "cudaMallocHost(stream staging)");
        pinned.emplace_back(static_cast<uint8_t*>(q), n);
        return static_cast<uint8_t*>(q);
    }
    void release(uint8_t* q) {
        if (!q) return;
        pinned.erase(std::find_if(pinned.begin(), pinned.end(), [q](const std::pair<uint8_t*, size_t>& b) { return b.first == q; }));
        cudaFreeHost(q);
    }

    // -- LineFeed's host: buffers and chunks
    FeedBuf fresh(size_t min_cap) {
        if (spare.empty() && ring->full()) deliver(ring->retire());
        FeedBuf b;
        if (!spare.empty()) { b = spare.back(); spare.pop_back(); }
        b.size = 0;
        if (b.cap < min_cap || b.cap > 2 * std::max(min_cap, big) + big / 2) {
            // every buffer holds a full chunk, so the ramp at the start allocates nothing twice (a buffer that grew for
            // a line longer than two chunks is not kept)
            release(b.data);
            b.cap = std::max(min_cap, big);
            b.data = alloc(b.cap);
        }
        return b;
    }
    void grow(FeedBuf& b, size_t min_cap) {
        size_t cap = std::max(min_cap, 2 * b.cap);
        uint8_t* q = alloc(cap);
        if (b.size) memcpy(q, b.data, b.size);
        release(b.data);
        b.data = q;
        b.cap = cap;
    }
    [[noreturn]] void too_long() { throw Error(kInvalidArgument, "InvalidArgumentError: utf8: a line is longer than 1 GiB"); }
    void emit(FeedBuf& b) {
        if (ring->full()) deliver(ring->retire());
        FeedBuf& slot_in = in[ring->n_chunks % kRingDepth];  // the slot the chunk goes to
        slot_in = b;
        b = FeedBuf();
        ring->submit(slot_in.data, slot_in.size);
    }

    // delivers a retired chunk: its output to `write` (tokenize; the ring keeps the evaluate totals)
    void deliver(LineRing::Slot& sl) {
        uint64_t nb = 0;
        if (ring->job.kind != VPT_STREAM_EVALUATE) {
            Scratch& s = *sl.lease->s;
            nb = s.totals->out_bytes;
            if (nb > out.cap) {
                release(out.data);
                out.cap = std::max(size_t(nb + nb / 4), big + big / 2);
                out.data = alloc(out.cap);
            }
            if (nb) cuda_check(cudaMemcpyAsync(out.data, s.out.get(), nb, cudaMemcpyDeviceToHost, s.stream_out), "D2H(text)");
            if (ring->trace) sl.ch.tr.mark(3, s.stream_out);
            cuda_check(cudaStreamSynchronize(s.stream_out), "sync(copy-out)");
        }
        if (ring->trace) ring->print(sl);
        FeedBuf& slot_in = in[sl.index % kRingDepth];
        spare.push_back(slot_in);
        slot_in = FeedBuf();
        if (nb && write(ctx, out.data, size_t(nb)) != 0) throw Error(kIoError, "write callback failed");
    }

    void drain() {
        ring->drain([this](LineRing::Slot& sl) { deliver(sl); });
    }
};

namespace {

// Runs `f` on a live stream: an error poisons the stream, and every later call returns it again.
int stream_call(vpt_line_stream* st, const std::function<void()>& f) {
    if (!st) return fail(Error(kInvalidArgument, "InvalidArgumentError: stream: must not be NULL"));
    if (st->status != kOk) {
        set_last_error(st->message);
        return st->status;
    }
    if (st->finished) return fail(Error(kInvalidArgument, "InvalidArgumentError: stream: already finished"));
    try {
        cuda_check(cudaSetDevice(st->p->device), "cudaSetDevice");
        f();
        return kOk;
    } catch (const Error& e) {
        st->status = e.code;
        st->message = e.what();
    } catch (const std::exception& e) {
        st->status = kInternal;
        st->message = std::string("internal error: ") + e.what();
    }
    set_last_error(st->message);
    return st->status;
}

}  // namespace

int vpt_line_stream_new(const vpt_predictor* p, int kind, int no_norm, uint32_t wsconst_types, int predict_tags,
                        vpt_stream_write_fn write, void* ctx, vpt_line_stream** out) {
    return vpt_line_stream_new_rules(p, nullptr, kind, no_norm, wsconst_types, predict_tags, write, ctx, out);
}

int vpt_line_stream_new_rules(const vpt_predictor* p, const vpt_tag_rules* rules, int kind, int no_norm,
                              uint32_t wsconst_types, int predict_tags, vpt_stream_write_fn write, void* ctx,
                              vpt_line_stream** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    if (kind != VPT_STREAM_TOKENIZE && kind != VPT_STREAM_EVALUATE)
        throw Error(kInvalidArgument, "InvalidArgumentError: kind: VPT_STREAM_TOKENIZE or VPT_STREAM_EVALUATE");
    const LineJob job = line_job(p, kind, no_norm, wsconst_types, predict_tags != 0, rules);
    if (kind == VPT_STREAM_TOKENIZE && !write) throw Error(kInvalidArgument, "InvalidArgumentError: write: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    *out = new vpt_line_stream(p, job, write, ctx);
    return kOk;
    VPT_API_END
}

int vpt_line_stream_new_scores(const vpt_predictor* p, const vpt_tag_rules* rules, int no_norm, uint32_t wsconst_types,
                               int predict_tags, uint32_t dumps, vpt_stream_write_fn write, void* ctx,
                               vpt_line_stream** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    LineJob job = line_job(p, VPT_STREAM_TOKENIZE, no_norm, wsconst_types, predict_tags != 0, rules);
    if (!write) throw Error(kInvalidArgument, "InvalidArgumentError: write: must not be NULL");
    if (dumps & ~uint32_t(VPT_DUMP_SCORES | VPT_DUMP_TAG_SCORES))
        throw Error(kInvalidArgument, "InvalidArgumentError: dumps: VPT_DUMP_SCORES and VPT_DUMP_TAG_SCORES only");
    // Token::tag_candidates panics on a sentence without tag scores (sentence.rs:1230-1233): fill_tags did not run, or
    // predicted nothing because the model has no tag slots (predictor.rs:553-555)
    if ((dumps & VPT_DUMP_TAG_SCORES) && !predict_tags)
        throw Error(kInvalidArgument, "InvalidArgumentError: dumps: VPT_DUMP_TAG_SCORES needs predict_tags");
    if ((dumps & VPT_DUMP_TAG_SCORES) && !job.tags)
        throw Error(kInvalidArgument, "InvalidArgumentError: dumps: VPT_DUMP_TAG_SCORES needs a model with tag slots");
    job.dumps = dumps;
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    *out = new vpt_line_stream(p, job, write, ctx);
    return kOk;
    VPT_API_END
}

int vpt_line_stream_new_partial(const vpt_predictor* p, const vpt_tag_rules* rules, int no_norm, uint32_t wsconst_types,
                                int predict_tags, vpt_stream_write_fn write, void* ctx, vpt_line_stream** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    const LineJob job = line_job(p, kJobPartial, no_norm, wsconst_types, predict_tags != 0, rules);
    if (!write) throw Error(kInvalidArgument, "InvalidArgumentError: write: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    *out = new vpt_line_stream(p, job, write, ctx);
    return kOk;
    VPT_API_END
}

int vpt_line_stream_new_annotate(const vpt_predictor* p, const vpt_tag_rules* rules, int no_norm, uint32_t wsconst_types,
                                 int predict_tags, int32_t margin, vpt_stream_write_fn write, void* ctx,
                                 vpt_line_stream** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    LineJob job = line_job(p, kJobAnnotate, no_norm, wsconst_types, predict_tags != 0, rules);
    if (margin < 0) throw Error(kInvalidArgument, "InvalidArgumentError: margin: must not be negative");
    job.margin = margin;
    if (!write) throw Error(kInvalidArgument, "InvalidArgumentError: write: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    *out = new vpt_line_stream(p, job, write, ctx);
    return kOk;
    VPT_API_END
}

int vpt_line_stream_new_reannotate(const vpt_predictor* p, const vpt_tag_rules* rules, int no_norm,
                                   uint32_t wsconst_types, int predict_tags, int32_t margin, int keep_tags,
                                   vpt_stream_write_fn write, void* ctx, vpt_line_stream** out) {
    VPT_API_BEGIN
    if (!out) throw Error(kInvalidArgument, "InvalidArgumentError: out: must not be NULL");
    *out = nullptr;
    LineJob job = line_job(p, kJobReannotate, no_norm, wsconst_types, predict_tags != 0, rules);
    if (margin < 0) throw Error(kInvalidArgument, "InvalidArgumentError: margin: must not be negative");
    job.margin = margin;
    job.keep_tags = keep_tags != 0;
    if (!write) throw Error(kInvalidArgument, "InvalidArgumentError: write: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    *out = new vpt_line_stream(p, job, write, ctx);
    return kOk;
    VPT_API_END
}

int vpt_line_stream_feed(vpt_line_stream* st, const uint8_t* bytes, size_t n) {
    return stream_call(st, [&] {
        if (n && !bytes) throw Error(kInvalidArgument, "InvalidArgumentError: bytes: must not be NULL");
        st->feed.feed(bytes, n);
    });
}

int vpt_line_stream_flush(vpt_line_stream* st) {
    return stream_call(st, [&] {
        st->feed.flush();
        st->drain();
    });
}

int vpt_line_stream_finish(vpt_line_stream* st, uint64_t* n_lines, vpt_eval_counts* counts) {
    if (n_lines) *n_lines = 0;
    if (counts) *counts = vpt_eval_counts();
    return stream_call(st, [&] {
        st->feed.finish();
        st->drain();
        st->finished = true;
        if (n_lines) *n_lines = st->ring->lines;
        if (counts && st->ring->job.kind == VPT_STREAM_EVALUATE) *counts = st->ring->counts();
    });
}

void vpt_line_stream_free(vpt_line_stream* st) {
    if (!st) return;
    cudaSetDevice(st->p->device);
    delete st;
}

namespace {

constexpr size_t kSingleMaxBytes = 2048;   // sentences up to this size take the one-round-trip path of vpt_predict
constexpr size_t kSingleIoBytes = 65536;

// Predictor::predict for ONE sentence (reference predictor.rs:518-543) with one launch and no copy calls: the text and the
// offsets are written into pinned host memory the kernel reads directly (zero-copy over PCIe; the tile loader's bulk copy
// takes a host address like any other), the results are stored straight into the same pinned block, and the look-back
// words + ticket live in a small device block that the kernel itself leaves zeroed (BatchArgs::self_clean).  The call is
// a memcpy into the pinned block, one kernel launch, one stream synchronisation.  (The batch pipeline costs several copies,
// a memset node and three synchronisations per call.)
bool predict_single_fast(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int32_t* scores_out, uint8_t* boundaries_out,
                         size_t out_capacity, uint32_t* char_states_out, uint32_t* type_states_out, size_t states_capacity,
                         uint64_t* n_chars_out) {
    if (n_bytes == 0 || n_bytes > kSingleMaxBytes || !fused_ok(p->dm) || (p->dm.ct.present && p->dm.ct.has_overflow)) return false;
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    ScratchLease lease(*p);
    Scratch& s = *lease.s;
    if (!s.d_io) {  // d_io is set last: after a first call that failed half-way, the next one allocates both again
        uint8_t* h = nullptr;
        cuda_check(cudaHostAlloc(reinterpret_cast<void**>(&h), kSingleIoBytes, cudaHostAllocMapped), "cudaHostAlloc");
        s.h_io.reset(h);
        uint8_t* d = nullptr;
        cuda_check(cudaMalloc(&d, 256), "cudaMalloc(single)");
        std::unique_ptr<uint8_t[], CudaFree> dev(d);
        cuda_check(cudaMemset(d, 0, 256), "cudaMemset(single)");
        s.d_io = std::move(dev);
    }
    uint8_t* const io = s.h_io.get();
    // layout of the pinned block: input part first, then the outputs
    const size_t o_text = 0;                                   // text, then 64 readable bytes
    const size_t o_off = align_up(n_bytes + 64, 16);           // u64 offsets[2]
    const size_t in_bytes = o_off + 16;
    const size_t o_boff = align_up(in_bytes, 16);              // u64 bound_offsets[2]
    const size_t o_coff = o_boff + 16;                         // u64 char_offsets[2]
    const size_t o_stat = o_coff + 16;                         // i32 status, u32 n_chars
    const size_t o_bnd = o_stat + 16;                          // u8 boundaries
    const size_t o_sc = align_up(o_bnd + n_bytes, 16);         // i32 scores
    const size_t o_cst = o_sc + 4 * n_bytes;                   // u32 states
    const size_t o_tst = o_cst + 4 * n_bytes;
    const size_t end = o_tst + 4 * n_bytes;
    if (end > kSingleIoBytes) return false;
    memcpy(io + o_text, utf8, n_bytes);
    memset(io + o_text + n_bytes, 0, o_off - n_bytes);
    uint64_t offs[2] = {0, n_bytes};
    memcpy(io + o_off, offs, 16);
    cudaStream_t st = s.stream;
    uint8_t* hd = nullptr;  // the device's address of the pinned block (the same value under unified addressing)
    cuda_check(cudaHostGetDevicePointer(reinterpret_cast<void**>(&hd), io, 0), "cudaHostGetDevicePointer");
    uint8_t* d = s.d_io.get();
    BatchArgs a;
    a.text = hd + o_text;
    a.offsets = reinterpret_cast<const uint64_t*>(hd + o_off);
    a.n_sent = 1;
    a.group_bound = reinterpret_cast<uint64_t*>(d);
    a.group_char = reinterpret_cast<uint64_t*>(d + 64);
    a.ticket = reinterpret_cast<uint32_t*>(d + 128);
    a.prezeroed = true;
    a.self_clean = true;
    a.n_chars = reinterpret_cast<uint32_t*>(hd + o_stat + 4);
    a.status = reinterpret_cast<int32_t*>(hd + o_stat);
    a.bound_offsets = reinterpret_cast<uint64_t*>(hd + o_boff);
    a.char_offsets = reinterpret_cast<uint64_t*>(hd + o_coff);
    a.boundaries = hd + o_bnd;
    a.scores = scores_out ? reinterpret_cast<int32_t*>(hd + o_sc) : nullptr;
    const bool want_states = char_states_out || type_states_out;
    if (want_states) {
        a.char_states = reinterpret_cast<uint32_t*>(hd + o_cst);
        a.type_states = reinterpret_cast<uint32_t*>(hd + o_tst);
    }
    cuda_check(launch_fused(p->dm, a, st), "launch(single)");
    cuda_check(cudaStreamSynchronize(st), "sync(single)");
    int32_t status;
    uint32_t n;
    memcpy(&status, io + o_stat, 4);
    memcpy(&n, io + o_stat + 4, 4);
    if (n_chars_out) *n_chars_out = n;
    if (status != 0) throw Error(kInternal, "internal error: device validation disagrees with host validation");
    const size_t nb = n > 0 ? n - 1 : 0;
    if (nb > out_capacity || (nb && !boundaries_out) || (want_states && n > states_capacity))
        throw Error(kInvalidArgument, "InvalidArgumentError: out_capacity/states_capacity: too small for the batch");
    if (nb) {
        memcpy(boundaries_out, io + o_bnd, nb);
        if (scores_out) memcpy(scores_out, io + o_sc, 4 * nb);
    }
    if (char_states_out) memcpy(char_states_out, io + o_cst, 4 * size_t(n));
    if (type_states_out) memcpy(type_states_out, io + o_tst, 4 * size_t(n));
    return true;
}

}  // namespace

int vpt_predict(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, int32_t* scores_out, uint8_t* boundaries_out,
                size_t out_capacity, uint32_t* char_states_out, uint32_t* type_states_out, size_t states_capacity,
                uint64_t* n_chars_out) {
    VPT_API_BEGIN
    if (!p) throw Error(kInvalidArgument, "InvalidArgumentError: predictor: must not be NULL");
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    check_raw_text(utf8, n_bytes);
    require_device(p);
    if (predict_single_fast(p, utf8, n_bytes, scores_out, boundaries_out, out_capacity, char_states_out, type_states_out,
                            states_capacity, n_chars_out))
        return kOk;
    const uint64_t offs[2] = {0, n_bytes};
    uint64_t boff[2], nb = 0, nc = 0;
    int32_t status = 0;
    uint8_t dummy = 0;
    int rc = vpt_predict_batch(p, utf8, offs, 1, scores_out, boundaries_out ? boundaries_out : &dummy, out_capacity, boff,
                               &status, char_states_out, type_states_out, states_capacity, nullptr, &nb, &nc);
    if (n_chars_out) *n_chars_out = nc;
    if (rc != kOk) return rc;
    if (status != 0) throw Error(kInternal, "internal error: device validation disagrees with host validation");
    return kOk;
    VPT_API_END
}

int vpt_char_types(const uint8_t* utf8, size_t n_bytes, uint8_t* types_out, size_t capacity, uint64_t* n_chars_out) {
    VPT_API_BEGIN
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    check_raw_text(utf8, n_bytes);
    std::vector<uint32_t> cps = utf8_to_codepoints(std::string(reinterpret_cast<const char*>(utf8), n_bytes));
    if (n_chars_out) *n_chars_out = cps.size();
    if (cps.size() > capacity) throw Error(kInvalidArgument, "InvalidArgumentError: capacity: too small");
    for (size_t i = 0; i < cps.size(); ++i) types_out[i] = host_char_type(cps[i]);
    return kOk;
    VPT_API_END
}

int vpt_split_linebreaks(const uint8_t* utf8, size_t n_bytes, uint8_t* boundaries, size_t n_boundaries) {
    VPT_API_BEGIN
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    check_raw_text(utf8, n_bytes);
    const std::vector<uint32_t> cps = utf8_to_codepoints(std::string(reinterpret_cast<const char*>(utf8), n_bytes));
    if (cps.size() != n_boundaries + 1 || (n_boundaries && !boundaries))
        throw Error(kInvalidArgument, "InvalidArgumentError: boundaries: one per pair of adjacent characters");
    auto lb = [](uint32_t c) { return c == 0x0D || c == 0x0A; };
    for (size_t i = 0; i + 1 < cps.size(); ++i)
        if (lb(cps[i]) || lb(cps[i + 1])) boundaries[i] = 1;
    return kOk;
    VPT_API_END
}

int vpt_concat_grapheme_clusters(const uint8_t* utf8, size_t n_bytes, uint8_t* boundaries, size_t n_boundaries) {
    VPT_API_BEGIN
    if (n_bytes && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    check_raw_text(utf8, n_bytes);
    const std::vector<uint32_t> cps = utf8_to_codepoints(std::string(reinterpret_cast<const char*>(utf8), n_bytes));
    if (cps.size() != n_boundaries + 1 || (n_boundaries && !boundaries))
        throw Error(kInvalidArgument, "InvalidArgumentError: boundaries: one per pair of adjacent characters");
    GraphemeState st;
    for (size_t i = 0; i < cps.size(); ++i) {
        const bool brk = grapheme_step(st, grapheme_class(kGraphemeTable, cps[i]));
        if (!brk && i > 0) boundaries[i - 1] = 0;
    }
    return kOk;
    VPT_API_END
}

uint32_t vpt_tag_n_tokens(const vpt_predictor* p) { return p ? uint32_t(p->tag_preds.size()) : 0; }

const char* vpt_tag_string(const vpt_predictor* p, uint32_t token_id, uint32_t slot, uint32_t cand) {
    if (!p || token_id >= p->tag_preds.size()) return nullptr;
    const auto& t = p->tag_preds[token_id].tags;
    if (slot >= t.size() || cand >= t[slot].size()) return nullptr;
    return t[slot][cand].c_str();
}

uint32_t vpt_tag_n_candidates(const vpt_predictor* p, uint32_t token_id, uint32_t slot) {
    if (!p || token_id >= p->tag_preds.size()) return 0;
    const auto& t = p->tag_preds[token_id].tags;
    return slot < t.size() ? uint32_t(t[slot].size()) : 0;
}

uint32_t vpt_tag_n_slots(const vpt_predictor* p, uint32_t token_id) {
    if (!p || token_id >= p->tag_preds.size()) return 0;
    return uint32_t(p->tag_preds[token_id].tags.size());
}

uint32_t vpt_tag_score_len(const vpt_predictor* p, uint32_t token_id) {
    if (!p || token_id >= p->tag_preds.size()) return 0;
    return uint32_t(p->tag_preds[token_id].bias.size());
}

int vpt_predict_tags_batch_dev(const vpt_predictor* p, const uint8_t* d_utf8, const uint64_t* d_byte_offsets, size_t n_sent,
                               const int32_t* d_status, const uint8_t* d_boundaries, const uint64_t* d_bound_offsets,
                               const uint64_t* d_char_offsets, const uint32_t* d_char_states, const uint32_t* d_type_states,
                               int32_t* d_tag_token, int32_t* d_tag_cand, uint32_t* d_unserved, void* cuda_stream) {
    VPT_API_BEGIN
    require_device(p);
    if (!p->predict_tags || p->from_blob)
        throw Error(kInvalidArgument, "InvalidArgumentError: this predictor is created with predict_tags = false");
    if (n_sent == 0) return kOk;
    if (!p->dt.tok_tab)
        throw Error(kUnsupported, "this tag model exceeds the limits of the device path (tags.hpp); use vpt_fill_tags");
    if (!d_utf8 || !d_byte_offsets || !d_status || !d_boundaries || !d_bound_offsets || !d_char_offsets || !d_tag_token || !d_tag_cand)
        throw Error(kInvalidArgument, "InvalidArgumentError: device buffers: must not be NULL");
    if (reinterpret_cast<uintptr_t>(d_utf8) & 15)
        throw Error(kInvalidArgument, "InvalidArgumentError: d_utf8: must be 16-byte aligned");
    if ((p->dt.char_rels && !d_char_states) || (p->dt.type_rels && !d_type_states))
        throw Error(kInvalidArgument, "InvalidArgumentError: states: required for tag prediction");
    TagArgs t;
    t.text = d_utf8;
    t.offsets = d_byte_offsets;
    t.n_sent = n_sent;
    t.status = d_status;
    t.boundaries = d_boundaries;
    t.bound_offsets = d_bound_offsets;
    t.char_offsets = d_char_offsets;
    t.char_states = p->dt.char_rels ? d_char_states : nullptr;
    t.type_states = p->dt.type_rels ? d_type_states : nullptr;
    t.tag_token = d_tag_token;
    t.tag_cand = d_tag_cand;
    t.n_unserved = d_unserved;
    cuda_check(launch_tags(p->dt, t, static_cast<cudaStream_t>(cuda_stream)), "launch(tags)");
    return kOk;
    VPT_API_END
}

int vpt_predict_batch_tags(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                           int32_t* scores_out, uint8_t* boundaries_out, size_t out_capacity, uint64_t* bound_offsets_out,
                           int32_t* status_out, int32_t* tag_token_out, int32_t* tag_cand_out, size_t chars_capacity,
                           uint64_t* char_offsets_out, uint64_t* n_boundaries_out, uint64_t* n_chars_out,
                           uint64_t* n_unserved_out) {
    VPT_API_BEGIN
    require_device(p);
    if (n_boundaries_out) *n_boundaries_out = 0;
    if (n_chars_out) *n_chars_out = 0;
    if (n_unserved_out) *n_unserved_out = 0;
    if (!p->predict_tags || p->from_blob)
        throw Error(kInvalidArgument, "InvalidArgumentError: this predictor is created with predict_tags = false");
    if (!p->dt.tok_tab)
        throw Error(kUnsupported, "this tag model exceeds the limits of the device path (tags.hpp); use vpt_fill_tags");
    if (!byte_offsets || !bound_offsets_out || !char_offsets_out || !tag_token_out || !tag_cand_out || !boundaries_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: output buffers: must not be NULL");
    if (n_sent == 0) { bound_offsets_out[0] = 0; char_offsets_out[0] = 0; return kOk; }
    if (byte_offsets[n_sent] < byte_offsets[0])
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets: must be non-decreasing");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    // one chunk: text in, scoring with the pattern-id states kept on the device, tag prediction, results out
    ScratchLease lease(*p);
    Scratch& s = *lease.s;
    cudaStream_t st = s.stream;
    const uint64_t byte_lo = byte_offsets[0], nbytes = byte_offsets[n_sent] - byte_lo;
    const size_t shift = size_t(byte_lo & 15);
    const WorkspaceLayout wl = workspace_layout(n_sent);
    const size_t nt = p->n_tags;
    BatchArgs a;
    uint8_t* const text = s.text.ensure(shift + nbytes + 64);
    uint64_t* const offsets = s.off.ensure(8 * (n_sent + 1));
    bind_workspace(a, s.ws.ensure(wl.total), n_sent);
    a.status = s.status.ensure(4 * n_sent);
    a.bound_offsets = s.boff.ensure(8 * (n_sent + 1));
    a.char_offsets = s.coff.ensure(8 * (n_sent + 1));
    a.scores = s.scores.ensure(4 * nbytes + 16);      // a character has at least one byte
    a.boundaries = s.bounds.ensure(nbytes + 16);
    a.char_states = s.cst.ensure(4 * nbytes + 16);
    a.type_states = s.tst.ensure(4 * nbytes + 16);
    int32_t* const tag_token = s.tok.ensure(4 * nbytes + 16);
    // the i32 candidates of every character, in the buffer that holds the u8 candidates of token records elsewhere
    int32_t* const tag_cand = reinterpret_cast<int32_t*>(s.cand.ensure(4 * nbytes * nt + 16));
    if (nbytes)
        cuda_check(cudaMemcpyAsync(text + shift, utf8 + byte_lo, nbytes, cudaMemcpyHostToDevice, st), "H2D(text)");
    cuda_check(cudaMemcpyAsync(offsets, byte_offsets, 8 * (n_sent + 1), cudaMemcpyHostToDevice, st), "H2D(offsets)");
    a.text = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(text) + shift - uintptr_t(byte_lo));
    a.offsets = offsets;
    a.n_sent = n_sent;
    a.totals_host = s.totals->bounds_chars;
    cuda_check(launch_batch(p->dm, a, st), "launch(batch)");
    // a word behind the ticket in the workspace's 256-byte ticket slot
    uint32_t* d_unserved = reinterpret_cast<uint32_t*>(s.ws.get() + wl.ticket + 128);
    cuda_check(cudaMemsetAsync(d_unserved, 0, 4, st), "memset");
    TagArgs t = tag_args(p->dt, a);
    t.tag_token = tag_token;
    t.tag_cand = tag_cand;
    t.n_unserved = d_unserved;
    cuda_check(launch_tags(p->dt, t, st), "launch(tags)");
    cuda_check(cudaStreamSynchronize(st), "sync(tags)");  // the totals are in pinned host memory now
    const uint64_t nb = s.totals->bounds_chars[0], nc = s.totals->bounds_chars[1];
    if (n_boundaries_out) *n_boundaries_out = nb;
    if (n_chars_out) *n_chars_out = nc;
    if (nb > out_capacity || nc > chars_capacity)
        throw Error(kInvalidArgument, "InvalidArgumentError: out_capacity/chars_capacity: too small for the batch");
    uint32_t unserved = 0;
    cuda_check(cudaMemcpyAsync(&unserved, d_unserved, 4, cudaMemcpyDeviceToHost, st), "D2H");
    if (nb) {
        if (scores_out) cuda_check(cudaMemcpyAsync(scores_out, a.scores, 4 * nb, cudaMemcpyDeviceToHost, st), "D2H(scores)");
        cuda_check(cudaMemcpyAsync(boundaries_out, a.boundaries, nb, cudaMemcpyDeviceToHost, st), "D2H(boundaries)");
    }
    cuda_check(cudaMemcpyAsync(bound_offsets_out, a.bound_offsets, 8 * (n_sent + 1), cudaMemcpyDeviceToHost, st), "D2H(offsets)");
    cuda_check(cudaMemcpyAsync(char_offsets_out, a.char_offsets, 8 * (n_sent + 1), cudaMemcpyDeviceToHost, st), "D2H(offsets)");
    if (status_out) cuda_check(cudaMemcpyAsync(status_out, a.status, 4 * n_sent, cudaMemcpyDeviceToHost, st), "D2H(status)");
    if (nc) {
        cuda_check(cudaMemcpyAsync(tag_token_out, tag_token, 4 * nc, cudaMemcpyDeviceToHost, st), "D2H(tags)");
        cuda_check(cudaMemcpyAsync(tag_cand_out, tag_cand, 4 * nc * nt, cudaMemcpyDeviceToHost, st), "D2H(tags)");
    }
    cuda_check(cudaStreamSynchronize(st), "sync(copy-out)");
    if (n_unserved_out) *n_unserved_out = unserved;
    return kOk;
    VPT_API_END
}

namespace {

// The longest score vector k_tok_score stores for a token of this predictor: the device path serves tokens of at most
// kTagMaxScores scores.  A chunk of `nc` characters has at most nc token records, so nc x this bounds its scores.
size_t device_score_len_bound(const vpt_predictor* p) {
    size_t m = 0;
    for (const TagPredictorHost& tp : p->tag_preds) m = std::max(m, tp.bias.size());
    return std::min<size_t>(m, size_t(kTagMaxScores));
}

// Scratch of the tag candidate scores of one chunk of at most `nc` token records; its total arrives in `tag_scores`.
TagScoreArgs bind_tag_scores(Scratch& s, uint64_t nc, size_t len_bound) {
    TagScoreArgs sc;
    sc.rec_off = s.scoff.ensure(4 * nc + 16);
    sc.blk = s.scblk.ensure(8 * (nc / kScoreScanBlock + 4));
    sc.scores = s.tagsc.ensure(4 * nc * len_bound + 16);
    s.totals->tag_scores = 0;
    sc.total_host = &s.totals->tag_scores;
    return sc;
}

}  // namespace

int vpt_predict_batch_compact(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                              uint32_t* boundary_bits_out, size_t bits_capacity_words, uint32_t* n_chars_out,
                              uint8_t* status_out, uint32_t* n_tokens_out, int32_t* token_ids_out, uint8_t* token_cands_out,
                              size_t token_capacity, uint64_t* n_boundaries_out, uint64_t* n_tokens_total_out,
                              uint64_t* n_unserved_out) {
    return vpt_predict_batch_compact_tag_scores(p, utf8, byte_offsets, n_sent, boundary_bits_out, bits_capacity_words, n_chars_out,
                                                status_out, n_tokens_out, token_ids_out, token_cands_out, token_capacity,
                                                n_boundaries_out, n_tokens_total_out, n_unserved_out, nullptr, 0, nullptr);
}

int vpt_predict_batch_compact_tag_scores(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_sent,
                                         uint32_t* boundary_bits_out, size_t bits_capacity_words, uint32_t* n_chars_out,
                                         uint8_t* status_out, uint32_t* n_tokens_out, int32_t* token_ids_out,
                                         uint8_t* token_cands_out, size_t token_capacity, uint64_t* n_boundaries_out,
                                         uint64_t* n_tokens_total_out, uint64_t* n_unserved_out, int32_t* tag_scores_out,
                                         size_t score_capacity, uint64_t* n_scores_total_out) {
    VPT_API_BEGIN
    require_device(p);
    if (n_boundaries_out) *n_boundaries_out = 0;
    if (n_tokens_total_out) *n_tokens_total_out = 0;
    if (n_unserved_out) *n_unserved_out = 0;
    if (n_scores_total_out) *n_scores_total_out = 0;
    const bool want_tags = token_ids_out != nullptr || token_cands_out != nullptr;
    const bool want_tokens = want_tags || n_tokens_out != nullptr;
    const bool want_scores = tag_scores_out != nullptr;
    if (want_scores && !want_tags)
        throw Error(kInvalidArgument, "InvalidArgumentError: tag_scores_out: needs token_ids_out (tag prediction)");
    if (want_tags) {
        if (!p->predict_tags || p->from_blob)
            throw Error(kInvalidArgument, "InvalidArgumentError: this predictor is created with predict_tags = false");
        if (!p->dt.tok_tab)
            throw Error(kUnsupported, "this tag model exceeds the limits of the device path (tags.hpp); use vpt_fill_tags");
        if (!token_ids_out || (p->n_tags && !token_cands_out) || !n_tokens_out)
            throw Error(kInvalidArgument, "InvalidArgumentError: token_ids_out/token_cands_out/n_tokens_out: must not be NULL");
    }
    if (!byte_offsets || !n_chars_out || !status_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets/n_chars_out/status_out: must not be NULL");
    if (n_sent == 0) return kOk;
    if (byte_offsets[n_sent] < byte_offsets[0])
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets: must be non-decreasing");
    if (byte_offsets[n_sent] > byte_offsets[0] && !utf8)
        throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");

    // Every chunk goes through the batch ring: copy-in + count pass (the boundaries and characters of the chunk), then
    // scoring (+ tag prediction) + compaction (the chunk's first boundary bit is known from the running total), then,
    // one chunk behind, the copy-out (bit words, per-sentence words, token records at the running token total).
    BatchRing ring(*p, "compact", "sync(score)", byte_offsets, sentence_chunks(byte_offsets, n_sent));
    const size_t nchunks = ring.chunks.size();
    const size_t nt = want_tags ? p->n_tags : 0;
    const size_t score_len = want_scores ? device_score_len_bound(p) : 0;
    uint64_t nb_total = 0, tok_total = 0, unserved_total = 0, score_total = 0;
    bool overflow = false;
    // pinned words that receive every chunk's first bit word (merged into the output at the end)
    Scratch& s0 = ring.scratch(0);
    if (s0.side_words < nchunks) {
        s0.h_side.reset();
        s0.side_words = 0;
        const size_t want = std::max<size_t>(256, 2 * nchunks);
        uint32_t* q = nullptr;
        cuda_check(cudaMallocHost(reinterpret_cast<void**>(&q), 4 * want), "cudaMallocHost");
        s0.h_side.reset(q);
        s0.side_words = want;
    }
    uint32_t* const h_side = s0.h_side.get();
    std::vector<uint32_t> h_unserved(nchunks, 0);
    std::vector<uint64_t> nb_base(nchunks, 0);  // the chunk's first boundary in the batch
    std::vector<char> copied(nchunks, 0);       // the chunk's first bit word is in h_side

    auto issue = [&](size_t c, ChunkState& ch, Scratch& s) {
        cudaStream_t st = s.stream;
        nb_base[c] = nb_total;
        nb_total += ch.nb;
        if ((nb_total + 31) / 32 > bits_capacity_words || (nb_total && !boundary_bits_out)) { overflow = true; return false; }
        BatchArgs& a = ch.a;
        a.boundaries = s.bounds.ensure(ch.nb + 4);
        a.scores = nullptr;
        if (!scores_optional(p->dm)) a.scores = s.scores.ensure(4 * ch.nb + 4);
        if (want_tags) {
            a.char_states = s.cst.ensure(4 * ch.nc + 4);
            a.type_states = s.tst.ensure(4 * ch.nc + 4);
        }
        // (chunk-local offsets: bound_base / char_base stay 0)
        if (pipeline_trace()) ch.tr.mark(1, st);
        cuda_check(launch_score(p->dm, a, st), "launch(score)");
        CompactArgs k;
        k.n_sent = ch.n;
        k.status = a.status;
        k.n_chars = a.n_chars;
        k.boundaries = a.boundaries;
        k.bound_offsets = a.bound_offsets;
        k.n_bound = ch.nb;
        k.bit_base = uint32_t(nb_base[c] & 31);
        const size_t nwords = size_t((k.bit_base + ch.nb + 31) / 32);
        k.bits = s.bits.ensure(4 * nwords + 16);
        k.status8 = s.st8.ensure(ch.n + 16);
        if (want_tokens) {
            bind_token_counts(s, k, ch.n);
            k.tok_total_host = &s.totals->tokens;
        }
        s.totals->tokens = 0;
        cuda_check(launch_compact(k, st), "launch(compact)");
        if (want_tags) {
            // a word behind the ticket in the workspace's 256-byte ticket slot
            uint32_t* d_unserved = reinterpret_cast<uint32_t*>(s.ws.get() + workspace_layout(ch.n).ticket + 128);
            cuda_check(cudaMemsetAsync(d_unserved, 0, 4, st), "memset");
            TagArgs t = tag_args(p->dt, a);
            t.n_unserved = d_unserved;
            t.tok_base = k.tok_base;
            bind_token_records(*p, s, t, ch.nc);  // a token has at least one character
            if (want_scores) {
                const TagScoreArgs sc = bind_tag_scores(s, ch.nc, score_len);
                cuda_check(launch_tags(p->dt, t, st, &sc), "launch(tags)");
            } else {
                cuda_check(launch_tags(p->dt, t, st), "launch(tags)");
            }
            cuda_check(cudaMemcpyAsync(&h_unserved[c], d_unserved, 4, cudaMemcpyDeviceToHost, st), "D2H(unserved)");
        }
        return true;
    };
    auto copy_out = [&](size_t c, ChunkState& ch, Scratch& s, cudaStream_t so) {
        const uint64_t ntok = want_tokens ? s.totals->tokens : 0;
        const uint64_t nsc = want_scores ? s.totals->tag_scores : 0;
        if (want_tags && tok_total + ntok > token_capacity) overflow = true;
        if (score_total + nsc > score_capacity) overflow = true;
        if (!overflow) {
            const uint32_t bit_base = uint32_t(nb_base[c] & 31);
            const size_t nwords = size_t((bit_base + ch.nb + 31) / 32);
            const uint64_t w0 = nb_base[c] >> 5;
            if (nwords) {
                // the chunk's first word may share its low bits with the previous chunk: it comes back through a pinned
                // word and is merged on the host at the end; the other words go straight to their place
                if (bit_base == 0) boundary_bits_out[w0] = 0;
                cuda_check(cudaMemcpyAsync(&h_side[c], s.bits.get(), 4, cudaMemcpyDeviceToHost, so), "D2H(bits)");
                if (nwords > 1)
                    cuda_check(cudaMemcpyAsync(boundary_bits_out + w0 + 1, s.bits.get() + 1, 4 * (nwords - 1),
                                               cudaMemcpyDeviceToHost, so), "D2H(bits)");
            }
            cuda_check(cudaMemcpyAsync(n_chars_out + ch.s_lo, ch.a.n_chars, 4 * ch.n, cudaMemcpyDeviceToHost, so), "D2H(n_chars)");
            cuda_check(cudaMemcpyAsync(status_out + ch.s_lo, s.st8.get(), ch.n, cudaMemcpyDeviceToHost, so), "D2H(status)");
            if (n_tokens_out) cuda_check(cudaMemcpyAsync(n_tokens_out + ch.s_lo, s.ntok.get(), 4 * ch.n, cudaMemcpyDeviceToHost, so), "D2H(n_tokens)");
            if (want_tags && ntok) {
                cuda_check(cudaMemcpyAsync(token_ids_out + tok_total, s.tok.get(), 4 * ntok, cudaMemcpyDeviceToHost, so), "D2H(tokens)");
                if (nt) cuda_check(cudaMemcpyAsync(token_cands_out + tok_total * nt, s.cand.get(), ntok * nt, cudaMemcpyDeviceToHost, so), "D2H(tokens)");
            }
            if (nsc)
                cuda_check(cudaMemcpyAsync(tag_scores_out + score_total, s.tagsc.get(), 4 * nsc, cudaMemcpyDeviceToHost, so), "D2H(tag scores)");
            copied[c] = ch.nb != 0;
        }
        tok_total += ntok;
        score_total += nsc;
    };
    ring.run(utf8, byte_offsets, true, issue, copy_out);
    for (uint32_t u : h_unserved) unserved_total += u;
    for (size_t c = 0; c < nchunks; ++c)
        if (copied[c]) boundary_bits_out[nb_base[c] >> 5] |= h_side[c];
    if (n_boundaries_out) *n_boundaries_out = nb_total;
    if (n_tokens_total_out) *n_tokens_total_out = tok_total;
    if (n_unserved_out) *n_unserved_out = unserved_total;
    if (n_scores_total_out) *n_scores_total_out = score_total;
    if (overflow) {
        if (score_total > score_capacity) throw Error(kInvalidArgument, "InvalidArgumentError: score_capacity: too small for the batch");
        throw Error(kInvalidArgument, "InvalidArgumentError: bits_capacity_words/token_capacity: too small for the batch");
    }
    return kOk;
    VPT_API_END
}

namespace {

// Pipeline chunks of vpt_token_spans as (first document, documents): the document counts of the ramp schedule over
// chunk_sentences(), each cut again where its text would pass the byte budget (VPT_CHUNK_BYTES, ramping up from 1/8 of
// it over the first chunks), whichever comes first.  A document over the budget is a chunk by itself.
std::vector<std::pair<size_t, size_t>> span_chunks(const uint64_t* byte_offsets, size_t n_docs) {
    const size_t cs = chunk_sentences();
    const uint64_t big = chunk_bytes();
    std::vector<std::pair<size_t, size_t>> out;
    size_t lo = 0;
    for (size_t sz : ramp_schedule(n_docs, cs, cs / 8, cs / 4)) {
        const size_t end = lo + sz;
        while (lo < end) {
            const uint64_t budget = out.size() < 3 ? std::max<uint64_t>(big >> (3 - out.size()), 1) : big;
            // the last document whose end is within the budget (at least one document)
            size_t hi = size_t(std::upper_bound(byte_offsets + lo + 1, byte_offsets + end + 1, byte_offsets[lo] + budget) -
                               byte_offsets) - 1;
            if (hi <= lo) hi = lo + 1;
            out.emplace_back(lo, hi - lo);
            lo = hi;
        }
    }
    return out;
}

// Device buffers of the span stage of vpt_token_spans and vpt_token_spans_dev
struct SpanStage {
    uint8_t* status8 = nullptr;
    uint32_t* n_tokens = nullptr;
    uint64_t* tok_base = nullptr;
    uint32_t* tok_local = nullptr;
    uint64_t* tok_blk = nullptr;
    uint64_t* tok_total_host = nullptr;  // nullable (SpanArgs::tok_total_host)
    uint32_t* token_ends = nullptr;
    // tag prediction (tok_ids == nullptr: none), as TagArgs
    int32_t* tok_ids = nullptr;
    uint8_t* tok_cands = nullptr;
    uint4* tok_desc = nullptr;
    uint32_t* tok_work = nullptr;
    uint64_t max_tokens = 0;
    const TagScoreArgs* scores = nullptr;  // nullable
};

// The kernels of token_stream behind the scoring pass of the documents `a`: SplitLinebreaksFilter, the wsconst post-filters,
// the token counts and their prefix, tags on the final boundaries (tokens looked up by their pre-filtered bytes, as
// vpt_tokenize_lines_tags), token ends.  `tr` (nullable): the trace mark between the token counts and the tags.
void launch_span_stage(const vpt_predictor* p, const BatchArgs& a, uint32_t wsconst_types, bool normalize, const SpanStage& b,
                       cudaStream_t st, TraceEvents* tr) {
    SpanArgs g;
    g.text = a.text;
    g.offsets = a.offsets;
    g.n_sent = a.n_sent;
    g.status = a.status;
    g.n_chars = a.n_chars;
    g.boundaries = a.boundaries;
    g.bound_offsets = a.bound_offsets;
    cuda_check(launch_split_linebreaks(g, st), "launch(split linebreaks)");
    TokArgs t;
    t.text = a.text;
    t.offsets = a.offsets;
    t.n_sent = a.n_sent;
    t.status = a.status;
    t.n_chars = a.n_chars;
    t.boundaries = a.boundaries;
    t.bound_offsets = a.bound_offsets;
    cuda_check(launch_wsconst(t, a.boundaries, wsconst_types, normalize, st), "launch(wsconst)");
    if (wsconst_types & 0x80u) cuda_check(launch_grapheme(t, a.boundaries, normalize, st), "launch(grapheme)");
    g.status8 = b.status8;
    g.n_tokens = b.n_tokens;
    g.tok_base = b.tok_base;
    g.tok_local = b.tok_local;
    g.tok_blk = b.tok_blk;
    g.tok_total_host = b.tok_total_host;
    cuda_check(launch_span_count(g, st), "launch(span count)");
    if (tr) tr->mark_sub(1, st);  // after the filters and the token counts
    if (b.tok_ids) {
        TagArgs ta = tag_args(p->dt, a);
        ta.tok_base = g.tok_base;
        ta.tok_ids = b.tok_ids;
        ta.tok_cands = b.tok_cands;
        ta.tok_desc = b.tok_desc;
        ta.max_tokens = b.max_tokens;
        ta.tok_work = b.tok_work;
        ta.norm = normalize ? 1 : 0;
        cuda_check(launch_tags(p->dt, ta, st, b.scores), "launch(tags)");
    }
    g.token_ends = b.token_ends;
    cuda_check(launch_token_ends(g, st), "launch(token ends)");
}

}  // namespace

int vpt_token_spans(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_docs, int no_norm,
                    uint32_t wsconst_types, uint32_t* n_tokens_out, uint8_t* status_out, uint32_t* token_ends_out,
                    int32_t* token_ids_out, uint8_t* token_cands_out, size_t token_capacity, uint64_t* n_tokens_total_out) {
    return vpt_token_spans_tag_scores(p, utf8, byte_offsets, n_docs, no_norm, wsconst_types, n_tokens_out, status_out,
                                      token_ends_out, token_ids_out, token_cands_out, token_capacity, n_tokens_total_out,
                                      nullptr, 0, nullptr);
}

int vpt_token_spans_tag_scores(const vpt_predictor* p, const uint8_t* utf8, const uint64_t* byte_offsets, size_t n_docs,
                               int no_norm, uint32_t wsconst_types, uint32_t* n_tokens_out, uint8_t* status_out,
                               uint32_t* token_ends_out, int32_t* token_ids_out, uint8_t* token_cands_out,
                               size_t token_capacity, uint64_t* n_tokens_total_out, int32_t* tag_scores_out,
                               size_t score_capacity, uint64_t* n_scores_total_out) {
    VPT_API_BEGIN
    if (n_tokens_total_out) *n_tokens_total_out = 0;
    if (n_scores_total_out) *n_scores_total_out = 0;
    const bool want_tags = token_ids_out != nullptr || token_cands_out != nullptr;
    if (tag_scores_out && !want_tags)
        throw Error(kInvalidArgument, "InvalidArgumentError: tag_scores_out: needs token_ids_out (tag prediction)");
    const bool tags = check_lines_flags(p, wsconst_types, want_tags);  // false with n_tags == 0: every token id is -1
    const size_t nt = tags ? p->n_tags : 0;
    const bool want_scores = tags && tag_scores_out != nullptr;  // (a model without tag slots has no scores)
    const size_t score_len = want_scores ? device_score_len_bound(p) : 0;
    if (want_tags && (!token_ids_out || (nt && !token_cands_out)))
        throw Error(kInvalidArgument, "InvalidArgumentError: token_ids_out/token_cands_out: must not be NULL");
    if (!byte_offsets || !n_tokens_out || !status_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets/n_tokens_out/status_out: must not be NULL");
    if (n_docs == 0) return kOk;
    for (size_t d = 0; d < n_docs; ++d) {
        if (byte_offsets[d + 1] < byte_offsets[d])
            throw Error(kInvalidArgument, "InvalidArgumentError: byte_offsets: must be non-decreasing");
        if (byte_offsets[d + 1] - byte_offsets[d] > kMaxLineChunk)
            throw Error(kInvalidArgument, "InvalidArgumentError: utf8: a document is longer than 1 GiB");
    }
    if (byte_offsets[n_docs] > byte_offsets[0] && !utf8) throw Error(kInvalidArgument, "InvalidArgumentError: utf8: must not be NULL");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    const bool normalize = no_norm == 0;
    DevModel dm = p->dm;
    dm.kytea_norm = normalize ? 1 : 0;

    // Every chunk goes through the batch ring: copy-in + count pass, then scoring, line breaks, post-filters, token
    // counts + prefix, (tags) and token ends (the chunk's tokens to pinned host memory), then, one chunk behind, the
    // copy-out (per-document words, token ends and tag records at the running token total).
    BatchRing ring(*p, "spans", "sync(spans)", byte_offsets, span_chunks(byte_offsets, n_docs));
    uint64_t tok_total = 0, score_total = 0;
    bool overflow = false;

    auto issue = [&](size_t, ChunkState& ch, Scratch& s) {
        cudaStream_t st = s.stream;
        const uint64_t nb = ch.nb, nc = ch.nc;
        BatchArgs& a = ch.a;
        a.boundaries = s.bounds.ensure(nb + 4);
        a.scores = nullptr;
        if (!scores_optional(dm)) a.scores = s.scores.ensure(4 * nb + 4);
        if (tags) {
            a.char_states = s.cst.ensure(4 * nc + 4);
            a.type_states = s.tst.ensure(4 * nc + 4);
        }
        SpanStage b;
        b.status8 = s.st8.ensure(ch.n + 16);
        b.token_ends = s.ends.ensure(4 * nc + 16);  // a token has at least one character
        bind_token_counts(s, b, ch.n);
        b.tok_total_host = &s.totals->tokens;
        s.totals->tokens = 0;
        TagScoreArgs sc;
        if (tags) {
            bind_token_records(*p, s, b, nc);
            if (want_scores) {
                sc = bind_tag_scores(s, nc, score_len);
                b.scores = &sc;
            }
        }
        // (chunk-local offsets: bound_base / char_base stay 0)
        if (pipeline_trace()) ch.tr.mark(1, st);
        cuda_check(launch_score(dm, a, st), "launch(score)");
        if (pipeline_trace()) ch.tr.mark_sub(0, st);  // after the scoring kernel
        launch_span_stage(p, a, wsconst_types, normalize, b, st, pipeline_trace() ? &ch.tr : nullptr);
        return true;
    };
    auto copy_out = [&](size_t, ChunkState& ch, Scratch& s, cudaStream_t so) {
        const uint64_t ntok = s.totals->tokens;
        const uint64_t nsc = want_scores ? s.totals->tag_scores : 0;
        if (tok_total + ntok > token_capacity || (ntok && !token_ends_out)) overflow = true;
        if (score_total + nsc > score_capacity) overflow = true;
        if (!overflow) {
            cuda_check(cudaMemcpyAsync(n_tokens_out + ch.s_lo, s.ntok.get(), 4 * ch.n, cudaMemcpyDeviceToHost, so), "D2H(n_tokens)");
            cuda_check(cudaMemcpyAsync(status_out + ch.s_lo, s.st8.get(), ch.n, cudaMemcpyDeviceToHost, so), "D2H(status)");
            if (ntok) {
                cuda_check(cudaMemcpyAsync(token_ends_out + tok_total, s.ends.get(), 4 * ntok, cudaMemcpyDeviceToHost, so), "D2H(ends)");
                if (tags) {
                    cuda_check(cudaMemcpyAsync(token_ids_out + tok_total, s.tok.get(), 4 * ntok, cudaMemcpyDeviceToHost, so), "D2H(tokens)");
                    if (nt) cuda_check(cudaMemcpyAsync(token_cands_out + tok_total * nt, s.cand.get(), ntok * nt, cudaMemcpyDeviceToHost, so), "D2H(tokens)");
                }
            }
            if (nsc)
                cuda_check(cudaMemcpyAsync(tag_scores_out + score_total, s.tagsc.get(), 4 * nsc, cudaMemcpyDeviceToHost, so), "D2H(tag scores)");
        }
        tok_total += ntok;
        score_total += nsc;
    };
    ring.run(utf8, byte_offsets, true, issue, copy_out);
    if (n_tokens_total_out) *n_tokens_total_out = tok_total;
    if (n_scores_total_out) *n_scores_total_out = score_total;
    if (overflow) {
        if (score_total > score_capacity) throw Error(kInvalidArgument, "InvalidArgumentError: score_capacity: too small for the batch");
        throw Error(kInvalidArgument, "InvalidArgumentError: token_capacity: too small for the batch");
    }
    if (want_tags && !tags) std::fill(token_ids_out, token_ids_out + tok_total, -1);  // a model without tag slots
    return kOk;
    VPT_API_END
}

namespace {

// Batch limit of vpt_token_spans_dev, for n_bytes and n_docs: the tag kernels index characters and token records of the
// whole batch with 32 bits (TagArgs::tok_desc .z, TagArgs::tok_work), and tokens <= characters <= bytes (+ 15 of shift)
constexpr uint64_t kMaxSpansDevBatch = (uint64_t(1) << 32) - 16;

// Scratch of vpt_token_spans_dev in the caller's workspace: byte offsets of every buffer; 0 size = not used
struct SpansDevLayout {
    size_t off, bad, dblk, ws, status, boff, coff, bounds, scores, cst, tst, tokdesc, tokwork, toklocal, tokblk, total;
};
SpansDevLayout spans_dev_layout(const vpt_predictor* p, uint64_t n_docs, uint64_t n_bytes, bool tags) {
    SpansDevLayout l;
    const uint64_t n = n_docs, b = n_bytes;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes, 256); return at; };
    l.off = take(8 * (n + 1));
    l.bad = take(n);
    l.dblk = take(8 * doc_offsets_blocks(n));
    l.ws = take(workspace_layout(n).total);
    l.status = take(4 * n);
    l.boff = take(8 * (n + 1));
    l.coff = tags ? take(8 * (n + 1)) : 0;
    l.bounds = take(b + 4);  // (the span kernels read boundaries as words)
    l.scores = scores_optional(p->dm) ? 0 : take(4 * b + 4);
    l.cst = tags ? take(4 * b + 4) : 0;
    l.tst = tags ? take(4 * b + 4) : 0;
    l.tokdesc = tags ? take(16 * b + 16) : 0;
    l.tokwork = tags ? take(4 * b + 32) : 0;
    l.toklocal = take(4 * n);
    l.tokblk = take(8 * (n / kSpanDocs + 4));
    l.total = o + 256;
    return l;
}

// `ptr` is device memory of the predictor's device (cudaPointerGetAttributes: no stream work, allowed under capture)
void require_device_ptr(const vpt_predictor* p, const void* ptr, const char* name) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess) {
        cudaGetLastError();
        throw Error(kInvalidArgument, std::string("InvalidArgumentError: ") + name + ": not device memory");
    }
    if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != p->device)
        throw Error(kInvalidArgument, std::string("InvalidArgumentError: ") + name +
                                          ": must be device memory of the predictor's device " + std::to_string(p->device));
}

}  // namespace

uint64_t vpt_token_spans_dev_workspace_size(const vpt_predictor* p, size_t n_docs, uint64_t n_bytes, int tags) {
    if (!p || p->device < 0) return 0;
    return spans_dev_layout(p, n_docs, n_bytes, tags != 0 && p->n_tags > 0).total;
}

int vpt_token_spans_dev(const vpt_predictor* p, const uint8_t* d_utf8, uint64_t n_bytes, const void* d_offsets,
                        int offset_bytes, size_t n_docs, int no_norm, uint32_t wsconst_types, uint64_t* d_token_offsets,
                        uint32_t* d_n_tokens, uint8_t* d_status, uint32_t* d_token_ends, int32_t* d_token_ids,
                        uint8_t* d_token_cands, void* d_workspace, uint64_t workspace_bytes, void* cuda_stream) {
    VPT_API_BEGIN
    // Every check reads the arguments only: nothing here synchronises, allocates or touches the device's data
    const bool want_tags = d_token_ids != nullptr || d_token_cands != nullptr;
    const bool tags = check_lines_flags(p, wsconst_types, want_tags);  // false with n_tags == 0: every token id is -1
    if (want_tags && (!d_token_ids || (tags && !d_token_cands)))
        throw Error(kInvalidArgument, "InvalidArgumentError: d_token_ids/d_token_cands: must not be NULL");
    if (offset_bytes != 4 && offset_bytes != 8)
        throw Error(kInvalidArgument, "InvalidArgumentError: offset_bytes: must be 4 (int32) or 8 (int64)");
    if (!d_offsets || !d_token_offsets || (n_docs > 0 && (!d_n_tokens || !d_status || !d_token_ends)))
        throw Error(kInvalidArgument, "InvalidArgumentError: device buffers: must not be NULL");
    if (n_bytes > 0 && !d_utf8) throw Error(kInvalidArgument, "InvalidArgumentError: d_utf8: must not be NULL");
    if (n_bytes > kMaxSpansDevBatch || n_docs > kMaxSpansDevBatch)
        throw Error(kInvalidArgument, "InvalidArgumentError: n_bytes/n_docs: over the batch limit of 2^32 - 16 (32-bit "
                                      "character and token indexes of the tag kernels)");
    const SpansDevLayout l = spans_dev_layout(p, n_docs, n_bytes, tags);
    if (n_docs > 0 && (!d_workspace || workspace_bytes < l.total))
        throw Error(kInvalidArgument, "InvalidArgumentError: workspace: too small (vpt_token_spans_dev_workspace_size)");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    if (n_bytes > 0) require_device_ptr(p, d_utf8, "d_utf8");
    require_device_ptr(p, d_offsets, "d_offsets");
    require_device_ptr(p, d_token_offsets, "d_token_offsets");
    if (n_docs > 0) {
        require_device_ptr(p, d_n_tokens, "d_n_tokens");
        require_device_ptr(p, d_status, "d_status");
        require_device_ptr(p, d_token_ends, "d_token_ends");
        require_device_ptr(p, d_workspace, "d_workspace");
    }
    if (d_token_ids) require_device_ptr(p, d_token_ids, "d_token_ids");
    if (tags) require_device_ptr(p, d_token_cands, "d_token_cands");
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (want_tags && !tags && n_bytes)  // a model without tag slots
        cuda_check(cudaMemsetAsync(d_token_ids, 0xFF, 4 * n_bytes, st), "memset(token ids)");
    if (n_docs == 0) {
        cuda_check(cudaMemsetAsync(d_token_offsets, 0, 8, st), "memset(token offsets)");
        return kOk;
    }
    uint8_t* w = static_cast<uint8_t*>(d_workspace);
    const bool normalize = no_norm == 0;
    DevModel dm = p->dm;
    dm.kytea_norm = normalize ? 1 : 0;

    // the caller's offsets -> offsets into the text rounded down to 16 bytes, and the documents out of range
    const uintptr_t text_addr = reinterpret_cast<uintptr_t>(d_utf8);
    DocArgs da;
    da.offsets = d_offsets;
    da.wide = offset_bytes == 8;
    da.n_docs = n_docs;
    da.n_bytes = n_bytes;
    da.shift = uint32_t(text_addr & 15);
    da.out = reinterpret_cast<uint64_t*>(w + l.off);
    da.bad = w + l.bad;
    da.blk = reinterpret_cast<uint64_t*>(w + l.dblk);
    cuda_check(launch_doc_offsets(da, st), "launch(doc offsets)");

    BatchArgs a;
    a.text = reinterpret_cast<const uint8_t*>(text_addr & ~uintptr_t(15));
    a.offsets = da.out;
    a.n_sent = n_docs;
    bind_workspace(a, w + l.ws, n_docs);
    a.status = reinterpret_cast<int32_t*>(w + l.status);
    a.bound_offsets = reinterpret_cast<uint64_t*>(w + l.boff);
    a.boundaries = w + l.bounds;
    a.scores = l.scores ? reinterpret_cast<int32_t*>(w + l.scores) : nullptr;
    SpanStage b;
    b.status8 = d_status;
    b.n_tokens = d_n_tokens;
    b.tok_base = d_token_offsets;
    b.tok_local = reinterpret_cast<uint32_t*>(w + l.toklocal);
    b.tok_blk = reinterpret_cast<uint64_t*>(w + l.tokblk);
    b.token_ends = d_token_ends;
    if (tags) {
        a.char_offsets = reinterpret_cast<uint64_t*>(w + l.coff);
        a.char_states = reinterpret_cast<uint32_t*>(w + l.cst);
        a.type_states = reinterpret_cast<uint32_t*>(w + l.tst);
        b.tok_ids = d_token_ids;
        b.tok_cands = d_token_cands;
        b.tok_desc = reinterpret_cast<uint4*>(w + l.tokdesc);
        b.tok_work = reinterpret_cast<uint32_t*>(w + l.tokwork);
        b.max_tokens = n_bytes;
    }
    cuda_check(launch_batch(dm, a, st), "launch(batch)");
    cuda_check(launch_doc_status(da, a.status, st), "launch(doc status)");
    launch_span_stage(p, a, wsconst_types, normalize, b, st, nullptr);
    return kOk;
    VPT_API_END
}

namespace {

// Scratch of vpt_tokenize_dev in the caller's workspace: byte offsets of every buffer; 0 size = not used
struct TokDevLayout {
    size_t off, bad, dblk, ws, status, boff, coff, bounds, scores, cst, tst, st8, ntok, tokbase, toklocal, tokblk, tokids,
        tokcands, tokdesc, tokwork, trule, tokg, total;
};
TokDevLayout tokenize_dev_layout(const vpt_predictor* p, uint64_t n_docs, uint64_t n_bytes, bool tags, bool rules) {
    TokDevLayout l = {};
    const uint64_t n = n_docs, b = n_bytes;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes, 256); return at; };
    l.off = take(8 * (n + 1));
    l.bad = take(n);
    l.dblk = take(8 * doc_offsets_blocks(n));
    l.ws = take(workspace_layout(n).total);
    l.status = take(4 * n);
    l.boff = take(8 * (n + 1));
    l.bounds = take(b + 4);  // (the writers read boundaries as words)
    l.scores = scores_optional(p->dm) ? 0 : take(4 * b + 4);
    if (tags) {
        l.coff = take(8 * (n + 1));
        l.cst = take(4 * b + 4);
        l.tst = take(4 * b + 4);
        // token counts and records: tokens <= characters <= bytes
        l.st8 = take(n + 16);
        l.ntok = take(4 * n + 16);
        l.tokbase = take(8 * (n + 1) + 16);
        l.toklocal = take(4 * n + 16);
        l.tokblk = take(8 * (n / kSpanDocs + 4));
        l.tokids = take(4 * b + 16);
        l.tokcands = take(b * std::max<size_t>(p->n_tags, 1) + 16);
        l.tokdesc = take(16 * b + 16);
        l.tokwork = take(4 * b + 32);
        l.trule = rules ? take(4 * b + 16) : 0;
    }
    l.tokg = take(8 * ((n + kGroup - 1) / kGroup + 2));  // the writer's look-back state words, then its ticket
    l.total = o + 256;
    return l;
}

// Whether vpt_tokenize_dev predicts tags / applies rules for these flags (the checks themselves are the call's)
bool tokenize_dev_tags(const vpt_predictor* p, int predict_tags) { return predict_tags != 0 && p->n_tags > 0; }
bool tokenize_dev_rules(const vpt_predictor* p, const vpt_tag_rules* rules, int predict_tags) {
    return rules && rules->n_rules && tokenize_dev_tags(p, predict_tags);
}

}  // namespace

uint64_t vpt_tokenize_dev_workspace_size(const vpt_predictor* p, const vpt_tag_rules* rules, size_t n_docs, uint64_t n_bytes,
                                         int predict_tags) {
    if (!p || p->device < 0) return 0;
    return tokenize_dev_layout(p, n_docs, n_bytes, tokenize_dev_tags(p, predict_tags),
                               tokenize_dev_rules(p, rules, predict_tags)).total;
}

uint64_t vpt_tokenize_dev_out_bound(const vpt_predictor* p, const vpt_tag_rules* rules, size_t /*n_docs*/, uint64_t n_bytes,
                                    int predict_tags) {
    if (!p) return 0;
    // surface bytes + at most one '\\' per byte + at most one ' ' per character; with tags every token (at most one per
    // byte) may get the longest "/tag.." suffix of the model and of the rules
    uint64_t bound = 3 * n_bytes;
    if (tokenize_dev_tags(p, predict_tags))
        bound += n_bytes * (uint64_t(p->dt.max_suffix) +
                            (tokenize_dev_rules(p, rules, predict_tags) ? uint64_t(rules->max_suffix) : 0));
    return bound;
}

int vpt_tokenize_dev(const vpt_predictor* p, const vpt_tag_rules* rules, const uint8_t* d_utf8, uint64_t n_bytes,
                     const void* d_offsets, int offset_bytes, size_t n_docs, int no_norm, uint32_t wsconst_types,
                     int predict_tags, int64_t* d_out_offsets, uint8_t* d_out, uint64_t out_capacity, uint8_t* d_status,
                     void* d_workspace, uint64_t workspace_bytes, void* cuda_stream) {
    VPT_API_BEGIN
    // Every check reads the arguments only: nothing here synchronises, allocates or touches the device's data
    const bool tags = check_lines_flags(p, wsconst_types, predict_tags != 0);
    if (rules && !predict_tags)
        throw Error(kInvalidArgument, "InvalidArgumentError: rules: need predict_tags (PatternMatchTagger fills predicted tags)");
    if (rules && rules->p != p) throw Error(kInvalidArgument, "InvalidArgumentError: rules: made for another predictor");
    const bool with_rules = tags && rules && rules->n_rules;
    if (offset_bytes != 4 && offset_bytes != 8)
        throw Error(kInvalidArgument, "InvalidArgumentError: offset_bytes: must be 4 (int32) or 8 (int64)");
    if (!d_offsets || !d_out_offsets || (n_docs > 0 && !d_status))
        throw Error(kInvalidArgument, "InvalidArgumentError: device buffers: must not be NULL");
    if (n_bytes > 0 && !d_utf8) throw Error(kInvalidArgument, "InvalidArgumentError: d_utf8: must not be NULL");
    if (out_capacity > 0 && !d_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: d_out: must not be NULL when out_capacity > 0");
    if (n_bytes > kMaxSpansDevBatch || n_docs > kMaxSpansDevBatch)
        throw Error(kInvalidArgument, "InvalidArgumentError: n_bytes/n_docs: over the batch limit of 2^32 - 16 (32-bit "
                                      "character and token indexes of the tag kernels)");
    const TokDevLayout l = tokenize_dev_layout(p, n_docs, n_bytes, tags, with_rules);
    if (n_docs > 0 && (!d_workspace || workspace_bytes < l.total))
        throw Error(kInvalidArgument, "InvalidArgumentError: workspace: too small (vpt_tokenize_dev_workspace_size)");
    cuda_check(cudaSetDevice(p->device), "cudaSetDevice");
    if (n_bytes > 0) require_device_ptr(p, d_utf8, "d_utf8");
    require_device_ptr(p, d_offsets, "d_offsets");
    require_device_ptr(p, d_out_offsets, "d_out_offsets");
    if (out_capacity > 0) require_device_ptr(p, d_out, "d_out");
    if (n_docs > 0) {
        require_device_ptr(p, d_status, "d_status");
        require_device_ptr(p, d_workspace, "d_workspace");
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    uint64_t* out_off = reinterpret_cast<uint64_t*>(d_out_offsets);
    if (n_docs == 0) {
        cuda_check(cudaMemsetAsync(out_off, 0, 8, st), "memset(out offsets)");
        return kOk;
    }
    uint8_t* w = static_cast<uint8_t*>(d_workspace);
    const bool normalize = no_norm == 0;
    DevModel dm = p->dm;
    dm.kytea_norm = normalize ? 1 : 0;

    // the caller's offsets -> offsets into the text rounded down to 16 bytes, and the documents out of range
    const uintptr_t text_addr = reinterpret_cast<uintptr_t>(d_utf8);
    DocArgs da;
    da.offsets = d_offsets;
    da.wide = offset_bytes == 8;
    da.n_docs = n_docs;
    da.n_bytes = n_bytes;
    da.shift = uint32_t(text_addr & 15);
    da.out = reinterpret_cast<uint64_t*>(w + l.off);
    da.bad = w + l.bad;
    da.blk = reinterpret_cast<uint64_t*>(w + l.dblk);
    cuda_check(launch_doc_offsets(da, st), "launch(doc offsets)");

    BatchArgs a;
    a.text = reinterpret_cast<const uint8_t*>(text_addr & ~uintptr_t(15));
    a.offsets = da.out;
    a.n_sent = n_docs;
    bind_workspace(a, w + l.ws, n_docs);
    a.status = reinterpret_cast<int32_t*>(w + l.status);
    a.bound_offsets = reinterpret_cast<uint64_t*>(w + l.boff);
    a.boundaries = w + l.bounds;
    a.scores = l.scores ? reinterpret_cast<int32_t*>(w + l.scores) : nullptr;
    if (tags) {
        a.char_offsets = reinterpret_cast<uint64_t*>(w + l.coff);
        a.char_states = reinterpret_cast<uint32_t*>(w + l.cst);
        a.type_states = reinterpret_cast<uint32_t*>(w + l.tst);
    }
    cuda_check(launch_batch(dm, a, st), "launch(batch)");
    cuda_check(launch_doc_status(da, a.status, st), "launch(doc status)");

    TokArgs t;
    t.text = a.text;
    t.offsets = a.offsets;
    t.n_sent = n_docs;
    t.status = a.status;
    t.n_chars = a.n_chars;
    t.boundaries = a.boundaries;
    t.bound_offsets = a.bound_offsets;
    cuda_check(launch_wsconst(t, a.boundaries, wsconst_types, normalize, st), "launch(wsconst)");
    if (wsconst_types & 0x80u) cuda_check(launch_grapheme(t, a.boundaries, normalize, st), "launch(grapheme)");
    TagRuleArgs ra;
    if (tags) {
        TagRecords r;
        r.status8 = w + l.st8;
        r.n_tokens = reinterpret_cast<uint32_t*>(w + l.ntok);
        r.tok_base = reinterpret_cast<uint64_t*>(w + l.tokbase);
        r.tok_local = reinterpret_cast<uint32_t*>(w + l.toklocal);
        r.tok_blk = reinterpret_cast<uint64_t*>(w + l.tokblk);
        r.tok_ids = reinterpret_cast<int32_t*>(w + l.tokids);
        r.tok_cands = w + l.tokcands;
        r.tok_desc = reinterpret_cast<uint4*>(w + l.tokdesc);
        r.tok_work = reinterpret_cast<uint32_t*>(w + l.tokwork);
        r.max_tokens = n_bytes;
        if (with_rules) {
            r.rules = rules;
            r.rule_words = reinterpret_cast<unsigned long long*>(w + l.trule);
        }
        launch_tag_records(*p, a, normalize, r, t, &ra, st);
    }
    // the column writer; its look-back state and ticket are zeroed by the launch
    t.tok_state = reinterpret_cast<uint64_t*>(w + l.tokg);
    t.ticket = reinterpret_cast<uint32_t*>(t.tok_state + (n_docs + kGroup - 1) / kGroup);
    t.total = out_off + n_docs;
    t.total_host = nullptr;
    t.out = d_out;
    ColOut col;
    col.offsets = out_off;
    col.capacity = out_capacity;
    col.status = d_status;
    cuda_check(launch_tokenize_column(t, ra, col, st), "launch(tok column)");
    return kOk;
    VPT_API_END
}

int vpt_unpack_boundaries(const uint32_t* boundary_bits, uint64_t first_bit, uint64_t n, uint8_t* boundaries_out) {
    VPT_API_BEGIN
    if (n && (!boundary_bits || !boundaries_out)) throw Error(kInvalidArgument, "InvalidArgumentError: buffers: must not be NULL");
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t b = first_bit + i;
        boundaries_out[i] = uint8_t((boundary_bits[b >> 5] >> (b & 31)) & 1u);
    }
    return kOk;
    VPT_API_END
}

int vpt_fill_tags(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, const uint8_t* boundaries,
                  const uint32_t* char_states, const uint32_t* type_states, int32_t* tag_token_out,
                  int32_t* tag_cand_out, int32_t* tag_scores_out, size_t score_stride) {
    VPT_API_BEGIN
    if (!p) throw Error(kInvalidArgument, "InvalidArgumentError: predictor: must not be NULL");
    if (!p->predict_tags || p->from_blob)
        throw Error(kInvalidArgument, "InvalidArgumentError: this predictor is created with predict_tags = false");
    if (!utf8 || !boundaries || !tag_token_out || !tag_cand_out)
        throw Error(kInvalidArgument, "InvalidArgumentError: utf8/boundaries/tag_token_out/tag_cand_out: must not be NULL");
    check_raw_text(utf8, n_bytes);
    const std::vector<uint32_t> pos = char_starts(utf8, n_bytes);
    const size_t n = pos.size() - 1;
    const size_t nt = p->n_tags;
    for (size_t i = 0; i < n; ++i) tag_token_out[i] = -1;
    for (size_t i = 0; i < n * nt; ++i) tag_cand_out[i] = -1;
    if (nt == 0) return kOk;  // predictor.rs:553-555
    if ((p->char_tags && !char_states) || (p->type_tags && !type_states))
        throw Error(kInvalidArgument, "InvalidArgumentError: states: required for tag prediction");
    std::vector<int32_t> scores;
    auto run = [&](size_t start, size_t last) {  // token = chars [start, last]
        std::string tok(reinterpret_cast<const char*>(utf8) + pos[start], pos[last + 1] - pos[start]);
        auto it = p->token_ids.find(tok);
        if (it == p->token_ids.end()) return;
        const uint32_t tid = it->second;
        const TagPredictorHost& tp = p->tag_preds[tid];
        scores.assign(tp.bias.size(), 0);
        add_truncated(tp.bias, scores);
        if (p->char_tags) add_tag_scores(p->char_tag_weight, p->char_suffix_link, tid, last, char_states, n, scores);
        if (p->type_tags) add_tag_scores(p->type_tag_weight, p->type_suffix_link, tid, last, type_states, n, scores);
        // TagPredictor::predict (predictor.rs:286-304): first strict maximum per slot with >= 2 candidates
        size_t off = 0;
        for (size_t k = 0; k < tp.tags.size() && k < nt; ++k) {
            const size_t ncand = tp.tags[k].size();
            if (ncand >= 2) {
                if (off + ncand > scores.size())
                    throw Error(kInvalidModel, "InvalidModelError: tag bias is shorter than the number of candidates");
                size_t best = 0;
                int32_t mx = INT32_MIN;
                for (size_t c = 0; c < ncand; ++c)
                    if (scores[off + c] > mx) { best = c; mx = scores[off + c]; }
                tag_cand_out[last * nt + k] = int32_t(best);
                off += ncand;
            } else {
                tag_cand_out[last * nt + k] = ncand == 1 ? 0 : -1;
            }
        }
        tag_token_out[last] = int32_t(tid);
        if (tag_scores_out) {
            const size_t m = std::min(score_stride, scores.size());
            memcpy(tag_scores_out + last * score_stride, scores.data(), m * 4);
        }
    };
    bool have = true;
    size_t start = 0;
    for (size_t i = 0; i + 1 < n; ++i) {
        const uint8_t b = boundaries[i];
        if (b == 2) have = false;
        else if (b == 1) {
            if (have) run(start, i);
            have = true;
            start = i + 1;
        }
    }
    if (have) run(start, n - 1);
    return kOk;
    VPT_API_END
}

int vpt_write_tokenized_text(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, const uint8_t* boundaries,
                             const int32_t* tag_token, const int32_t* tag_cand, char* buf, size_t capacity,
                             uint64_t* len_out) {
    VPT_API_BEGIN
    if (!utf8 || !boundaries) throw Error(kInvalidArgument, "InvalidArgumentError: utf8/boundaries: must not be NULL");
    check_raw_text(utf8, n_bytes);
    const std::vector<uint32_t> pos = char_starts(utf8, n_bytes);
    const size_t n = pos.size() - 1;
    const size_t nt = (p && tag_token && tag_cand) ? p->n_tags : 0;
    std::string out;
    auto put = [&](const char* s, size_t l) {
        for (size_t i = 0; i < l; ++i) {
            if (s[i] == ' ' || s[i] == '\\' || s[i] == '/') out.push_back('\\');
            out.push_back(s[i]);
        }
    };
    auto emit = [&](size_t st, size_t en) {  // chars [st, en)
        if (!out.empty()) out.push_back(' ');
        put(reinterpret_cast<const char*>(utf8) + pos[st], pos[en] - pos[st]);
        if (nt) {
            const size_t i = en - 1;
            int last = -1;
            for (size_t k = 0; k < nt; ++k) if (tag_cand[i * nt + k] >= 0) last = int(k);
            for (int k = 0; k <= last; ++k) {
                out.push_back('/');
                const int32_t c = tag_cand[i * nt + size_t(k)];
                if (c >= 0) {
                    const char* t = vpt_tag_string(p, uint32_t(tag_token[i]), uint32_t(k), uint32_t(c));
                    if (t) put(t, strlen(t));
                }
            }
        }
    };
    // TokenIterator (sentence.rs:1273-1299): tokens adjacent to Unknown boundaries are skipped
    size_t start = 0;
    bool skip = false;
    for (size_t i = 0; i + 1 < n; ++i) {
        const uint8_t b = boundaries[i];
        if (b == 1) {
            if (!skip) emit(start, i + 1);
            skip = false;
            start = i + 1;
        } else if (b == 2) skip = true;
    }
    if (!skip) emit(start, n);
    if (len_out) *len_out = out.size();
    if (buf && capacity) {
        const size_t m = std::min(capacity - 1, out.size());
        memcpy(buf, out.data(), m);
        buf[m] = 0;
    }
    return kOk;
    VPT_API_END
}

int vpt_write_partial_annotation_text(const vpt_predictor* p, const uint8_t* utf8, size_t n_bytes, const uint8_t* boundaries,
                                      const int32_t* tag_token, const int32_t* tag_cand, char* buf, size_t capacity,
                                      uint64_t* len_out) {
    VPT_API_BEGIN
    if (!utf8 || !boundaries) throw Error(kInvalidArgument, "InvalidArgumentError: utf8/boundaries: must not be NULL");
    check_raw_text(utf8, n_bytes);
    const std::vector<uint32_t> pos = char_starts(utf8, n_bytes);
    const size_t n = pos.size() - 1;
    const size_t nt = (p && tag_token && tag_cand) ? p->n_tags : 0;
    std::string out;
    for (size_t i = 0; i < n; ++i) {
        if (i > 0) {
            const uint8_t b = boundaries[i - 1];
            out.push_back(b == 0 ? '-' : b == 1 ? '|' : ' ');
        }
        out.append(reinterpret_cast<const char*>(utf8) + pos[i], pos[i + 1] - pos[i]);
        // the tags of character i, unescaped, up to the last slot that has one (sentence.rs:907-944)
        int last = -1;
        for (size_t k = 0; k < nt; ++k) if (tag_cand[i * nt + k] >= 0) last = int(k);
        for (int k = 0; k <= last; ++k) {
            out.push_back('/');
            const int32_t c = tag_cand[i * nt + size_t(k)];
            if (c >= 0) {
                const char* t = vpt_tag_string(p, uint32_t(tag_token[i]), uint32_t(k), uint32_t(c));
                if (t) out.append(t);
            }
        }
    }
    if (len_out) *len_out = out.size();
    if (buf && capacity) {
        const size_t m = std::min(capacity - 1, out.size());
        memcpy(buf, out.data(), m);
        buf[m] = 0;
    }
    return kOk;
    VPT_API_END
}

}  // extern "C"
