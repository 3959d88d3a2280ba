// Tag prediction of one token from the flat tag tables (tags.hpp): the per-thread code of the tag kernels (tags.cu: k_tags,
// k_tok_lookup, k_tok_score).  It has no warp operations, so it also compiles for the host: tests/native/host_emul.cpp runs
// THIS code over the tables tags_build.cpp makes and compares with the oracle's predict_tags (tests/test_host_tables.py).
#pragma once
#include <cstdint>

#include "keys.hpp"
#include "tags.hpp"
#include "textnorm.hpp"

#if defined(__CUDA_ARCH__)
#define VPT_LDG(p) __ldg(p)
#define VPT_COUNT(p) atomicAdd((p), 1u)
#else
#define VPT_LDG(p) (*(p))
#define VPT_COUNT(p) (++*(p))
#endif

#if !defined(__CUDACC__)
#include <algorithm>
#include <climits>
#endif

namespace vpt {

#if !defined(__CUDACC__)
using std::min;  // (a built-in of the CUDA compiler)
#endif

// Calls f(byte) for every byte of the token -- of its KyteaFullwidthFilter image when norm != 0 (one character maps to
// one character, the byte length may change) -- and returns how many bytes that were.
template <typename F>
VPT_HD uint32_t token_bytes(const uint8_t* __restrict__ bytes, uint32_t len, int norm, F f) {
    if (!norm) {
        for (uint32_t i = 0; i < len; ++i) f(uint32_t(VPT_LDG(bytes + i)));
        return len;
    }
    uint32_t out = 0;
    for (uint32_t i = 0; i < len;) {
        const uint32_t b0 = VPT_LDG(bytes + i);
        const uint32_t l = b0 < 0x80u ? 1u : b0 < 0xE0u ? 2u : b0 < 0xF0u ? 3u : 4u;
        uint32_t c = l == 1 ? b0 : b0 & (0x3Fu >> (l - 1));
        for (uint32_t k = 1; k < l && i + k < len; ++k) c = (c << 6) | (VPT_LDG(bytes + i + k) & 0x3Fu);
        i += l;
        c = kytea_fullwidth(c);
        if (c < 0x80u) { f(c); out += 1; }
        else if (c < 0x800u) { f(0xC0u | (c >> 6)); f(0x80u | (c & 0x3Fu)); out += 2; }
        else if (c < 0x10000u) { f(0xE0u | (c >> 12)); f(0x80u | ((c >> 6) & 0x3Fu)); f(0x80u | (c & 0x3Fu)); out += 3; }
        else { f(0xF0u | (c >> 18)); f(0x80u | ((c >> 12) & 0x3Fu)); f(0x80u | ((c >> 6) & 0x3Fu)); f(0x80u | (c & 0x3Fu)); out += 4; }
    }
    return out;
}

VPT_HD bool token_lookup(const DevTags& t, const uint8_t* __restrict__ bytes, uint32_t len, int norm, uint32_t& tid) {
    if (len == 0 || len > 4u * t.max_token_bytes) return false;
    uint64_t h = kTagHashInit;
    const uint32_t nlen = token_bytes(bytes, len, norm, [&](uint32_t b) { h = tag_hash_step(h, b); });
    if (nlen > t.max_token_bytes) return false;
    h = tag_hash_finish(h);
    for (uint32_t s = uint32_t(h >> 20) & t.tok_mask;; s = (s + 1) & t.tok_mask) {
        const TagTokenEntry e = t.tok_tab[s];
        if (e.hash == 0) return false;
        if (e.hash == h && e.len == nlen) {
            bool same = true;
            uint32_t idx = 0;
            token_bytes(bytes, len, norm, [&](uint32_t b) { same = same && VPT_LDG(t.tok_bytes + e.str_off + idx) == b; ++idx; });
            if (same) { tid = e.tid; return true; }
        }
    }
}

constexpr int kTagRelRegs = 4;  // rel positions whose chains are kept in registers (window 3: rel 0..3)

// true when pattern `want` lies on the suffix chain that starts at `pid` (positions 0..4 from the chain record, the rest
// through the link table: only patterns longer than five suffix levels, i.e. dictionary words, get there)
VPT_HD bool on_chain(uint32_t want, uint32_t pid, const uint4 ch, const uint32_t* __restrict__ link) {
    if (want == pid || want == ch.x || want == ch.y || want == ch.z || want == ch.w) return true;
    if (ch.w == kNoPattern) return false;
    for (uint32_t q = VPT_LDG(link + ch.w); q != kNoPattern; q = VPT_LDG(link + q))
        if (q == want) return true;
    return false;
}

// scores += the tag weights of one scorer for the token whose last character is `i` (add_tag_scores,
// char_scorer/boundary_tag_scorer.rs:154-174, type_scorer/boundary_tag_scorer.rs:123-143): for every rel position the
// pattern found at character i + rel contributes its own vector and those of its suffix patterns (merged in the
// reference at build time), element k of a shorter pattern's vector only while every longer one on the chain is longer
// than k.  The token's key list is sorted by rel, longest pattern first: one pass per rel position applies the rule.
// cnt[r]: entries with rel position r (0 .. 3); rest: entries with rel position >= 4 behind them.
VPT_HD void add_scorer(const TagKey* __restrict__ keys, const uint8_t* cnt, uint32_t rest,
                                           const TagChain* __restrict__ chains, const uint32_t* __restrict__ link,
                                           const int32_t* __restrict__ pool, const uint32_t* __restrict__ states, uint32_t npat,
                                           uint32_t rels, uint32_t i, uint32_t n, int32_t* scores, uint32_t nscores) {
    // the patterns at the rel positions and their chains: all loads first (they are independent)
    uint32_t pid[kTagRelRegs];
    uint4 ch[kTagRelRegs];
#pragma unroll
    for (int r = 0; r < kTagRelRegs; ++r) {
        pid[r] = kNoPattern;
        if (cnt[r] != 0 && uint32_t(r) < rels && i + uint32_t(r) < n) pid[r] = states[i + r];
        if (pid[r] >= npat) pid[r] = kNoPattern;
    }
#pragma unroll
    for (int r = 0; r < kTagRelRegs; ++r) {
        ch[r] = make_uint4(kNoPattern, kNoPattern, kNoPattern, kNoPattern);
        if (pid[r] != kNoPattern) ch[r] = VPT_LDG(reinterpret_cast<const uint4*>(chains + pid[r]));
    }
#pragma unroll
    for (int r = 0; r < kTagRelRegs; ++r) {
        const uint32_t nk = cnt[r];
        if (pid[r] != kNoPattern) {
            uint32_t limit = nscores;
            for (uint32_t j = 0; j < nk && limit; ++j) {
                const uint4 e = VPT_LDG(reinterpret_cast<const uint4*>(keys + j));  // pid, off, len, rel
                if (on_chain(e.x, pid[r], ch[r], link)) {
                    const uint32_t upto = min(limit, e.z);
                    for (uint32_t k = 0; k < upto; ++k) scores[k] = int32_t(uint32_t(scores[k]) + uint32_t(VPT_LDG(pool + e.y + k)));
                    limit = upto;
                }
            }
        }
        keys += nk;
    }
    // wider windows: rel positions from 4 on, the chain straight from the tables
    uint32_t cur_rel = 0xFFFFFFFFu, limit = 0;
    for (uint32_t j = 0; j < rest; ++j) {
        const uint4 e = VPT_LDG(reinterpret_cast<const uint4*>(keys + j));
        if (e.w != cur_rel) { cur_rel = e.w; limit = nscores; }
        if (limit == 0 || e.w >= rels || i + e.w >= n) continue;
        const uint32_t q = states[i + e.w];
        if (q < npat && on_chain(e.x, q, VPT_LDG(reinterpret_cast<const uint4*>(chains + q)), link)) {
            const uint32_t upto = min(limit, e.z);
            for (uint32_t k = 0; k < upto; ++k) scores[k] = int32_t(uint32_t(scores[k]) + uint32_t(VPT_LDG(pool + e.y + k)));
            limit = upto;
        }
    }
}

// Number of scores a token of the table gets: its whole score vector (bias_len entries), or 0 when its slots' candidates
// overrun the vector -- exactly the tokens tag_score_token answers -1 for after the `usable` check.  k_tok_lookup sizes
// the score output with it before k_tok_score computes the scores.
VPT_HD uint32_t tag_score_count(const TagTokenInfo& ti, uint32_t nt) {
    uint32_t off = 0;
    for (uint32_t k = 0; k < ti.n_slots && k < nt; ++k) {
        const uint32_t nc = ti.cand[k];
        if (nc >= 2) {
            if (off + nc > ti.bias_len) return 0;
            off += nc;
        }
    }
    return ti.bias_len;
}

// Tag prediction of one token (bytes [bytes, bytes + len) of the text; `i` = index of its last character inside the
// sentence's `n` characters whose pattern-id states start at cst / tst): token lookup, bias + tag weights of both scorers,
// first strict maximum per tag slot (TagPredictor::predict, predictor.rs:286-304).  Returns the token id or -1 and the
// chosen candidates in cand[].  kStoreScores: a token answered with its id also gets its whole score vector (the
// `scores` Predictor::predict_tags keeps with store_tag_scores, tag_score_count(ti) entries) in scores_out[].
// (the part behind the token lookup: `tid` is a token of the table)
template <bool kStoreScores = false>
VPT_HD int32_t tag_score_token(const DevTags& t, uint32_t tid, const uint32_t* __restrict__ cst,
                                                   const uint32_t* __restrict__ tst, uint32_t i, uint32_t n, int32_t* cand,
                                                   uint32_t* n_unserved, int32_t* __restrict__ scores_out = nullptr) {
    TagTokenInfo ti;
    {
        const uint4* q = reinterpret_cast<const uint4*>(t.tok_info + tid);
        *reinterpret_cast<uint4*>(&ti) = VPT_LDG(q);
        *(reinterpret_cast<uint4*>(&ti) + 1) = VPT_LDG(q + 1);
    }
    if (!ti.usable) {
        if (n_unserved) VPT_COUNT(n_unserved);
        return -1;
    }
    int32_t scores[kTagMaxScores];
    const uint32_t ns = ti.bias_len;
    for (uint32_t k = 0; k < ns; ++k) scores[k] = VPT_LDG(t.pool + ti.bias_off + k);
    const uint32_t n_ckeys = uint32_t(ti.ckeys[0]) + ti.ckeys[1] + ti.ckeys[2] + ti.ckeys[3] + ti.c_rest;
    const uint32_t n_tkeys = uint32_t(ti.tkeys[0]) + ti.tkeys[1] + ti.tkeys[2] + ti.tkeys[3] + ti.t_rest;
    if (cst && n_ckeys)
        add_scorer(t.keys + ti.key_off, ti.ckeys, ti.c_rest, t.c_chain, t.c_link, t.pool, cst, t.n_char_patterns, t.char_rels, i, n,
                   scores, ns);
    if (tst && n_tkeys)
        add_scorer(t.keys + ti.key_off + n_ckeys, ti.tkeys, ti.t_rest, t.t_chain, t.t_link, t.pool, tst, t.n_type_patterns,
                   t.type_rels, i, n, scores, ns);
    uint32_t off = 0;
    const uint32_t nt = t.n_tags;
    for (uint32_t k = 0; k < ti.n_slots && k < nt; ++k) {
        const uint32_t nc = ti.cand[k];
        if (nc >= 2) {
            if (off + nc > ns) {
                if (n_unserved) VPT_COUNT(n_unserved);  // the host path reports the model error
                return -1;
            }
            uint32_t best = 0;
            int32_t mx = INT32_MIN;
            for (uint32_t c = 0; c < nc; ++c)
                if (scores[off + c] > mx) { best = c; mx = scores[off + c]; }
            cand[k] = int32_t(best);
            off += nc;
        } else {
            cand[k] = nc == 1 ? 0 : -1;
        }
    }
    if (kStoreScores)
        for (uint32_t k = 0; k < ns; ++k) scores_out[k] = scores[k];
    return int32_t(tid);
}

VPT_HD int32_t tag_token_at(const DevTags& t, const uint8_t* __restrict__ bytes, uint32_t len,
                                                const uint32_t* __restrict__ cst, const uint32_t* __restrict__ tst, uint32_t i,
                                                uint32_t n, int32_t* cand, uint32_t* n_unserved, int norm) {
    uint32_t tid = 0;
    if (!token_lookup(t, bytes, len, norm, tid)) return -1;
    return tag_score_token(t, tid, cst, tst, i, n, cand, n_unserved);
}

}  // namespace vpt
