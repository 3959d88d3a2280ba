// evaluate.cu — the reference's `evaluate` command on the device (evaluate/src/main.rs:69-195):
//
//   * k_gold_parse: `Sentence::from_tokenized` (sentence.rs:285-467) for every line of a chunk: the raw sentence text
//     (compacted, so the scoring kernels run on it unchanged), the gold boundaries, where each gold token's tag fields
//     start, the tag width of every line, and the first error of the chunk (the lowest line; inside it, the first
//     violation the reference's character loop meets; invalid UTF-8 before everything, since `lines()` fails first);
//   * k_eval: the char metric (TP/TN/FP/FN, main.rs:121-147) and Nagata's word metric (main.rs:149-191) of the gold
//     boundaries and tags against the system's, per line and summed over the chunk.
//
// Both are byte-streaming work in the style of lines.cu: one warp per line, 128 bytes (k_eval: 32 boundaries) per
// step, warp scans inside a step and warp-uniform carries across steps, so a line of any length works.
#include <cuda_runtime.h>

#include <cstdint>

#include "byte_window.cuh"
#include "device_model.hpp"

namespace vpt {

namespace {

using bw::byte_of;
using bw::inside80;
using bw::kFull;
using bw::warp_incl_scan_u32;

constexpr int kEvThreads = 256;
constexpr int kWarps = kEvThreads / 32;
constexpr uint64_t kStAgg = 1ull << 62, kStIncl = 2ull << 62, kStMask = (1ull << 62) - 1;

// inclusive "last non-zero value" scan: the latest event of a lane or of the lanes before it (0: none)
__device__ __forceinline__ uint32_t warp_last_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d && v == 0) v = o;
    }
    return v;
}

__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) {
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}
__device__ __forceinline__ uint32_t eq_bytes(uint32_t x, uint32_t c) { return zero_bytes(x ^ (c * 0x01010101u)); }

struct GoldLine {
    uint32_t surf = 0, chars = 0, width = 0;
    uint64_t err = kGoldNoError;  // (position in the line + 1) << 3 | kind; kind kGoldUtf8 has position 0
};

// One line by one warp.  kWrite: also writes the surface bytes at `surf_out`, the gold boundary flag of every character
// at gold_bnd[char_base + k] and the tag positions (kWrite is only used once the bases are known).
//
// Per byte: escaped = odd run of '\' right before it; an unescaped ' ' ends a token, an unescaped '/' starts a tag
// field that runs to the next unescaped ' ', an unescaped '\' is dropped; every other byte belongs to the surface
// unless it is inside a tag field.  The character loop's state at a byte (escape parity, in a tag field, a ' ' since
// the last surface character, tag fields of the current token) is a scan over the bytes before it.
template <bool kWrite>
__device__ GoldLine gold_line(const EvalArgs& e, uint64_t o0, uint64_t o1, uint32_t trim, uint64_t surf_base,
                              uint64_t char_base, int lane) {
    GoldLine r;
    const uint64_t a0 = o0 & ~3ull;
    const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(o1 - a0) - trim;
    if (b1 <= b0) return r;  // empty line: skipped by the CLI
    const uint8_t* __restrict__ base = e.text + a0;
    uint32_t c_bs = 0, c_tag = 0, c_psp = 0, c_fields = 0, first_err = 0;
    bool utf8_bad = false;
    for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t lo = 0, hi = 0, in80 = 0;
        if (addr < b1) {
            lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
            if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(base + addr + 4));
            in80 = inside80(addr, b0, b1);
        }
        // ---- UTF-8: every non-continuation byte checks its own sequence and that no extra continuation byte follows
        bool bad = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (!(in80 & (0x80u << (8 * j)))) continue;
            const uint32_t c0 = byte_of(lo, hi, j);
            auto cont = [&](int k) { return addr + uint32_t(k) < b1 && (byte_of(lo, hi, k) & 0xC0u) == 0x80u; };
            if ((c0 & 0xC0u) == 0x80u) {
                if (addr + uint32_t(j) == b0) bad = true;  // a line cannot start inside a character
                continue;
            }
            const int len = c0 < 0x80u ? 1 : c0 < 0xC2u ? 0 : c0 < 0xE0u ? 2 : c0 < 0xF0u ? 3 : c0 < 0xF5u ? 4 : 0;
            if (len == 0) { bad = true; continue; }
            for (int k = 1; k < len; ++k) bad |= !cont(j + k);
            bad |= cont(j + len);
            if (len >= 3 && cont(j + 1)) {
                const uint32_t c1 = byte_of(lo, hi, j + 1);
                if ((c0 == 0xE0u && c1 < 0xA0u) || (c0 == 0xEDu && c1 >= 0xA0u) || (c0 == 0xF0u && c1 < 0x90u) ||
                    (c0 == 0xF4u && c1 >= 0x90u))
                    bad = true;
            }
        }
        utf8_bad |= __any_sync(kFull, bad) != 0;

        // ---- 1. escapes: parity of the run of '\' before each byte (segmented scan, carried across steps)
        const uint32_t bs80 = eq_bytes(lo, 0x5Cu) & in80;
        uint32_t run = 0;
#pragma unroll
        for (int j = 3; j >= 0; --j) {
            if (!(bs80 & (0x80u << (8 * j)))) break;
            ++run;
        }
        uint32_t s_all = run == 4 ? 1u : 0u, s_par = run & 1u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t oa = __shfl_up_sync(kFull, s_all, d), op = __shfl_up_sync(kFull, s_par, d);
            if (lane >= d && s_all) { s_par ^= op; s_all = oa; }
        }
        uint32_t x_all = __shfl_up_sync(kFull, s_all, 1), x_par = __shfl_up_sync(kFull, s_par, 1);
        if (lane == 0) { x_all = 1; x_par = 0; }
        uint32_t esc = x_all ? (c_bs ^ x_par) : x_par;
        uint32_t sp80 = 0, sl80 = 0, drop80 = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (!(in80 & bit)) { esc = 0; continue; }
            const uint32_t c = byte_of(lo, hi, j);
            if (!esc) {
                if (c == 0x20u) sp80 |= bit;
                else if (c == 0x2Fu) sl80 |= bit;
                else if (c == 0x5Cu) drop80 |= bit;
            }
            esc = (c == 0x5Cu) ? esc ^ 1u : 0u;
        }
        {
            const uint32_t a31 = __shfl_sync(kFull, s_all, 31), p31 = __shfl_sync(kFull, s_par, 31);
            c_bs = a31 ? (c_bs ^ p31) : p31;
        }

        // ---- 2. tag fields: the last unescaped ' ' (1) or '/' (2) before each byte
        uint32_t ev = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (sp80 & bit) ev = 1;
            if (sl80 & bit) ev = 2;
        }
        const uint32_t tag_incl = warp_last_scan(ev, lane);
        uint32_t tag_x = __shfl_up_sync(kFull, tag_incl, 1);
        if (lane == 0) tag_x = 0;
        uint32_t in_tag = tag_x ? (tag_x == 2) : c_tag;
        uint32_t surf80 = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if ((in80 & bit) && !((sp80 | sl80 | drop80) & bit) && !in_tag) surf80 |= bit;
            if (sp80 & bit) in_tag = 0;
            if (sl80 & bit) in_tag = 1;
        }
        {
            const uint32_t t31 = __shfl_sync(kFull, tag_incl, 31);
            if (t31) c_tag = t31 == 2;
        }
        const uint32_t st80 = surf80 & ~(lo & ~(lo << 1));  // surface bytes that start a character

        // ---- 3. counts, ' ' since the last character (prev_boundary), tag fields of the current token
        const uint32_t nsurf = __popc(surf80), nst = __popc(st80);
        const uint32_t surf_incl = warp_incl_scan_u32(nsurf, lane), st_incl = warp_incl_scan_u32(nst, lane);
        uint32_t pev = 0;  // last ' ' (1) or character start (2) of the lane
        uint32_t f_reset = 0, f_cnt = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (sp80 & bit) { pev = 1; f_reset = 1; f_cnt = 0; }
            if (st80 & bit) pev = 2;
            if (sl80 & bit) ++f_cnt;
        }
        const uint32_t psp_incl = warp_last_scan(pev, lane);
        uint32_t psp_x = __shfl_up_sync(kFull, psp_incl, 1);
        if (lane == 0) psp_x = 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t orr = __shfl_up_sync(kFull, f_reset, d), oc = __shfl_up_sync(kFull, f_cnt, d);
            if (lane >= d && !f_reset) { f_reset = orr; f_cnt += oc; }
        }
        uint32_t fx_reset = __shfl_up_sync(kFull, f_reset, 1), fx_cnt = __shfl_up_sync(kFull, f_cnt, 1);
        if (lane == 0) { fx_reset = 0; fx_cnt = 0; }

        uint32_t psp = psp_x ? (psp_x == 1) : c_psp;
        uint32_t fields = fx_reset ? fx_cnt : c_fields + fx_cnt;
        uint32_t cb = r.chars + st_incl - nst;       // characters of the line before this byte
        uint64_t so = r.surf + surf_incl - nsurf;    // surface bytes of the line before this byte
        uint32_t width = 0, err = 0xFFFFFFFFu;       // err: (position in this step) << 3 | kind
        uint32_t sl_char[4] = {0, 0, 0, 0};
        uint32_t sl_first = 0;                        // bytes that open the first tag field of a token (kWrite)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (!(in80 & bit)) continue;
            const uint32_t c = byte_of(lo, hi, j);
            const uint32_t at = ((4u * uint32_t(lane) + uint32_t(j)) << 3);
            if (c == 0) err = min(err, at | kGoldNul);
            if (sp80 & bit) {
                if (cb == 0) err = min(err, at | kGoldStartWs);
                else if (psp) err = min(err, at | kGoldDoubleWs);
                psp = 1;
                width = max(width, fields);
                fields = 0;
            } else if (sl80 & bit) {
                if (cb == 0 || psp) err = min(err, at | kGoldSlash);
                if (fields == 0 && cb > 0) { sl_first |= bit; sl_char[j] = cb - 1; }
                ++fields;
            } else if (st80 & bit) {
                if (kWrite) {
                    e.gold_bnd[char_base + cb] = (cb > 0 && psp) ? 1 : 0;
                    if (e.tag_pos) e.tag_pos[char_base + cb] = 0xFFFFFFFFu;
                }
                psp = 0;
                ++cb;
            }
            if (kWrite && (surf80 & bit)) e.surface[surf_base + so++] = uint8_t(c);
        }
        if (kWrite && e.tag_pos) {
            __syncwarp();  // a character's "no tags" mark above is written before the tag position of its token
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (sl_first & (0x80u << (8 * j))) e.tag_pos[char_base + sl_char[j]] = uint32_t(a0 + addr + j);
        }
        r.width = max(r.width, __reduce_max_sync(kFull, width));
        const uint32_t werr = __reduce_min_sync(kFull, err);
        if (first_err == 0 && werr != 0xFFFFFFFFu) {
            const uint32_t pos = w0 + (werr >> 3) - b0;
            r.err = (uint64_t(pos + 1) << 3) | (werr & 7u);
            first_err = 1;
        }
        // carries: the state after the last byte of the step is the last lane's
        c_psp = __shfl_sync(kFull, psp, 31);
        c_fields = __shfl_sync(kFull, fields, 31);
        r.surf += __shfl_sync(kFull, surf_incl, 31);
        r.chars += __shfl_sync(kFull, st_incl, 31);
    }
    r.width = max(r.width, c_fields);
    const uint64_t end = uint64_t(b1 - b0 + 1) << 3;
    if (!first_err) {
        if (r.chars == 0) r.err = end | kGoldEmpty;  // a lone '\' (the reference divides by zero here)
        else if (c_psp) r.err = end | kGoldEndWs;
    }
    if (utf8_bad) r.err = kGoldUtf8;
    return r;
}

// One CTA per 64-line group (ticket order, as k_tok_write): 1. each warp parses its lines and counts their surface
// bytes and characters; 2. the group's offsets come from a decoupled look-back over the predecessors' totals (state
// word: 2 flag bits | surface bytes << 31 | characters, both below 2^31 in a chunk of at most 1 GiB); 3. the lines
// are parsed again and written.
__global__ void __launch_bounds__(kEvThreads) k_gold_parse(EvalArgs e, uint64_t ngroups) {
    __shared__ uint64_t s_off[kGroup + 1];
    __shared__ uint32_t s_surf[kGroup], s_ch[kGroup], s_xs[kGroup], s_xc[kGroup];
    __shared__ uint8_t s_trim[kGroup];
    __shared__ uint64_t s_base;
    __shared__ uint32_t s_grp;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_grp = atomicAdd(e.ticket, 1u);
    __syncthreads();
    const uint64_t grp = s_grp;
    const uint64_t gbase = grp * kGroup;
    const int ns = int(min(uint64_t(kGroup), e.n_sent - gbase));
    if (threadIdx.x <= ns) s_off[threadIdx.x] = e.offsets[gbase + threadIdx.x];
    if (threadIdx.x < kGroup) { s_surf[threadIdx.x] = 0; s_ch[threadIdx.x] = 0; }
    if (threadIdx.x < ns) s_trim[threadIdx.x] = e.trims[gbase + threadIdx.x];
    __syncthreads();
    // 1. counts, widths, errors
    for (int i = warp; i < ns; i += kWarps) {
        const GoldLine g = gold_line<false>(e, s_off[i], s_off[i + 1], s_trim[i], 0, 0, lane);
        if (lane == 0) {
            s_surf[i] = g.surf;
            s_ch[i] = g.chars;
            e.width[gbase + i] = g.width;
            if (g.err != kGoldNoError) atomicMin(reinterpret_cast<unsigned long long*>(e.err), ((gbase + i) << 34) | g.err);
        }
    }
    __syncthreads();
    // 2. offsets
    if (warp == 0) {
        const uint32_t s0 = s_surf[2 * lane], s1 = s_surf[2 * lane + 1];
        const uint32_t c0 = s_ch[2 * lane], c1 = s_ch[2 * lane + 1];
        const uint32_t is = warp_incl_scan_u32(s0 + s1, lane), ic = warp_incl_scan_u32(c0 + c1, lane);
        s_xs[2 * lane] = is - s0 - s1;
        s_xs[2 * lane + 1] = is - s1;
        s_xc[2 * lane] = ic - c0 - c1;
        s_xc[2 * lane + 1] = ic - c1;
        const uint64_t total = (uint64_t(__shfl_sync(kFull, is, 31)) << 31) | __shfl_sync(kFull, ic, 31);
        volatile uint64_t* state = e.state;
        if (lane == 0) state[grp] = (grp == 0 ? kStIncl : kStAgg) | total;
        uint64_t prefix = 0;
        if (grp > 0) {
            int64_t idx = int64_t(grp) - 1;
            for (;;) {
                const int64_t j = idx - lane;
                uint64_t v = kStIncl;
                if (j >= 0) {
                    do { v = state[j]; } while ((v >> 62) == 0);
                }
                const unsigned incl = __ballot_sync(kFull, (v >> 62) == 2);
                const int stop = incl ? __ffs(incl) - 1 : 32;
                uint64_t add = lane <= stop ? (v & kStMask) : 0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
                prefix += add;
                if (incl) break;
                idx -= 32;
            }
            if (lane == 0) state[grp] = kStIncl | (prefix + total);
        }
        if (lane == 0) {
            s_base = prefix;
            if (grp + 1 == ngroups) {
                e.surf_offsets[e.n_sent] = (prefix + total) >> 31;
                e.char_offsets[e.n_sent] = (prefix + total) & 0x7FFFFFFFu;
            }
        }
    }
    __syncthreads();
    // 3. write
    const uint64_t sb = s_base >> 31, cbase = s_base & 0x7FFFFFFFu;
    for (int i = warp; i < ns; i += kWarps) {
        const uint64_t so = sb + s_xs[i], co = cbase + s_xc[i];
        if (lane == 0) {
            e.surf_offsets[gbase + i] = so;
            e.char_offsets[gbase + i] = co;
        }
        gold_line<true>(e, s_off[i], s_off[i + 1], s_trim[i], so, co, lane);
    }
}

// the next character of an escaped string ('\x' is x; a '\' at the end escapes nothing)
__device__ __forceinline__ bool next_unescaped(const uint8_t* s, uint32_t n, uint32_t& i, uint32_t& c) {
    if (i < n && s[i] == 0x5Cu) ++i;
    if (i >= n) return false;
    c = s[i++];
    return true;
}

// Vec<Option<String>> equality of the gold and system tags of the character that ends a gold and a system token
// (main.rs:110-120): the gold fields are read from the input line, the system's are the chosen candidates' strings.
__device__ bool tags_equal(const EvalArgs& e, uint64_t line, uint64_t ch, uint64_t rec) {
    if (e.tag_mode == kTagsAlwaysEqual) return true;
    const uint32_t width = e.width[line];
    if (e.tag_mode == kTagsGoldEmpty) return width == 0;
    if (width != e.n_tags) return false;
    const uint8_t* text = e.text;
    const uint64_t end = e.offsets[line + 1] - e.trims[line];
    uint64_t p = e.tag_pos[ch];  // the token's first '/', or none
    if (p == 0xFFFFFFFFu) p = end;
    const int32_t tid = e.tok_ids[rec];
    const uint32_t sb = tid >= 0 ? __ldg(e.ts_slot + tid) : 0u;
    for (uint32_t k = 0; k < e.n_tags; ++k) {
        // gold field k: [f0, f1) in escaped form, or none
        uint64_t f0 = end, f1 = end;
        if (p < end && text[p] == 0x2Fu) {
            f0 = p + 1;
            uint64_t q = f0;
            while (q < end) {
                const uint8_t b = text[q];
                if (b == 0x5Cu) { q = q + 2 < end ? q + 2 : end; continue; }
                if (b == 0x2Fu || b == 0x20u) break;
                ++q;
            }
            f1 = q;
            p = q;
        } else {
            p = end;
        }
        uint32_t gi = 0, gc = 0;
        const uint32_t gn = uint32_t(f1 - f0);
        const bool gold_none = !next_unescaped(text + f0, gn, gi, gc);
        const uint32_t c = tid >= 0 ? e.tok_cands[rec * e.n_tags + k] : 255u;
        if (c == 255u) {
            if (!gold_none) return false;
            continue;
        }
        if (gold_none) return false;
        const uint2 ref = __ldg(e.ts_ref + __ldg(e.ts_cand + sb + k) + c);
        const uint8_t* ts = e.ts_bytes + ref.x;
        uint32_t si = 0, sc = 0;
        if (!next_unescaped(ts, ref.y, si, sc) || sc != gc) return false;
        for (;;) {
            const bool more_g = next_unescaped(text + f0, gn, gi, gc), more_s = next_unescaped(ts, ref.y, si, sc);
            if (more_g != more_s) return false;
            if (!more_g) break;
            if (gc != sc) return false;
        }
    }
    return true;
}

// One warp per line, 32 boundaries per step.  Word metric: at a position where gold and system both end a token (or
// at the sentence end) the token counts as correct when no boundary disagreed since the last position where both had
// one -- the reference's `matched` flag -- and the tags there are equal.
__global__ void __launch_bounds__(kEvThreads) k_eval(EvalArgs e) {
    __shared__ unsigned long long s_tot[kEvalTotals];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < kEvalTotals) s_tot[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t gbase = uint64_t(blockIdx.x) * kGroup;
    const int ns = int(min(uint64_t(kGroup), e.n_sent - gbase));
    uint64_t acc[kEvalTotals] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = warp; i < ns; i += kWarps) {
        const uint64_t l = gbase + i;
        const uint32_t nch = e.status[l] == 0 ? e.n_chars[l] : 0u;
        uint32_t cnt[7] = {0, 0, 0, 0, 0, 0, 0};  // tp tn fp fn n_sys n_ref n_cor
        if (nch > 0) {
            const uint8_t* __restrict__ sys = e.boundaries + e.bound_offsets[l];
            const uint8_t* __restrict__ gold = e.gold_bnd + e.char_offsets[l] + 1;
            const uint64_t c0 = e.char_offsets[l];
            const uint64_t rec0 = e.tok_base ? e.tok_base[l] : 0;
            const uint32_t nb = nch - 1;
            uint32_t c_ev = 0, c_nsys = 0;
            for (uint32_t w0 = 0; w0 < nb; w0 += 32) {
                const uint32_t j = w0 + uint32_t(lane);
                const bool valid = j < nb;
                const uint32_t s = valid ? sys[j] : 0u, g = valid ? gold[j] : 0u;
                cnt[0] += s & g;
                cnt[1] += valid & !s & !g;
                cnt[2] += s & !g;
                cnt[3] += !s & g;
                cnt[5] += g;
                const uint32_t ev = s != g ? 1u : (s & g) ? 2u : 0u;  // 1: disagreement, 2: both end a token
                const uint32_t ev_incl = warp_last_scan(ev, lane);
                uint32_t prev = __shfl_up_sync(kFull, ev_incl, 1);
                if (lane == 0 || prev == 0) prev = c_ev;
                const uint32_t sys_incl = warp_incl_scan_u32(s, lane);
                if (ev == 2 && prev != 1 && tags_equal(e, l, c0 + j, rec0 + c_nsys + sys_incl - s)) ++cnt[6];
                const uint32_t last = __shfl_sync(kFull, ev_incl, 31);
                if (last) c_ev = last;
                c_nsys += __shfl_sync(kFull, sys_incl, 31);
            }
            if (lane == 0 && c_ev != 1 && tags_equal(e, l, c0 + nb, rec0 + c_nsys)) ++cnt[6];
#pragma unroll
            for (int k = 0; k < 7; ++k) cnt[k] = __reduce_add_sync(kFull, cnt[k]);
            cnt[4] = c_nsys + 1;
            cnt[5] += 1;
        }
        if (lane == 0) {
            if (e.line_counts)
                for (int k = 0; k < 7; ++k) e.line_counts[l * 7 + k] = cnt[k];
            for (int k = 0; k < 7; ++k) acc[k] += cnt[k];
            acc[7] += nch > 0;
        }
    }
    if (lane == 0)
        for (int k = 0; k < kEvalTotals; ++k)
            if (acc[k]) atomicAdd(&s_tot[k], static_cast<unsigned long long>(acc[k]));
    __syncthreads();
    if (threadIdx.x < kEvalTotals && s_tot[threadIdx.x])
        atomicAdd(reinterpret_cast<unsigned long long*>(e.totals) + threadIdx.x, s_tot[threadIdx.x]);
}

}  // namespace

cudaError_t launch_gold_parse(const EvalArgs& e, cudaStream_t stream) {
    if (e.n_sent == 0) return cudaSuccess;
    const uint64_t ngroups = (e.n_sent + kGroup - 1) / kGroup;
    // look-back state words + the ticket that follows them
    cudaError_t err = cudaMemsetAsync(e.state, 0, 8 * (ngroups + 1), stream);
    if (err != cudaSuccess) return err;
    k_gold_parse<<<unsigned(ngroups), kEvThreads, 0, stream>>>(e, ngroups);
    return cudaGetLastError();
}

cudaError_t launch_eval(const EvalArgs& e, cudaStream_t stream) {
    if (e.n_sent == 0) return cudaSuccess;
    const uint64_t ngroups = (e.n_sent + kGroup - 1) / kGroup;
    k_eval<<<unsigned(ngroups), kEvThreads, 0, stream>>>(e);
    return cudaGetLastError();
}

}  // namespace vpt
