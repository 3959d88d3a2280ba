// partial.cu — partially annotated lines on the device (vpt_tokenize_partial_lines):
//
//   * k_part_parse: `Sentence::from_partial_annotation` (reference sentence.rs:516-631) for every line of a chunk: the
//     raw sentence text (compacted, so the scoring kernels run on it unchanged), the marker before every character, and
//     the first error of the chunk (the lowest line; inside it, the first violation the reference's character loop
//     meets; invalid UTF-8 before everything, since `lines()` fails first);
//   * k_part_apply: after scoring and the post-filters, every '|' / '-' the caller wrote replaces the boundary it marks.
//
// k_part_parse streams a line through one warp, 128 bytes per step, as k_gold_parse does: the state of the character
// loop at every byte is a warp scan of the byte automaton of partial_parse.hpp, carried across steps.
#include <cuda_runtime.h>

#include <cstdint>

#include "byte_window.cuh"
#include "device_model.hpp"
#include "partial_parse.hpp"

namespace vpt {

namespace {

using bw::byte_of;
using bw::inside80;
using bw::kFull;
using bw::warp_incl_scan_u32;

constexpr int kPaThreads = 256;
constexpr int kWarps = kPaThreads / 32;
constexpr uint64_t kStAgg = 1ull << 62, kStIncl = 2ull << 62, kStMask = (1ull << 62) - 1;

struct PartLine {
    uint32_t surf = 0, chars = 0;
    uint64_t err = kGoldNoError;  // (position in the line + 1) << 3 | kind; kind kPartUtf8 has position 0
};

// One line by one warp.  kWrite: also writes the surface bytes at `surf_out` and the marker code before every
// character at given[char_base + k] (kWrite is only used once the bases are known).
template <bool kWrite>
__device__ PartLine part_line(const PartArgs& e, uint64_t o0, uint64_t o1, uint32_t trim, uint64_t surf_base,
                              uint64_t char_base, int lane) {
    PartLine r;
    const uint64_t a0 = o0 & ~3ull;
    const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(o1 - a0) - trim;
    if (b1 <= b0) return r;  // empty line: an empty output line
    const uint8_t* __restrict__ base = e.text + a0;
    uint32_t c_state = kPaChar, first_err = 0;
    bool utf8_bad = false;
    for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t lo = 0, hi = 0, in80 = 0;
        if (addr < b1) {
            lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
            if (addr + 4 < b1) hi = __ldg(reinterpret_cast<const uint32_t*>(base + addr + 4));
            in80 = inside80(addr, b0, b1);
        }
        utf8_bad |= __any_sync(kFull, bw::utf8_word_bad(lo, hi, addr, b0, b1, in80)) != 0;

        // the state before the lane's first byte: the composed moves of the lanes before it, on the carried state
        const uint32_t m = pa_word_map(lo, in80);
        uint32_t incl = m;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl = pa_compose(o, incl);
        }
        uint32_t x = __shfl_up_sync(kFull, incl, 1);
        if (lane == 0) x = kPaIdentity;
        uint32_t s = pa_apply(x, c_state);

        uint32_t surf80 = 0, st80 = 0, err = 0xFFFFFFFFu;  // err: (position in this step) << 3 | kind
        uint32_t codes = 0xFFFFFFFFu;                        // byte j: the marker code of byte j, or 0xFF
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (!(in80 & bit)) continue;
            const PaByte pb = pa_byte(s, byte_of(lo, hi, j));
            s = pb.next;
            if (pb.surf) surf80 |= bit;
            if (pb.start) st80 |= bit;
            codes &= ~(0xFFu << (8 * j)) | (pb.code << (8 * j));
            if (pb.err) err = min(err, ((4u * uint32_t(lane) + uint32_t(j)) << 3) | pb.err);
        }
        const uint32_t nsurf = __popc(surf80), nst = __popc(st80);
        const uint32_t surf_incl = warp_incl_scan_u32(nsurf, lane), st_incl = warp_incl_scan_u32(nst, lane);
        if (kWrite) {
            uint32_t cb = r.chars + st_incl - nst;      // characters of the line before this byte
            uint64_t so = r.surf + surf_incl - nsurf;   // surface bytes of the line before this byte
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bit = 0x80u << (8 * j);
                if (st80 & bit) ++cb;
                if (surf80 & bit) e.surface[surf_base + so++] = uint8_t(byte_of(lo, hi, j));
                const uint32_t code = (codes >> (8 * j)) & 0xFFu;
                if (code != 0xFFu) e.given[char_base + cb] = uint8_t(code);  // the boundary before the next character
            }
        }
        const uint32_t werr = __reduce_min_sync(kFull, err);
        if (first_err == 0 && werr != 0xFFFFFFFFu) {
            const uint32_t pos = w0 + (werr >> 3) - b0;
            r.err = (uint64_t(pos + 1) << 3) | (werr & 7u);
            first_err = 1;
        }
        // carries: the state after the step is the whole warp's move on the carried state
        c_state = pa_apply(__shfl_sync(kFull, incl, 31), c_state);
        r.surf += __shfl_sync(kFull, surf_incl, 31);
        r.chars += __shfl_sync(kFull, st_incl, 31);
    }
    if (!first_err && c_state == kPaChar) r.err = (uint64_t(b1 - b0 + 1) << 3) | kPartEnd;
    if (utf8_bad) r.err = kPartUtf8;
    return r;
}

// One CTA per 64-line group (ticket order, as k_gold_parse): 1. each warp parses its lines and counts their surface
// bytes and characters; 2. the group's offsets come from a decoupled look-back over the predecessors' totals (state
// word: 2 flag bits | surface bytes << 31 | characters, both below 2^31 in a chunk of at most 1 GiB); 3. the lines
// are parsed again and written.
__global__ void __launch_bounds__(kPaThreads) k_part_parse(PartArgs e, uint64_t ngroups) {
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
    // 1. counts, errors
    for (int i = warp; i < ns; i += kWarps) {
        const PartLine g = part_line<false>(e, s_off[i], s_off[i + 1], s_trim[i], 0, 0, lane);
        if (lane == 0) {
            s_surf[i] = g.surf;
            s_ch[i] = g.chars;
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
        part_line<true>(e, s_off[i], s_off[i + 1], s_trim[i], so, co, lane);
    }
}

// One warp per line, 32 boundaries per step: boundary j of a line lies between its characters j and j + 1, and the
// marker before character j + 1 is at given[char_offsets[line] + j + 1].
__global__ void __launch_bounds__(kPaThreads) k_part_apply(PartArgs e) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t l = uint64_t(blockIdx.x) * kWarps + warp;
    if (l >= e.n_sent || e.status[l] != 0) return;
    const uint32_t nb = e.n_chars[l] - 1;
    const uint8_t* __restrict__ given = e.given + e.char_offsets[l] + 1;
    uint8_t* __restrict__ bnd = e.boundaries + e.bound_offsets[l];
    for (uint32_t j = lane; j < nb; j += 32) {
        const uint8_t c = given[j];
        if (c != kPaUnknown) bnd[j] = c;
    }
}

// One warp per line, 128 bytes per step, as part_line: the automaton's state before every byte from the same scan, then
// every byte's tag class (pa_tag_class).  Each lane walks its bytes from the max of the carried walk and the lanes before
// it (pa_tag_max); at every marker after a character, and at the line's end, the character's region is written.  Lines
// with an error (the call fails on them) still write only inside their characters.
__global__ void __launch_bounds__(kPaThreads) k_part_tags(PartTagArgs e) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t l = uint64_t(blockIdx.x) * kWarps + warp;
    if (l >= e.n_sent) return;
    const uint64_t o0 = e.offsets[l], o1 = e.offsets[l + 1];
    const uint64_t a0 = o0 & ~3ull;
    const uint32_t b0 = uint32_t(o0 - a0), b1 = uint32_t(o1 - a0) - e.trims[l];
    if (b1 <= b0) return;
    const uint8_t* __restrict__ base = e.text + a0;
    uint2* __restrict__ regions = e.regions + e.char_offsets[l];
    uint32_t c_state = kPaChar, chars = 0;
    PaTagRun carry;
    for (uint32_t w0 = 0; w0 < b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t lo = 0, in80 = 0;
        if (addr < b1) {
            lo = __ldg(reinterpret_cast<const uint32_t*>(base + addr));
            in80 = inside80(addr, b0, b1);
        }
        const uint32_t m = pa_word_map(lo, in80);
        uint32_t incl = m;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl = pa_compose(o, incl);
        }
        uint32_t x = __shfl_up_sync(kFull, incl, 1);
        if (lane == 0) x = kPaIdentity;
        const uint32_t s0 = pa_apply(x, c_state);
        // the lane's own walk from nothing: its character starts and its maxima
        uint32_t s = s0, st80 = 0;
        PaTagRun own;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (!(in80 & bit)) continue;
            const uint32_t b = (lo >> (8 * j)) & 0xFFu;
            const PaByte pb = pa_byte(s, b);
            if (pb.start) st80 |= bit;
            pa_tag_step(own, pb.start, pa_tag_class(s, b), addr + uint32_t(j) - b0);
            s = pb.next;
        }
        const uint32_t nst = __popc(st80);
        const uint32_t st_incl = warp_incl_scan_u32(nst, lane);
        // the walk before the lane: max over the carry and the lanes before it
        PaTagRun run = own;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            PaTagRun o;
            o.start = __shfl_up_sync(kFull, run.start, d);
            o.open = __shfl_up_sync(kFull, run.open, d);
            o.content = __shfl_up_sync(kFull, run.content, d);
            if (lane >= d) pa_tag_max(run, o);
        }
        PaTagRun before;
        before.start = __shfl_up_sync(kFull, run.start, 1);
        before.open = __shfl_up_sync(kFull, run.open, 1);
        before.content = __shfl_up_sync(kFull, run.content, 1);
        if (lane == 0) before = PaTagRun();
        pa_tag_max(before, carry);
        // the walk again, writing the region of the character before every marker
        uint32_t k = chars + st_incl - nst;  // characters of the line before this byte
        s = s0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t bit = 0x80u << (8 * j);
            if (!(in80 & bit)) continue;
            const uint32_t b = (lo >> (8 * j)) & 0xFFu;
            const uint32_t cls = pa_tag_class(s, b);
            if (st80 & bit) ++k;
            pa_tag_step(before, (st80 & bit) != 0, cls, addr + uint32_t(j) - b0);
            if (cls == kPaTagClose) {
                uint32_t first;
                const uint32_t len = pa_tag_region(before, first);
                regions[k - 1] = make_uint2(uint32_t(a0) + b0 + first, len);
            }
            s = pa_apply(pa_byte_map(b), s);
        }
        c_state = pa_apply(__shfl_sync(kFull, incl, 31), c_state);
        chars += __shfl_sync(kFull, st_incl, 31);
        PaTagRun step;
        step.start = __shfl_sync(kFull, run.start, 31);
        step.open = __shfl_sync(kFull, run.open, 31);
        step.content = __shfl_sync(kFull, run.content, 31);
        pa_tag_max(carry, step);
    }
    // the last character: its region ends with the line
    if (lane == 0 && chars > 0 && c_state != kPaChar && c_state != kPaErr) {
        uint32_t first;
        const uint32_t len = pa_tag_region(carry, first);
        regions[chars - 1] = make_uint2(uint32_t(a0) + b0 + first, len);
    }
}

}  // namespace

cudaError_t launch_part_tags(const PartTagArgs& e, cudaStream_t stream) {
    if (e.n_sent == 0) return cudaSuccess;
    k_part_tags<<<unsigned((e.n_sent + kWarps - 1) / kWarps), kPaThreads, 0, stream>>>(e);
    return cudaGetLastError();
}

cudaError_t launch_part_parse(const PartArgs& e, cudaStream_t stream) {
    if (e.n_sent == 0) return cudaSuccess;
    const uint64_t ngroups = (e.n_sent + kGroup - 1) / kGroup;
    // look-back state words + the ticket that follows them
    cudaError_t err = cudaMemsetAsync(e.state, 0, 8 * (ngroups + 1), stream);
    if (err != cudaSuccess) return err;
    k_part_parse<<<unsigned(ngroups), kPaThreads, 0, stream>>>(e, ngroups);
    return cudaGetLastError();
}

cudaError_t launch_part_apply(const PartArgs& e, cudaStream_t stream) {
    if (e.n_sent == 0) return cudaSuccess;
    k_part_apply<<<unsigned((e.n_sent + kWarps - 1) / kWarps), kPaThreads, 0, stream>>>(e);
    return cudaGetLastError();
}

}  // namespace vpt
