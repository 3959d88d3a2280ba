// spans.cu — documents to token byte spans on the device: the part of vaporetto_tantivy's `token_stream`
// (vaporetto_tantivy/src/lib.rs:157-199) that follows `predict`, for a batch of documents (vpt_token_spans).
//
//   k_split_linebreaks  SplitLinebreaksFilter (vaporetto_rules/src/sentence_filters/split_linebreaks.rs:9-37): the
//                       boundary on either side of every '\r' / '\n' becomes WordBoundary.  It runs after scoring and
//                       before the --wsconst filters, which only clear boundaries (lib.rs:69-85 puts it first).
//   k_span_count        tokens per document (boundaries set + 1), one warp per document; block prefix
//   k_span_scan         prefix of the block totals (one block), the chunk's total to pinned host memory
//   k_span_base         first token record of every document
//   k_token_ends        `boundary_pos` (lib.rs:179-188): the byte offset, from the document's start, of every token's
//                       exclusive end; one warp per document, 128-byte windows, token ranks by a warp scan carried
//                       from window to window.
// The window arithmetic is spans.hpp (also compiled for the host by tests/native/spans_test.cpp).
#include <cuda_runtime.h>

#include <cstdint>

#include "device_model.hpp"
#include "spans.hpp"

namespace vpt {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kSpanThreads = 256;
constexpr int kSpanWarps = kSpanThreads / 32;
static_assert(kSpanDocs == kSpanThreads, "k_span_count: one thread per document in the block prefix");

__device__ __forceinline__ uint32_t span_warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

// the document's bytes in window coordinates: [b0, b1) from the 4-byte aligned address a0
struct DocWindow {
    const uint8_t* base;
    uint32_t b0, b1;
};
__device__ __forceinline__ DocWindow doc_window(const SpanArgs& a, uint64_t s) {
    const uint64_t o0 = a.offsets[s];
    const uint64_t a0 = o0 & ~3ull;
    return DocWindow{a.text + a0, uint32_t(o0 - a0), uint32_t(a.offsets[s + 1] - a0)};
}

__global__ void __launch_bounds__(kSpanThreads) k_split_linebreaks(SpanArgs a) {
    const int lane = threadIdx.x & 31;
    const uint64_t s = uint64_t(blockIdx.x) * kSpanWarps + (threadIdx.x >> 5);
    if (s >= a.n_sent || a.status[s] != 0) return;
    const uint32_t n = a.n_chars[s];
    if (n < 2) return;
    const DocWindow d = doc_window(a, s);
    uint8_t* __restrict__ bnd = a.boundaries + a.bound_offsets[s];
    uint32_t chars = 0;  // characters before this window
    for (uint32_t w0 = 0; w0 < d.b1; w0 += 128) {
        const uint32_t addr = w0 + 4u * uint32_t(lane);
        uint32_t w = 0, in80 = 0;
        if (addr < d.b1) {
            w = __ldg(reinterpret_cast<const uint32_t*>(d.base + addr));
            in80 = span_inside80(addr, d.b0, d.b1);
        }
        const uint32_t st80 = span_starts80(w, in80);
        const uint32_t nst = span_popc(st80);
        const uint32_t incl = span_warp_incl_scan(nst, lane);
        const uint32_t lb80 = span_linebreaks80(w, in80);
        if (lb80) span_set_linebreaks(st80, lb80, chars + incl - nst, n, bnd);
        chars += __shfl_sync(kFull, incl, 31);
    }
}

__global__ void __launch_bounds__(kSpanThreads) k_span_count(SpanArgs a) {
    __shared__ uint32_t s_ntok[kSpanDocs];
    __shared__ uint32_t s_w[kSpanWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t gbase = uint64_t(blockIdx.x) * kSpanDocs;
    const int nd = int(min(uint64_t(kSpanDocs), a.n_sent - gbase));
    for (int i = warp; i < nd; i += kSpanWarps) {
        const uint64_t s = gbase + i;
        const int32_t st = a.status[s];
        const uint32_t n = a.n_chars[s];
        uint32_t ntok = 0;
        if (st == 0 && n > 0) {
            // boundaries [bo, bo + n - 1), bytes 0 / 1, read as aligned words
            const uint64_t bo = a.bound_offsets[s];
            const uint64_t p0 = bo & ~3ull;
            const uint32_t b0 = uint32_t(bo - p0), b1 = b0 + (n - 1);
            const uint8_t* __restrict__ base = a.boundaries + p0;
            uint32_t cnt = 0;
            for (uint32_t addr = 4u * uint32_t(lane); addr < b1; addr += 128) {
                const uint32_t w = *reinterpret_cast<const uint32_t*>(base + addr);
                cnt += span_popc(w & (span_inside80(addr, b0, b1) >> 7));
            }
            ntok = __reduce_add_sync(kFull, cnt) + 1;
        }
        if (lane == 0) {
            a.status8[s] = uint8_t(st);
            a.n_tokens[s] = ntok;
            s_ntok[i] = ntok;
        }
    }
    __syncthreads();
    const uint32_t v = int(threadIdx.x) < nd ? s_ntok[threadIdx.x] : 0u;
    const uint32_t incl = span_warp_incl_scan(v, lane);
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kSpanWarps; ++w) {
        if (w < warp) base += s_w[w];
        tot += s_w[w];
    }
    if (int(threadIdx.x) < nd) a.tok_local[gbase + threadIdx.x] = base + incl - v;
    if (threadIdx.x == 0) a.tok_blk[blockIdx.x] = tot;
}

// exclusive prefix of the block totals (one block, 1024 totals per round); the grand total behind them
__global__ void __launch_bounds__(1024) k_span_scan(SpanArgs a) {
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const uint64_t nblk = (a.n_sent + kSpanDocs - 1) / kSpanDocs;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint64_t lo = 0; lo < nblk; lo += 1024) {
        const uint64_t i = lo + threadIdx.x;
        const uint64_t v = i < nblk ? a.tok_blk[i] : 0;
        uint64_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t o = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl += o;
        }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        uint64_t base = s_carry;
        for (int w = 0; w < warp; ++w) base += s_w[w];
        if (i < nblk) a.tok_blk[i] = base + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = base + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        a.tok_base[a.n_sent] = s_carry;
        if (a.tok_total_host) *a.tok_total_host = s_carry;
    }
}

__global__ void __launch_bounds__(kSpanThreads) k_span_base(SpanArgs a) {
    const uint64_t s = uint64_t(blockIdx.x) * kSpanThreads + threadIdx.x;
    if (s < a.n_sent) a.tok_base[s] = a.tok_blk[s / kSpanDocs] + a.tok_local[s];
}

__global__ void __launch_bounds__(kSpanThreads) k_token_ends(SpanArgs a) {
    const int lane = threadIdx.x & 31;
    const uint64_t s = uint64_t(blockIdx.x) * kSpanWarps + (threadIdx.x >> 5);
    if (s >= a.n_sent || a.status[s] != 0) return;
    const uint32_t n = a.n_chars[s];
    if (n == 0) return;
    const DocWindow d = doc_window(a, s);
    uint32_t* __restrict__ ends = a.token_ends + a.tok_base[s];
    if (n >= 2) {
        const uint8_t* __restrict__ bnd = a.boundaries + a.bound_offsets[s];
        uint32_t chars = 0, rank = 0;  // characters and token starts before this window
        for (uint32_t w0 = 0; w0 < d.b1; w0 += 128) {
            const uint32_t addr = w0 + 4u * uint32_t(lane);
            uint32_t w = 0, in80 = 0;
            if (addr < d.b1) {
                w = __ldg(reinterpret_cast<const uint32_t*>(d.base + addr));
                in80 = span_inside80(addr, d.b0, d.b1);
            }
            const uint32_t st80 = span_starts80(w, in80);
            const uint32_t nst = span_popc(st80);
            const uint32_t incl = span_warp_incl_scan(nst, lane);
            const uint32_t ts80 = st80 ? span_token_starts80(st80, chars + incl - nst, bnd) : 0u;
            const uint32_t nts = span_popc(ts80);
            const uint32_t tincl = span_warp_incl_scan(nts, lane);
            if (ts80) span_store_ends(ts80, addr, d.b0, ends + rank + tincl - nts);
            chars += __shfl_sync(kFull, incl, 31);
            rank += __shfl_sync(kFull, tincl, 31);
        }
        // (rank + 1 == the document's token count)
        if (lane == 0) ends[rank] = d.b1 - d.b0;
    } else if (lane == 0) {
        ends[0] = d.b1 - d.b0;
    }
}

}  // namespace

cudaError_t launch_split_linebreaks(const SpanArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    k_split_linebreaks<<<unsigned((a.n_sent + kSpanWarps - 1) / kSpanWarps), kSpanThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_span_count(const SpanArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    const uint64_t nblk = (a.n_sent + kSpanDocs - 1) / kSpanDocs;
    k_span_count<<<unsigned(nblk), kSpanThreads, 0, stream>>>(a);
    k_span_scan<<<1, 1024, 0, stream>>>(a);
    k_span_base<<<unsigned((a.n_sent + kSpanThreads - 1) / kSpanThreads), kSpanThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_token_ends(const SpanArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    k_token_ends<<<unsigned((a.n_sent + kSpanWarps - 1) / kSpanWarps), kSpanThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace vpt
