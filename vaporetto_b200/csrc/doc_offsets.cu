// doc_offsets.cu — the caller's document offsets of vpt_token_spans_dev, read on the device (the host never sees them):
//
//   k_doc_max      largest key of every block of kDocThreads offsets
//   k_doc_scan     exclusive prefix maximum of the block maxima (one block)
//   k_doc_offsets  rebased u64 offsets (the prefix maximum + shift) and the flag of every document out of range
//   k_doc_status   after the scoring pass: status VPT_SENT_BAD_RANGE for every flagged document, before the span kernels
//                  count its tokens (a status other than 0 gives 0 tokens)
// The per-offset arithmetic is doc_offsets.hpp (also compiled for the host by tests/native/doc_offsets_test.cpp).
#include <cuda_runtime.h>

#include <cstdint>

#include "device_model.hpp"
#include "doc_offsets.hpp"

namespace vpt {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kDocThreads = 256;
constexpr int kDocWarps = kDocThreads / 32;
constexpr int32_t kSentBadRange = 4;  // VPT_SENT_BAD_RANGE

__device__ __forceinline__ int64_t doc_offset(const DocArgs& a, uint64_t i) {
    return a.wide ? static_cast<const int64_t*>(a.offsets)[i] : int64_t(static_cast<const int32_t*>(a.offsets)[i]);
}

__device__ __forceinline__ uint64_t warp_incl_max(uint64_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v = max(v, o);
    }
    return v;
}

__global__ void __launch_bounds__(kDocThreads) k_doc_max(DocArgs a) {
    __shared__ uint64_t s_w[kDocWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t i = uint64_t(blockIdx.x) * kDocThreads + threadIdx.x;
    uint64_t v = i <= a.n_docs ? doc_key(doc_offset(a, i), a.n_bytes) : 0u;
    v = warp_incl_max(v, lane);
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t m = 0;
#pragma unroll
        for (int w = 0; w < kDocWarps; ++w) m = max(m, s_w[w]);
        a.blk[blockIdx.x] = m;
    }
}

// exclusive prefix maximum of the block maxima, 1024 per round
__global__ void __launch_bounds__(1024) k_doc_scan(DocArgs a) {
    __shared__ uint64_t s_w[32];
    __shared__ uint64_t s_carry;
    const uint64_t nblk = (a.n_docs + 1 + kDocThreads - 1) / kDocThreads;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint64_t lo = 0; lo < nblk; lo += 1024) {
        const uint64_t i = lo + threadIdx.x;
        const uint64_t v = i < nblk ? a.blk[i] : 0u;
        const uint64_t incl = warp_incl_max(v, lane);
        const uint64_t up = __shfl_up_sync(kFull, incl, 1);  // (every lane takes part in the shuffle)
        const uint64_t excl_w = max(s_carry, lane ? up : 0u);
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        uint64_t base = excl_w;
        for (int w = 0; w < warp; ++w) base = max(base, s_w[w]);
        if (i < nblk) a.blk[i] = base;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = max(base, v);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kDocThreads) k_doc_offsets(DocArgs a) {
    __shared__ uint64_t s_w[kDocWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t i = uint64_t(blockIdx.x) * kDocThreads + threadIdx.x;
    const int64_t o = i <= a.n_docs ? doc_offset(a, i) : 0;
    const uint64_t c = i <= a.n_docs ? doc_key(o, a.n_bytes) : 0u;
    const uint64_t incl_w = warp_incl_max(c, lane);
    const uint64_t up = __shfl_up_sync(kFull, incl_w, 1);  // (every lane takes part in the shuffle)
    const uint64_t excl_w = lane ? up : 0u;
    if (lane == 31) s_w[warp] = incl_w;
    __syncthreads();
    uint64_t before = a.blk[blockIdx.x];  // largest key in front of this thread's, of earlier blocks / warps
    for (int w = 0; w < warp; ++w) before = max(before, s_w[w]);
    before = max(before, excl_w);
    if (i <= a.n_docs) a.out[i] = max(before, c) + a.shift;
    if (i < a.n_docs) a.bad[i] = doc_bad(o, doc_offset(a, i + 1), a.n_bytes, before) ? 1 : 0;
}

__global__ void __launch_bounds__(kDocThreads) k_doc_status(DocArgs a, int32_t* status) {
    const uint64_t d = uint64_t(blockIdx.x) * kDocThreads + threadIdx.x;
    if (d < a.n_docs && a.bad[d]) status[d] = kSentBadRange;
}

}  // namespace

uint64_t doc_offsets_blocks(uint64_t n_docs) { return (n_docs + 1 + kDocThreads - 1) / kDocThreads; }

cudaError_t launch_doc_offsets(const DocArgs& a, cudaStream_t stream) {
    const unsigned nblk = unsigned(doc_offsets_blocks(a.n_docs));
    k_doc_max<<<nblk, kDocThreads, 0, stream>>>(a);
    k_doc_scan<<<1, 1024, 0, stream>>>(a);
    k_doc_offsets<<<nblk, kDocThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_doc_status(const DocArgs& a, int32_t* status, cudaStream_t stream) {
    if (a.n_docs == 0) return cudaSuccess;
    k_doc_status<<<unsigned((a.n_docs + kDocThreads - 1) / kDocThreads), kDocThreads, 0, stream>>>(a, status);
    return cudaGetLastError();
}

}  // namespace vpt
