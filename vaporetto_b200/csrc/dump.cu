// The predict CLI's --scores / --tag-scores dumps of the lines path (dump.hpp has the per-line code and the contract).
// Behind the token-line writer of a chunk, three kernels, one thread per line:
//   k_dump_size    every line's token line bytes (token_line_len) and dump bytes (dump_line with the counting sink),
//                  their prefixes inside a block of kDumpBlock lines and the block's totals
//   k_dump_scan    one block: the prefixes of the block totals; the chunk's totals to pinned host words
//   k_dump_write   line l at (its token line's offset) - l + (its dump prefix): its token line without the '\n', then
//                  dump_line's bytes (the '\n' included)
// The host reads the totals between the scan and the writer, to size the output exactly.
#include <cuda_runtime.h>

#include "dump.hpp"
#include "kernels_common.cuh"

namespace vpt {

// inclusive prefix of (x, y) over a warp
__device__ __forceinline__ void warp_scan2(uint64_t& x, uint64_t& y, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t ox = __shfl_up_sync(kFull, x, d), oy = __shfl_up_sync(kFull, y, d);
        if (lane >= d) { x += ox; y += oy; }
    }
}

__global__ void __launch_bounds__(kDumpBlock) k_dump_size(DumpArgs a) {
    __shared__ uint64_t s_w[2][kDumpBlock / 32];
    const uint64_t l = uint64_t(blockIdx.x) * kDumpBlock + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    DumpCount c;
    uint64_t tl = 0;
    if (l < a.n_sent) {
        dump_line(a, l, c);
        tl = token_line_len(a, l);
    }
    uint64_t incl = c.n, tincl = tl;
    warp_scan2(incl, tincl, lane);
    if (lane == 31) { s_w[0][warp] = incl; s_w[1][warp] = tincl; }
    __syncthreads();
    uint64_t base = 0, tot = 0, tbase = 0, ttot = 0;
#pragma unroll
    for (int w = 0; w < kDumpBlock / 32; ++w) {
        if (w < warp) { base += s_w[0][w]; tbase += s_w[1][w]; }
        tot += s_w[0][w];
        ttot += s_w[1][w];
    }
    if (l < a.n_sent) {
        a.size[l] = base + incl - c.n;
        a.tl_len[l] = tl;
        a.tl_off[l] = tbase + tincl - tl;
    }
    if (threadIdx.x == 0) { a.blk[2 * blockIdx.x] = tot; a.blk[2 * blockIdx.x + 1] = ttot; }
}

__global__ void __launch_bounds__(1024) k_dump_scan(DumpArgs a, uint64_t nblk) {
    __shared__ uint64_t s_w[2][32];
    __shared__ uint64_t s_carry[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 2) s_carry[threadIdx.x] = 0;
    __syncthreads();
    for (uint64_t lo = 0; lo < nblk; lo += 1024) {
        const uint64_t i = lo + threadIdx.x;
        const uint64_t v = i < nblk ? a.blk[2 * i] : 0, tv = i < nblk ? a.blk[2 * i + 1] : 0;
        uint64_t incl = v, tincl = tv;
        warp_scan2(incl, tincl, lane);
        if (lane == 31) { s_w[0][warp] = incl; s_w[1][warp] = tincl; }
        __syncthreads();
        uint64_t base = s_carry[0], tbase = s_carry[1];
        for (int w = 0; w < warp; ++w) { base += s_w[0][w]; tbase += s_w[1][w]; }
        if (i < nblk) { a.blk[2 * i] = base + incl - v; a.blk[2 * i + 1] = tbase + tincl - tv; }
        __syncthreads();
        if (threadIdx.x == 1023) { s_carry[0] = base + incl; s_carry[1] = tbase + tincl; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { a.total_host[0] = s_carry[0]; a.total_host[1] = s_carry[1]; }
}

__global__ void __launch_bounds__(kDumpBlock) k_dump_write(DumpArgs a) {
    const uint64_t l = uint64_t(blockIdx.x) * kDumpBlock + threadIdx.x;
    if (l >= a.n_sent) return;
    const uint64_t b = l / kDumpBlock;
    const uint64_t lo = a.blk[2 * b + 1] + a.tl_off[l], hi = lo + a.tl_len[l] - 1;  // the token line without its '\n'
    // (dump_line writes the token line's '\n' itself, where the mode puts it: l newlines come before line l)
    DumpWrite w{a.out + lo - l + a.blk[2 * b] + a.size[l]};
    for (uint64_t i = lo; i < hi; ++i) w.byte(a.tok_lines[i]);
    dump_line(a, l, w);
}

cudaError_t launch_dump_size(const DumpArgs& a, cudaStream_t stream) {
    const uint64_t nblk = (a.n_sent + kDumpBlock - 1) / kDumpBlock;
    if (nblk == 0) return cudaSuccess;
    k_dump_size<<<unsigned(nblk), kDumpBlock, 0, stream>>>(a);
    k_dump_scan<<<1, 1024, 0, stream>>>(a, nblk);
    return cudaGetLastError();
}

cudaError_t launch_dump_write(const DumpArgs& a, cudaStream_t stream) {
    const uint64_t nblk = (a.n_sent + kDumpBlock - 1) / kDumpBlock;
    if (nblk == 0) return cudaSuccess;
    k_dump_write<<<unsigned(nblk), kDumpBlock, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace vpt
