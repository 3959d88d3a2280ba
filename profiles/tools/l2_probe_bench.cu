// l2_probe_bench — what an H100 delivers for the access pattern of the node-table probes: random, independent
// 32-byte records (two 128-bit loads each, as load_record in vaporetto_b200/csrc/kernels_common.cuh) out of a table
// that stays resident in L2 (or does not), and random single-byte reads from a shared-memory seed table.  Standalone;
// build + run:
//   mkdir -p build && nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/l2_probe_bench profiles/tools/l2_probe_bench.cu
//   build/l2_probe_bench > build/l2_probe_bench.jsonl
//   build/l2_probe_bench --probe-seq build/probe_slots.u32   (k_fused's own probe slots, from probe_slots.py: only
//                                                             the `probe_seq` record_load test)
// Output: one JSON object per line {"test": ..., "table_mb": ..., "ilp": ..., "gprobes_s": ..., "gbs": ...}.
// The numbers give the peak of the scoring kernel's second roofline (bench.py: roofline_l1_lines).  "record_load" is
// the test with load_record's own instructions and k_fused's geometry; the older "record32" kernels and the 32- and
// 128-byte "variant" kernels read only some words of a record, and ptxas narrows those loads to 32-bit ones.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e_ = (x);                                                          \
        if (e_ != cudaSuccess) {                                                       \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); \
            exit(1);                                                                   \
        }                                                                              \
    } while (0)

struct Rec32 {
    uint32_t v[8];
};

__device__ __forceinline__ Rec32 load_record(const void* base, uint32_t slot) {
    Rec32 r;
    const char* p = static_cast<const char*>(base) + (size_t(slot) << 5);
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4+16];" : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]) : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t mix(uint32_t x) {
    x *= 0x9E3779B1u;
    x ^= x >> 15;
    x *= 0x85EBCA77u;
    x ^= x >> 13;
    return x;
}

// kIlp independent random record loads in flight per thread, `iters` rounds; kDependent chains the next index on
// the loaded data (latency-bound variant: one probe depends on the previous, as the 3->2->1 fallback chain does).
template <int kIlp, bool kDependent>
__global__ void __launch_bounds__(1024) k_probe(const void* table, uint32_t nslots, int iters, uint32_t* sink) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t acc = 0;
    uint32_t idx[kIlp];
#pragma unroll
    for (int j = 0; j < kIlp; ++j) idx[j] = mix(tid * kIlp + j + 1);
    for (int i = 0; i < iters; ++i) {
        Rec32 r[kIlp];
#pragma unroll
        for (int j = 0; j < kIlp; ++j) r[j] = load_record(table, uint32_t((uint64_t(idx[j]) * nslots) >> 32));
#pragma unroll
        for (int j = 0; j < kIlp; ++j) {
            const uint32_t s = r[j].v[0] ^ r[j].v[3] ^ r[j].v[7];
            acc += s;
            idx[j] = mix(idx[j] + (kDependent ? s : 0u) + 0x632BE5ABu);
        }
    }
    if (acc == 0x12345678u) *sink = acc;
}

// Variants that tell WHAT the limit is: kBytes per lane (8 / 16 / 32 / 128) and kShare lanes per 128-byte line
// (1 = every lane its own random line, 2 / 4 = neighbouring lanes read different records of the same line).
template <int kBytes, int kShare>
__global__ void __launch_bounds__(1024) k_probe_var(const void* table, uint32_t nlines, int iters, uint32_t* sink) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t acc = 0;
    uint32_t idx = mix((tid / kShare) + 1);
    const uint32_t sub = (tid % kShare) * (128 / kShare);
    for (int i = 0; i < iters; ++i) {
        const uint32_t line = uint32_t((uint64_t(idx) * nlines) >> 32);
        const char* p = static_cast<const char*>(table) + (size_t(line) << 7) + sub;
        uint32_t s;
        if (kBytes == 8) {
            uint32_t a, b;
            asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
            s = a ^ b;
        } else if (kBytes == 16) {
            uint32_t a, b, c, d;
            asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "l"(p));
            s = a ^ b ^ c ^ d;
        } else if (kBytes == 32) {
            const Rec32 r = load_record(p, 0);
            s = r.v[0] ^ r.v[3] ^ r.v[7];
        } else {
            const Rec32 r0 = load_record(p, 0), r1 = load_record(p, 1), r2 = load_record(p, 2), r3 = load_record(p, 3);
            s = r0.v[0] ^ r1.v[3] ^ r2.v[7] ^ r3.v[1];
        }
        acc += s;
        idx = mix(idx + 0x632BE5ABu);
    }
    if (acc == 0x12345678u) *sink = acc;
}

// ---- record load forms (load_record in vaporetto_b200/csrc/kernels_common.cuh), at k_fused's geometry ---------------
// na2     two v4 loads, L1::no_allocate + evict-last L2 hint (the kernel's load): two L2 sector requests per record
// l1a2    the same two loads allocating in L1 (the second may hit the line the first brought in)
// l1a2ef  as l1a2 with L1::evict_first
// pair    lanes 2k / 2k+1 read the two halves of one record in one instruction (one sector request per record), four
//         shuffles give each lane the half its partner read
// one16   one v4 load per record: the one-request lower bound (not a record format)
enum Mode { kNa2, kL1a2, kL1a2ef, kPair, kOne16 };

__device__ __forceinline__ uint64_t pol_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t pol_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

template <int kMode>
__device__ __forceinline__ void ld16(const char* p, uint64_t pol, uint32_t (&v)[4]) {
    if (kMode == kL1a2)
        asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p), "l"(pol));
    else if (kMode == kL1a2ef)
        asm volatile("ld.global.nc.L1::evict_first.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p), "l"(pol));
    else
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p), "l"(pol));
}

// the record of `slot`, loaded in form kMode (called by the whole warp for kPair)
template <int kMode>
__device__ __forceinline__ Rec32 load_mode(const char* table, uint32_t slot, uint32_t lane, uint64_t pol) {
    Rec32 r;
    uint32_t a[4], b[4];
    if (kMode == kPair) {
        const uint32_t odd = lane & 1u;
        const uint32_t se = __shfl_sync(0xFFFFFFFFu, slot, lane & ~1u), so = __shfl_sync(0xFFFFFFFFu, slot, lane | 1u);
        // both lanes of a pair read the even lane's record, then the odd lane's; each keeps half 0 of its own record
        ld16<kNa2>(table + (size_t(se) << 5) + 16u * odd, pol, a);
        ld16<kNa2>(table + (size_t(so) << 5) + 16u * (odd ^ 1u), pol, b);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t keep = odd ? b[j] : a[j], send = odd ? a[j] : b[j];
            r.v[j] = keep;
            r.v[4 + j] = __shfl_xor_sync(0xFFFFFFFFu, send, 1);
        }
    } else if (kMode == kOne16) {
        ld16<kNa2>(table + (size_t(slot) << 5), pol, a);
#pragma unroll
        for (int j = 0; j < 4; ++j) { r.v[j] = a[j]; r.v[4 + j] = a[j] >> 1; }
    } else {
        ld16<kMode>(table + (size_t(slot) << 5), pol, a);
        ld16<kMode>(table + (size_t(slot) << 5) + 16, pol, b);
#pragma unroll
        for (int j = 0; j < 4; ++j) { r.v[j] = a[j]; r.v[4 + j] = b[j]; }
    }
    return r;
}

// One 1024-thread CTA per SM with k_fused's shared-memory footprint (so L1 is as small as the kernel's).  With kStream,
// every fourth warp streams instead of probing: 16 B per lane and iteration read with an evict-first hint (the text's
// bulk copy) and 16 B written with a streaming store (the outputs), through buffers larger than L2 -- about 5 B per
// probe, k_fused's ratio of streamed bytes to record probes.  Without it those warps idle, so the probe count is the same.
template <int kMode, bool kStream>
__global__ void __launch_bounds__(1024, 1) k_probe_mode(const char* table, uint32_t nslots, int iters, const uint4* sin,
                                                         uint4* sout, size_t nvec, uint32_t* sink) {
    extern __shared__ uint8_t s_pad[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t acc = 0;
    if ((warp & 3) == 3) {
        if (!kStream) return;
        const uint64_t pf = pol_first();
        const size_t sw = size_t(blockIdx.x) * 8 + (warp >> 2), nsw = size_t(gridDim.x) * 8;
        for (int i = 0; i < iters; ++i) {
            const size_t k = ((size_t(i) * nsw + sw) * 32 + lane) % nvec;
            uint32_t v[4];
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                         : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(sin + k), "l"(pf));
            __stcs(sout + k, make_uint4(v[0] + i, v[1], v[2], v[3]));
        }
        return;
    }
    const uint64_t pol = pol_last();
    uint32_t idx[2] = {mix(tid * 2 + 1), mix(tid * 2 + 2)};
    for (int i = 0; i < iters; ++i) {
        Rec32 r[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) r[j] = load_mode<kMode>(table, uint32_t((uint64_t(idx[j]) * nslots) >> 32), lane, pol);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            // (every word: ptxas narrows a vector load whose other words are unused)
#pragma unroll
            for (int w = 0; w < 8; ++w) acc += r[j].v[w] << w;
            idx[j] = mix(idx[j] + 0x632BE5ABu);
        }
    }
    if (acc == 0x12345678u) *sink = acc + s_pad[0];
}

// As k_probe_mode<kL1a2, true> (load_record's form: allocating in L1, evict-last in L2), but the slots are k_fused's
// own probe sequence on the config-2 text (profiles/tools/probe_slots.py) instead of uniformly random ones.  Probing
// lane g takes entries g, g + P, g + 2P, ... (P probing lanes in the grid); the entry of the next round is loaded one
// round ahead, without allocating in L1, so that only the records compete for the L1 the shared memory leaves.
__global__ void __launch_bounds__(1024, 1) k_probe_seq(const char* table, const uint32_t* seq, uint32_t nseq, int iters,
                                                        const uint4* sin, uint4* sout, size_t nvec, uint32_t* sink) {
    extern __shared__ uint8_t s_pad[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t acc = 0;
    if ((warp & 3) == 3) {
        const uint64_t pf = pol_first();
        const size_t sw = size_t(blockIdx.x) * 8 + (warp >> 2), nsw = size_t(gridDim.x) * 8;
        for (int i = 0; i < iters; ++i) {
            const size_t k = ((size_t(i) * nsw + sw) * 32 + lane) % nvec;
            uint32_t v[4];
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                         : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(sin + k), "l"(pf));
            __stcs(sout + k, make_uint4(v[0] + i, v[1], v[2], v[3]));
        }
        return;
    }
    const uint64_t pol = pol_last();
    const uint64_t nprobe = uint64_t(gridDim.x) * 768;  // probing lanes in the grid
    const uint64_t g = uint64_t(blockIdx.x) * 768 + (warp - (warp >> 2)) * 32 + lane;
    auto next = [&](uint64_t e) {
        uint32_t s;
        asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(s) : "l"(seq + (e % nseq)));
        return s;
    };
    uint32_t sl[2] = {next(g), next(g + nprobe)};
    for (int i = 0; i < iters; ++i) {
        const uint64_t e = (uint64_t(i + 1) * 2) * nprobe + g;
        const uint32_t n0 = next(e), n1 = next(e + nprobe);
        Rec32 r[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) r[j] = load_mode<kL1a2>(table, sl[j], lane, pol);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int w = 0; w < 8; ++w) acc += r[j].v[w] << w;
        sl[0] = n0;
        sl[1] = n1;
    }
    if (acc == 0x12345678u) *sink = acc + s_pad[0];
}

// random byte reads from a 37 KB shared-memory table (the perfect-hash seeds): LDS.U8 with random bank pattern
__global__ void __launch_bounds__(1024) k_smem_seed(int iters, uint32_t* sink) {
    __shared__ uint8_t s_seed[37632];
    for (int i = threadIdx.x; i < 37632; i += blockDim.x) s_seed[i] = uint8_t(i * 7);
    __syncthreads();
    uint32_t x = mix(blockIdx.x * blockDim.x + threadIdx.x + 1), acc = 0;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            acc += s_seed[(uint64_t(x) * 37632u) >> 32];
            x = x * 0x9E3779B1u + 0x7F4A7C15u;
        }
    }
    if (acc == 0x12345678u) *sink = acc;
}

// pure issue-rate reference: dependent-free integer work (IMAD + LOP3 mix), 8 chains per thread
__global__ void __launch_bounds__(1024) k_issue(int iters, uint32_t* sink) {
    uint32_t a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = threadIdx.x + j;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            a[j] = a[j] * 0x9E3779B1u + 12345u;  // IMAD
            a[j] ^= a[j] >> 7;                   // SHF + LOP3
        }
    }
    uint32_t acc = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc ^= a[j];
    if (acc == 0x12345678u) *sink = acc;
}

template <typename F>
static float time_ms(F&& launch, int reps) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    launch();
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    for (int r = 0; r < reps; ++r) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return ms / reps;
}

// k_fused's probe sequence (probe_slots.py's output) at four shared-memory footprints, one per H100 carve-out (228, 196,
// 164 and 132 KB), with the carve-out each needs: the ratio of the rates is what the L1 the smaller footprint leaves is
// worth to the probes.
static void probe_seq_test(const char* path, const char* table, uint32_t* sink, int n_sm) {
    FILE* f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "%s: cannot open\n", path); exit(1); }
    std::vector<uint32_t> h;
    uint32_t buf[4096];
    size_t got;
    while ((got = fread(buf, 4, 4096, f)) > 0) h.insert(h.end(), buf, buf + got);
    fclose(f);
    uint32_t* seq;
    CK(cudaMalloc(&seq, h.size() * 4));
    CK(cudaMemcpy(seq, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    const size_t stream_bytes = size_t(64) << 20;
    uint4 *sin, *sout;
    CK(cudaMalloc(&sin, stream_bytes));
    CK(cudaMalloc(&sout, stream_bytes));
    CK(cudaMemset(sin, 0x11, stream_bytes));
    int smem_sm = 0;
    CK(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, 0));
    const int iters = 256;
    const double probes = double(n_sm) * 768 * iters * 2;
    const int smem_kb[] = {217, 177, 146, 130};
    for (int rep = 0; rep < 3; ++rep) {
        for (int kb : smem_kb) {
            const int smem = kb * 1024;
            // the smallest carve-out that holds the CTA's shared memory and the 1 KB the system reserves per CTA
            const int carve = std::min(100, ((smem + 1024) * 100 + smem_sm - 1) / smem_sm);
            CK(cudaFuncSetAttribute(k_probe_seq, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            CK(cudaFuncSetAttribute(k_probe_seq, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
            const float ms = time_ms([&] {
                k_probe_seq<<<n_sm, 1024, smem>>>(table, seq, uint32_t(h.size()), iters, sin, sout, stream_bytes / 16, sink);
            }, 20);
            printf("{\"test\": \"record_load\", \"mode\": \"probe_seq\", \"smem_kb\": %d, \"carveout\": %d, \"probes\": %zu, "
                   "\"ms\": %.4f, \"gprobes_s\": %.2f}\n",
                   kb, carve, h.size(), ms, probes / ms / 1e6);
            fflush(stdout);
        }
    }
    CK(cudaGetLastError());
    CK(cudaFree(seq));
    CK(cudaFree(sin));
    CK(cudaFree(sout));
}

int main(int argc, char** argv) {
    int dev = 0, n_sm = 0, clk_khz = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, dev));
    uint32_t* sink;
    CK(cudaMalloc(&sink, 4));
    const size_t max_bytes = size_t(1024) << 20;
    void* table;
    CK(cudaMalloc(&table, max_bytes));
    CK(cudaMemset(table, 0x5A, max_bytes));
    const int threads = 1024, blocks_per_sm = 2;
    const int grid = n_sm * blocks_per_sm;
    const double nthreads = double(grid) * threads;
    printf("{\"test\": \"device\", \"sms\": %d, \"clock_mhz\": %.0f}\n", n_sm, clk_khz / 1000.0);
    if (argc == 3 && std::string(argv[1]) == "--probe-seq") {
        probe_seq_test(argv[2], static_cast<const char*>(table), sink, n_sm);
        CK(cudaFree(table));
        CK(cudaFree(sink));
        return 0;
    }

    {   // what the limit is made of: bytes per lane and lanes per line, L2-resident 23 MB table and an L1-sized 64 KB one
        const int iters = 64;
        const double sizes_mb[] = {0.0625, 23};
        for (double mb : sizes_mb) {
            const uint32_t nlines = uint32_t(mb * 1048576.0 / 128.0);
            struct V { const char* name; float ms; } v[7];
            v[0] = {"8B_share1", time_ms([&] { k_probe_var<8, 1><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[1] = {"16B_share1", time_ms([&] { k_probe_var<16, 1><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[2] = {"32B_share1", time_ms([&] { k_probe_var<32, 1><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[3] = {"128B_share1", time_ms([&] { k_probe_var<128, 1><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[4] = {"32B_share2", time_ms([&] { k_probe_var<32, 2><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[5] = {"32B_share4", time_ms([&] { k_probe_var<32, 4><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            v[6] = {"8B_share4", time_ms([&] { k_probe_var<8, 4><<<grid, threads>>>(table, nlines, iters, sink); }, 5)};
            for (const V& x : v) {
                const double probes = nthreads * iters;
                printf("{\"test\": \"variant\", \"variant\": \"%s\", \"table_mb\": %.4f, \"ms\": %.4f, \"glane_loads_s\": %.2f, "
                       "\"per_clk_per_sm\": %.3f}\n",
                       x.name, mb, x.ms, probes / x.ms / 1e6, probes / x.ms / 1e3 / n_sm / clk_khz);
            }
            fflush(stdout);
        }
    }
    const double table_mb[] = {0.0625, 0.5, 2, 8, 23, 48, 96, 256, 1024};
    for (double mb : table_mb) {
        const uint32_t nslots = uint32_t(mb * 1048576.0 / 32.0);
        const int iters = 64;
        struct V { const char* name; int ilp; bool dep; float ms; } v[] = {
            {"ilp1", 1, false, 0}, {"ilp2", 2, false, 0}, {"ilp4", 4, false, 0}, {"dep1", 1, true, 0}, {"dep2", 2, true, 0}};
        v[0].ms = time_ms([&] { k_probe<1, false><<<grid, threads>>>(table, nslots, iters, sink); }, 5);
        v[1].ms = time_ms([&] { k_probe<2, false><<<grid, threads>>>(table, nslots, iters, sink); }, 5);
        v[2].ms = time_ms([&] { k_probe<4, false><<<grid, threads>>>(table, nslots, iters, sink); }, 5);
        v[3].ms = time_ms([&] { k_probe<1, true><<<grid, threads>>>(table, nslots, iters, sink); }, 5);
        v[4].ms = time_ms([&] { k_probe<2, true><<<grid, threads>>>(table, nslots, iters, sink); }, 5);
        for (const V& x : v) {
            const double probes = nthreads * iters * x.ilp;
            printf("{\"test\": \"record32\", \"variant\": \"%s\", \"table_mb\": %.0f, \"ms\": %.4f, \"gprobes_s\": %.2f, "
                   "\"gbs\": %.1f, \"per_clk_per_sm\": %.3f}\n",
                   x.name, mb, x.ms, probes / x.ms / 1e6, probes * 32.0 / x.ms / 1e6, probes / x.ms / 1e3 / n_sm / clk_khz);
        }
        fflush(stdout);
    }
    {   // the record load forms at k_fused's geometry, alone and beside streaming traffic
        const size_t stream_bytes = size_t(64) << 20;  // each of the two streamed buffers: larger than the 50 MB L2
        uint4 *sin, *sout;
        CK(cudaMalloc(&sin, stream_bytes));
        CK(cudaMalloc(&sout, stream_bytes));
        CK(cudaMemset(sin, 0x11, stream_bytes));
        const size_t nvec = stream_bytes / 16;
        const int smem = 220 * 1024;  // k_fused's 217-227 KB: the L1 that is left is the kernel's
        const int iters = 256;
        struct M { const char* name; void (*k0)(const char*, uint32_t, int, const uint4*, uint4*, size_t, uint32_t*);
                   void (*k1)(const char*, uint32_t, int, const uint4*, uint4*, size_t, uint32_t*); } modes[] = {
            {"na2", k_probe_mode<kNa2, false>, k_probe_mode<kNa2, true>},
            {"l1a2", k_probe_mode<kL1a2, false>, k_probe_mode<kL1a2, true>},
            {"l1a2ef", k_probe_mode<kL1a2ef, false>, k_probe_mode<kL1a2ef, true>},
            {"pair", k_probe_mode<kPair, false>, k_probe_mode<kPair, true>},
            {"one16", k_probe_mode<kOne16, false>, k_probe_mode<kOne16, true>}};
        for (const M& x : modes)
            for (auto k : {x.k0, x.k1}) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        const double mode_mb[] = {8, 17.1, 23};
        // probing warps: three of every four, two independent records in flight per lane
        const double probes = double(n_sm) * 1024 * 3 / 4 * iters * 2;
        for (double mb : mode_mb) {
            const uint32_t nslots = uint32_t(mb * 1048576.0 / 32.0);
            for (int stream = 0; stream < 2; ++stream) {
                for (const M& x : modes) {
                    auto k = stream ? x.k1 : x.k0;
                    const float ms = time_ms([&] { k<<<n_sm, 1024, smem>>>(static_cast<const char*>(table), nslots, iters, sin, sout, nvec, sink); }, 10);
                    printf("{\"test\": \"record_load\", \"mode\": \"%s\", \"table_mb\": %.1f, \"streaming\": %s, \"ms\": %.4f, "
                           "\"gprobes_s\": %.2f, \"stream_gbs\": %.1f}\n",
                           x.name, mb, stream ? "true" : "false", ms, probes / ms / 1e6,
                           stream ? double(n_sm) * 8 * iters * 1024.0 / ms / 1e6 : 0.0);
                }
                fflush(stdout);
            }
        }
        CK(cudaGetLastError());
        CK(cudaFree(sin));
        CK(cudaFree(sout));
    }
    {
        const int iters = 256;
        const float ms = time_ms([&] { k_smem_seed<<<n_sm, 1024>>>(iters, sink); }, 5);
        const double reads = double(n_sm) * 1024 * iters * 4;
        printf("{\"test\": \"smem_seed_u8\", \"ms\": %.4f, \"greads_s\": %.2f, \"reads_per_clk_per_sm\": %.2f}\n", ms,
               reads / ms / 1e6, reads / ms / 1e3 / n_sm / double(clk_khz));
    }
    {
        const int iters = 2048;
        const float ms = time_ms([&] { k_issue<<<grid, threads>>>(iters, sink); }, 5);
        const double warp_instr = nthreads / 32.0 * iters * 8 * 3;
        printf("{\"test\": \"issue\", \"ms\": %.4f, \"gwarp_instr_s\": %.1f, \"per_clk_per_sm\": %.2f}\n", ms,
               warp_instr / ms / 1e6, warp_instr / ms / 1e3 / n_sm / double(clk_khz));
    }
    CK(cudaFree(table));
    CK(cudaFree(sink));
    return 0;
}
