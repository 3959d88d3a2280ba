// vaporetto_b200 — host side of k_fused (fused_kernel.cuh): the dispatch to the kernel variants plan() chooses
// (kernel_plan.hpp), which are instantiated in fused_ss.cu / fused_sg.cu / fused_gs.cu / fused_gg.cu (one translation
// unit per (seeds in shared memory, common shape) pair, so that they compile in parallel).
#include <atomic>
#include <algorithm>

#include "device_model.hpp"
#include "fused_launch.hpp"
#include "kernel_plan.hpp"

namespace vpt {

bool fused_ok(const DevModel& m) { return plan_detail::fused_shape_ok(m); }

// One launch for the whole batch (plus the memset node that clears the look-back descriptors and the ticket).
cudaError_t launch_fused(const DevModel& m, const BatchArgs& a, cudaStream_t stream) {
    if (a.n_sent == 0) return cudaSuccess;
    const KernelPlan pl = plan(m, a.char_states != nullptr || a.type_states != nullptr);
    if (pl.kernel != kPlanFused) return cudaErrorInvalidValue;  // (callers check fused_ok first)
    static std::atomic<int> sm_count[fused_detail::kMaxDevices] = {};  // (idempotent cache: every writer stores the same value)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= fused_detail::kMaxDevices) return cudaErrorInvalidDevice;
    if (sm_count[dev] == 0) {
        int v = 0;
        e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        sm_count[dev] = v;
    }
    // group_bound, group_char and the ticket are one contiguous, 256-byte aligned region of the workspace
    const size_t clear_bytes = size_t(reinterpret_cast<const uint8_t*>(a.ticket) - reinterpret_cast<const uint8_t*>(a.group_bound)) + 256;
    if (!a.prezeroed) {
        e = cudaMemsetAsync(a.group_bound, 0, clear_bytes, stream);
        if (e != cudaSuccess) return e;
    }
    StreamCfg cfg;
    cfg.lag = pl.lag;
    cfg.r0 = m.ct.present ? m.ct.r0 : 0;
    cfg.gap = pl.gap;
    cfg.tw = m.type_cache_window;
    cfg.norm = m.kytea_norm != 0;
    const int n_sm = sm_count[dev];
    if (pl.seeds_smem) return pl.common ? fused_detail::launch_fused_group<true, true>(pl, m, a, cfg, stream, dev, n_sm) : fused_detail::launch_fused_group<true, false>(pl, m, a, cfg, stream, dev, n_sm);
    return pl.common ? fused_detail::launch_fused_group<false, true>(pl, m, a, cfg, stream, dev, n_sm) : fused_detail::launch_fused_group<false, false>(pl, m, a, cfg, stream, dev, n_sm);
}

}  // namespace vpt
