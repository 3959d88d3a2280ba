// Interface between the host dispatcher (fused.cu) and the translation units that instantiate k_fused.
#pragma once
#include <cuda_runtime.h>

#include "device_model.hpp"

namespace vpt {

struct StreamCfg {
    int lag;        // a boundary is finished `lag` slots after its own slot
    int r0;         // inline window start
    int gap;
    int tw;         // type table window (0 = none)
    bool norm;
};

struct KernelPlan;  // kernel_plan.hpp

namespace fused_detail {

constexpr int kSeedCap = 37632;   // seed bytes the kernel keeps in shared memory
#ifndef VPT_FUSED_GROUP
#define VPT_FUSED_GROUP 64
#endif
constexpr int kGroupSentences = VPT_FUSED_GROUP;   // sentences per tile of k_fused (>= 32: vpt_workspace_size)
constexpr int kMaxDevices = 64;
constexpr int kCommonGap = 2;     // separator slots between sentences for the common shape (char window 3, type window 3)

template <bool kSeeds, bool kCommon>
cudaError_t launch_fused_group(const KernelPlan& pl, const DevModel& m, const BatchArgs& a, const StreamCfg& cfg, cudaStream_t stream, int dev, int n_sm);

extern template cudaError_t launch_fused_group<true, true>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);
extern template cudaError_t launch_fused_group<true, false>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);
extern template cudaError_t launch_fused_group<false, true>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);
extern template cudaError_t launch_fused_group<false, false>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);

}  // namespace fused_detail

}  // namespace vpt
