// k_fused variants with seeds in global memory, generic model shape (see fused.cu).
#include "fused_kernel.cuh"

namespace vpt {
namespace fused_detail {
template cudaError_t launch_fused_group<false, false>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);
}  // namespace fused_detail
}  // namespace vpt
