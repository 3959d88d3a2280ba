// k_fused variants with seeds in shared memory, common model shape (see fused.cu).
#include "fused_kernel.cuh"

namespace vpt {
namespace fused_detail {
template cudaError_t launch_fused_group<true, true>(const KernelPlan&, const DevModel&, const BatchArgs&, const StreamCfg&, cudaStream_t, int, int);
}  // namespace fused_detail
}  // namespace vpt
