// memory_chain: kernels and host path for bfloat16 observations (obs_dtype, Philox), apart from the float32 ones.
#include "bsb_dispatch.cuh"

namespace bsb {
template int run_reduced<MemoryChain>(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs*);
}  // namespace bsb
