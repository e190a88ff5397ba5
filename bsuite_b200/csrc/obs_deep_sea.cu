// deep_sea: kernels and host path for bfloat16 and uint8 observations (obs_dtype, Philox), apart from the float32 ones.
#include "bsb_dispatch.cuh"

namespace bsb {
template int run_reduced<DeepSea>(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs*);
}  // namespace bsb
