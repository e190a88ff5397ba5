// deep_sea: instantiations of both kernels (Philox / MT19937 x RewardNoise x Logging accumulators) and host path.
#include <cstring>

#include "bsb_dispatch.cuh"

namespace bsb {
int run_deep_sea(bsb_env* e, const LaunchArgs& a, cudaStream_t stream, const TwoPhaseArgs* two_phase) {
  return run_family<DeepSea>(e, a, stream, two_phase);
}
}  // namespace bsb
