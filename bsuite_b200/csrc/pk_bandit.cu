// bandit: packed kernels and host path (bsb_create_packed: float32, next-step, Philox), apart from the ordinary ones.
#include "bsb_dispatch.cuh"

namespace bsb {
template int run_packed<Bandit>(bsb_env*, const LaunchArgs&, cudaStream_t);
}  // namespace bsb
