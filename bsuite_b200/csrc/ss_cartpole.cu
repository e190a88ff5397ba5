// cartpole: same-step auto-reset kernels and host path (BSB_FLAG_SAME_STEP_RESET, Philox, every obs_dtype), apart from
// the next-step ones.
#include "bsb_dispatch.cuh"

namespace bsb {
template int run_same_step<Cartpole>(bsb_env*, const LaunchArgs&, cudaStream_t);
}  // namespace bsb
