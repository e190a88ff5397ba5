// Kernels and host path of the kernel variants of one translation unit.  build.py compiles this file once per unit,
// with -DBSB_UNIT=BSB_UNIT_<unit> naming the unit's slice of the variant list (bsb_kernels.cuh), so that every
// variant is instantiated in exactly one unit and the units compile in parallel.
#include <cstring>

#include "bsb_dispatch.cuh"

namespace bsb {
#define BSB_INSTANTIATE(F, O, mode, mt, two_phase) \
  template int run_variant<Variant<F, O, mode> >(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs*); \
  template int run_masked<Variant<F, O, mode> >(bsb_env*, const LaunchArgs&, const uint8_t*, int64_t*, uint8_t*, \
                                                const bsb_outputs*, const bsb_policy*, const bsb_replay*, \
                                                const bsb_sequence*, const bsb_ensemble_policy*, cudaStream_t);
BSB_UNIT(BSB_INSTANTIATE)
#undef BSB_INSTANTIATE
}  // namespace bsb
