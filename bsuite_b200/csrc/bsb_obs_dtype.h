// Observation element types narrower than float32 (bsb_config.obs_dtype) and the one conversion from the float32
// observation to each.  Plain C++: the kernels, the host path and tests/obs_dtype_harness.cpp include it alike, so a
// reduced observation is the same function of the float32 one wherever it is produced.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define BSB_OBS_HD __host__ __device__ __forceinline__
#else
#define BSB_OBS_HD inline
#endif

namespace bsb {

// Storage of one bfloat16 (the upper half of a float32).
struct Bf16 { uint16_t bits; };

BSB_OBS_HD uint32_t f32_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, sizeof(u));
  return u;
#endif
}

// float32 -> bfloat16 with round-to-nearest-even, as torch.Tensor.to(torch.bfloat16) rounds (c10::BFloat16):
// subnormals round like any other value and finite values past the largest bfloat16 round to infinity.  Every NaN
// becomes 0x7fc0, c10::BFloat16's quiet NaN; torch's own conversions do not agree on NaN (its CUDA kernels give
// 0x7fff, its vectorised CPU path 0xffff), so for NaN the result is a NaN, not a particular pattern.  No family's
// observation is ever NaN.
BSB_OBS_HD uint16_t f32_to_bf16_bits(float f) {
  const uint32_t u = f32_bits(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fc0u;
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

// float32 -> uint8 for the 0 / 1 observations of deep_sea and catch: exact for every integer in [0, 255], which is
// what torch gives too.  Anything else saturates (NaN -> 0), a defined result where a plain cast would not be.
BSB_OBS_HD uint8_t f32_to_u8(float f) { return f > 0.f ? (f < 255.f ? (uint8_t)(int32_t)f : (uint8_t)255) : (uint8_t)0; }

// The observation element of type O that stands for the float32 value v.
template <class O> BSB_OBS_HD O obs_cast(float v);
template <> BSB_OBS_HD float obs_cast<float>(float v) { return v; }
template <> BSB_OBS_HD Bf16 obs_cast<Bf16>(float v) { Bf16 b; b.bits = f32_to_bf16_bits(v); return b; }
template <> BSB_OBS_HD uint8_t obs_cast<uint8_t>(float v) { return f32_to_u8(v); }

}  // namespace bsb
