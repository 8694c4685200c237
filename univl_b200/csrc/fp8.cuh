// univl_b200 — e4m3 block scaling shared by the quantizers (quant_fp8.cu) and the FP8 GEMM's GELU epilogue.
//
// A block of values (1 x 128 activations, 128 x 128 weights) is stored as e4m3 codes q and one fp32 scale s with
// value = q * s.  s is the power of two 2^ceil(log2(amax / 448)), amax the block's largest magnitude: the block's
// largest value lands in (224, 448], e4m3's top binade.  An all-zero block gets s = 1, and s is at least 2^-126 (the
// smallest normal fp32) so that 1 / s is finite.  Being powers of two, x / s and q * s are exact in fp32; the
// conversion to e4m3 rounds to nearest even and saturates at +-448.
#pragma once

#include <cuda_fp8.h>

#include "common.cuh"

namespace univl {

constexpr float E4M3_MAX = 448.f;

// the scale of a block whose largest magnitude is amax, from the bits of the correctly rounded amax / 448
__device__ __forceinline__ float e4m3_scale(float amax) {
  if (!(amax > 0.f)) return 1.f;
  const uint32_t b = __float_as_uint(__fdiv_rn(amax, E4M3_MAX));
  int e = (int)((b >> 23) & 0xff) - 127 + ((b & 0x7fffff) != 0);  // ceil(log2(.)) for a normal value
  e = max(e, -126);                                                 // subnormal or zero quotient
  return __uint_as_float((uint32_t)(e + 127) << 23);
}

// 1 / s, exact for the scales e4m3_scale returns
__device__ __forceinline__ float e4m3_inv_scale(float s) { return __uint_as_float((254u << 23) - __float_as_uint(s)); }

// two values (already divided by the scale) -> two e4m3 codes, lo in the low byte
__device__ __forceinline__ uint16_t e4m3x2(float lo, float hi) {
  return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, __NV_E4M3);
}

}  // namespace univl
