// The absmax e4m3 quantisation rule, shared by every quantiser that feeds the fp8 GEMMs (the per-token group quantiser in
// gemm_fp8_block_sm90.cu, the row and transposing quantisers in fp8_quant.cu) so that they cannot drift apart.
//
//   scale = max(amax / 448, 1e-12)          (NaN when amax is NaN or ±inf)
//   code  = RNE(clamp(x / scale, ±448))     (NaN → the e4m3 NaN code 0x7F)
//
// Bit for bit the torch oracle ``ops.gemm_fp8._quantize_groups_reference`` on a CUDA tensor.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

namespace nxd {

// fmaxf / fminf return the other operand when one is NaN, which would turn NaN into a finite code, so the clamp, the amax and
// its reductions use the NaN-propagating forms; their .ftz matches what fmaxf / fminf compile to under --use_fast_math.
NXD_DEVICE float max_nan(float a, float b) {
  float r;
  asm("max.ftz.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
NXD_DEVICE float min_nan(float a, float b) {
  float r;
  asm("min.ftz.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

NXD_DEVICE bool e4m3_amax_finite(float amax) { return amax <= 3.402823466e38f; }

// torch evaluates `amax / 448` on a CUDA tensor as a product with the rounded reciprocal: the same here, bit for bit
NXD_DEVICE float e4m3_absmax_scale(float amax) {
  if (!e4m3_amax_finite(amax)) return __int_as_float(0x7fffffff);   // NaN, or ±inf: NaN scale, NaN codes
  return fmaxf(amax * (1.f / 448.f), 1e-12f);
}

// true division (not a reciprocal multiply) so the codes are bit-identical to the torch quantisers
NXD_DEVICE uint32_t e4m3_code(float v, float scale) {
  const float c = min_nan(max_nan(__fdiv_rn(v, scale), -448.f), 448.f);
  return (uint32_t)__nv_cvt_float_to_fp8(c, __NV_SATFINITE, __NV_E4M3);
}

}  // namespace nxd
