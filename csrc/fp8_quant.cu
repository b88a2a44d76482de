// Per-row e4m3 quantisers that feed the fp8 GEMM of gemm_sm90.cu in training (row-wise scaled FP8 linears).
//
//   rows(t)   : bf16 [M, K] → e4m3 [M, K] + fp32 [M]       one absmax scale per row
//   cols_t(t) : bf16 [R, C] → e4m3 [C, R] + fp32 [C]       rows(tᵀ): one scale per column, written transposed so that a GEMM
//                                                          contracting over R reads it K-major (e4m3 wgmma takes no other)
//
// The scale and code rule is fp8_rule.cuh, the one the group quantiser uses; both kernels are bandwidth-bound with one read
// pass for the absmax and one for the codes.
#include <cuda_fp8.h>

#include "common.cuh"
#include "fp8_rule.cuh"
#include "kernels.h"

namespace nxd {
namespace fp8q {

constexpr int kThreads = 256;

// One CTA per row; thread t takes the 16-byte vectors t, t + 256, … of the row.  The second pass re-reads the row (from L2).
__global__ void __launch_bounds__(kThreads)
quantize_rows_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ s, int K) {
  __shared__ float red[kThreads / 32];
  const size_t row = blockIdx.x;
  const uint4* xr = (const uint4*)(x + row * K);
  uint2* qr = (uint2*)(q + row * K);
  const int nvec = K / 8;
  float amax = 0.f;
  for (int i = threadIdx.x; i < nvec; i += kThreads) {
    const uint4 raw = __ldg(xr + i);
    const __nv_bfloat162* h = (const __nv_bfloat162*)&raw;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(h[j]);
      amax = max_nan(amax, max_nan(fabsf(f.x), fabsf(f.y)));
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = max_nan(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) amax = max_nan(amax, red[w]);
  const float scale = e4m3_absmax_scale(amax);
  if (threadIdx.x == 0) s[row] = scale;
  for (int i = threadIdx.x; i < nvec; i += kThreads) {
    const uint4 raw = __ldg(xr + i);
    const __nv_bfloat162* h = (const __nv_bfloat162*)&raw;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(h[j]);
      const uint32_t b = e4m3_code(f.x, scale) | (e4m3_code(f.y, scale) << 8);
      if (j < 2) lo |= b << (16 * j); else hi |= b << (16 * (j - 2));
    }
    qr[i] = make_uint2(lo, hi);
  }
}

// Pass 1 of cols_t: column absmax.  A CTA covers 256 columns (8 per lane, one 16-byte load) of kColRows rows, warp w taking
// rows w, w + 8, …; the partial maxima meet in shared memory and leave with one atomicMax per column.  The max runs on the bf16
// bit patterns with the sign cleared: for non-negative values the pattern order is the magnitude order, NaN sorts above ±inf
// (so a column with a NaN gets a NaN scale), and a max does not depend on the order of the atomics.
constexpr int kColRows = 128;

__global__ void __launch_bounds__(kThreads)
col_absmax_kernel(const __nv_bfloat16* __restrict__ x, uint32_t* __restrict__ amax_bits, int R, int C) {
  __shared__ uint32_t part[kThreads / 32][kThreads];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * kColRows, r1 = min(r0 + kColRows, R);
  uint32_t m[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < C) {
    for (int r = r0 + warp; r < r1; r += kThreads / 32) {
      const uint4 raw = __ldg((const uint4*)(x + (size_t)r * C + c0));
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m[2 * j] = max(m[2 * j], w[j] & 0x7fffu);
        m[2 * j + 1] = max(m[2 * j + 1], (w[j] >> 16) & 0x7fffu);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[warp][lane * 8 + j] = m[j];
  __syncthreads();
  uint32_t v = part[0][threadIdx.x];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) v = max(v, part[w][threadIdx.x]);
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col < C && v != 0) atomicMax(amax_bits + col, v << 16);        // bf16 → fp32 bit pattern; the buffer starts at zero
}

// Pass 2 of cols_t: a CTA quantises a [128 rows (R), 64 columns (C)] tile and writes it transposed.  Thread t = 8·rq + cv loads
// columns 8cv..8cv+7 of rows 4rq..4rq+3 (a warp reads four 128-byte row segments per load), packs the four codes of each column
// into one word of the shared tile [column][row / 4] (33 words per column, so a warp's stores hit distinct banks but for pairs),
// then the CTA writes 64 output rows of 128 bytes in 16-byte vectors.  R % 16 == 0: a vector is wholly inside or past the end.
constexpr int kTileR = 128, kTileC = 64;

__global__ void __launch_bounds__(kThreads)
quantize_cols_t_kernel(const __nv_bfloat16* __restrict__ x, const uint32_t* __restrict__ amax_bits, uint8_t* __restrict__ q,
                       float* __restrict__ s, int R, int C) {
  __shared__ float sc[kTileC];
  __shared__ uint32_t tile[kTileC][kTileR / 4 + 1];
  const int t = threadIdx.x;
  const int c_base = blockIdx.x * kTileC, r_base = blockIdx.y * kTileR;
  if (t < kTileC) {
    const int col = c_base + t;
    const float scale = col < C ? e4m3_absmax_scale(__uint_as_float(amax_bits[col])) : 1.f;
    sc[t] = scale;
    if (blockIdx.y == 0 && col < C) s[col] = scale;
  }
  __syncthreads();
  const int cv = t & 7, rq = t >> 3;
  const int c0 = c_base + cv * 8;
  uint32_t packed[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < C) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r_base + rq * 4 + i;
      if (r >= R) break;
      const uint4 raw = __ldg((const uint4*)(x + (size_t)r * C + c0));
      const __nv_bfloat162* h = (const __nv_bfloat162*)&raw;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(h[j]);
        packed[2 * j] |= e4m3_code(f.x, sc[cv * 8 + 2 * j]) << (8 * i);
        packed[2 * j + 1] |= e4m3_code(f.y, sc[cv * 8 + 2 * j + 1]) << (8 * i);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) tile[cv * 8 + j][rq] = packed[j];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kTileC * (kTileR / 16) / kThreads; ++k) {
    const int idx = t + k * kThreads;
    const int orow = idx >> 3, v = idx & 7;
    const int col = c_base + orow, r = r_base + v * 16;
    if (col < C && r < R) {
      const uint32_t* w = &tile[orow][4 * v];
      *(uint4*)(q + (size_t)col * R + r) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

}  // namespace fp8q

void quantize_fp8_rows(const void* x, void* q, float* scale, int M, int K, cudaStream_t st) {
  if (K % 8) nxd_throw("fp8 row quantiser needs K % 8 == 0", __FILE__, __LINE__);
  if (M == 0 || K == 0) return;
  fp8q::quantize_rows_kernel<<<M, fp8q::kThreads, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, scale, K);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void quantize_fp8_cols_t(const void* x, void* q, float* scale, uint32_t* amax_bits, int R, int C, cudaStream_t st) {
  if (R % 16 || C % 8) nxd_throw("fp8 transposing quantiser needs R % 16 == 0 and C % 8 == 0", __FILE__, __LINE__);
  if (R == 0 || C == 0) return;
  const dim3 g1((C + 255) / 256, (R + fp8q::kColRows - 1) / fp8q::kColRows);
  fp8q::col_absmax_kernel<<<g1, fp8q::kThreads, 0, st>>>((const __nv_bfloat16*)x, amax_bits, R, C);
  NXD_CUDA_CHECK(cudaGetLastError());
  const dim3 g2((C + fp8q::kTileC - 1) / fp8q::kTileC, (R + fp8q::kTileR - 1) / fp8q::kTileR);
  fp8q::quantize_cols_t_kernel<<<g2, fp8q::kThreads, 0, st>>>((const __nv_bfloat16*)x, amax_bits, (uint8_t*)q, scale, R, C);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
