// Block-scaled FP8 GEMM for sm_90a (block-wise FP8 and MXFP8 linear layers) and the per-token group quantiser that feeds it.
//
//   D[M,N] (bf16) = Σ_g (Aq[:, g] · Bq[:, g]ᵀ) ∘ sa[:, g] ⊗ sb[:, g]        g = scale group of G consecutive k
//
// Aq e4m3 [M, K] and Bq e4m3 [N, K] are both K-major; sa / sb are fp32 with one scale per (row, group) and (column, group),
// stored group-major ([K/G, M] with a padded row stride, [K/G, N]) so that TMA brings the slice of a k-block in one box.
//
// Hopper has no block-scaled MMA, so each group is a separate wgmma chain into a temporary fp32 accumulator that is promoted
// into the main accumulator in registers with the product of its row and column scales.  Nothing is de-quantised in memory
// and the sum over groups stays in fp32.
//
// One persistent CTA per SM, 384 threads:
//   warpgroup 0     TMA producer : one thread fills a ring of stages; a stage is one 128-byte k-block (128 e4m3 elements) of
//                                  the 128 x 128 A / B tiles (128B swizzle) plus the tile's 128/G scale rows of A and of B
//   warpgroups 1-2  consumers    : consumer c owns rows 64c..64c+63 of the tile; per group it issues G/32 wgmma m64n128k32
//                                  (the first with scale_d = 0), waits, and promotes; the stage is released after its last
//                                  group.  The two consumers are independent, so one's promotion overlaps the other's MMAs.
//
// Grouped mode (GROUPED = true, MoE experts): the rows of A come in `block_rows`-row blocks and block i is multiplied by expert
// block_expert[i].  B is every expert's K-major [N, K] weight stacked into one [E·N, K] tensor map and the weight scales are
// stacked into one [E·K/G, N] map, so the tile's expert only shifts two TMA row coordinates: e·N for the B tile and e·K/G for
// the scale rows.  block_rows % 128 == 0, so a 128-row tile lies inside one block and its expert is block_expert[m0 / block_rows].
// Ragged N (N % 128 != 0): the last column tile of expert e reads B rows e·N + n0 + j with n0 + j >= N, which are the first rows
// of expert e + 1 (only the last expert's over-read is past the map and zero-filled).  Column j of a tile depends only on B row
// n0 + j and scale column n0 + j (whose over-read is always past the scale map's N columns, so zero), and columns >= N are never
// stored: the neighbour's rows, NaN included, cannot reach a stored element.
#include <cuda.h>
#include <cuda_fp8.h>

#include "common.cuh"
#include "fp8_rule.cuh"
#include "kernels.h"
#include "sm90_ptx.cuh"

namespace nxd {
namespace fp8b {

constexpr int BM = 128, BN = 128;
constexpr int BK = 128;                         // e4m3 elements (= bytes) per k-block: one 128-byte swizzle row
constexpr int kThreads = 384;
constexpr int kStages = 6;
constexpr int kTileBytes = BM * BK;             // 16 KB for A, the same for B

template <int G>
struct Cfg {
  static constexpr int kGroups = BK / G;                           // scale groups per k-block
  static constexpr int kScaleBytes = kGroups * BM * 4;             // one operand's scale slice
  static constexpr int kStageBytes = 2 * kTileBytes + 2 * kScaleBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kStageBytes % 1024 == 0, "swizzled tiles need 1 KB aligned stages");
};

// tile index → (m_blk, n_blk): 8 M-blocks at a time so that B tiles are re-used from L2
NXD_DEVICE void tile_coords(int tile, int tiles_m, int tiles_n, int& m_blk, int& n_blk) {
  constexpr int GROUP = 8;
  const int per_group = GROUP * tiles_n;
  const int g = tile / per_group, first_m = g * GROUP;
  const int gsz = min(GROUP, tiles_m - first_m);
  const int in = tile - g * per_group;
  m_blk = first_m + in % gsz;
  n_blk = in / gsz;
}

template <int G, bool GROUPED>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_block_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                      const __grid_constant__ CUtensorMap tma_sa, const __grid_constant__ CUtensorMap tma_sb,
                      __nv_bfloat16* __restrict__ out, int M, int N, int K, const int* __restrict__ block_expert,
                      int block_rows) {
  using C = Cfg<G>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1 KB alignment
  uint64_t* bars = (uint64_t*)(smem + kStages * C::kStageBytes);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + kStages);
  const uint32_t smem_base = smem_u32(smem);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = K / BK;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tma_a); prefetch_tmap(&tma_b); prefetch_tmap(&tma_sa); prefetch_tmap(&tma_sb);
    // empty: one arrival per consumer warp (8), after the warp's last read of the stage's scales
    for (int i = 0; i < kStages; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===== TMA producer: hands its registers to the consumers, which hold two 64-float accumulators =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(tile, tiles_m, tiles_n, m_blk, n_blk);
        const int m0 = m_blk * BM, n0 = n_blk * BN;
        int b_row = n0, sb_row = 0;                     // grouped: the tile's expert shifts the B and weight-scale rows
        if constexpr (GROUPED) {
          const int e = block_expert[m0 / block_rows];
          b_row += e * N;
          sb_row = e * (K / G);
        }
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_bounded(bar_empty + 8 * stage, phase ^ 1);
          const uint32_t full = bar_full + 8 * stage;
          mbar_expect_tx(full, C::kStageBytes);          // out-of-bounds box elements are zero-filled and still counted
          const uint32_t sa = smem_base + stage * C::kStageBytes, sb = sa + kTileBytes;
          const uint32_t ssa = sb + kTileBytes, ssb = ssa + C::kScaleBytes;
          tma_load_2d(sa, &tma_a, full, kb * BK, m0);                       // box {128 k, 128 m}
          tma_load_2d(sb, &tma_b, full, kb * BK, b_row);                    // box {128 k, 128 n}
          tma_load_2d(ssa, &tma_sa, full, m0, kb * C::kGroups);             // box {128 m, groups}
          tma_load_2d(ssb, &tma_sb, full, n0, sb_row + kb * C::kGroups);    // box {128 n, groups}
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
    return;
  }

  // ===== consumers =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = (threadIdx.x - 128) >> 7;              // consumer warpgroup 0 / 1 → rows 64*cw ..
  const int wq = warp & 3;                              // warp inside the warpgroup → 16-row slice
  const int r_loc = cw * 64 + wq * 16 + (lane >> 2);    // this thread's first row inside the tile (second: + 8)
  const int c_loc = 2 * (lane & 3);                     // this thread's first column inside each 8-column slice
  int stage = 0; uint32_t phase = 0;
  float acc[64], part[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) part[i] = 0.f;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int m_blk, n_blk;
    tile_coords(tile, tiles_m, tiles_n, m_blk, n_blk);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_bounded(bar_full + 8 * stage, phase);
      const uint32_t st_addr = smem_base + stage * C::kStageBytes;
      const uint32_t sa = st_addr + cw * 8192, sb = st_addr + kTileBytes;
      const float* ssa = (const float*)(smem + stage * C::kStageBytes + 2 * kTileBytes);
      const float* ssb = ssa + C::kGroups * BM;
#pragma unroll
      for (int g = 0; g < C::kGroups; ++g) {
        fence_acc(part);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < G / 32; ++k) {
          const int kk = g * (G / 32) + k;                // 32-byte step inside the 128-byte swizzle row
          wgmma_m64n128k32_e4m3(part, make_smem_desc(sa + kk * 32, 16, 1024), make_smem_desc(sb + kk * 32, 16, 1024),
                                k == 0 ? 0u : 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(part);
        // promotion: acc += part · sa[row, g] · sb[col, g]  (register 4j + {0,1}: row r_loc, columns 8j + c_loc + {0,1};
        // 4j + {2,3}: the same columns eight rows further down)
        const float a0 = ssa[g * BM + r_loc], a1 = ssa[g * BM + r_loc + 8];
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const float2 b = *(const float2*)(ssb + g * BN + 8 * j + c_loc);
          acc[4 * j] = fmaf(part[4 * j], a0 * b.x, acc[4 * j]);
          acc[4 * j + 1] = fmaf(part[4 * j + 1], a0 * b.y, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(part[4 * j + 2], a1 * b.x, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(part[4 * j + 3], a1 * b.y, acc[4 * j + 3]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }

    // epilogue straight from registers: bf16 pairs, rows >= M and columns >= N are not stored
    const int row0 = m_blk * BM + r_loc, n0 = n_blk * BN;
    const bool ok0 = row0 < M, ok1 = row0 + 8 < M;
    __nv_bfloat16* o0 = out + (size_t)row0 * N;
    __nv_bfloat16* o1 = out + (size_t)(row0 + 8) * N;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n0 + 8 * j + c_loc;
      if (col >= N) continue;                                  // N is even: col < N → col + 1 < N
      if (ok0) *(__nv_bfloat162*)(o0 + col) = __floats2bfloat162_rn(acc[4 * j], acc[4 * j + 1]);
      if (ok1) *(__nv_bfloat162*)(o1 + col) = __floats2bfloat162_rn(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
}

// ---- per-token group quantiser ----------------------------------------------------------------------------------------
// One warp quantises a 256-element segment of one row: lane l holds elements 8l..8l+7 (one 16-byte load), the G/8 lanes of a
// group reduce their absmax with shuffles.  Warps are ordered row-fastest so that neighbouring warps write neighbouring
// scales of the group-major scale buffer.
//
// Non-finite input: a group holding a NaN, or ±inf with no clamp, gets a NaN scale and NaN codes, so every output that reads
// it is NaN (the clamp, the amax and its shuffle reduction propagate NaN: fp8_rule.cuh; the MX exponent of an infinite amax
// would overflow the int shift into a finite scale, so it is tested first).  The absmax scale and the codes are the shared
// rule of fp8_rule.cuh.
template <int G, bool MX>
__global__ void __launch_bounds__(256)
quantize_fp8_groups_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ s, int M, int K,
                           long s_ld, float clamp_bound) {
  const long w = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long segs = (K + 255) / 256;
  if (w >= (long)M * segs) return;
  const int row = (int)(w % M);
  const int col = (int)(w / M) * 256 + lane * 8;
  const bool live = col < K;                                   // K % G == 0: a group is wholly live or wholly not
  float v[8];
  float amax = 0.f;
  if (live) {
    const uint4 raw = __ldg((const uint4*)(x + (size_t)row * K + col));
    const __nv_bfloat162* h = (const __nv_bfloat162*)&raw;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      v[2 * i] = min_nan(max_nan(f.x, -clamp_bound), clamp_bound);
      v[2 * i + 1] = min_nan(max_nan(f.y, -clamp_bound), clamp_bound);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = max_nan(amax, fabsf(v[i]));
  }
#pragma unroll
  for (int off = 1; off < G / 8; off <<= 1) amax = max_nan(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if (!live) return;
  float scale;
  if constexpr (MX) {
    if (!e4m3_amax_finite(amax)) {
      scale = __int_as_float(0x7fffffff);                      // NaN, or ±inf with no clamp: NaN scale, NaN codes
    } else {
      // OCP MX: 2^(floor(log2 amax) - 8), amax clamped to 2^-100; log2 rounded to fp32 first, as the torch quantiser does.
      // amax is finite here, so -100 <= e <= 127 and the biased exponent e - 8 + 127 is in [19, 246]: no overflow
      const float e = floorf((float)log2((double)fmaxf(amax, 0x1p-100f)));
      scale = __int_as_float(((int)e - 8 + 127) << 23);
    }
  } else {
    scale = e4m3_absmax_scale(amax);
  }
  uint32_t lo = 0, hi = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t b = e4m3_code(v[i], scale);
    if (i < 4) lo |= b << (8 * i); else hi |= b << (8 * (i - 4));
  }
  *(uint2*)(q + (size_t)row * K + col) = make_uint2(lo, hi);
  if ((lane & (G / 8 - 1)) == 0) s[(long)(col / G) * s_ld + row] = scale;
}

// E = 1 and block_expert = nullptr: the dense GEMM.  Otherwise b is [E·N, K] and sb [E·K/G, N] (grouped mode).
template <int G, bool GROUPED>
void launch_gemm(const void* a, const void* b, void* out, const float* sa, long sa_ld, const float* sb, int M, int N, int K,
                 int E, const int* block_expert, int block_rows, cudaStream_t st) {
  using C = Cfg<G>;
  const int groups = K / G;
  const CUtensorMap ta = make_tmap_2d(a, CU_TENSOR_MAP_DATA_TYPE_UINT8, M, K, K, BK, BM, CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMap tb = make_tmap_2d(b, CU_TENSOR_MAP_DATA_TYPE_UINT8, (uint64_t)E * N, K, K, BK, BN,
                                      CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMap tsa = make_tmap_2d(sa, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, groups, M, sa_ld * 4, BM, C::kGroups,
                                       CU_TENSOR_MAP_SWIZZLE_NONE);
  const CUtensorMap tsb = make_tmap_2d(sb, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (uint64_t)E * groups, N, (uint64_t)N * 4, BN,
                                       C::kGroups, CU_TENSOR_MAP_SWIZZLE_NONE);
  auto kern = gemm_fp8_block_kernel<G, GROUPED>;
  static bool configured = false;
  if (!configured) {
    NXD_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    configured = true;
  }
  const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int sms = device_sm_count();
  kern<<<tiles < sms ? tiles : sms, kThreads, C::kSmemBytes, st>>>(ta, tb, tsa, tsb, (__nv_bfloat16*)out, M, N, K,
                                                                   block_expert, block_rows);
  NXD_CUDA_CHECK(cudaGetLastError());
}

template <int G>
void launch_quantize(const void* x, void* q, float* s, int M, int K, long s_ld, bool mx, float clamp_bound, cudaStream_t st) {
  const long warps = (long)M * ((K + 255) / 256);
  const unsigned blocks = (unsigned)((warps + 7) / 8);
  if (mx) quantize_fp8_groups_kernel<G, true><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, s, M, K, s_ld, clamp_bound);
  else quantize_fp8_groups_kernel<G, false><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)x, (uint8_t*)q, s, M, K, s_ld, clamp_bound);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace fp8b

void gemm_fp8_block(const void* a, const void* b, void* out, const float* scale_a, long scale_a_ld, const float* scale_b,
                    int M, int N, int K, int group, cudaStream_t st) {
  if (K % fp8b::BK || N % 8) nxd_throw("block-scaled fp8 GEMM needs K % 128 == 0 and N % 8 == 0", __FILE__, __LINE__);
  if (scale_a_ld % 4 || scale_a_ld < M) nxd_throw("block-scaled fp8 GEMM: A-scale row stride must be >= M and a multiple of 4",
                                                  __FILE__, __LINE__);
  if (M == 0) return;
  switch (group) {
    case 32: fp8b::launch_gemm<32, false>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, 1, nullptr, 0, st); break;
    case 64: fp8b::launch_gemm<64, false>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, 1, nullptr, 0, st); break;
    case 128: fp8b::launch_gemm<128, false>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, 1, nullptr, 0, st); break;
    default: nxd_throw("block-scaled fp8 GEMM: group size must be 32, 64 or 128", __FILE__, __LINE__);
  }
}

void grouped_gemm_fp8_block(const void* a, const void* b, void* out, const float* scale_a, long scale_a_ld,
                            const float* scale_b, int M, int N, int K, int E, const int* block_expert, int block_rows,
                            int group, cudaStream_t st) {
  if (K % fp8b::BK || N % 8) nxd_throw("grouped block-scaled fp8 GEMM needs K % 128 == 0 and N % 8 == 0", __FILE__, __LINE__);
  if (block_rows <= 0 || block_rows % fp8b::BM || M % block_rows)
    nxd_throw("grouped block-scaled fp8 GEMM: block_rows must be a positive multiple of 128 dividing M", __FILE__, __LINE__);
  if (scale_a_ld % 4 || scale_a_ld < M)
    nxd_throw("grouped block-scaled fp8 GEMM: A-scale row stride must be >= M and a multiple of 4", __FILE__, __LINE__);
  if (E <= 0) nxd_throw("grouped block-scaled fp8 GEMM: needs at least one expert", __FILE__, __LINE__);
  if (M == 0) return;
  switch (group) {
    case 32: fp8b::launch_gemm<32, true>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, E, block_expert, block_rows, st); break;
    case 64: fp8b::launch_gemm<64, true>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, E, block_expert, block_rows, st); break;
    case 128: fp8b::launch_gemm<128, true>(a, b, out, scale_a, scale_a_ld, scale_b, M, N, K, E, block_expert, block_rows, st); break;
    default: nxd_throw("grouped block-scaled fp8 GEMM: group size must be 32, 64 or 128", __FILE__, __LINE__);
  }
}

void quantize_fp8_groups(const void* x, void* q, float* scale, int M, int K, long scale_ld, int group, bool mx, float clamp_bound,
                         cudaStream_t st) {
  if (K % group || K % 8) nxd_throw("fp8 group quantiser needs K % group == 0", __FILE__, __LINE__);
  if (M == 0) return;
  switch (group) {
    case 32: fp8b::launch_quantize<32>(x, q, scale, M, K, scale_ld, mx, clamp_bound, st); break;
    case 64: fp8b::launch_quantize<64>(x, q, scale, M, K, scale_ld, mx, clamp_bound, st); break;
    case 128: fp8b::launch_quantize<128>(x, q, scale, M, K, scale_ld, mx, clamp_bound, st); break;
    default: nxd_throw("fp8 group quantiser: group size must be 32, 64 or 128", __FILE__, __LINE__);
  }
}

}  // namespace nxd
