// Row-wise selection kernels for on-device sampling (roles of the reference's NKI `cascaded_max` K10, `nkilib.core.topk`
// K11 and the torch_neuronx TopK / Argmax custom calls K12 — operators/argmax.py:129, operators/topk.py:17-21,
// utils/sampling.py:50-60).  A vocab(-shard) row is a one-pass HBM-bound reduction: one CTA per row, 16-byte loads.
//   row_argmax   x [R, V] → value fp32 [R], index int64 [R] (+ index_offset: global id of this rank's first column)
//   row_topk     x [R, V] → values fp32 [R, k], indices int64 [R, k], sorted descending; k <= 128, V*4 bytes <= 200 KB:
//                the row is staged once in shared memory as order keys and k block-wide arg-max passes pick the winners.
//
// Selection rule (torch's, and what the distributed wrappers in operators/ rely on): descending order; NaN ranks above
// +inf; -0 and +0 are equal; among equal values the smaller index comes first (torch leaves that order unspecified, the
// wrappers need "smallest global index wins").  top-k returns k distinct indices and the values x[idx] in fp32, -inf and
// NaN included; the arg-max of an all -inf row is index 0 with value -inf.
// Every element is ranked by a 32-bit order key (the fp32 bit pattern made monotonic as an unsigned integer, NaN mapped to
// the top key).  The smallest real key is that of -inf, 0x007fffff, so key 0 is free: it marks a top-k entry already taken
// and "nothing seen yet", and can never win against a real element.  Key and index travel as one 64-bit word
// (key << 32 | ~index), so "larger word" is exactly the rule above.
#include "common.cuh"
#include "kernels.h"

namespace nxd {

namespace {

NXD_DEVICE uint32_t order_key(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0xffffffffu;      // any NaN: above +inf (0xff800000)
  if (u == 0x80000000u) u = 0u;                                 // -0 ranks equal to +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
NXD_DEVICE unsigned long long pack_key(uint32_t key, int i) { return (unsigned long long)key << 32 | (uint32_t)~i; }
NXD_DEVICE int packed_index(unsigned long long p) { return (int)~(uint32_t)p; }

NXD_DEVICE unsigned long long warp_best(unsigned long long x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, o);
    x = y > x ? y : x;
  }
  return x;
}
NXD_DEVICE unsigned long long block_best(unsigned long long x, unsigned long long* smem) {   // smem: >= 32 entries; all threads
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  x = warp_best(x);
  __syncthreads();
  if (lane == 0) smem[warp] = x;
  __syncthreads();
  return warp_best(lane < nw ? smem[lane] : 0ull);
}

template <typename T>
__global__ void __launch_bounds__(256) row_argmax_kernel(const T* __restrict__ x, float* __restrict__ val, long* __restrict__ idx,
                                                         int V, long row_stride, long index_offset) {
  __shared__ unsigned long long red[32];
  const T* row = x + (long)blockIdx.x * row_stride;
  unsigned long long best = 0ull;                               // below every real element (V >= 1)
  constexpr int N = 16 / sizeof(T);
  const bool vec_ok = ((uintptr_t)row % 16 == 0);
  const int nvec = vec_ok ? V / N : 0;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    Pack16<T> p;
    p.load(row + (long)v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const unsigned long long c = pack_key(order_key(p.f(j)), v * N + j);
      best = c > best ? c : best;
    }
  }
  for (int c = nvec * N + threadIdx.x; c < V; c += blockDim.x) {
    const unsigned long long q = pack_key(order_key(to_f32<T>(row[c])), c);
    best = q > best ? q : best;
  }
  best = block_best(best, red);
  if (threadIdx.x == 0) {
    const int i = packed_index(best);
    val[blockIdx.x] = to_f32<T>(row[i]);
    idx[blockIdx.x] = (long)i + index_offset;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) row_topk_kernel(const T* __restrict__ x, float* __restrict__ vals, long* __restrict__ idxs,
                                                       int V, int k, long row_stride, long index_offset) {
  extern __shared__ uint32_t skey[];
  __shared__ unsigned long long red[32];
  const T* row = x + (long)blockIdx.x * row_stride;
  for (int c = threadIdx.x; c < V; c += blockDim.x) skey[c] = order_key(to_f32<T>(row[c]));
  __syncthreads();
  for (int j = 0; j < k; ++j) {                                 // k <= V: an untaken real element always wins
    unsigned long long best = 0ull;
    for (int c = threadIdx.x; c < V; c += blockDim.x) {
      const unsigned long long q = pack_key(skey[c], c);
      best = q > best ? q : best;
    }
    best = block_best(best, red);
    if (threadIdx.x == 0) {
      const int i = packed_index(best);
      vals[(long)blockIdx.x * k + j] = to_f32<T>(row[i]);
      idxs[(long)blockIdx.x * k + j] = (long)i + index_offset;
      skey[i] = 0u;                                             // taken
    }
    __syncthreads();
  }
}

}  // namespace

void row_argmax(const void* x, float* val, long* idx, int rows, int V, long row_stride, long index_offset, int dt, cudaStream_t st) {
  if (rows == 0) return;
  if (V < 1) nxd_throw("row_argmax: a row needs at least one element", __FILE__, __LINE__);
  if (dt == kBF16) row_argmax_kernel<__nv_bfloat16><<<rows, 256, 0, st>>>((const __nv_bfloat16*)x, val, idx, V, row_stride, index_offset);
  else if (dt == kF16) row_argmax_kernel<__half><<<rows, 256, 0, st>>>((const __half*)x, val, idx, V, row_stride, index_offset);
  else row_argmax_kernel<float><<<rows, 256, 0, st>>>((const float*)x, val, idx, V, row_stride, index_offset);
  NXD_CUDA_CHECK(cudaGetLastError());
}

bool row_topk_supported(int V, int k) { return k >= 1 && k <= 128 && (size_t)V * 4 <= 200 * 1024 && k <= V; }

void row_topk(const void* x, float* vals, long* idxs, int rows, int V, int k, long row_stride, long index_offset, int dt,
              cudaStream_t st) {
  if (rows == 0) return;
  if (!row_topk_supported(V, k)) nxd_throw("row_topk: k <= 128 and a row of at most 51200 elements", __FILE__, __LINE__);
  const size_t smem = (size_t)V * 4;
#define NXD_TOPK(T)                                                                                              \
  do {                                                                                                           \
    auto kern = row_topk_kernel<T>;                                                                              \
    if (smem > 48 * 1024) NXD_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<rows, 256, smem, st>>>((const T*)x, vals, idxs, V, k, row_stride, index_offset);                      \
  } while (0)
  if (dt == kBF16) NXD_TOPK(__nv_bfloat16);
  else if (dt == kF16) NXD_TOPK(__half);
  else NXD_TOPK(float);
#undef NXD_TOPK
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd

// =====================================================================================================================
// MoE block-metadata build (role of the reference's `find_nonzero_indices` / `indexed_flatten` NKI kernels K9,
// modules/moe/expert_mlps_v2.py:1079-1206): from the routed expert ids [T, k] produce, in ONE launch and without a sort,
//   tokens_per_expert [E], block_to_expert [nb], token_position_to_id [nb * B]  (-1 = padding)
// with every expert's tokens in ascending token order (the stable order of the torch.argsort-based path it replaces).
// One CTA of 1024 threads: smem histogram → per-expert block ranges → chunked stable scatter (warp match + cross-warp prefix).
namespace nxd {
namespace {

constexpr int kMoeThreads = 1024;
constexpr int kMoeMaxExperts = 256;

template <typename IdxT>
__global__ void __launch_bounds__(kMoeThreads) moe_block_metadata_kernel(const IdxT* __restrict__ expert_index, long n, int k, int E,
                                                                         int B, int nb, long* __restrict__ block_to_expert,
                                                                         long* __restrict__ tp2id, long* __restrict__ counts_out) {
  __shared__ int counts[kMoeMaxExperts];
  __shared__ int base[kMoeMaxExperts];
  __shared__ int wc[32][kMoeMaxExperts];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int e = tid; e < E; e += kMoeThreads) counts[e] = 0;
  for (long s = tid; s < (long)nb * B; s += kMoeThreads) tp2id[s] = -1;
  __syncthreads();
  for (long i = tid; i < n; i += kMoeThreads) {
    const int e = (int)expert_index[i];
    if (e >= 0 && e < E) atomicAdd(&counts[e], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int blk = 0;
    for (int e = 0; e < E; ++e) {
      const int nblk = (counts[e] + B - 1) / B;
      base[e] = blk * B;                               // first slot of expert e
      for (int b = blk; b < blk + nblk && b < nb; ++b) block_to_expert[b] = e;
      blk += nblk;
    }
    for (int b = blk; b < nb; ++b) block_to_expert[b] = E - 1;        // unused tail blocks (all padding)
  }
  for (int e = tid; e < E; e += kMoeThreads) counts_out[e] = counts[e];
  __syncthreads();
  for (long chunk = 0; chunk < n; chunk += kMoeThreads) {
    for (int j = tid; j < 32 * E; j += kMoeThreads) wc[j / E][j % E] = 0;
    __syncthreads();
    const long i = chunk + tid;
    int e = -1;
    if (i < n) { e = (int)expert_index[i]; if (e < 0 || e >= E) e = -1; }
    const unsigned mask = __match_any_sync(0xffffffffu, e);
    const int rank_in_warp = __popc(mask & ((1u << lane) - 1u));
    if (e >= 0 && rank_in_warp == 0) wc[warp][e] = __popc(mask);
    __syncthreads();
    if (e >= 0) {
      int before = 0;
      for (int w = 0; w < warp; ++w) before += wc[w][e];
      const long slot = (long)base[e] + before + rank_in_warp;
      if (slot < (long)nb * B) tp2id[slot] = i / k;
    }
    __syncthreads();
    for (int ee = tid; ee < E; ee += kMoeThreads) {
      int tot = 0;
      for (int w = 0; w < 32; ++w) tot += wc[w][ee];
      base[ee] += tot;
    }
    __syncthreads();
  }
}

}  // namespace

void moe_block_metadata(const void* expert_index, bool idx64, long n, int k, int E, int B, int nb, long* block_to_expert, long* tp2id,
                        long* counts, cudaStream_t st) {
  if (E > kMoeMaxExperts) nxd_throw("moe_block_metadata: at most 256 experts", __FILE__, __LINE__);
  if (idx64) moe_block_metadata_kernel<long><<<1, kMoeThreads, 0, st>>>((const long*)expert_index, n, k, E, B, nb, block_to_expert, tp2id, counts);
  else moe_block_metadata_kernel<int><<<1, kMoeThreads, 0, st>>>((const int*)expert_index, n, k, E, B, nb, block_to_expert, tp2id, counts);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
