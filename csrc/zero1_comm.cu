// ZeRO-1 data-parallel collectives over NVLink peer memory (no NCCL):
//   zero1_reduce_scatter : every rank PULLS its contiguous shard of the flat gradient buffer from all peers' symmetric
//                          buffers, sums in fp32, applies the 1/dp (and optional clip) scale and writes its fp32 shard —
//                          bucket cast + scale + reduce-scatter in one kernel (reference: torch_xla ZeRO reduce-scatter in
//                          coalesced fp32 buckets, trainer.py:258-285).
//   zero1_all_gather     : every rank PUSHES its updated fp32 master shard, cast to the model dtype on the fly, into all
//                          peers' flat parameter buffers (all-gather fused with the fp32→bf16 cast).
// Cross-rank ordering uses epoch flags in the symmetric flag region: an entry barrier ("my gradients are final") and an exit
// barrier ("I no longer read/you have received everything").
#include "common.cuh"
#include "kernels.h"

namespace nxd {

// all threads of all blocks call; thread p < world of every block spins on flag p
NXD_DEVICE void cross_rank_wait(const uint32_t* my_flags, int world, uint32_t epoch) {
  if ((int)threadIdx.x < world) wait_flag_ge(my_flags + threadIdx.x, epoch);
  __syncthreads();
}

template <typename G>
__global__ void __launch_bounds__(512) zero1_rs_kernel(const int64_t* __restrict__ peer_bufs, long grad_off_bytes,
                                                       const int64_t* __restrict__ peer_flags, int flag_off, uint32_t epoch,
                                                       int rank, int world, long shard_numel, long sub_begin,
                                                       long sub_len, float scale, float* __restrict__ out,
                                                       uint32_t* __restrict__ done_ctr) {
  // [sub_begin, sub_begin + sub_len) of this rank's shard is reduced (bucketed calls overlap the backward pass; a rank
  // whose shard does not intersect the bucket passes sub_len = 0 and only takes part in the two barriers)
  // ---- entry barrier: tell every peer my gradient buffer is final, wait until all peers said so ----
  if (blockIdx.x == 0 && (int)threadIdx.x < world) {
    __threadfence_system();
    st_release_sys((uint32_t*)peer_flags[threadIdx.x] + flag_off + rank, epoch);
  }
  cross_rank_wait((const uint32_t*)peer_flags[rank] + flag_off, world, epoch);

  constexpr int VEC = 16 / sizeof(G);
  const long nvec = sub_len / VEC;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
    // issue all peers' loads before consuming any (world independent 16-byte loads in flight)
    uint4 raw[8];
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      if (p < world) {
        const int src = (rank + p) % world;      // start with the local copy, spread peers across ranks
        const G* base = (const G*)((const uint8_t*)peer_bufs[src] + grad_off_bytes) + (long)rank * shard_numel + sub_begin;
        raw[p] = *(const uint4*)(base + v * VEC);
      }
    }
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      if (p < world) {
        const G* g = (const G*)&raw[p];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] += to_f32<G>(g[j]);
      }
    }
    float* o = out + sub_begin + v * VEC;
#pragma unroll
    for (int j = 0; j < VEC; j += 4)
      *(float4*)(o + j) = make_float4(acc[j] * scale, acc[j + 1] * scale, acc[j + 2] * scale, acc[j + 3] * scale);
  }
  // ---- exit barrier: peers may overwrite their gradient buffers only after everyone finished reading ----
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(done_ctr, 1u) == gridDim.x - 1);
  __syncthreads();
  if (last) {
    if (threadIdx.x == 0) *done_ctr = 0;
    if ((int)threadIdx.x < world) st_release_sys((uint32_t*)peer_flags[threadIdx.x] + flag_off + 8 + rank, epoch);
    cross_rank_wait((const uint32_t*)peer_flags[rank] + flag_off + 8, world, epoch);
  }
}

template <typename P>
__global__ void __launch_bounds__(512) zero1_ag_kernel(const float* __restrict__ master, const int64_t* __restrict__ peer_bufs,
                                                       long param_off_bytes, const int64_t* __restrict__ peer_flags,
                                                       int flag_off, uint32_t epoch, int rank, int world, long shard_numel,
                                                       uint32_t* __restrict__ done_ctr) {
  constexpr int VEC = 8;   // 8 fp32 in → 8 elements out
  const long nvec = shard_numel / VEC;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const float4 a = *(const float4*)(master + v * VEC), b = *(const float4*)(master + v * VEC + 4);
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    if constexpr (sizeof(P) == 2) {
      uint4 o; P* h = (P*)&o;
#pragma unroll
      for (int j = 0; j < 8; ++j) h[j] = from_f32<P>(f[j]);
      for (int p = 0; p < world; ++p) {
        const int dst = (rank + p) % world;
        P* base = (P*)((uint8_t*)peer_bufs[dst] + param_off_bytes) + (long)rank * shard_numel;
        *(uint4*)(base + v * VEC) = o;
      }
    } else {
      for (int p = 0; p < world; ++p) {
        const int dst = (rank + p) % world;
        float* base = (float*)((uint8_t*)peer_bufs[dst] + param_off_bytes) + (long)rank * shard_numel;
        *(float4*)(base + v * VEC) = a;
        *(float4*)(base + v * VEC + 4) = b;
      }
    }
  }
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(done_ctr, 1u) == gridDim.x - 1);
  __syncthreads();
  if (last) {
    if (threadIdx.x == 0) *done_ctr = 0;
    if ((int)threadIdx.x < world) st_release_sys((uint32_t*)peer_flags[threadIdx.x] + flag_off + 16 + rank, epoch);
    cross_rank_wait((const uint32_t*)peer_flags[rank] + flag_off + 16, world, epoch);
  }
}

static int sms() {
  static int n = 0;
  if (!n) { int dev; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
  return n;
}

void zero1_reduce_scatter(const int64_t* peer_bufs, long grad_off_bytes, const int64_t* peer_flags, int flag_off,
                          uint32_t epoch, int rank, int world, long shard_numel, long sub_begin, long sub_len, float scale,
                          float* out, uint32_t* done_ctr, int grad_dt, int max_ctas, cudaStream_t st) {
  if (world > 8) nxd_throw("zero1 kernels support up to 8 ranks per group", __FILE__, __LINE__);
  // one CTA per SM by default; overlapped (bucketed) calls pass a small max_ctas so the backward GEMMs keep the SMs
  const int grid = max_ctas > 0 && max_ctas < sms() ? max_ctas : sms();
  if (grad_dt == kF32)
    zero1_rs_kernel<float><<<grid, 512, 0, st>>>(peer_bufs, grad_off_bytes, peer_flags, flag_off, epoch, rank, world,
                                                 shard_numel, sub_begin, sub_len, scale, out, done_ctr);
  else
    zero1_rs_kernel<__nv_bfloat16><<<grid, 512, 0, st>>>(peer_bufs, grad_off_bytes, peer_flags, flag_off, epoch, rank, world,
                                                         shard_numel, sub_begin, sub_len, scale, out, done_ctr);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void zero1_all_gather(const float* master, const int64_t* peer_bufs, long param_off_bytes, const int64_t* peer_flags,
                      int flag_off, uint32_t epoch, int rank, int world, long shard_numel, uint32_t* done_ctr, int param_dt,
                      cudaStream_t st) {
  if (world > 8) nxd_throw("zero1 kernels support up to 8 ranks per group", __FILE__, __LINE__);
  const int grid = sms();
  if (param_dt == kBF16)
    zero1_ag_kernel<__nv_bfloat16><<<grid, 512, 0, st>>>(master, peer_bufs, param_off_bytes, peer_flags, flag_off, epoch, rank,
                                                         world, shard_numel, done_ctr);
  else
    zero1_ag_kernel<float><<<grid, 512, 0, st>>>(master, peer_bufs, param_off_bytes, peer_flags, flag_off, epoch, rank, world,
                                                 shard_numel, done_ctr);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
