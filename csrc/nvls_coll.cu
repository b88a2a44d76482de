// Stand-alone collectives over an NVLS symmetric region (csrc/symm_vmm.cpp): one kernel each, no NCCL.
//   nvls_allreduce       latency-bound all-reduce (decode-time RowParallelLinear / ParallelEmbedding without sequence
//                        parallel; reference layers.py:1040-1043, mappings.py:196-211): every rank copies its vector into its
//                        OWN slot, one `multimem.red` per CTA signals all ranks at once, then every rank reads the in-switch
//                        sum with `multimem.ld_reduce` (fp32 accumulation) — one local write + one reduced read per element,
//                        versus world peer writes + world local reads in the unicast kernel (allreduce.cu).
//   nvls_all_gather      `multimem.st` of the local shard to all ranks + cross-rank CTA barrier.
//   nvls_reduce_scatter  `multimem.ld_reduce` of this rank's chunk of a symmetric input.
// All three are CUDA-graph capturable: the call counter (epoch) lives in device memory and is advanced by the last CTA.
// Region layout is chosen by the caller (ops/nvls.py): `flag_off` = kNvlsCollMaxCtas u32 barrier counters, payload
// double-buffered by epoch parity.  With `mc_base == nullptr` the kernels use unicast peer accesses (same protocol).
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace nxd {

constexpr int kNvlsCollMaxCtas = 1024;

NXD_DEVICE void mm_red_add_release_u32(uint32_t* mc, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
NXD_DEVICE void mm_st_v4(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
               ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
template <typename T> NXD_DEVICE uint4 mm_ld_reduce(const void* mc);
template <> NXD_DEVICE uint4 mm_ld_reduce<__nv_bfloat16>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
template <> NXD_DEVICE uint4 mm_ld_reduce<float>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}

struct NvlsRegion {
  const int64_t* peer_bases;   // [world] unicast VAs
  uint8_t* mc_base;            // multicast VA or nullptr
  uint8_t* local_base;
  long flag_off;               // kNvlsCollMaxCtas u32 counters
  long data_off;               // payload: 2 parity halves of `half_bytes`
  long half_bytes;
  int rank, world;
};

// Cross-rank barrier between CTA `blockIdx.x` of every rank: counter[cta] += 1 on all ranks, wait until it shows `world`
// arrivals for this CTA's n-th barrier (n is kept per CTA in state[2 + cta], so calls may use different grid sizes as long
// as every rank uses the same one).  Caller has fenced its payload writes (fence.sys) and synchronised the CTA.
NXD_DEVICE void cta_barrier_all_ranks(const NvlsRegion& r, uint32_t* state) {
  if (r.mc_base != nullptr) {
    if (threadIdx.x == 0) mm_red_add_release_u32((uint32_t*)(r.mc_base + r.flag_off) + blockIdx.x, 1u);
  } else if ((int)threadIdx.x < r.world) {
    red_add_release_sys((uint32_t*)((uint8_t*)r.peer_bases[threadIdx.x] + r.flag_off) + blockIdx.x, 1u);
  }
  if (threadIdx.x == 0) {
    const uint32_t n = state[2 + blockIdx.x] + 1u;
    state[2 + blockIdx.x] = n;
    wait_flag_ge((const uint32_t*)(r.local_base + r.flag_off) + blockIdx.x, n * (uint32_t)r.world);
  }
  __syncthreads();
}

NXD_DEVICE void finish_call(uint32_t* state, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(state + 1, 1u) == gridDim.x - 1) {
      state[1] = 0;
      __threadfence();
      st_release_sys(state, epoch);
    }
  }
}

// out = sum over ranks of x (+ residual).  numel * sizeof(T) multiple of 16 and <= half_bytes.
template <typename T>
__global__ void __launch_bounds__(512) nvls_allreduce_kernel(const T* __restrict__ x, const T* __restrict__ residual,
                                                             T* __restrict__ out, NvlsRegion r, uint32_t* __restrict__ state,
                                                             long numel) {
  const uint32_t epoch = ld_acquire_sys(state) + 1u;
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  constexpr int VEC = 16 / sizeof(T);
  const long nvec = numel / VEC;
  const long per_cta = (nvec + gridDim.x - 1) / gridDim.x;
  const long v0 = (long)blockIdx.x * per_cta, v1 = min(nvec, v0 + per_cta);
  uint4* mine = (uint4*)(r.local_base + base);
  for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) mine[v] = ((const uint4*)x)[v];
  __threadfence_system();
  __syncthreads();
  cta_barrier_all_ranks(r, state);
  for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
    uint4 o;
    if (r.mc_base != nullptr) {
      o = mm_ld_reduce<T>(r.mc_base + base + v * 16);
    } else {
      float acc[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
      for (int p = 0; p < r.world; ++p) {
        uint4 raw;
        const void* src = (const uint8_t*)r.peer_bases[p] + base + v * 16;
        asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(raw.x), "=r"(raw.y), "=r"(raw.z), "=r"(raw.w) : "l"(src) : "memory");
        const T* e = (const T*)&raw;
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] += to_f32<T>(e[j]);
      }
      T* oe = (T*)&o;
#pragma unroll
      for (int j = 0; j < VEC; ++j) oe[j] = from_f32<T>(acc[j]);
    }
    if (residual != nullptr) {
      const uint4 rr = ((const uint4*)residual)[v];
      const T* re = (const T*)&rr;
      T* oe = (T*)&o;
#pragma unroll
      for (int j = 0; j < VEC; ++j) oe[j] = from_f32<T>(to_f32<T>(oe[j]) + to_f32<T>(re[j]));
    }
    ((uint4*)out)[v] = o;
  }
  finish_call(state, epoch);
}

// Every rank contributes `bytes` (multiple of 16); afterwards payload[parity][p*bytes .. ) holds rank p's data on all ranks.
// `out` (optional) receives a private copy of the gathered buffer.
__global__ void __launch_bounds__(512) nvls_all_gather_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ out,
                                                              NvlsRegion r, uint32_t* __restrict__ state, long bytes) {
  const uint32_t epoch = ld_acquire_sys(state) + 1u;
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  const long nvec = bytes / 16;
  const long per_cta = (nvec + gridDim.x - 1) / gridDim.x;
  const long v0 = (long)blockIdx.x * per_cta, v1 = min(nvec, v0 + per_cta);
  const long dst_off = base + (long)r.rank * bytes;
  constexpr int U = 4;
  for (long b = v0 + threadIdx.x; b < v1; b += (long)U * blockDim.x) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const long i = b + (long)u * blockDim.x; if (i < v1) v[u] = ((const uint4*)x)[i]; }
    if (r.mc_base != nullptr) {
#pragma unroll
      for (int u = 0; u < U; ++u) { const long i = b + (long)u * blockDim.x; if (i < v1) mm_st_v4(r.mc_base + dst_off + i * 16, v[u]); }
    } else {
      for (int p = 0; p < r.world; ++p) {
        uint4* d = (uint4*)((uint8_t*)r.peer_bases[p] + dst_off);
#pragma unroll
        for (int u = 0; u < U; ++u) { const long i = b + (long)u * blockDim.x; if (i < v1) d[i] = v[u]; }
      }
    }
  }
  __threadfence_system();
  __syncthreads();
  cta_barrier_all_ranks(r, state);
  if (out != nullptr) {
    // slice [v0, v1) of every rank's contribution has landed (CTA i of every rank moved the same slice)
    for (int p = 0; p < r.world; ++p) {
      const uint4* s = (const uint4*)(r.local_base + base + (long)p * bytes);
      uint4* d = (uint4*)(out + (long)p * bytes);
      for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
        uint4 t;
        asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(s + v) : "memory");
        d[v] = t;
      }
    }
  }
  finish_call(state, epoch);
}

// x = [world * chunk] elements on every rank; out[chunk] = sum over ranks of x[rank*chunk .. (rank+1)*chunk).
template <typename T>
__global__ void __launch_bounds__(512) nvls_reduce_scatter_kernel(const T* __restrict__ x, T* __restrict__ out, NvlsRegion r,
                                                                  uint32_t* __restrict__ state, long chunk) {
  const uint32_t epoch = ld_acquire_sys(state) + 1u;
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  constexpr int VEC = 16 / sizeof(T);
  const long cvec = chunk / VEC;
  const long per_cta = (cvec + gridDim.x - 1) / gridDim.x;
  const long v0 = (long)blockIdx.x * per_cta, v1 = min(cvec, v0 + per_cta);
  // copy slice [v0, v1) of EVERY chunk into the own slot: CTA i of rank q later reads slice i of chunk q from all ranks
  for (int p = 0; p < r.world; ++p) {
    const uint4* s = (const uint4*)x + (long)p * cvec;
    uint4* d = (uint4*)(r.local_base + base) + (long)p * cvec;
    for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) d[v] = s[v];
  }
  __threadfence_system();
  __syncthreads();
  cta_barrier_all_ranks(r, state);
  const long my = base + (long)r.rank * chunk * (long)sizeof(T);
  for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
    uint4 o;
    if (r.mc_base != nullptr) {
      o = mm_ld_reduce<T>(r.mc_base + my + v * 16);
    } else {
      float acc[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
      for (int p = 0; p < r.world; ++p) {
        uint4 raw;
        const void* src = (const uint8_t*)r.peer_bases[p] + my + v * 16;
        asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(raw.x), "=r"(raw.y), "=r"(raw.z), "=r"(raw.w) : "l"(src) : "memory");
        const T* e = (const T*)&raw;
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] += to_f32<T>(e[j]);
      }
      T* oe = (T*)&o;
#pragma unroll
      for (int j = 0; j < VEC; ++j) oe[j] = from_f32<T>(acc[j]);
    }
    ((uint4*)out)[v] = o;
  }
  finish_call(state, epoch);
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused decode-time GEMV → all-reduce (RowParallelLinear without sequence parallel at batch 1..8: o_proj / down_proj of every
// layer; reference layers.py:1040-1043).  y[M<=8, N] = sum over ranks of x_r[M, K] · W_r[N, K]ᵀ (+ residual).
// One warp per output column streams its weight row once (16-byte loads, fp32 accumulation), the fp32 partials go to this
// rank's OWN symmetric slot, CTA i of every rank meets in a cross-rank barrier (one multimem.red per CTA), and the same CTA
// then reads the in-switch fp32 sum of its columns with multimem.ld_reduce — one launch instead of GEMV + copy-in +
// all-reduce, partials never rounded to bf16 (the reference's reduce_dtype=fp32).
template <int M>
__global__ void __launch_bounds__(256) gemv_allreduce_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                             const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ y,
                                                             int N, int K, NvlsRegion r, uint32_t* __restrict__ state) {
  const uint32_t epoch = ld_acquire_sys(state) + 1u;
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  float* slot = (float*)(r.local_base + base);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = (N + 7) / 8;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    const int n = g * 8 + warp;
    if (n >= N) continue;
    float acc[M];
#pragma unroll
    for (int m = 0; m < M; ++m) acc[m] = 0.f;
    const __nv_bfloat16* wr = w + (long)n * K;
#pragma unroll 4
    for (int k = lane * 8; k < K; k += 256) {
      const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + k));
      const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(&wv);
      float wf[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(w2[i]); wf[2 * i] = f.x; wf[2 * i + 1] = f.y; }
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const uint4 xv = *reinterpret_cast<const uint4*>(x + (long)m * K + k);
        const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&xv);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __bfloat1622float2(x2[i]);
          acc[m] = fmaf(f.x, wf[2 * i], acc[m]);
          acc[m] = fmaf(f.y, wf[2 * i + 1], acc[m]);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const float v = warp_sum(acc[m]);
      if (lane == 0) slot[(long)m * N + n] = v;
    }
  }
  __threadfence_system();
  __syncthreads();
  cta_barrier_all_ranks(r, state);
  // reduce the same column groups: thread t handles (row t/2, 4 columns of the group's 8)
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    if ((int)threadIdx.x < 2 * M) {
      const int m = threadIdx.x >> 1, c0 = g * 8 + (threadIdx.x & 1) * 4;
      if (c0 < N) {                                     // N % 4 == 0 (checked by the launcher)
        const long off = base + ((long)m * N + c0) * 4;
        float4 v;
        if (r.mc_base != nullptr) {
          const uint4 raw = mm_ld_reduce<float>(r.mc_base + off);
          v = make_float4(__uint_as_float(raw.x), __uint_as_float(raw.y), __uint_as_float(raw.z), __uint_as_float(raw.w));
        } else {
          v = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int p = 0; p < r.world; ++p) {
            uint4 raw;
            const void* src = (const uint8_t*)r.peer_bases[p] + off;
            asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(raw.x), "=r"(raw.y), "=r"(raw.z), "=r"(raw.w) : "l"(src) : "memory");
            v.x += __uint_as_float(raw.x); v.y += __uint_as_float(raw.y); v.z += __uint_as_float(raw.z); v.w += __uint_as_float(raw.w);
          }
        }
        if (residual != nullptr) {
          const uint2 rr = *reinterpret_cast<const uint2*>(residual + (long)m * N + c0);
          const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&rr);
          const float2 a = __bfloat1622float2(r2[0]), b = __bfloat1622float2(r2[1]);
          v.x += a.x; v.y += a.y; v.z += b.x; v.w += b.y;
        }
        uint2 o;
        __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
        o2[0] = __floats2bfloat162_rn(v.x, v.y);
        o2[1] = __floats2bfloat162_rn(v.z, v.w);
        *reinterpret_cast<uint2*>(y + (long)m * N + c0) = o;
      }
    }
  }
  finish_call(state, epoch);
}

// ---- vocab-parallel embedding lookup for a sequence-parallel consumer (SURVEY §7.4 `embedding_rs`) -------------------------
// The reference looks every token up in the local vocab shard (zero rows for foreign ids), producing the full [S, B, H]
// partial, and reduce-scatters it (layers.py:334-378): S·B·H elements written, masked and pushed through a collective although
// every output row has exactly ONE non-zero contributor.  With NVSwitch peer memory the lookup itself can be remote:
//   1. nvls_publish_kernel      every rank copies its table shard into its symmetric slot (parity by call) and meets the same CTA
//                               of every other rank; when the kernel has finished on a rank, all shards are visible to it;
//   2. peer_row_gather_kernel   one warp per token of THIS rank's sequence shard loads the row from the owner's slot over
//                               NVLink (16-byte loads) and stores it locally.  No reduction, S/tp·B·H elements moved once.
__global__ void __launch_bounds__(512) nvls_publish_kernel(const uint8_t* __restrict__ x, NvlsRegion r, uint32_t* __restrict__ state,
                                                           long bytes, int forced_parity) {
  // forced_parity >= 0: the host chose the half (it needs the address to build views / TMA maps of the peers' copies);
  // otherwise the half follows the device-side call counter (CUDA-graph capturable)
  const uint32_t epoch = ld_acquire_sys(state) + 1u;
  const long base = r.data_off + (long)(forced_parity >= 0 ? (uint32_t)forced_parity : (epoch & 1u)) * r.half_bytes;
  const long nvec = bytes / 16;
  const long per_cta = (nvec + gridDim.x - 1) / gridDim.x;
  const long v0 = (long)blockIdx.x * per_cta, v1 = min(nvec, v0 + per_cta);
  uint4* mine = (uint4*)(r.local_base + base);
  for (long v = v0 + threadIdx.x; v < v1; v += blockDim.x) mine[v] = ((const uint4*)x)[v];
  __threadfence_system();
  __syncthreads();
  cta_barrier_all_ranks(r, state);
  finish_call(state, epoch);
}

__global__ void __launch_bounds__(256) peer_row_gather_kernel(const long* __restrict__ ids, uint8_t* __restrict__ out, NvlsRegion r,
                                                              const uint32_t* __restrict__ state, long rows_per_rank, long row_bytes,
                                                              long ntok) {
  const uint32_t epoch = ld_acquire_sys(state);                    // the publish kernel of this call has advanced it
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long t = warp; t < ntok; t += nwarps) {
    const long id = ids[t];
    const long owner = id / rows_per_rank;
    uint4* dst = (uint4*)(out + t * row_bytes);
    if (id < 0 || owner >= r.world) {                              // not a vocabulary id: zero row (what the masked lookup gives)
      for (long i = lane; i < row_bytes / 16; i += 32) dst[i] = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const uint4* src = (const uint4*)((const uint8_t*)r.peer_bases[owner] + base + (id - owner * rows_per_rank) * row_bytes);
    for (long i = lane; i < row_bytes / 16; i += 32) {
      uint4 v;
      asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i) : "memory");
      dst[i] = v;
    }
  }
}

// ---- all-to-all with equal splits (EP dispatch / combine; reference mappings.py:160-172 `xm.all_to_all`) ----------------------
// After `nvls_publish_kernel` every rank's whole send buffer [world][chunk] sits in its slot; rank r pulls chunk r of every peer
// straight into its output (16-byte loads over NVLink, all peers in flight at once): out[p] = send_p[r].
__global__ void __launch_bounds__(512) peer_chunk_pull_kernel(uint8_t* __restrict__ out, NvlsRegion r, const uint32_t* __restrict__ state,
                                                              long chunk_bytes) {
  const uint32_t epoch = ld_acquire_sys(state);
  const long base = r.data_off + (long)(epoch & 1u) * r.half_bytes;
  const long nvec = chunk_bytes / 16, total = nvec * r.world;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i / nvec);
    const long v = i - (long)p * nvec;
    const uint4* src = (const uint4*)((const uint8_t*)r.peer_bases[p] + base + (long)r.rank * chunk_bytes) + v;
    uint4 t;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(src) : "memory");
    ((uint4*)(out + (long)p * chunk_bytes))[v] = t;
  }
}

static NvlsRegion make_region(const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off, long data_off,
                              long half_bytes, int rank, int world) {
  NvlsRegion r;
  r.peer_bases = peer_bases; r.mc_base = (uint8_t*)mc_base; r.local_base = (uint8_t*)local_base; r.flag_off = flag_off;
  r.data_off = data_off; r.half_bytes = half_bytes; r.rank = rank; r.world = world;
  return r;
}

void nvls_allreduce(const void* x, const void* residual, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base,
                    long flag_off, long data_off, long half_bytes, uint32_t* state, int rank, int world, long numel, int dt,
                    int ctas, cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  const long bytes = numel * (dt == kF32 ? 4 : 2);
  if (bytes % 16 || bytes > half_bytes) nxd_throw("nvls_allreduce: size must be a multiple of 16 bytes and fit the slot", __FILE__, __LINE__);
  if (dt == kBF16)
    nvls_allreduce_kernel<__nv_bfloat16><<<ctas, 512, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)residual,
                                                               (__nv_bfloat16*)out, r, state, numel);
  else if (dt == kF32)
    nvls_allreduce_kernel<float><<<ctas, 512, 0, st>>>((const float*)x, (const float*)residual, (float*)out, r, state, numel);
  else
    nxd_throw("nvls_allreduce: bf16 or fp32 only", __FILE__, __LINE__);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void gemv_allreduce(const void* x, const void* w, const void* residual, void* y, int M, int N, int K, const int64_t* peer_bases,
                    int64_t mc_base, int64_t local_base, long flag_off, long data_off, long half_bytes, uint32_t* state, int rank,
                    int world, int max_ctas, cudaStream_t st) {
  if (N % 8 || K % 8 || (long)M * N * 4 > half_bytes) nxd_throw("gemv_allreduce: N, K multiples of 8 and M*N*4 bytes within the slot", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  int grid = (N + 7) / 8;
  if (grid > max_ctas) grid = max_ctas;                  // every CTA must be resident: they meet in a cross-rank barrier
  if (grid > kNvlsCollMaxCtas) grid = kNvlsCollMaxCtas;
#define NXD_GAR(Mv)                                                                                                       \
  gemv_allreduce_kernel<Mv><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)residual, \
                                                  (__nv_bfloat16*)y, N, K, r, state)
  switch (M) {
    case 1: NXD_GAR(1); break;
    case 2: NXD_GAR(2); break;
    case 3: NXD_GAR(3); break;
    case 4: NXD_GAR(4); break;
    case 5: NXD_GAR(5); break;
    case 6: NXD_GAR(6); break;
    case 7: NXD_GAR(7); break;
    case 8: NXD_GAR(8); break;
    default: nxd_throw("gemv_allreduce: M must be 1..8", __FILE__, __LINE__);
  }
#undef NXD_GAR
  NXD_CUDA_CHECK(cudaGetLastError());
}

void nvls_all_gather(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                     long data_off, long half_bytes, uint32_t* state, int rank, int world, long bytes, int ctas, cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  if (bytes % 16 || bytes * world > half_bytes) nxd_throw("nvls_all_gather: bad size", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  nvls_all_gather_kernel<<<ctas, 512, 0, st>>>((const uint8_t*)x, (uint8_t*)out, r, state, bytes);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void nvls_reduce_scatter(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                         long data_off, long half_bytes, uint32_t* state, int rank, int world, long chunk_numel, int dt, int ctas,
                         cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  const long bytes = chunk_numel * (dt == kF32 ? 4 : 2);
  if (bytes % 16 || bytes * world > half_bytes) nxd_throw("nvls_reduce_scatter: bad size", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  if (dt == kBF16)
    nvls_reduce_scatter_kernel<__nv_bfloat16><<<ctas, 512, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)out, r, state, chunk_numel);
  else if (dt == kF32)
    nvls_reduce_scatter_kernel<float><<<ctas, 512, 0, st>>>((const float*)x, (float*)out, r, state, chunk_numel);
  else
    nxd_throw("nvls_reduce_scatter: bf16 or fp32 only", __FILE__, __LINE__);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd

namespace nxd {

void nvls_all_to_all(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                     long data_off, long half_bytes, uint32_t* state, int rank, int world, long bytes, int ctas, cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  if (bytes % (16L * world) || bytes > half_bytes) nxd_throw("nvls_all_to_all: per-peer chunks of 16-byte multiples, buffer must fit the slot", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  nvls_publish_kernel<<<ctas, 512, 0, st>>>((const uint8_t*)x, r, state, bytes, -1);
  peer_chunk_pull_kernel<<<ctas, 512, 0, st>>>((uint8_t*)out, r, state, bytes / world);
  NXD_CUDA_CHECK(cudaGetLastError());
}

// Copy `x` into this rank's half `parity` of the slot and meet every rank: after the kernel, every peer's copy can be read at
// peer_base + data_off + parity * half_bytes (e.g. by the attention kernel's TMA loads: context-parallel attention without a ring).
void nvls_publish(const void* x, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off, long data_off,
                  long half_bytes, uint32_t* state, int rank, int world, long bytes, int parity, int ctas, cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  if (bytes % 16 || bytes > half_bytes) nxd_throw("nvls_publish: multiple of 16 bytes that fits the slot", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  nvls_publish_kernel<<<ctas, 512, 0, st>>>((const uint8_t*)x, r, state, bytes, parity);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void nvls_embedding_gather(const void* table, const long* ids, void* out, const int64_t* peer_bases, int64_t mc_base,
                           int64_t local_base, long flag_off, long data_off, long half_bytes, uint32_t* state, int rank, int world,
                           long rows_per_rank, long row_bytes, long ntok, int ctas, cudaStream_t st) {
  if (ctas > kNvlsCollMaxCtas) ctas = kNvlsCollMaxCtas;
  const long bytes = rows_per_rank * row_bytes;
  if (row_bytes % 16 || bytes > half_bytes) nxd_throw("nvls_embedding_gather: rows of 16-byte multiples, shard must fit the slot", __FILE__, __LINE__);
  const NvlsRegion r = make_region(peer_bases, mc_base, local_base, flag_off, data_off, half_bytes, rank, world);
  nvls_publish_kernel<<<ctas, 512, 0, st>>>((const uint8_t*)table, r, state, bytes, -1);
  NXD_CUDA_CHECK(cudaGetLastError());
  if (ntok > 0) {
    const int grid = (int)std::min<long>((ntok + 7) / 8, 132L * 8);     // 8 CTAs per H100 SM
    peer_row_gather_kernel<<<grid, 256, 0, st>>>(ids, (uint8_t*)out, r, state, rows_per_rank, row_bytes, ntok);
    NXD_CUDA_CHECK(cudaGetLastError());
  }
}

}  // namespace nxd
