// Shared device helpers for the sm_90a kernels of neuronx_distributed_b200.
// Everything here is plain CUDA C++ + inline PTX (no CUTLASS/CuTe dependency).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define NXD_DEVICE __device__ __forceinline__

#define NXD_CUDA_CHECK(expr)                                                                     \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      nxd_throw(std::string(#expr) + " failed: " + cudaGetErrorString(_e), __FILE__, __LINE__);  \
    }                                                                                            \
  } while (0)

#ifdef __cplusplus
#include <stdexcept>
#include <string>
inline void nxd_throw(const std::string& msg, const char* file, int line) {
  throw std::runtime_error(msg + " (" + file + ":" + std::to_string(line) + ")");
}
#include <type_traits>
#endif

namespace nxd {

// f(std::integral_constant<int, HD>{}) for a runtime head dimension: the head sizes every attention kernel (flash forward and
// backward, decode, verification) is instantiated for.  `fn` names the caller in the error for any other size.
template <class F>
inline void dispatch_head_dim(int D, const char* fn, F&& f) {
  switch (D) {
    case 64: f(std::integral_constant<int, 64>{}); break;
    case 80: f(std::integral_constant<int, 80>{}); break;
    case 96: f(std::integral_constant<int, 96>{}); break;
    case 128: f(std::integral_constant<int, 128>{}); break;
    default: nxd_throw(std::string(fn) + ": head_dim must be 64, 80, 96 or 128", __FILE__, __LINE__);
  }
}

// f(std::integral_constant<int, G>{}) for a runtime GQA group size G = H / Hkv: the groups the token-generation kernels
// (decode, flash-decoding, verification) are instantiated for (ops.attention.DECODE_GQA_GROUPS).  They keep G query rows
// in registers, so G > 8 would spill.
template <class F>
inline void dispatch_gqa_group(int G, const char* fn, F&& f) {
  switch (G) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 3: f(std::integral_constant<int, 3>{}); break;
    case 4: f(std::integral_constant<int, 4>{}); break;
    case 5: f(std::integral_constant<int, 5>{}); break;
    case 6: f(std::integral_constant<int, 6>{}); break;
    case 7: f(std::integral_constant<int, 7>{}); break;
    case 8: f(std::integral_constant<int, 8>{}); break;
    default: nxd_throw(std::string(fn) + ": the GQA group size must be 1 to 8", __FILE__, __LINE__);
  }
}

// ---------------------------------------------------------------- type helpers
template <typename T> struct Vec8;  // 8 elements of a 16-bit type = 16 bytes
template <> struct Vec8<__nv_bfloat16> { uint4 raw; };
template <> struct Vec8<__half> { uint4 raw; };

template <typename T> NXD_DEVICE float to_f32(T v);
template <> NXD_DEVICE float to_f32<float>(float v) { return v; }
template <> NXD_DEVICE float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> NXD_DEVICE float to_f32<__half>(__half v) { return __half2float(v); }

template <typename T> NXD_DEVICE T from_f32(float v);
template <> NXD_DEVICE float from_f32<float>(float v) { return v; }
template <> NXD_DEVICE __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> NXD_DEVICE __half from_f32<__half>(float v) { return __float2half_rn(v); }

// A 16-byte packet of T (8 x 16-bit or 4 x 32-bit) with load/store + float conversion.
template <typename T> struct Pack16 {
  static constexpr int N = 16 / sizeof(T);
  T v[N];
  NXD_DEVICE void load(const T* p) { *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(p); }
  NXD_DEVICE void load_nc(const T* p) { *reinterpret_cast<uint4*>(v) = __ldg(reinterpret_cast<const uint4*>(p)); }
  NXD_DEVICE void store(T* p) const { *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(v); }
  NXD_DEVICE float f(int i) const { return to_f32<T>(v[i]); }
  NXD_DEVICE void set(int i, float x) { v[i] = from_f32<T>(x); }
};

NXD_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
NXD_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum; `smem` must hold >= 32 floats. All threads get the result.
NXD_DEVICE float block_sum(float v, float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? smem[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
NXD_DEVICE float block_max(float v, float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? smem[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

// ---------------------------------------------------------------- system-scope flags (NVLink peers)
NXD_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
NXD_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
NXD_DEVICE void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
NXD_DEVICE uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
NXD_DEVICE void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
// generic-proxy writes → visible to the async proxy (TMA) and vice versa
NXD_DEVICE void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
NXD_DEVICE void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// spin until *p >= target (monotonic epochs; wrap-safe signed compare)
NXD_DEVICE void wait_flag_ge(const uint32_t* p, uint32_t target) {
  while ((int32_t)(ld_acquire_sys(p) - target) < 0) { __nanosleep(64); }
}

}  // namespace nxd
