// Residual-add fused with RMSNorm (sm_90a, HBM-bound: one pass, 16-byte accesses, fp32 math).
//
//   forward :  h = x + r                      (the updated residual stream, written once)
//              y = h * rsqrt(mean(h^2) + eps) * w
//   backward:  dh = gh + rstd * (gy*w - hhat * mean_H(gy*w*hhat))     (gh: gradient arriving on the residual path)
//              dw = sum_rows gy * hhat                                   dx = dr = dh
//
// Unfused this is an add kernel (read x, r; write h) plus the norm (read h; write y) = 5 row passes forward and, backward,
// the norm backward (read gy, h; write d) plus an add (read d, gh; write dh) = 6; fused: 4 and 4.
// The norm math is the one of elementwise.cu (rmsnorm_fwd_kernel / rmsnorm_bwd_kernel); h is rounded to the storage dtype
// BEFORE the statistics so that y is exactly rmsnorm(h_stored), i.e. bit-compatible with the unfused sequence.
#include "common.cuh"
#include "kernels.h"

namespace nxd {

template <typename T, int MAXV, bool WIDE>
__global__ void __launch_bounds__(256) add_rmsnorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ r,
                                                              const T* __restrict__ w, T* __restrict__ h,
                                                              T* __restrict__ y, float* __restrict__ rstd_out, int H,
                                                              float eps) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  __shared__ float red[32];
  const int row = blockIdx.x;
  const size_t base = (size_t)row * H;
  const int nvec = H / N;
  P cache[MAXV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
    if (v < nvec) {
      P px, pr;
      px.load(x + base + v * N);
      pr.load(r + base + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        cache[i].set(j, px.f(j) + pr.f(j));
        const float f = cache[i].f(j);          // the rounded value: statistics of what is stored
        ss += f * f;
      }
      cache[i].store(h + base + v * N);
    }
  }
  // tail beyond the register cache (very wide rows): h is re-read in the second pass, as rmsnorm_fwd_kernel re-reads x
  for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
    P px, pr, ph;
    px.load(x + base + v * N);
    pr.load(r + base + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      ph.set(j, px.f(j) + pr.f(j));
      const float f = ph.f(j);
      ss += f * f;
    }
    ph.store(h + base + v * N);
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0) rstd_out[row] = rstd;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
    if (v < nvec) {
      P pw, po;
      pw.load_nc(w + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) po.set(j, cache[i].f(j) * rstd * pw.f(j));
      po.store(y + base + v * N);
    }
  }
  for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
    P ph, pw, po;
    ph.load(h + base + v * N);
    pw.load_nc(w + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) po.set(j, ph.f(j) * rstd * pw.f(j));
    po.store(y + base + v * N);
  }
}

// Persistent CTAs stride over rows; each thread owns fixed columns so the dW partial lives in registers across rows.
// Packets beyond the register cache are re-read and accumulate dW in place in the CTA's own partial row.
template <typename T, int MAXV, bool WIDE>
__global__ void __launch_bounds__(256) add_rmsnorm_bwd_kernel(const T* __restrict__ gy, const T* __restrict__ gh,
                                                              const T* __restrict__ h, const T* __restrict__ w,
                                                              const float* __restrict__ rstd, T* __restrict__ dh,
                                                              float* __restrict__ partial_dw, int rows, int H) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  __shared__ float red[32];
  const int nvec = H / N;
  float* pdw = partial_dw + (size_t)blockIdx.x * H;
  float dw[MAXV][N];
  P pw[MAXV];
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
#pragma unroll
    for (int j = 0; j < N; ++j) dw[i][j] = 0.f;
    if (v < nvec) pw[i].load_nc(w + v * N);
  }
  for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x)
#pragma unroll
    for (int j = 0; j < N; ++j) pdw[v * N + j] = 0.f;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const size_t base = (size_t)row * H;
    const float rs = rstd[row];
    P ph[MAXV], pg[MAXV];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = threadIdx.x + i * blockDim.x;
      if (v < nvec) {
        ph[i].load(h + base + v * N);
        pg[i].load(gy + base + v * N);
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float hh = ph[i].f(j) * rs, gg = pg[i].f(j);
          dot += gg * pw[i].f(j) * hh;
          dw[i][j] += gg * hh;
        }
      }
    }
    for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
      P qh, qg, qw; qh.load(h + base + v * N); qg.load(gy + base + v * N); qw.load_nc(w + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) { const float hh = qh.f(j) * rs; dot += qg.f(j) * qw.f(j) * hh; }
    }
    dot = block_sum(dot, red) / (float)H;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = threadIdx.x + i * blockDim.x;
      if (v < nvec) {
        P pr, po;
        pr.load(gh + base + v * N);
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float hh = ph[i].f(j) * rs;
          po.set(j, pr.f(j) + rs * (pg[i].f(j) * pw[i].f(j) - hh * dot));
        }
        po.store(dh + base + v * N);
      }
    }
    for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
      P qh, qg, qw, pr, po;
      qh.load(h + base + v * N); qg.load(gy + base + v * N); qw.load_nc(w + v * N); pr.load(gh + base + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float hh = qh.f(j) * rs, gg = qg.f(j);
        po.set(j, pr.f(j) + rs * (gg * qw.f(j) - hh * dot));
        pdw[v * N + j] += gg * hh;
      }
      po.store(dh + base + v * N);
    }
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
    if (v < nvec) {
#pragma unroll
      for (int j = 0; j < N; ++j) pdw[v * N + j] = dw[i][j];
    }
  }
}

static __global__ void fused_norm_reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                         int nparts, int H) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float s = 0.f;
  for (int p = 0; p < nparts; ++p) s += partial[(size_t)p * H + c];
  out[c] = s;
}

template <typename T> static int fn_pick_threads(int H) {
  const int nvec = H / Pack16<T>::N;
  int t = 32;
  while (t < 256 && t * 4 < nvec) t <<= 1;
  return t;
}

#define FN_DISPATCH_DTYPE(dt, ...)                                      \
  switch (dt) {                                                         \
    case kF32: { using T = float; __VA_ARGS__; break; }                 \
    case kBF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }        \
    case kF16: { using T = __half; __VA_ARGS__; break; }                \
    default: nxd_throw("unsupported dtype", __FILE__, __LINE__);        \
  }

void add_rmsnorm_fwd(const void* x, const void* r, const void* w, void* h, void* y, float* rstd, int rows, int H,
                     float eps, int dt, cudaStream_t st) {
  FN_DISPATCH_DTYPE(dt, {
    if (H % Pack16<T>::N) nxd_throw("add_rmsnorm: H must be a multiple of the 16-byte vector width", __FILE__, __LINE__);
    const int th = fn_pick_threads<T>(H);
    // the wide-row loops cost registers (one CTA per SM fewer), so rows that fit the register cache do not carry them
    if (H / Pack16<T>::N > 4 * th)
      add_rmsnorm_fwd_kernel<T, 4, true><<<rows, th, 0, st>>>((const T*)x, (const T*)r, (const T*)w, (T*)h, (T*)y, rstd, H, eps);
    else
      add_rmsnorm_fwd_kernel<T, 4, false><<<rows, th, 0, st>>>((const T*)x, (const T*)r, (const T*)w, (T*)h, (T*)y, rstd, H, eps);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void add_rmsnorm_bwd(const void* gy, const void* gh, const void* h, const void* w, const float* rstd, void* dh,
                     float* partial, float* dw, int rows, int H, int dt, cudaStream_t st) {
  const int grid = rmsnorm_bwd_num_partials(rows);
  FN_DISPATCH_DTYPE(dt, {
    if (H % Pack16<T>::N) nxd_throw("add_rmsnorm_bwd: H must be a multiple of the 16-byte vector width", __FILE__, __LINE__);
    const int th = fn_pick_threads<T>(H);
    // the wide-row loops cost registers (one CTA per SM fewer), so rows that fit the register cache do not carry them
    if (H / Pack16<T>::N > 4 * th)
      add_rmsnorm_bwd_kernel<T, 4, true><<<grid, th, 0, st>>>((const T*)gy, (const T*)gh, (const T*)h, (const T*)w, rstd,
                                                              (T*)dh, partial, rows, H);
    else
      add_rmsnorm_bwd_kernel<T, 4, false><<<grid, th, 0, st>>>((const T*)gy, (const T*)gh, (const T*)h, (const T*)w, rstd,
                                                               (T*)dh, partial, rows, H);
  });
  fused_norm_reduce_partials_kernel<<<(H + 255) / 256, 256, 0, st>>>(partial, dw, grid, H);
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
