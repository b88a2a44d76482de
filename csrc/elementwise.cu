// Hand-written sm_90a elementwise / normalisation / loss kernels.
//   rmsnorm fwd+bwd   (reference call site: modules/rms_norm.py:10-33)
//   swiglu  fwd+bwd   (examples/training/llama/modeling_llama_nxd.py:208-219)
//   rope apply        (overrides/transformer_overrides.py:20-32)
//   vocab-parallel cross-entropy stats + backward (parallel_layers/loss_functions.py:12-129)
// All are HBM-bound: 16-byte vector accesses, one pass over the data, fp32 math.
#include "common.cuh"
#include "kernels.h"

namespace nxd {

// =====================================================================================
// RMSNorm forward: one CTA per row, row cached in registers (up to MAXV 16-byte packets/thread)
// =====================================================================================
template <typename T, int MAXV>
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                          T* __restrict__ y, float* __restrict__ rstd_out, int H,
                                                          float eps) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  __shared__ float red[32];
  const int row = blockIdx.x;
  const T* xr = x + (size_t)row * H;
  T* yr = y + (size_t)row * H;
  const int nvec = H / N;
  P cache[MAXV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
    if (v < nvec) {
      cache[i].load(xr + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) { const float f = cache[i].f(j); ss += f * f; }
    }
  }
  // tail beyond the register cache (very wide rows): re-read in the second pass
  for (int v = threadIdx.x + MAXV * blockDim.x; v < nvec; v += blockDim.x) {
    P p; p.load(xr + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) { const float f = p.f(j); ss += f * f; }
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0) rstd_out[row] = rstd;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = threadIdx.x + i * blockDim.x;
    if (v < nvec) {
      P pw, po; pw.load_nc(w + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) po.set(j, cache[i].f(j) * rstd * pw.f(j));
      po.store(yr + v * N);
    }
  }
  for (int v = threadIdx.x + MAXV * blockDim.x; v < nvec; v += blockDim.x) {
    P p, pw, po; p.load(xr + v * N); pw.load_nc(w + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) po.set(j, p.f(j) * rstd * pw.f(j));
    po.store(yr + v * N);
  }
}

// =====================================================================================
// RMSNorm backward. Persistent CTAs stride over rows; each thread owns fixed columns so the
// dW partial lives in registers across rows.  partial_dw: [gridDim.x, H] fp32.
//   dx = rstd * (g*w - xhat * mean_H(g*w*xhat)),  dw = sum_rows g*xhat
// Packets beyond the register cache (very wide rows) are re-read in the second pass and accumulate dW in place in the
// CTA's own partial row, which no other CTA touches.
// =====================================================================================
template <typename T, int MAXV, bool WIDE>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const T* __restrict__ g, const T* __restrict__ x,
                                                          const T* __restrict__ w, const float* __restrict__ rstd,
                                                          T* __restrict__ dx, float* __restrict__ partial_dw, int rows,
                                                          int H) {
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
    const T* xr = x + (size_t)row * H;
    const T* gr = g + (size_t)row * H;
    T* dxr = dx + (size_t)row * H;
    const float rs = rstd[row];
    P px[MAXV], pg[MAXV];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = threadIdx.x + i * blockDim.x;
      if (v < nvec) {
        px[i].load(xr + v * N);
        pg[i].load(gr + v * N);
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float xh = px[i].f(j) * rs, gg = pg[i].f(j);
          dot += gg * pw[i].f(j) * xh;
          dw[i][j] += gg * xh;
        }
      }
    }
    for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
      P qx, qg, qw; qx.load(xr + v * N); qg.load(gr + v * N); qw.load_nc(w + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) { const float xh = qx.f(j) * rs; dot += qg.f(j) * qw.f(j) * xh; }
    }
    dot = block_sum(dot, red) / (float)H;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = threadIdx.x + i * blockDim.x;
      if (v < nvec) {
        P po;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float xh = px[i].f(j) * rs;
          po.set(j, rs * (pg[i].f(j) * pw[i].f(j) - xh * dot));
        }
        po.store(dxr + v * N);
      }
    }
    for (int v = threadIdx.x + MAXV * blockDim.x; WIDE && v < nvec; v += blockDim.x) {
      P qx, qg, qw, po; qx.load(xr + v * N); qg.load(gr + v * N); qw.load_nc(w + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float xh = qx.f(j) * rs, gg = qg.f(j);
        po.set(j, rs * (gg * qw.f(j) - xh * dot));
        pdw[v * N + j] += gg * xh;
      }
      po.store(dxr + v * N);
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

__global__ void reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out, int nparts, int H) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float s = 0.f;
  for (int p = 0; p < nparts; ++p) s += partial[(size_t)p * H + c];
  out[c] = s;
}

// =====================================================================================
// SwiGLU: out[t, i] = silu(gu[t, i]) * gu[t, I + i]
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const T* __restrict__ gu, T* __restrict__ out, size_t rows, int I) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  const int vec_per_row = I / N;
  const size_t total = rows * (size_t)vec_per_row;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t r = idx / vec_per_row;
    const int c = (int)(idx % vec_per_row) * N;
    P pg, pu, po;
    pg.load(gu + r * 2 * I + c);
    pu.load(gu + r * 2 * I + I + c);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float g = pg.f(j);
      po.set(j, g / (1.f + __expf(-g)) * pu.f(j));
    }
    po.store(out + r * I + c);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const T* __restrict__ go, const T* __restrict__ gu,
                                                         T* __restrict__ dgu, size_t rows, int I) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  const int vec_per_row = I / N;
  const size_t total = rows * (size_t)vec_per_row;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t r = idx / vec_per_row;
    const int c = (int)(idx % vec_per_row) * N;
    P pg, pu, pd, og, ou;
    pg.load(gu + r * 2 * I + c);
    pu.load(gu + r * 2 * I + I + c);
    pd.load(go + r * I + c);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float g = pg.f(j), u = pu.f(j), d = pd.f(j);
      const float sig = 1.f / (1.f + __expf(-g));
      const float silu = g * sig;
      og.set(j, d * u * (sig + silu * (1.f - sig)));
      ou.set(j, d * silu);
    }
    og.store(dgu + r * 2 * I + c);
    ou.store(dgu + r * 2 * I + I + c);
  }
}

// =====================================================================================
// RoPE (rotate-half).  x: [B,S,H,D] with arbitrary B/S/H strides (D contiguous) → out contiguous.
// sign=+1 forward, -1 backward (inverse rotation).  One thread: 8 elements of each half.
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256) rope_kernel(const T* __restrict__ x, T* __restrict__ out,
                                                   const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                   int B, int S, int Hh, int D, long sb, long ss, long sh, float sign) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  const int half = D / 2;
  const int vec_per_head = half / N;
  const size_t total = (size_t)B * S * Hh * vec_per_head;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % vec_per_head) * N;
    size_t t = idx / vec_per_head;
    const int h = (int)(t % Hh); t /= Hh;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const T* src = x + b * sb + s * ss + h * sh;
    T* dst = out + (((size_t)b * S + s) * Hh + h) * D;
    P p1, p2, o1, o2;
    p1.load(src + c);
    p2.load(src + half + c);
    const float* cr = cos_t + (size_t)s * half + c;
    const float* sr = sin_t + (size_t)s * half + c;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float cs = cr[j], sn = sr[j] * sign;
      const float a = p1.f(j), bb = p2.f(j);
      o1.set(j, a * cs - bb * sn);
      o2.set(j, bb * cs + a * sn);
    }
    o1.store(dst + c);
    o2.store(dst + half + c);
  }
}

// =====================================================================================
// Cross-entropy statistics: per row (max, sum exp(x-max), target logit if owned, sum x).
// One CTA per row; online softmax per thread then block merge.
// VEC: rows are read as 16-byte packets, which needs a 16-byte aligned base and V % (16 / sizeof(T)) == 0 (every row
// start aligned).  Otherwise the whole row goes through the element loop.
// =====================================================================================
template <typename T, bool VEC>
__global__ void __launch_bounds__(256) ce_stats_kernel(const T* __restrict__ logits, const int64_t* __restrict__ target,
                                                       float* __restrict__ stats, int V, int vocab_start) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  __shared__ float red[32];
  const int row = blockIdx.x;
  const T* xr = logits + (size_t)row * V;
  float m = -INFINITY, s = 0.f, sx = 0.f;
  const int nvec = VEC ? V / N : 0;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    P p; p.load(xr + v * N);
    float lm = p.f(0);
#pragma unroll
    for (int j = 1; j < N; ++j) lm = fmaxf(lm, p.f(j));
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) { const float f = p.f(j); acc += __expf(f - nm); sx += f; }
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  for (int c = nvec * N + threadIdx.x; c < V; c += blockDim.x) {  // ragged tail, or the whole row without VEC
    const float f = to_f32<T>(xr[c]);
    const float nm = fmaxf(m, f);
    s = s * __expf(m - nm) + __expf(f - nm);
    m = nm; sx += f;
  }
  const float gm = block_max(m, red);
  const float contrib = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
  const float gs = block_sum(contrib, red);
  const float gsx = block_sum(sx, red);
  if (threadIdx.x == 0) {
    const long local = (long)target[row] - vocab_start;
    const float tl = (local >= 0 && local < V) ? to_f32<T>(xr[local]) : 0.f;
    float* o = stats + (size_t)row * 4;
    o[0] = gm; o[1] = gs; o[2] = tl; o[3] = gsx;
  }
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(256) ce_bwd_kernel(const T* __restrict__ logits, const int64_t* __restrict__ target,
                                                     const float* __restrict__ lse, const float* __restrict__ gout,
                                                     T* __restrict__ grad, int V, int vocab_start, float smoothing,
                                                     float inv_vocab) {
  using P = Pack16<T>;
  constexpr int N = P::N;
  const int row = blockIdx.x;
  const T* xr = logits + (size_t)row * V;
  T* gr = grad + (size_t)row * V;
  const float l = lse[row], g = gout[row];
  const long local = (long)target[row] - vocab_start;
  const float sm_term = smoothing * inv_vocab;
  const int nvec = VEC ? V / N : 0;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    P p, o; p.load(xr + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      float d = __expf(p.f(j) - l) - sm_term;
      if ((long)(v * N + j) == local) d -= (1.f - smoothing);
      o.set(j, d * g);
    }
    o.store(gr + v * N);
  }
  for (int c = nvec * N + threadIdx.x; c < V; c += blockDim.x) {
    float d = __expf(to_f32<T>(xr[c]) - l) - sm_term;
    if ((long)c == local) d -= (1.f - smoothing);
    gr[c] = from_f32<T>(d * g);
  }
}

// ---------------------------------------------------------------- launchers
template <typename T> static int pick_threads(int H) {
  const int nvec = H / Pack16<T>::N;
  int t = 32;
  while (t < 256 && t * 4 < nvec) t <<= 1;   // aim for <= 4 packets / thread
  return t;
}

#define DISPATCH_DTYPE(dt, ...)                                         \
  switch (dt) {                                                         \
    case kF32: { using T = float; __VA_ARGS__; break; }                 \
    case kBF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }        \
    case kF16: { using T = __half; __VA_ARGS__; break; }                \
    default: nxd_throw("unsupported dtype", __FILE__, __LINE__);        \
  }

static int num_sms() {
  static int n = 0;
  if (!n) { int dev; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
  return n;
}

void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H, float eps, int dt, cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    if (H % Pack16<T>::N) nxd_throw("rmsnorm: H must be a multiple of the 16-byte vector width", __FILE__, __LINE__);
    const int th = pick_threads<T>(H);
    rmsnorm_fwd_kernel<T, 4><<<rows, th, 0, st>>>((const T*)x, (const T*)w, (T*)y, rstd, H, eps);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

int rmsnorm_bwd_num_partials(int rows) { return min(rows, num_sms() * 4); }

void rmsnorm_bwd(const void* g, const void* x, const void* w, const float* rstd, void* dx, float* partial, float* dw,
                 int rows, int H, int dt, cudaStream_t st) {
  const int grid = rmsnorm_bwd_num_partials(rows);
  DISPATCH_DTYPE(dt, {
    if (H % Pack16<T>::N) nxd_throw("rmsnorm_bwd: H must be a multiple of the 16-byte vector width", __FILE__, __LINE__);
    const int th = pick_threads<T>(H);
    // the wide-row loops cost registers (one CTA per SM fewer), so rows that fit the register cache do not carry them
    if (H / Pack16<T>::N > 4 * th)
      rmsnorm_bwd_kernel<T, 4, true><<<grid, th, 0, st>>>((const T*)g, (const T*)x, (const T*)w, rstd, (T*)dx, partial, rows, H);
    else
      rmsnorm_bwd_kernel<T, 4, false><<<grid, th, 0, st>>>((const T*)g, (const T*)x, (const T*)w, rstd, (T*)dx, partial, rows, H);
  });
  reduce_partials_kernel<<<(H + 255) / 256, 256, 0, st>>>(partial, dw, grid, H);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void swiglu_fwd(const void* gu, void* out, long rows, int I, int dt, cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    const size_t total = (size_t)rows * (I / Pack16<T>::N);
    const int grid = (int)min((size_t)num_sms() * 16, (total + 255) / 256);
    swiglu_fwd_kernel<T><<<max(grid, 1), 256, 0, st>>>((const T*)gu, (T*)out, (size_t)rows, I);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void swiglu_bwd(const void* go, const void* gu, void* dgu, long rows, int I, int dt, cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    const size_t total = (size_t)rows * (I / Pack16<T>::N);
    const int grid = (int)min((size_t)num_sms() * 16, (total + 255) / 256);
    swiglu_bwd_kernel<T><<<max(grid, 1), 256, 0, st>>>((const T*)go, (const T*)gu, (T*)dgu, (size_t)rows, I);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

// any even D (partial rotary dims such as GPT-NeoX-20B's 24 of 96): one element pair per thread
template <typename T>
__global__ void __launch_bounds__(256) rope_scalar_kernel(const T* __restrict__ x, T* __restrict__ out,
                                                          const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                          int B, int S, int Hh, int D, long sb, long ss, long sh, float sign) {
  const int half = D / 2;
  const size_t total = (size_t)B * S * Hh * half;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % half);
    size_t t = idx / half;
    const int h = (int)(t % Hh); t /= Hh;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const T* src = x + b * sb + s * ss + h * sh;
    T* dst = out + (((size_t)b * S + s) * Hh + h) * D;
    const float cs = cos_t[(size_t)s * half + c], sn = sin_t[(size_t)s * half + c] * sign;
    const float a = to_f32<T>(src[c]), bb = to_f32<T>(src[half + c]);
    dst[c] = from_f32<T>(a * cs - bb * sn);
    dst[half + c] = from_f32<T>(bb * cs + a * sn);
  }
}

void rope_apply(const void* x, void* out, const float* cos_t, const float* sin_t, int B, int S, int Hh, int D, long sb,
                long ss, long sh, float sign, int dt, cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    if (D % 2) nxd_throw("rope: D must be even", __FILE__, __LINE__);
    if ((D / 2) % Pack16<T>::N || ((uintptr_t)x % 16) || (sb * sizeof(T)) % 16 || (ss * sizeof(T)) % 16 || (sh * sizeof(T)) % 16) {
      const size_t total = (size_t)B * S * Hh * (D / 2);
      const int grid = (int)min((size_t)num_sms() * 16, (total + 255) / 256);
      rope_scalar_kernel<T><<<max(grid, 1), 256, 0, st>>>((const T*)x, (T*)out, cos_t, sin_t, B, S, Hh, D, sb, ss, sh, sign);
      NXD_CUDA_CHECK(cudaGetLastError());
      return;
    }
    const size_t total = (size_t)B * S * Hh * ((D / 2) / Pack16<T>::N);
    const int grid = (int)min((size_t)num_sms() * 16, (total + 255) / 256);
    rope_kernel<T><<<max(grid, 1), 256, 0, st>>>((const T*)x, (T*)out, cos_t, sin_t, B, S, Hh, D, sb, ss, sh, sign);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

// Vocab shards need not be a multiple of the vector width (Llama-2-13B's 32016 over TP=4 is 8004 columns per rank;
// BERT's 30522 and GPT-2's 50257 at any TP), and logits may be a view at any element offset.
template <typename T> static bool ce_vec_ok(const void* p, int V) {
  return (uintptr_t)p % 16 == 0 && V % Pack16<T>::N == 0;
}

void ce_stats(const void* logits, const int64_t* target, float* stats, int rows, int V, int vocab_start, int dt,
              cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    if (ce_vec_ok<T>(logits, V))
      ce_stats_kernel<T, true><<<rows, 256, 0, st>>>((const T*)logits, target, stats, V, vocab_start);
    else
      ce_stats_kernel<T, false><<<rows, 256, 0, st>>>((const T*)logits, target, stats, V, vocab_start);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void ce_backward(const void* logits, const int64_t* target, const float* lse, const float* gout, void* grad, int rows,
                 int V, int vocab_start, float smoothing, int vocab, int dt, cudaStream_t st) {
  DISPATCH_DTYPE(dt, {
    if (ce_vec_ok<T>(logits, V) && ce_vec_ok<T>(grad, V))
      ce_bwd_kernel<T, true><<<rows, 256, 0, st>>>((const T*)logits, target, lse, gout, (T*)grad, V, vocab_start,
                                                   smoothing, 1.f / (float)vocab);
    else
      ce_bwd_kernel<T, false><<<rows, 256, 0, st>>>((const T*)logits, target, lse, gout, (T*)grad, V, vocab_start,
                                                    smoothing, 1.f / (float)vocab);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
