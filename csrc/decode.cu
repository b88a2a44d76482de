// Token-generation (decode) kernels for sm_90a — both are HBM-bandwidth problems, so they are plain CUDA tuned for wide
// coalesced loads rather than tensor-core kernels:
//   decode_attention : one query token per sequence against the KV cache (flash-decoding: split over the cache length,
//                      GQA group processed together so K/V are read once per kv head), + a combine pass over the splits.
//                      Role of the reference's token-generation attention (modules/attention, models' TKG path).
//                      Optional sliding window W: only cache rows positions[b] − W < j ≤ positions[b] are read.
//                      The cache is bf16 or fp8 e4m3 with one fp32 scale per tensor (inference/kv_cache.py owns that format).
//   gemv_bf16        : y[M≤8, N] = x[M, K] · W[N, K]ᵀ (+ optional residual) for batch-1..8 decode; every weight byte is read once
//                      with 16-byte loads, fp32 accumulation.
#include <cuda.h>
#include <cuda_fp8.h>

#include "common.cuh"
#include "kernels.h"

namespace nxd {

namespace {

constexpr int kDecThreads = 128;
// Without a minimum-blocks hint ptxas held three HD ≠ 128 instantiations (G = 2) to 64 or 80 registers, which spilled; a
// floor of one CTA per SM lets it allocate what they need.  0 (no hint) keeps the HD = 128 instantiations as they were.
template <int HD> constexpr int kDecMinBlocks = HD == 128 ? 0 : 1;

// 8 consecutive elements → fp32 (bf16: one 16-byte load; e4m3: one 8-byte load and the hardware fp8x2 → f16x2 unpack)
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8], float mul) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&a);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x * mul; f[2 * i + 1] = t.y * mul; }
}
__device__ __forceinline__ void load8(const __nv_fp8_e4m3* p, float (&f)[8], float mul) {
  const uint2 a = *reinterpret_cast<const uint2*>(p);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned w = i < 2 ? a.x : a.y;
    const float2 t = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> (16 * (i & 1))), __NV_E4M3)));
    f[2 * i] = t.x * mul; f[2 * i + 1] = t.y * mul;
  }
}

// HD = 128: 16 lanes share one kv position (8 dims each); a warp covers 2 positions per step, the CTA 8.  A bf16 lane loads
// 16 bytes of K and of V per position and takes one position per step (P = 1).  An e4m3 lane gets 8 bytes per position, so
// it takes P = 2 positions per step (a warp covers 4, the CTA 16): each lane still has 32 bytes of K/V in flight per step, as
// on bf16, and keeps the bf16 kernel's per-lane softmax state (P = 1 would halve the bytes in flight of a kernel that is
// latency-bound per CTA).  The other way to keep 16-byte loads, 8 lanes × 16 dims, doubles each lane's q and o registers:
// G = 8 uses 184 registers on bf16 already, so it would spill there.  For G ≤ 4 that mapping fits and would halve the softmax
// updates per position (16 lanes repeat the same one here); it has not been timed against this one (DESIGN §6).
// Other head sizes keep 8 dims (16 bytes of bf16, 8 of e4m3) and the same softmax state per lane:
//   HD = 64: 8 lanes per position, so a warp covers 4 positions per step (8 on e4m3); the dot product reduces over xor 1, 2
//            and 4, and the 4 position slots of a warp merge over xor 8 and 16 before the merge across the 4 warps.
//   HD = 80 / 96: 16-lane groups of which HD / 8 = 10 / 12 lanes hold dims.  The others load nothing, hold zeros and still
//            take part in the shuffles; they idle 37.5 % (80) / 25 % (96) of the load slots.  5- or 6-dim lanes would not
//            keep 16-byte loads.
// k_scale is folded into scale_log2 by the host; v_scale multiplies the partial o (1 on bf16).
// ROLL: the cache is a ring of L rows (inference/kv_cache.py, rolling mode) and logical position s lives in row s mod L.  The
// visible range stays in logical positions and is not clipped to L; the host guarantees 0 < window < L, so it spans fewer
// than L positions and row(s) = s − wrap0, minus L once past the end, with wrap0 = lo − lo mod L.
template <int HD, typename T, int G, bool ROLL>
__global__ void __launch_bounds__(kDecThreads, kDecMinBlocks<HD>) decode_attn_kernel(
    const __nv_bfloat16* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
    const long* __restrict__ positions, float* __restrict__ part_o, float* __restrict__ part_ml, int B, int H, int Hkv, int L,
    long k_sb, long k_ss, long k_sh, long v_sb, long v_ss, long v_sh, long q_sb, long q_sh, float scale_log2, int splits,
    int window, float v_scale) {
  constexpr bool kE4M3 = sizeof(T) == 1;
  constexpr int P = kE4M3 ? 2 : 1;                          // positions per lane per step
  constexpr int kLaneBits = HD == 64 ? 3 : 4;               // lanes per position = 1 << kLaneBits
  constexpr int kLanes = 1 << kLaneBits, kSlots = 32 / kLanes;   // position slots of a warp step
  static_assert(HD % 8 == 0 && HD / 8 <= kLanes && HD <= kDecThreads, "decode_attn_kernel: unsupported head_dim");
  const int kvh = blockIdx.x, b = blockIdx.y, split = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane >> kLaneBits, l16 = lane & (kLanes - 1);   // position slot within the warp step, 8-dim slice
  const bool act = HD / 8 == kLanes || l16 < HD / 8;        // the lane holds dims (HD = 80 / 96: 10 / 12 of 16 lanes do)
  // visible rows [lo, hi): the splits divide this range.  Positions may lie outside [0, L) (the local positions of a sequence
  // shard); then the range is clipped to the cache, and it is empty when the window ends before row 0 or starts past L.
  const long pos = positions[b];
  const int hi = ROLL ? (int)(pos + 1) : (int)min(pos + 1, (long)L);
  const int lo = ROLL ? (int)max(pos - window + 1, 0L) : window > 0 ? (int)min(max(pos - window + 1, 0L), (long)L) : 0;
  const int n_valid = max(hi - lo, 0);
  const int per = (n_valid + splits - 1) / splits;
  const int s0 = lo + split * per, s1 = min(hi, s0 + per);
  const int wrap0 = ROLL ? lo - lo % L : 0;
  auto row = [&](int s) {
    int r = s - wrap0;
    if (ROLL && r >= L) r -= L;
    return r;
  };

  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (act) {
      load8(q + b * q_sb + (long)(kvh * G + g) * q_sh + l16 * 8, qf[g], scale_log2);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) qf[g][i] = 0.f;
    }
  }
  float m[G], l[G], o[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = -INFINITY; l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) o[g][i] = 0.f;
  }
  const T* kb = kc + b * k_sb + (long)kvh * k_sh + l16 * 8;
  const T* vb = vc + b * v_sb + (long)kvh * v_sh + l16 * 8;
  for (int sbase = s0 + warp * kSlots * P; sbase < s1; sbase += 4 * kSlots * P) {   // warp-uniform trip count (full-mask shuffles inside)
    bool live[P];
    float kf[P][8], vf[P][8];
#pragma unroll
    for (int j = 0; j < P; ++j) {                         // all loads of the step are issued before any math
      const int s = sbase + kSlots * j + sub;
      live[j] = s < s1;
      if (kE4M3 && act) {                                 // a position past s1 re-reads row s1 − 1; its score is not used
        load8(kb + (long)row(min(s, s1 - 1)) * k_ss, kf[j], 1.f);
        load8(vb + (long)row(min(s, s1 - 1)) * v_ss, vf[j], 1.f);
      } else if (!kE4M3 && live[j] && act) {
        load8(kb + (long)row(s) * k_ss, kf[j], 1.f);
        load8(vb + (long)row(s) * v_ss, vf[j], 1.f);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) { kf[j][i] = 0.f; vf[j][i] = 0.f; }
      }
    }
#pragma unroll
    for (int j = 0; j < P; ++j) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) d = fmaf(qf[g][i], kf[j][i], d);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 4);
        if constexpr (kLanes == 16) d += __shfl_xor_sync(0xffffffffu, d, 8);
        // d: score·log2e of (position s, head g) in all lanes of the position
        if (live[j]) {
          const float mn = fmaxf(m[g], d);
          const float corr = exp2f(m[g] - mn), p = exp2f(d - mn);
          m[g] = mn;
          l[g] = l[g] * corr + p;
#pragma unroll
          for (int i = 0; i < 8; ++i) o[g][i] = fmaf(o[g][i], corr, p * vf[j][i]);
        }
      }
    }
  }
  // merge the position slots of the warp (HD = 64: lanes l16 + 8·sub over xor 8 and 16; else l16, l16 + 16 over xor 16),
  // then the 4 warps through smem
  __shared__ float sm_o[4][G][HD];
  __shared__ float sm_m[4][G], sm_l[4][G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
#pragma unroll
    for (int x = kLanes; x < 32; x *= 2) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m[g], x), l2 = __shfl_xor_sync(0xffffffffu, l[g], x);
      const float mn = fmaxf(m[g], m2);
      const float c1 = mn == -INFINITY ? 0.f : exp2f(m[g] - mn), c2 = mn == -INFINITY ? 0.f : exp2f(m2 - mn);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float o2 = __shfl_xor_sync(0xffffffffu, o[g][i], x);
        o[g][i] = o[g][i] * c1 + o2 * c2;
      }
      l[g] = l[g] * c1 + l2 * c2;
      m[g] = mn;
    }
    if (sub == 0) {
      if (act) {
#pragma unroll
        for (int i = 0; i < 8; ++i) sm_o[warp][g][l16 * 8 + i] = o[g][i];
      }
      if (l16 == 0) { sm_m[warp][g] = m[g]; sm_l[warp][g] = l[g]; }
    }
  }
  __syncthreads();
  // thread t = dim (threads ≥ HD write nothing); loop over heads of the group
  const int d = threadIdx.x;
  if (HD < kDecThreads && d >= HD) return;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    float mn = fmaxf(fmaxf(sm_m[0][g], sm_m[1][g]), fmaxf(sm_m[2][g], sm_m[3][g]));
    float acc = 0.f, ls = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float c = mn == -INFINITY ? 0.f : exp2f(sm_m[w][g] - mn);
      acc += sm_o[w][g][d] * c;
      ls += sm_l[w][g] * c;
    }
    const long idx = (((long)b * H + kvh * G + g) * splits + split);
    if constexpr (kE4M3) part_o[idx * HD + d] = acc * v_scale;
    else part_o[idx * HD + d] = acc;
    if (d == 0) { part_ml[idx * 2] = mn; part_ml[idx * 2 + 1] = ls; }
  }
}

// one CTA of HD threads per output row; partial rows [rows·splits, HD]
template <int HD>
__global__ void __launch_bounds__(HD) decode_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                            __nv_bfloat16* __restrict__ out, int splits, long o_sb, long o_sh,
                                                            int H) {
  const int bh = blockIdx.x, d = threadIdx.x;
  float mn = -INFINITY;
  for (int s = 0; s < splits; ++s) mn = fmaxf(mn, part_ml[((long)bh * splits + s) * 2]);
  float acc = 0.f, ls = 0.f;
  for (int s = 0; s < splits; ++s) {
    const long idx = (long)bh * splits + s;
    const float c = mn == -INFINITY ? 0.f : exp2f(part_ml[idx * 2] - mn);
    acc += part_o[idx * HD + d] * c;
    ls += part_ml[idx * 2 + 1] * c;
  }
  const int b = bh / H, h = bh % H;
  out[b * o_sb + h * o_sh + d] = __float2bfloat16_rn(ls > 0.f ? acc / ls : 0.f);
}

// Same merge over the splits, but the result stays un-normalised: o (relative to the row maximum), the maximum (natural-log
// units) and the row sum — what a rank contributes to distributed flash-decoding, where the final normalisation happens after
// the cross-rank log-sum-exp merge (modules/attention/flash_decode.py).
template <int HD>
__global__ void __launch_bounds__(HD) decode_combine_partial_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                                    float* __restrict__ fin_o, float* __restrict__ fin_ml, int splits) {
  const int bh = blockIdx.x, d = threadIdx.x;
  float mn = -INFINITY;
  for (int s = 0; s < splits; ++s) mn = fmaxf(mn, part_ml[((long)bh * splits + s) * 2]);
  float acc = 0.f, ls = 0.f;
  for (int s = 0; s < splits; ++s) {
    const long idx = (long)bh * splits + s;
    const float c = mn == -INFINITY ? 0.f : exp2f(part_ml[idx * 2] - mn);
    acc += part_o[idx * HD + d] * c;
    ls += part_ml[idx * 2 + 1] * c;
  }
  fin_o[(long)bh * HD + d] = acc;
  if (d == 0) { fin_ml[bh * 2] = mn * 0.6931471805599453f; fin_ml[bh * 2 + 1] = ls; }
}

__device__ __forceinline__ float gemv_act(float h, int act) {
  switch (act) {
    case 1: return 0.5f * h * (1.f + erff(h * 0.70710678118654752f));
    case 2: return 0.5f * h * (1.f + tanhf(0.7978845608028654f * (h + 0.044715f * h * h * h)));
    default: return h;
  }
}

// y[m, n] = Σ_k x[m, k] · W[n, k]; one warp per output column n (8 columns per 256-thread CTA), M ≤ 8 rows of x kept hot in L1.
// EPI: the epilogue also adds bias[n] (when given) and applies act (gemv_act; 1: exact GELU, 2: tanh GELU, as in
// csrc/moe_tkg.cu) before the residual, y = act(x·Wᵀ + bias) + residual with one bf16 rounding.  EPI = false is the plain
// kernel; its two extra parameters are not read.
template <int M, bool EPI>
__global__ void __launch_bounds__(256) gemv_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                   const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ y,
                                                   int N, int K, const __nv_bfloat16* __restrict__ bias, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.f;
  const __nv_bfloat16* wr = w + (long)n * K;
#pragma unroll 4
  for (int k = lane * 8; k < K; k += 256) {
    const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + k));       // weights stream through once
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
    if (lane == 0) {
      float r = v;
      if constexpr (EPI) {
        if (bias) r += __bfloat162float(bias[n]);
        r = gemv_act(r, act);
      }
      if (residual) r += __bfloat162float(residual[(long)m * N + n]);
      y[(long)m * N + n] = __float2bfloat16_rn(r);
    }
  }
}

// KVCacheManager._q on CUDA, bit for bit: x · (1/scale) in fp32 (torch divides by a Python scalar through its fp32
// reciprocal), then torch's float → e4m3 cast.  That cast rounds to nearest even and does not saturate: a value past 464
// (which rounds beyond 448), ±inf and NaN become the NaN byte 0x7F with the input's sign, where the hardware's satfinite
// conversion would clamp to ±448.
__device__ __forceinline__ __nv_fp8_e4m3 quant_e4m3(__nv_bfloat16 x, float inv) {
  const float f = __bfloat162float(x) * inv;
  __nv_fp8_e4m3 r;
  r.__x = fabsf(f) <= 464.f ? __nv_cvt_float_to_fp8(f, __NV_SATFINITE, __NV_E4M3)
                            : (__nv_fp8_storage_t)(((__float_as_uint(f) >> 24) & 0x80u) | 0x7Fu);
  return r;
}

// Decode-time RoPE + KV-cache append in ONE launch (was ~25 tiny elementwise / index_put kernels per layer in the token-
// generation graph): q [B,W,H,D] rotated into q_out, k rotated and v copied into the cache.  Token w of sequence b is
// rotated at position positions[b] + depth[w] (no depth: + w), clamped to [0, n_pos), and written to slot positions[b] + w,
// clamped to the cache (W = 1: the token at positions[b]; W > 1: a speculation window or a Medusa tree).  ROLL: the cache is
// a ring of L rows and the slot is (positions[b] + w) mod L.  One warp per head row; cos/sin rows gathered by position.
// HF rotate-half convention (csrc/elementwise.cu rope_kernel).  An e4m3 cache gets the bf16 rows a bf16 cache would hold,
// quantised by quant_e4m3 with k_inv = 1/k_scale and v_inv = 1/v_scale.
// PARTIAL (GPT-NeoX rotary_pct < 1): only dims [0, 2·rot_half) of q and k are rotated, rotate-half within them (pairs
// (c, rot_half + c), tables of width rot_half); dims [2·rot_half, D) are copied (k quantised on an e4m3 cache).  The full-
// rotary kernels (PARTIAL = false) do not read rot_half.
template <typename T, bool ROLL, bool PARTIAL>
__global__ void __launch_bounds__(128) decode_rope_kv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                            const __nv_bfloat16* __restrict__ v, const long* __restrict__ positions,
                                                            const long* __restrict__ depth, const float* __restrict__ cos_t,
                                                            const float* __restrict__ sin_t, __nv_bfloat16* __restrict__ q_out,
                                                            T* __restrict__ kc, T* __restrict__ vc, int B, int W, int H, int Hkv,
                                                            int D, int L, int n_pos, long q_sb, long q_ss, long q_sh, long k_sb,
                                                            long k_ss, long k_sh, long v_sb, long v_ss, long v_sh, long c_sb,
                                                            long c_ss, long c_sh, float k_inv, float v_inv, int rot_half) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int rows = B * W * (H + 2 * Hkv);
  if (warp >= rows) return;
  const int bw = warp / (H + 2 * Hkv), r = warp % (H + 2 * Hkv), b = bw / W, w = bw % W;
  const long p = positions[b];
  long pos = p + (depth ? depth[w] : w), slot = p + w;
  pos = pos < 0 ? 0 : (pos >= n_pos ? n_pos - 1 : pos);
  if constexpr (ROLL) {
    slot %= L;
    if (slot < 0) slot += L;
  } else {
    slot = slot < 0 ? 0 : (slot >= L ? L - 1 : slot);
  }
  q += b * q_sb + w * q_ss;
  k += b * k_sb + w * k_ss;
  v += b * v_sb + w * v_ss;
  const int half = PARTIAL ? rot_half : D / 2;
  if (r < H + Hkv) {                                   // q or k head: rotate
    const bool is_q = r < H;
    const int h = is_q ? r : r - H;
    const __nv_bfloat16* src = is_q ? q + (long)h * q_sh : k + (long)h * k_sh;
    __nv_bfloat16* dst = is_q ? q_out + ((long)bw * H + h) * D : reinterpret_cast<__nv_bfloat16*>(kc + b * c_sb + slot * c_ss + (long)h * c_sh);
    const float* cr = cos_t + pos * half;
    const float* sr = sin_t + pos * half;
    if constexpr (sizeof(T) == 2) {
      for (int c = lane; c < half; c += 32) {
        const float a = __bfloat162float(src[c]), bb = __bfloat162float(src[half + c]);
        const float cs = cr[c], sn = sr[c];
        dst[c] = __float2bfloat16_rn(a * cs - bb * sn);
        dst[half + c] = __float2bfloat16_rn(bb * cs + a * sn);
      }
    } else {                                           // q rows stay bf16; k rows are rounded to bf16, then quantised
      T* kd = reinterpret_cast<T*>(dst);
      for (int c = lane; c < half; c += 32) {
        const float a = __bfloat162float(src[c]), bb = __bfloat162float(src[half + c]);
        const float cs = cr[c], sn = sr[c];
        const __nv_bfloat16 x0 = __float2bfloat16_rn(a * cs - bb * sn), x1 = __float2bfloat16_rn(bb * cs + a * sn);
        if (is_q) {
          dst[c] = x0;
          dst[half + c] = x1;
        } else {
          kd[c] = quant_e4m3(x0, k_inv);
          kd[half + c] = quant_e4m3(x1, k_inv);
        }
      }
    }
    if constexpr (PARTIAL) {                           // pass-through dims
      for (int c = 2 * half + lane; c < D; c += 32) {
        if constexpr (sizeof(T) == 2) {
          dst[c] = src[c];
        } else {
          if (is_q) dst[c] = src[c];
          else reinterpret_cast<T*>(dst)[c] = quant_e4m3(src[c], k_inv);
        }
      }
    }
  } else {                                             // v head: copy
    const int h = r - H - Hkv;
    const __nv_bfloat16* src = v + (long)h * v_sh;
    T* dst = vc + b * c_sb + slot * c_ss + (long)h * c_sh;
    if constexpr (sizeof(T) == 2) {
      for (int c = lane; c < D; c += 32) dst[c] = src[c];
    } else {
      for (int c = lane; c < D; c += 32) dst[c] = quant_e4m3(src[c], v_inv);
    }
  }
}

}  // namespace

void decode_rope_kv(const void* q, const void* k, const void* v, const long* positions, const long* depth, const float* cos_t,
                    const float* sin_t, void* q_out, void* kc, void* vc, int B, int W, int H, int Hkv, int D, int L, int n_pos,
                    const long* qs, const long* ks, const long* vs, long c_sb, long c_ss, long c_sh, cudaStream_t st, bool kv_e4m3,
                    float k_inv, float v_inv, bool rolling, int rot) {
  const int rows = B * W * (H + 2 * Hkv);
  const int grid = (rows * 32 + 127) / 128;
#define NXD_ROPE_KV_P(T, R, P)                                                                                                   \
  decode_rope_kv_kernel<T, R, P><<<grid, 128, 0, st>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, \
      positions, depth, cos_t, sin_t, (__nv_bfloat16*)q_out, (T*)kc, (T*)vc, B, W, H, Hkv, D, L, n_pos, qs[0], qs[1], qs[2],      \
      ks[0], ks[1], ks[2], vs[0], vs[1], vs[2], c_sb, c_ss, c_sh, k_inv, v_inv, rot / 2)
#define NXD_ROPE_KV(T, R)                        \
  if (rot < D) NXD_ROPE_KV_P(T, R, true);        \
  else NXD_ROPE_KV_P(T, R, false)
  if (kv_e4m3) {
    if (rolling) { NXD_ROPE_KV(__nv_fp8_e4m3, true); }
    else { NXD_ROPE_KV(__nv_fp8_e4m3, false); }
  } else {
    if (rolling) { NXD_ROPE_KV(__nv_bfloat16, true); }
    else { NXD_ROPE_KV(__nv_bfloat16, false); }
  }
#undef NXD_ROPE_KV
#undef NXD_ROPE_KV_P
  NXD_CUDA_CHECK(cudaGetLastError());
}

void decode_attention(const void* q, const void* k, const void* v, const long* positions, void* out, float* part_o,
                      float* part_ml, int B, int H, int Hkv, int D, int L, const long* ks, const long* vs, long q_sb, long q_sh,
                      long o_sb, long o_sh, float scale, int splits, int window, cudaStream_t st, float* fin_o, float* fin_ml,
                      bool kv_e4m3, float k_scale, float v_scale, bool rolling) {
  const int G = H / Hkv;
  dim3 grid(Hkv, B, splits);
  const float sl2 = scale * 1.4426950408889634f * k_scale;
  dispatch_head_dim(D, "decode_attention", [&](auto hd) {
    constexpr int HD = decltype(hd)::value;
#define NXD_DEC(T, Gv, R)                                                                                                     \
  decode_attn_kernel<HD, T, Gv, R><<<grid, kDecThreads, 0, st>>>((const __nv_bfloat16*)q, (const T*)k, (const T*)v, positions, \
      part_o, part_ml, B, H, Hkv, L, ks[0], ks[1], ks[2], vs[0], vs[1], vs[2], q_sb, q_sh, sl2, splits, window, v_scale)
#define NXD_DEC_R(T, Gv)             \
  if (rolling) NXD_DEC(T, Gv, true); \
  else NXD_DEC(T, Gv, false)
    dispatch_gqa_group(G, "decode_attention", [&](auto g) {
      constexpr int Gv = decltype(g)::value;
      if (kv_e4m3) NXD_DEC_R(__nv_fp8_e4m3, Gv);
      else NXD_DEC_R(__nv_bfloat16, Gv);
    });
#undef NXD_DEC_R
#undef NXD_DEC
    if (fin_o != nullptr) decode_combine_partial_kernel<HD><<<B * H, HD, 0, st>>>(part_o, part_ml, fin_o, fin_ml, splits);
    else decode_combine_kernel<HD><<<B * H, HD, 0, st>>>(part_o, part_ml, (__nv_bfloat16*)out, splits, o_sb, o_sh, H);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void decode_combine(const float* part_o, const float* part_ml, void* out, int rows, int splits, int D, long o_sb, long o_sh,
                    int H, cudaStream_t st) {
  dispatch_head_dim(D, "decode_combine", [&](auto hd) {
    constexpr int HD = decltype(hd)::value;
    decode_combine_kernel<HD><<<rows, HD, 0, st>>>(part_o, part_ml, (__nv_bfloat16*)out, splits, o_sb, o_sh, H);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void gemv_bf16(const void* x, const void* w, const void* residual, void* y, int M, int N, int K, cudaStream_t st,
               const void* bias, int act) {
  const int grid = (N + 7) / 8;
  const bool epi = bias != nullptr || act != 0;
#define NXD_GEMV_E(Mv, E)                                                                                              \
  gemv_kernel<Mv, E><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)residual, \
                                           (__nv_bfloat16*)y, N, K, (const __nv_bfloat16*)bias, act)
#define NXD_GEMV(Mv)           \
  if (epi) NXD_GEMV_E(Mv, true); \
  else NXD_GEMV_E(Mv, false)
  switch (M) {
    case 1: NXD_GEMV(1); break;
    case 2: NXD_GEMV(2); break;
    case 3: NXD_GEMV(3); break;
    case 4: NXD_GEMV(4); break;
    case 5: NXD_GEMV(5); break;
    case 6: NXD_GEMV(6); break;
    case 7: NXD_GEMV(7); break;
    case 8: NXD_GEMV(8); break;
    default: nxd_throw("gemv_bf16: M must be 1..8", __FILE__, __LINE__);
  }
#undef NXD_GEMV
#undef NXD_GEMV_E
  NXD_CUDA_CHECK(cudaGetLastError());
}

}  // namespace nxd
