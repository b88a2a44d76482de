// Flash attention for sm_90a (head_dim 64, 80, 96 or 128, bf16): warpgroup tensor-core MMAs (wgmma.mma_async) on
// 128B-swizzled shared-memory tiles filled by cp.async (double-buffered), fp32 online softmax.  Role parity: reference
// kernels/flash_attn.py:162-212 (nki_flash_attn_func → flash_fwd / flash_attn_bwd) and modules/attention call sites.
//
// Every kernel runs two warpgroups per CTA; warpgroup g owns rows 64g..64g+63 of the CTA's 128-row tile, and warp w of it
// rows 16w..16w+15 of those, in the register layout of the mma.sync m16n8 fragments (which is the wgmma m64 layout).
// Forward, one CTA per (128-query tile, head, batch), looping over 64-key tiles:
//   S = Q·K_jᵀ (SS wgmma), running max / sum in registers, P packed to bf16 straight from the S fragments into the A
//   operand of O += P·V_j (RS wgmma).  Outputs: O (bf16, arbitrary b/s/h strides) and LSE (fp32 [B, H, S], natural log).
// Backward, three launches:
//   prep   δ = rowsum(dO ∘ O) − dLSE                                         (one warp per query row)
//   dK/dV  one CTA per (128-key tile, kv head, batch), loops over the 64-query tiles of every query head of the group:
//          Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ (SS), Pᵀ = exp(Sᵀ − LSE), dSᵀ = Pᵀ∘(dPᵀ − δ), dV += Pᵀ·dO, dK += dSᵀ·Q (RS)
//   dQ     one CTA per (128-query tile, head, batch), loops over the 64-key tiles: S, dP = dO·Vᵀ (SS), P, dS, dQ += dS·K (RS)
//   Every gradient element is owned by one thread of one CTA (no atomics), so the backward is bit-reproducible.
// Every kernel is a template on the head dimension HD with the same tiles and the same MMA sequence for all of them: the
// products with k = HD take HD/16 k-steps, and those with n = HD always compute 64 columns per 64-column panel (the
// columns past HD are discarded), so a D < 128 run equals the first D columns of a D = 128 run on zero-padded inputs.
// Visibility: query row i < S_q sees key j < S_kv iff
//   - MASK (key-padding mask, uint8 [B, S_kv]): mask[b, j] != 0;
//   - causal: j ≤ i + off;
//   - WINDOW (sliding window W, causal only): j > i + off − W.
// off = q_offset ≥ 0 (WINDOW kernels only, 0 otherwise) is the global position of query row 0 minus that of key row 0: one
// off-diagonal block of context-parallel attention, whose queries sit `off` positions after its keys.  W ≥ S_kv + off is
// plain causal attention.  The mask term is tested at each call site (the forward and dQ kernels stage each key tile's 64
// flags in shared memory, a dK/dV thread reads the flags of its two key rows once); the causal / window / offset terms are
// `sees`, and the tiles a CTA visits are the union of `key_tiles` / `query_tiles` over its two 64-row halves, which skip
// only tiles that hold no visible pair.
// An invisible pair contributes nothing: a query row that sees no key gets O = 0, LSE = −inf and dQ = 0, and a key no row
// sees gets dK = dV = 0.  A tile one warpgroup sees nothing of adds exact zeros to its accumulators.
// DROPOUT kernels apply attention dropout with the rule written above `Dropout`: the forward zeroes the dropped entries of
// P before O += P·V (the row sums, the running max and the LSE use the undropped P, so the LSE equals that of p = 0) and
// folds 1/(1 − p) into the final normalisation; the backward uses dV += (P∘Z)ᵀ·dO / (1 − p) and dS = P∘(dP∘Z/(1 − p) − δ),
// where δ = rowsum(dO∘O) of the dropped output is unchanged.
// spec_attn_kernel runs a forward loop on warp-level mma.sync (m16n8k16, ldmatrix from padded shared memory, 4 warps per
// 64-row tile) for W new tokens per sequence against a bf16 or e4m3 KV cache (speculation and Medusa verification); its
// visibility rule is written above it.
#include <cuda.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "sm90_ptx.cuh"

namespace nxd {
namespace fa {

constexpr int BT = 64;                       // rows of a query or key tile
constexpr int kThreads = 128;                // spec_attn_kernel
constexpr int kWgThreads = 256;              // flash kernels: two warpgroups
// padded shared-memory row of spec_attn_kernel (elements): 144 / 176 / 208 / 272 B for HD = 64 / 80 / 96 / 128.  Each
// stride is 16 B more than a multiple of 32 B, so the 8 row addresses of one ldmatrix 8x8 matrix start in distinct 4-bank
// groups (conflict-free).
template <int HD> constexpr int LDS = HD + 8;
template <int HD> constexpr int kTile = BT * LDS<HD>;              // elements of one staged tile
// wgmma operand tiles of the flash kernels: R rows × HD columns staged as kPanels [R × 64] bf16 panels in the 128-byte
// swizzle (row r of a panel is 128 B at r·128, its 16-byte chunk c sits at chunk c ^ (r & 7)); panels start 1 KB aligned.
template <int HD> constexpr int kPanels = (HD + 63) / 64;
template <int R, int HD> constexpr int kPTile = R * 64 * kPanels<HD>;           // elements
template <int HD> constexpr int kSmemFwd = (kPTile<2 * BT, HD> + 4 * kPTile<BT, HD>) * 2 + 1024;      // Q, K×2, V×2
template <int HD> constexpr int kSmemDkv = (2 * kPTile<2 * BT, HD> + 4 * kPTile<BT, HD>) * 2 + 4 * BT * 4 + 1024;
                                                                             // K, V, Q×2, dO×2, LSE×2, δ×2
template <int HD> constexpr int kSmemDq = (2 * kPTile<2 * BT, HD> + 4 * kPTile<BT, HD>) * 2 + 1024;   // Q, dO, K×2, V×2
constexpr int kSmemFlags = 2 * BT;                                                 // key-mask flags ×2 (MASK kernels)
constexpr float kLog2e = 1.4426950408889634f;

typedef __nv_bfloat16 bf16;

struct View { const bf16* p; long sb, ss, sh; };

NXD_DEVICE uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// two floats → bf16x2, `lo` in the low half (the lower address)
NXD_DEVICE uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

NXD_DEVICE void cp_async16(bf16* dst, const bf16* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
NXD_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
NXD_DEVICE void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// row (s0 + r) mod L of a ring of L rows, from w0 = s0 mod L (computed once per tile): r < 64, so one subtraction when L ≥ 64
NXD_DEVICE int ring_row(int w0, int r, int L) {
  const int x = w0 + r;
  return x < L ? x : (L >= BT ? x - L : x % L);
}

// rows [s0, s0+64) of one (batch, head) slice → padded shared tile; rows ≥ S are zero-filled.  ROLL: the slice is a ring of
// L rows and row s is read at s mod L.
template <int HD, bool ROLL = false>
NXD_DEVICE void load_tile(bf16* sm, const bf16* base, long ss, int s0, int S, int L = 0) {
  constexpr int kChunks = HD / 8;                                   // 16-byte chunks per row
  constexpr bool kPow2 = (kChunks & (kChunks - 1)) == 0;
  const int w0 = ROLL ? s0 % L : 0;
  for (int i = threadIdx.x; i < BT * kChunks; i += kThreads) {
    const int r = kPow2 ? i >> (kChunks == 16 ? 4 : 3) : i / kChunks, c = kPow2 ? i & (kChunks - 1) : i % kChunks;
    const bool ok = s0 + r < S;
    cp_async16(sm + r * LDS<HD> + c * 8, base + (long)(ok ? (ROLL ? ring_row(w0, r, L) : s0 + r) : 0) * ss + c * 8, ok);
  }
}

// rows [s0, s0+R) of one (batch, head) slice → swizzled panels; rows ≥ S are zero-filled.  NT threads share the copies.
template <int R, int HD, int NT = kWgThreads>
NXD_DEVICE void load_panels(bf16* sm, const bf16* base, long ss, int s0, int S) {
  constexpr int kChunks = HD / 8;                                   // 16-byte chunks per row
  for (int i = threadIdx.x; i < R * kChunks; i += NT) {
    const int r = i / kChunks, c = i - r * kChunks;
    const bool ok = s0 + r < S;
    cp_async16(sm + (c >> 3) * (R * 64) + r * 64 + (((c ^ r) & 7) << 3), base + (long)(ok ? s0 + r : 0) * ss + c * 8, ok);
  }
}

// aligns the dynamic shared memory to the 1 KB the 128-byte swizzle needs (the kernels request 1 KB of slack)
NXD_DEVICE bf16* panel_base(uint8_t* smem) { return (bf16*)(((uintptr_t)smem + 1023) & ~(uintptr_t)1023); }

// wgmma descriptor of a K-major operand (k = HD contiguous): rows [r0, r0 + 64) of an R-row panel tile, k-step ks
// (16 columns: panel ks / 4, 32 B into its rows)
template <int R>
NXD_DEVICE uint64_t desc_k(const bf16* tile, int r0, int ks) {
  return make_smem_desc(smem_u32(tile + (ks >> 2) * (R * 64) + r0 * 64) + (ks & 3) * 32, 16, 1024);
}
// wgmma descriptor of an MN-major operand (n = HD contiguous) of a 64-row panel tile: k rows [16ks, 16ks + 16), every
// panel (LBO = one panel)
NXD_DEVICE uint64_t desc_mn(const bf16* tile, int ks) {
  return make_smem_desc(smem_u32(tile + ks * 16 * 64), BT * 128, 1024);
}

// visibility flags of keys [s0, s0+64) (1 = visible; keys ≥ S are 0) → shared memory.  Plain loads: the mask row has no
// alignment guarantee.  Read after the next __syncthreads.
NXD_DEVICE void load_flags(uint8_t* sm, const uint8_t* mask, int s0, int S) {
  if (threadIdx.x < BT) {
    const int s = s0 + threadIdx.x;
    sm[threadIdx.x] = s < S && mask[s] != 0;
  }
}

NXD_DEVICE void ldsm_x4(uint32_t (&r)[4], const bf16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}
NXD_DEVICE void ldsm_x4_t(uint32_t (&r)[4], const bf16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}
NXD_DEVICE void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// C[16 x 64] = A[16 rows from a_row0][HD] · Bᵀ where B is a 64-row tile, both with the HD-long k dimension contiguous
// (QKᵀ, KQᵀ, VdOᵀ, dOVᵀ).  C fragment j holds columns 8j..8j+7: c0,c1 row lane/4, c2,c3 row lane/4+8, columns 2(lane%4)+{0,1}.
template <int HD>
NXD_DEVICE void mma_abt(float (&c)[8][4], const bf16* sa, int a_row0, const bf16* sb) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 8; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks) {
    uint32_t a[4];
    ldsm_x4(a, sa + (a_row0 + (lane & 15)) * LDS<HD> + ks * 16 + (lane >> 4) * 8);
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t b[4];
      ldsm_x4(b, sb + (jp * 16 + (lane & 7) + (lane >> 4) * 8) * LDS<HD> + ks * 16 + ((lane >> 3) & 1) * 8);
      mma16816(c[2 * jp], a, b[0], b[1]);
      mma16816(c[2 * jp + 1], a, b[2], b[3]);
    }
  }
}

// C[16 x HD] += P[16 x 64] · B where P comes as bf16 A fragments (4 k-steps) and B is a 64-row tile with the HD-wide
// output dimension contiguous (P·V, Pᵀ·dO, dSᵀ·Q, dS·K).
template <int HD>
NXD_DEVICE void mma_pb(float (&c)[HD / 8][4], const uint32_t (&p)[4][4], const bf16* sb) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int ks = 0; ks < BT / 16; ++ks) {
#pragma unroll
    for (int dp = 0; dp < HD / 16; ++dp) {
      uint32_t b[4];
      ldsm_x4_t(b, sb + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS<HD> + dp * 16 + (lane >> 4) * 8);
      mma16816(c[2 * dp], p[ks], b[0], b[1]);
      mma16816(c[2 * dp + 1], p[ks], b[2], b[3]);
    }
  }
}

// fp32 C fragments of a 16 x 64 block → bf16 A fragments of the next MMA (same thread ↔ element mapping)
NXD_DEVICE void to_a_frags(const float (&c)[8][4], uint32_t (&p)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    p[ks][0] = pack_bf16(c[2 * ks][0], c[2 * ks][1]);
    p[ks][1] = pack_bf16(c[2 * ks][2], c[2 * ks][3]);
    p[ks][2] = pack_bf16(c[2 * ks + 1][0], c[2 * ks + 1][1]);
    p[ks][3] = pack_bf16(c[2 * ks + 1][2], c[2 * ks + 1][3]);
  }
}

// the first HD columns of 16 x NB·8 fp32 fragments (rows row0 + lane/4 and +8) × scale → bf16 rows of a [B,S,H,HD] view
template <int HD, int NB>
NXD_DEVICE void store_rows(const float (&c)[NB][4], bf16* base, long ss, int row0, int S, float scale0, float scale1) {
  const int lane = threadIdx.x & 31;
  const int r0 = row0 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int dt = 0; dt < HD / 8; ++dt) {
    const int d = dt * 8 + 2 * (lane & 3);
    if (r0 < S) *(uint32_t*)(base + (long)r0 * ss + d) = pack_bf16(c[dt][0] * scale0, c[dt][1] * scale0);
    if (r1 < S) *(uint32_t*)(base + (long)r1 * ss + d) = pack_bf16(c[dt][2] * scale1, c[dt][3] * scale1);
  }
}

// the fields every kernel reads
struct Params {
  View q, k, v;
  int B, H, Hkv, S_q, S_kv, causal;
  float scale_log2;
  const uint8_t* mask; long mask_sb;            // key-padding mask [B, S_kv] (MASK kernels only)
  int window;                                   // sliding window W, 1 ≤ W ≤ S_kv + q_offset (WINDOW kernels only)
  int q_offset;                                 // query row 0 minus key row 0 in global positions (WINDOW kernels only)
};

// the causal / window / offset terms of the visibility rule: query row i sees key j
template <bool WINDOW>
NXD_DEVICE bool sees(const Params& p, int i, int j) {
  const int off = WINDOW ? p.q_offset : 0;
  return !(p.causal && j > i + off) && !(WINDOW && j <= i + off - p.window);
}

// Attention dropout.  Element (b, h, i, j) — query row i, key row j, h the global query head (head_offset + the head index
// of this call) — is kept iff word 2·((i >> 3) & 1) + ((j >> 3) & 1) of Philox4x32-10 with key (seed low word, seed high
// word) and counter (j & ~8, i & ~8, h, b) is below keep_threshold = round((1 − p)·2³²) (at most 2³² − 1), and a kept
// element is scaled by 1/(1 − p).  The rule depends on nothing but these coordinates (not on tiling, head size, layout,
// GQA grouping or the head count, so tensor-parallel shards with their head offsets drop what one unsharded run drops).
// One Philox call decides the 2×2 block {i0, i0 + 8} × {j0, j0 + 8}, which one thread holds whole in the accumulator
// fragments of all three kernels (rows r, r + 8 and columns c, c + 8).  ops.attention.attention_dropout_keep is the same
// rule on the host.
struct Dropout {
  const void* seed; int seed64;                 // the seed: one int64 (seed64) or int32 in device memory
  uint32_t keep_threshold;
  float rscale;                                 // 1 / (1 − p)
  int head_offset;
};

NXD_DEVICE uint2 dropout_key(const Dropout& d) {
  const uint64_t s = d.seed64 ? *(const unsigned long long*)d.seed : (uint64_t)(int64_t)*(const int*)d.seed;
  return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

NXD_DEVICE uint4 philox4x32_10(uint2 key, uint4 c) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { key.x += 0x9E3779B9u; key.y += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ key.x, lo1, hi0 ^ c.w ^ key.y, lo0);
  }
  return c;
}

// keep flags of the block {i0, i0 + 8} × {j0, j0 + 8} (bit 3 of i0 and j0 clear): bit 2·(i ≠ i0) + (j ≠ j0)
NXD_DEVICE uint32_t keep_bits(const Dropout& d, uint2 key, int b, int h, int i0, int j0) {
  const uint4 w = philox4x32_10(key, make_uint4((uint32_t)j0, (uint32_t)i0, (uint32_t)(h + d.head_offset), (uint32_t)b));
  const uint32_t t = d.keep_threshold;
  return (uint32_t)(w.x < t) | (uint32_t)(w.y < t) << 1 | (uint32_t)(w.z < t) << 2 | (uint32_t)(w.w < t) << 3;
}

// the dropout of a [16 × 64] fragment with query rows {i, i + 8} and key columns j0(jj, c) + {0, 8} (forward, dQ): f(x, keep)
// for every element x of c[8][4]
template <class F>
NXD_DEVICE void drop_rows(const Dropout& d, uint2 key, int b, int h, int i, int k0, float (&c)[8][4], F&& f) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int jj = 0; jj < 8; jj += 2) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint32_t z = keep_bits(d, key, b, h, i, k0 + jj * 8 + 2 * (lane & 3) + e);
      f(c[jj][e], z & 1);
      f(c[jj + 1][e], z & 2);
      f(c[jj][2 + e], z & 4);
      f(c[jj + 1][2 + e], z & 8);
    }
  }
}

// Tiles lo ≤ t < hi a CTA visits (none when hi ≤ lo); tile t holds rows [64t, 64t + 64).
// key_tiles: the rows of query tile [q0, q0 + 64) see keys q0 + off − W < j (its first row's window start) up to
// j ≤ q0 + 63 + off (causal: its last row's diagonal), so every visible key lies in the tiles returned.
template <bool WINDOW>
NXD_DEVICE void key_tiles(const Params& p, int q0, int& lo, int& hi) {
  const int off = WINDOW ? p.q_offset : 0, n = (p.S_kv + BT - 1) / BT;
  lo = WINDOW ? max(0, q0 + off - p.window + 1) / BT : 0;
  hi = p.causal ? min(n, (q0 + BT - 1 + off) / BT + 1) : n;
}
// query_tiles: the keys of key tile [k0, k0 + 64) are seen by rows i ≥ k0 − off (causal: the first key's diagonal) up to
// i ≤ k0 + 63 + W − 1 − off (the last key's window end), so every row that sees one of them lies in the tiles returned.  A
// negative last row leaves the range empty.
template <bool WINDOW>
NXD_DEVICE void query_tiles(const Params& p, int k0, int& lo, int& hi) {
  const int off = WINDOW ? p.q_offset : 0, n = (p.S_q + BT - 1) / BT;
  lo = p.causal ? max(0, k0 - off) / BT : 0;
  hi = WINDOW ? min(n, (k0 + 2 * BT - 2 + p.window - off) / BT) : n;
}

// K / V tile t of one (batch, kv head) and, with the mask, its key flags → buffer t & 1 of the double-buffered sK, sV, sM
// (forward and dQ)
template <int HD, bool MASK>
NXD_DEVICE void load_kv(bf16* sK, bf16* sV, uint8_t* sM, const bf16* kb, const bf16* vb, const uint8_t* mb, const Params& p,
                        int t) {
  const int buf = t & 1;
  load_panels<BT, HD>(sK + buf * kPTile<BT, HD>, kb, p.k.ss, t * BT, p.S_kv);
  load_panels<BT, HD>(sV + buf * kPTile<BT, HD>, vb, p.v.ss, t * BT, p.S_kv);
  cp_async_commit();
  if (MASK) load_flags(sM + buf * BT, mb, t * BT, p.S_kv);
}

struct FwdParams : Params {
  bf16* o; long o_sb, o_ss, o_sh;
  float* lse;
  Dropout drop;                                 // DROPOUT kernels only
};

template <int HD, bool MASK, bool WINDOW, bool DROPOUT>
__global__ void __launch_bounds__(kWgThreads) fa_fwd_kernel(const FwdParams p) {
  constexpr int kT = kPTile<BT, HD>, kNB = 8 * kPanels<HD>;
  extern __shared__ uint8_t smem_raw[];
  bf16* sQ = panel_base(smem_raw);              // 128 rows
  bf16* sK = sQ + kPTile<2 * BT, HD>;           // 2 buffers
  bf16* sV = sK + 2 * kT;                       // 2 buffers
  uint8_t* sM = (uint8_t*)(sV + 2 * kT);        // 2 × 64 key flags (MASK)
  // causal: the last query tiles see the most keys, so they are scheduled first
  const int qt = gridDim.x - 1 - blockIdx.x, h = blockIdx.y, b = blockIdx.z, hk = h / (p.H / p.Hkv);
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int q0 = qt * 2 * BT, r0 = q0 + wg * BT + warp * 16;
  const bf16* qb = p.q.p + b * p.q.sb + h * p.q.sh;
  const bf16* kb = p.k.p + b * p.k.sb + hk * p.k.sh;
  const bf16* vb = p.v.p + b * p.v.sb + hk * p.v.sh;
  const uint8_t* mb = MASK ? p.mask + b * p.mask_sb : nullptr;
  int t_lo, n_kv, lo1, hi0;                     // the key tiles of either 64-row half (monotone in the first row)
  key_tiles<WINDOW>(p, q0, t_lo, hi0);
  key_tiles<WINDOW>(p, q0 + BT, lo1, n_kv);

  load_panels<2 * BT, HD>(sQ, qb, p.q.ss, q0, p.S_q);
  load_kv<HD, MASK>(sK, sV, sM, kb, vb, mb, p, t_lo);

  float o[kNB][4];
#pragma unroll
  for (int i = 0; i < kNB; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int row[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};
  const uint2 dkey = DROPOUT ? dropout_key(p.drop) : make_uint2(0, 0);

  for (int t = t_lo; t < n_kv; ++t) {
    const int buf = t & 1;
    if (t + 1 < n_kv) {
      load_kv<HD, MASK>(sK, sV, sM, kb, vb, mb, p, t + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint8_t* fl = sM + buf * BT;
    float s[8][4];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks)
      wgmma_m64n64k16_ss(s, desc_k<2 * BT>(sQ, wg * BT, ks), desc_k<BT>(sK + buf * kT, 0, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = t * BT + j * 8 + 2 * (lane & 3) + (e & 1);
        const bool vis = key < p.S_kv && (!MASK || fl[j * 8 + 2 * (lane & 3) + (e & 1)]) && sees<WINDOW>(p, row[e >> 1], key);
        const float x = vis ? s[j][e] * p.scale_log2 : -INFINITY;
        s[j][e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float alpha[2], mu[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);
      mu[r] = mn == -INFINITY ? 0.f : mn;         // a row with no visible key so far keeps P = 0
      alpha[r] = exp2f(m[r] - mu[r]);
      m[r] = mn;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = exp2f(s[j][e] - mu[e >> 1]);
        s[j][e] = x;
        rs[e >> 1] += x;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + rs[r];
#pragma unroll
    for (int i = 0; i < kNB; ++i) { o[i][0] *= alpha[0]; o[i][1] *= alpha[0]; o[i][2] *= alpha[1]; o[i][3] *= alpha[1]; }
    if constexpr (DROPOUT) drop_rows(p.drop, dkey, b, h, row[0], t * BT, s, [](float& x, bool keep) { x = keep ? x : 0.f; });
    uint32_t pf[4][4];
    to_a_frags(s, pf);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BT / 16; ++ks) wgmma_m64k16_rs(o, pf[ks], desc_mn(sV + buf * kT, ks));
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(o);
    __syncthreads();                              // buffer `buf` is refilled at the next iteration
  }
  if (WINDOW) cp_async_wait<0>();                 // an offset tile that sees no key skips the loop with its first loads in flight
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    inv[r] = l[r] > 0.f ? (DROPOUT ? p.drop.rscale : 1.f) / l[r] : 0.f;
  }
  store_rows<HD>(o, p.o + b * p.o_sb + h * p.o_sh, p.o_ss, r0, p.S_q, inv[0], inv[1]);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
      if (row[r] < p.S_q)
        p.lse[((long)b * p.H + h) * p.S_q + row[r]] = l[r] > 0.f ? (m[r] + __log2f(l[r])) / kLog2e : -INFINITY;
  }
}

// ---- verification of W new tokens per sequence against a KV cache (speculation chains, Medusa trees) ----------------------
// Sequence b's window holds cache slots p = positions[b] .. p + W − 1.  Window row w sits at sequence position p + d[w]
// (d = depth, or w for a chain) and has tree-mask row M[w] (a chain: u ≤ w).  Row w sees slot c < min(p + W, L) iff
//   - c < p (committed): with a sliding window SW, c > p + d[w] − SW;
//   - c = p + u (window): M[w, u] and, with SW, d[u] > d[w] − SW.
// A row that sees nothing gets O = 0.  The W·G (token w, head g of the GQA group) rows of one kv head are cut into 64-row
// tiles (row w·G + g), and one CTA per (row tile, split, kv head, sequence) runs the forward kernel's loop over 64-slot K/V
// tiles, so each K/V row is read once for every row of the tile.  The splits divide only the slots a row of the tile can
// see (from p + min d − SW + 1 with a window).  An e4m3 cache is staged raw by cp.async and converted to bf16 in shared
// memory, which is exact; k_scale is folded into the softmax scale and v_scale multiplies the partial output.  A window
// slot no row of the tile sees gets its V row zeroed, so its bytes never reach the output (K is masked by a select).
// Partials (o relative to the row maximum, maximum and sum in log2 units) are merged by decode.cu's combine kernel.
// ROLL: the cache is a ring of L rows and slot c (a logical position) lives in row c mod L.  Everything above stays in
// logical positions, without the upper clamp at L; only the row address of a tile load wraps, per row, because a 64-row
// tile can straddle the end of the ring.  The host guarantees window > 0 and window + W − 1 ≤ L, so the slots a tile reads
// (at most p + dmin − window + 1 … p + W − 1) map to distinct rows.
constexpr int kSpecMaxW = 64;
template <int HD> constexpr int kRawTile = BT * HD;     // bytes of one staged e4m3 tile
template <int HD, bool E4M3>
constexpr int kSmemSpec = (E4M3 ? 3 * kTile<HD> * 2 + 4 * kRawTile<HD> : 5 * kTile<HD> * 2) + kSpecMaxW * (8 + 4);

struct SpecParams {
  const bf16* q; long q_sb, q_ss, q_sh;
  const void *k, *v; long k_sb, k_ss, k_sh, v_sb, v_ss, v_sh;
  const long* positions;
  const uint8_t* mask;                          // [W, W], row w sees window column u iff nonzero; null: chain
  const long* depth;                            // [W]; null: chain (d[w] = w)
  float *part_o, *part_ml;
  int W, H, L, splits, row_tiles, window;
  float scale_log2, v_scale;
};

NXD_DEVICE void cp_async8(void* dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(valid ? 8 : 0) : "memory");
}

// rows [s0, s0+64) of one e4m3 (batch, kv head) slice → unpadded HD-byte shared rows; rows ≥ S are zero-filled.  HD / 8
// copies of 8 bytes per row: an e4m3 cache is only required to be 8-byte aligned (so are 80-byte rows).  ROLL as in load_tile.
template <int HD, bool ROLL>
NXD_DEVICE void load_raw_e4m3(uint8_t* sm, const uint8_t* base, long ss, int s0, int S, int L) {
  constexpr int kChunks = HD / 8;                                   // 8-byte chunks per row
  constexpr bool kPow2 = (kChunks & (kChunks - 1)) == 0;
  const int w0 = ROLL ? s0 % L : 0;
  for (int i = threadIdx.x; i < BT * kChunks; i += kThreads) {
    const int r = kPow2 ? i >> (kChunks == 16 ? 4 : 3) : i / kChunks, c = kPow2 ? i & (kChunks - 1) : i % kChunks;
    const bool ok = s0 + r < S;
    cp_async8(sm + r * HD + c * 8, base + (long)(ok ? (ROLL ? ring_row(w0, r, L) : s0 + r) : 0) * ss + c * 8, ok);
  }
}

// staged e4m3 tile → padded bf16 tile (every e4m3 value is a bf16 value)
template <int HD>
NXD_DEVICE void e4m3_to_bf16(bf16* dst, const uint8_t* src) {
  constexpr int kChunks = HD / 8;
  constexpr bool kPow2 = (kChunks & (kChunks - 1)) == 0;
  for (int i = threadIdx.x; i < BT * kChunks; i += kThreads) {
    const int r = kPow2 ? i >> (kChunks == 16 ? 4 : 3) : i / kChunks, c = kPow2 ? i & (kChunks - 1) : i % kChunks;
    const uint2 a = *(const uint2*)(src + r * HD + c * 8);
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned w = j < 2 ? a.x : a.y;
      const float2 f = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> (16 * (j & 1))), __NV_E4M3)));
      o[j] = pack_bf16(f.x, f.y);
    }
    *(uint4*)(dst + r * LDS<HD> + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

template <int HD, int G, bool E4M3, bool ROLL>
__global__ void __launch_bounds__(kThreads) spec_attn_kernel(const SpecParams p) {
  constexpr int kTl = kTile<HD>, kBufs = E4M3 ? 1 : 2;
  constexpr int kChunks = HD / 8;                               // 16-byte chunks of a bf16 row
  constexpr bool kPow2 = (kChunks & (kChunks - 1)) == 0;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  bf16* sQ = (bf16*)smem_raw;
  bf16* sK = sQ + kTl;                          // kBufs buffers
  bf16* sV = sK + kBufs * kTl;                  // kBufs buffers
  uint8_t* sRaw = (uint8_t*)(sV + kBufs * kTl); // e4m3: raw K, V × 2 buffers
  uint64_t* sBits = (uint64_t*)(sRaw + (E4M3 ? 4 * kRawTile<HD> : 0));   // window columns row w sees
  int* sDepth = (int*)(sBits + kSpecMaxW);
  const int rt = blockIdx.x % p.row_tiles, split = blockIdx.x / p.row_tiles, kvh = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int W = p.W, r0 = rt * BT, n_rows = W * G;
  const long pos = p.positions[b];
  // p clamped to [−64, L] (ROLL: to ≥ −64): the same slots are committed / window slots below L, and slot − p stays in int
  // range
  const int p32 = ROLL ? (int)max(pos, (long)-kSpecMaxW) : (int)min(max(pos, (long)-kSpecMaxW), (long)p.L);

  if (threadIdx.x < W) sDepth[threadIdx.x] = p.depth ? (int)p.depth[threadIdx.x] : threadIdx.x;
  __syncthreads();
  if (threadIdx.x < W) {
    const int w = threadIdx.x;
    const long dw = sDepth[w];
    uint64_t bits = 0;
    for (int u = 0; u < W; ++u) {
      const bool m = p.mask ? p.mask[w * W + u] != 0 : u <= w;
      if (m && (p.window == 0 || sDepth[u] > dw - p.window)) bits |= 1ull << u;
    }
    sBits[w] = bits;
  }
  __syncthreads();
  // tokens [w_lo, w_hi) with a row in this tile: their smallest depth and the window columns any of them sees.  When G does
  // not divide 64, a token's G rows can straddle two tiles, and the one holding its first rows must count it too (round up).
  constexpr int kRoundUp = BT % G == 0 ? 0 : G - 1;
  const int w_lo = r0 / G, w_hi = min((r0 + BT + kRoundUp) / G, W);
  int dmin = INT32_MAX;
  uint64_t seen = 0;
  for (int w = w_lo; w < w_hi; ++w) { dmin = min(dmin, sDepth[w]); seen |= sBits[w]; }
  const uint64_t unseen = ~seen & (W == 64 ? ~0ull : (1ull << W) - 1);
  // slots [lo, hi) some row of the tile sees; the splits divide them in whole 64-slot tiles
  const long lo_l = p.window > 0 ? min(pos, pos + dmin - p.window + 1) : 0;
  const int lo = ROLL ? (int)max(lo_l, 0L) : (int)min(max(lo_l, 0L), (long)p.L);
  const int hi = ROLL ? (int)max(pos + W, (long)lo) : (int)max(min(pos + W, (long)p.L), (long)lo);
  const int per = ((hi - lo + p.splits - 1) / p.splits + BT - 1) / BT * BT;
  const int s0 = lo + split * per, s1 = min(hi, s0 + per);
  const int n_t = s1 > s0 ? (s1 - s0 + BT - 1) / BT : 0;

  // this thread's two rows: committed slots c > cmin are visible, window slot p + u iff bit u of wbits
  int cmin[2];
  uint64_t wbits[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r0 + warp * 16 + (lane >> 2) + 8 * r;
    const bool ok = row < n_rows;
    wbits[r] = ok ? sBits[row / G] : 0;
    const long c = p.window > 0 ? (long)p32 + sDepth[ok ? row / G : 0] - p.window : (long)INT32_MIN;
    cmin[r] = ok ? (int)max(c, (long)INT32_MIN) : INT32_MAX;
  }

  const bf16* qb = p.q + b * p.q_sb + (long)kvh * G * p.q_sh;
  const uint8_t* kb = (const uint8_t*)p.k + (b * p.k_sb + (long)kvh * p.k_sh) * (E4M3 ? 1 : 2);
  const uint8_t* vb = (const uint8_t*)p.v + (b * p.v_sb + (long)kvh * p.v_sh) * (E4M3 ? 1 : 2);
  auto issue = [&](int t) {                     // K / V tile t of the split → buffer t & 1
    const int s = s0 + t * BT, buf = t & 1;
    if constexpr (E4M3) {
      load_raw_e4m3<HD, ROLL>(sRaw + 2 * buf * kRawTile<HD>, kb, p.k_ss, s, s1, p.L);
      load_raw_e4m3<HD, ROLL>(sRaw + (2 * buf + 1) * kRawTile<HD>, vb, p.v_ss, s, s1, p.L);
    } else {
      load_tile<HD, ROLL>(sK + buf * kTl, (const bf16*)kb, p.k_ss, s, s1, p.L);
      load_tile<HD, ROLL>(sV + buf * kTl, (const bf16*)vb, p.v_ss, s, s1, p.L);
    }
    cp_async_commit();
  };
  if (n_t > 0) {
    for (int i = threadIdx.x; i < BT * kChunks; i += kThreads) {   // Q rows (token w, head g) of the tile; rows past W·G are 0
      const int r = kPow2 ? i >> (kChunks == 16 ? 4 : 3) : i / kChunks, c = kPow2 ? i & (kChunks - 1) : i % kChunks;
      const int row = r0 + r;
      const bool ok = row < n_rows;
      cp_async16(sQ + r * LDS<HD> + c * 8, qb + (ok ? (row / G) * p.q_ss + (row % G) * p.q_sh : 0) + c * 8, ok);
    }
    issue(0);
  }

  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

  for (int t = 0; t < n_t; ++t) {
    const int buf = t & 1, c0 = s0 + t * BT;
    if (t + 1 < n_t) {
      issue(t + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    bf16* k = sK + (E4M3 ? 0 : buf * kTl);
    bf16* v = sV + (E4M3 ? 0 : buf * kTl);
    if constexpr (E4M3) {
      e4m3_to_bf16<HD>(k, sRaw + 2 * buf * kRawTile<HD>);
      e4m3_to_bf16<HD>(v, sRaw + (2 * buf + 1) * kRawTile<HD>);
    }
    // tile rows holding a window slot no row of the tile sees
    const int sh = c0 - p32;
    const uint64_t zero = sh >= 0 ? (sh < 64 ? unseen >> sh : 0) : (sh > -64 ? unseen << -sh : 0);
    if (zero) {
      for (int i = threadIdx.x; i < BT * kChunks; i += kThreads) {
        const int r = kPow2 ? i >> (kChunks == 16 ? 4 : 3) : i / kChunks, c = kPow2 ? i & (kChunks - 1) : i % kChunks;
        if ((zero >> r) & 1) *(uint4*)(v + r * LDS<HD> + c * 8) = make_uint4(0, 0, 0, 0);
      }
    }
    if (E4M3 || zero) __syncthreads();
    float s[8][4];
    mma_abt<HD>(s, sQ, warp * 16, k);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = c0 + j * 8 + 2 * (lane & 3) + (e & 1), r = e >> 1;
        const bool vis = c < s1 && (c < p32 ? c > cmin[r] : (wbits[r] >> ((c - p32) & 63)) & 1);
        const float x = vis ? s[j][e] * p.scale_log2 : -INFINITY;
        s[j][e] = x;
        mx[r] = fmaxf(mx[r], x);
      }
    }
    float alpha[2], mu[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);
      mu[r] = mn == -INFINITY ? 0.f : mn;
      alpha[r] = exp2f(m[r] - mu[r]);
      m[r] = mn;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = exp2f(s[j][e] - mu[e >> 1]);
        s[j][e] = x;
        rs[e >> 1] += x;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + rs[r];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] *= alpha[0]; o[i][1] *= alpha[0]; o[i][2] *= alpha[1]; o[i][3] *= alpha[1]; }
    uint32_t pf[4][4];
    to_a_frags(s, pf);
    mma_pb<HD>(o, pf, v);
    __syncthreads();                              // the buffers are refilled at the next iteration
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    const int row = r0 + warp * 16 + (lane >> 2) + 8 * r;
    if (row >= n_rows) continue;
    const long idx = (((long)b * W + row / G) * p.H + kvh * G + row % G) * p.splits + split;
#pragma unroll
    for (int dt = 0; dt < HD / 8; ++dt)
      *(float2*)(p.part_o + idx * HD + dt * 8 + 2 * (lane & 3)) = make_float2(o[dt][2 * r] * p.v_scale, o[dt][2 * r + 1] * p.v_scale);
    if ((lane & 3) == 0) { p.part_ml[idx * 2] = m[r]; p.part_ml[idx * 2 + 1] = l[r]; }
  }
}

// δ[b,h,s] = Σ_d dO·O − dLSE   (one warp per query row; lane i reads elements 4i..4i+3, lanes past HD/4 read nothing)
template <int HD>
__global__ void fa_bwd_prep_kernel(const bf16* __restrict__ o, const bf16* __restrict__ go, const float* __restrict__ dlse,
                                   float* __restrict__ delta, int B, int S, int H, long o_sb, long o_ss, long o_sh, long g_sb,
                                   long g_ss, long g_sh) {
  const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long)B * H * S) return;
  const int s = (int)(w % S), h = (int)((w / S) % H), b = (int)(w / ((long)S * H));
  float acc = 0.f;
  if (HD == 128 || lane < HD / 4) {
    const uint2 ov = *(const uint2*)(o + b * o_sb + s * o_ss + h * o_sh + lane * 4);
    const uint2 gv = *(const uint2*)(go + b * g_sb + s * g_ss + h * g_sh + lane * 4);
    const __nv_bfloat162* oh = (const __nv_bfloat162*)&ov;
    const __nv_bfloat162* gh = (const __nv_bfloat162*)&gv;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float2 a = __bfloat1622float2(oh[j]), c = __bfloat1622float2(gh[j]);
      acc += a.x * c.x + a.y * c.y;
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  // w enumerates (b, h, s) in the [B, H, S] order of LSE / δ
  if (lane == 0) delta[w] = acc - (dlse ? dlse[w] : 0.f);
}

struct BwdParams : Params {
  View g;
  bf16 *dq, *dk, *dv;
  long dq_sb, dq_ss, dq_sh, dk_sb, dk_ss, dk_sh, dv_sb, dv_ss, dv_sh;
  const float *lse, *delta;
  float scale;
  Dropout drop;                                 // DROPOUT kernels only
};

template <int HD, bool MASK, bool WINDOW, bool DROPOUT>
__global__ void __launch_bounds__(kWgThreads, 1) fa_bwd_dkdv_kernel(const BwdParams p) {
  constexpr int kT = kPTile<BT, HD>, kNB = 8 * kPanels<HD>;
  extern __shared__ uint8_t smem_raw[];
  bf16* sK = panel_base(smem_raw);              // 128 rows
  bf16* sV = sK + kPTile<2 * BT, HD>;           // 128 rows
  bf16* sQ = sV + kPTile<2 * BT, HD>;           // 2 buffers
  bf16* sG = sQ + 2 * kT;                       // 2 buffers
  float* sL = (float*)(sG + 2 * kT);            // 2 × 64 LSE (log2 units)
  float* sD = sL + 2 * BT;                      // 2 × 64 δ
  const int kt = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int G = p.H / p.Hkv;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int k0 = kt * 2 * BT, r0 = k0 + wg * BT + warp * 16;
  int qt0, qt_end, lo1, hi0;                    // the query tiles of either 64-key half (monotone in the first key)
  query_tiles<WINDOW>(p, k0, qt0, hi0);
  query_tiles<WINDOW>(p, k0 + BT, lo1, qt_end);
  const int per_head = qt_end > qt0 ? qt_end - qt0 : 0;
  const int n_it = G * per_head;

  load_panels<2 * BT, HD>(sK, p.k.p + b * p.k.sb + hk * p.k.sh, p.k.ss, k0, p.S_kv);
  load_panels<2 * BT, HD>(sV, p.v.p + b * p.v.sb + hk * p.v.sh, p.v.ss, k0, p.S_kv);
  auto issue = [&](int it, int buf) {
    const int h = hk * G + it / per_head, q0 = (qt0 + it % per_head) * BT;
    load_panels<BT, HD>(sQ + buf * kT, p.q.p + b * p.q.sb + h * p.q.sh, p.q.ss, q0, p.S_q);
    load_panels<BT, HD>(sG + buf * kT, p.g.p + b * p.g.sb + h * p.g.sh, p.g.ss, q0, p.S_q);
    if (threadIdx.x < BT) {
      const int s = q0 + threadIdx.x;
      const long i = ((long)b * p.H + h) * p.S_q + s;
      sL[buf * BT + threadIdx.x] = s < p.S_q ? p.lse[i] * kLog2e : 0.f;
      sD[buf * BT + threadIdx.x] = s < p.S_q ? p.delta[i] : 0.f;
    }
  };
  if (n_it > 0) issue(0, 0);
  cp_async_commit();

  float dk[kNB][4], dv[kNB][4];
#pragma unroll
  for (int i = 0; i < kNB; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }
  const int key[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};
  bool kvis[2] = {true, true};                       // this thread's two key rows are not masked
  if (MASK) {
#pragma unroll
    for (int r = 0; r < 2; ++r) kvis[r] = key[r] < p.S_kv && p.mask[b * p.mask_sb + key[r]] != 0;
  }
  const uint2 dkey = DROPOUT ? dropout_key(p.drop) : make_uint2(0, 0);

  for (int it = 0; it < n_it; ++it) {
    const int buf = it & 1;
    const int q0 = (qt0 + it % per_head) * BT;
    if (it + 1 < n_it) {
      issue(it + 1, buf ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const bf16* q = sQ + buf * kT;
    const bf16* g = sG + buf * kT;
    const float* L = sL + buf * BT;
    const float* D = sD + buf * BT;
    float pt[8][4], dpt[8][4];                       // Sᵀ, dPᵀ: rows = keys, columns = queries
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) wgmma_m64n64k16_ss(pt, desc_k<2 * BT>(sK, wg * BT, ks), desc_k<BT>(q, 0, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) wgmma_m64n64k16_ss(dpt, desc_k<2 * BT>(sV, wg * BT, ks), desc_k<BT>(g, 0, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(pt);
    fence_acc(dpt);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = j * 8 + 2 * (lane & 3) + (e & 1);
        const int qi = q0 + qc;
        const bool vis = qi < p.S_q && sees<WINDOW>(p, qi, key[e >> 1]) && (!MASK || kvis[e >> 1]);
        pt[j][e] = vis ? exp2f(pt[j][e] * p.scale_log2 - L[qc]) : 0.f;
      }
    }
    uint32_t pf[4][4], sf[4][4];
    if constexpr (DROPOUT) {
      // dSᵀ = Pᵀ∘(dPᵀ∘Z/(1 − p) − δ) and Pᵀ∘Z for dV (its 1/(1 − p) is applied at the store), packed to bf16 one k-step at
      // a time so the fp32 fragments die early.  Rows are keys and columns queries here: the block of query columns
      // qc, qc + 8 and key rows key[0], key[1] is bits 0, 2 | 1, 3.
      const int h = hk * G + it / per_head;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int jj = 2 * ks;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qc = jj * 8 + 2 * (lane & 3) + e;
          const uint32_t z = keep_bits(p.drop, dkey, b, h, q0 + qc, key[0]);
          auto f = [&](float& x, float& dx, bool keep, float delta) {
            dx = x * (keep ? dx * p.drop.rscale - delta : -delta);
            x = keep ? x : 0.f;
          };
          f(pt[jj][e], dpt[jj][e], z & 1, D[qc]);
          f(pt[jj][2 + e], dpt[jj][2 + e], z & 2, D[qc]);
          f(pt[jj + 1][e], dpt[jj + 1][e], z & 4, D[qc + 8]);
          f(pt[jj + 1][2 + e], dpt[jj + 1][2 + e], z & 8, D[qc + 8]);
        }
        pf[ks][0] = pack_bf16(pt[jj][0], pt[jj][1]);
        pf[ks][1] = pack_bf16(pt[jj][2], pt[jj][3]);
        pf[ks][2] = pack_bf16(pt[jj + 1][0], pt[jj + 1][1]);
        pf[ks][3] = pack_bf16(pt[jj + 1][2], pt[jj + 1][3]);
        sf[ks][0] = pack_bf16(dpt[jj][0], dpt[jj][1]);
        sf[ks][1] = pack_bf16(dpt[jj][2], dpt[jj][3]);
        sf[ks][2] = pack_bf16(dpt[jj + 1][0], dpt[jj + 1][1]);
        sf[ks][3] = pack_bf16(dpt[jj + 1][2], dpt[jj + 1][3]);
      }
    } else {
      to_a_frags(pt, pf);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BT / 16; ++ks) wgmma_m64k16_rs(dv, pf[ks], desc_mn(g, ks));     // dV += Pᵀ·dO
    wgmma_commit();
    if constexpr (!DROPOUT) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = j * 8 + 2 * (lane & 3) + (e & 1);
          dpt[j][e] = pt[j][e] * (dpt[j][e] - D[qc]);
        }
      }
      to_a_frags(dpt, sf);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BT / 16; ++ks) wgmma_m64k16_rs(dk, sf[ks], desc_mn(q, ks));     // dK += dSᵀ·Q
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(dv);
    fence_acc(dk);
    __syncthreads();
  }
  if (WINDOW) cp_async_wait<0>();                    // a key tile no offset query sees skips the loop with K / V in flight
  store_rows<HD>(dk, p.dk + b * p.dk_sb + hk * p.dk_sh, p.dk_ss, r0, p.S_kv, p.scale, p.scale);
  const float dv_scale = DROPOUT ? p.drop.rscale : 1.f;
  store_rows<HD>(dv, p.dv + b * p.dv_sb + hk * p.dv_sh, p.dv_ss, r0, p.S_kv, dv_scale, dv_scale);
}

template <int HD, bool MASK, bool WINDOW, bool DROPOUT>
__global__ void __launch_bounds__(kWgThreads, 1) fa_bwd_dq_kernel(const BwdParams p) {
  constexpr int kT = kPTile<BT, HD>, kNB = 8 * kPanels<HD>;
  extern __shared__ uint8_t smem_raw[];
  bf16* sQ = panel_base(smem_raw);              // 128 rows
  bf16* sG = sQ + kPTile<2 * BT, HD>;           // 128 rows
  bf16* sK = sG + kPTile<2 * BT, HD>;           // 2 buffers
  bf16* sV = sK + 2 * kT;                       // 2 buffers
  uint8_t* sM = (uint8_t*)(sV + 2 * kT);        // 2 × 64 key flags (MASK)
  // causal: the last query tiles see the most keys, so they are scheduled first
  const int qt = gridDim.x - 1 - blockIdx.x, h = blockIdx.y, b = blockIdx.z, hk = h / (p.H / p.Hkv);
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int q0 = qt * 2 * BT, r0 = q0 + wg * BT + warp * 16;
  const bf16* kb = p.k.p + b * p.k.sb + hk * p.k.sh;
  const bf16* vb = p.v.p + b * p.v.sb + hk * p.v.sh;
  const uint8_t* mb = MASK ? p.mask + b * p.mask_sb : nullptr;
  int t_lo, n_kv, lo1, hi0;                     // as in the forward
  key_tiles<WINDOW>(p, q0, t_lo, hi0);
  key_tiles<WINDOW>(p, q0 + BT, lo1, n_kv);

  load_panels<2 * BT, HD>(sQ, p.q.p + b * p.q.sb + h * p.q.sh, p.q.ss, q0, p.S_q);
  load_panels<2 * BT, HD>(sG, p.g.p + b * p.g.sb + h * p.g.sh, p.g.ss, q0, p.S_q);
  load_kv<HD, MASK>(sK, sV, sM, kb, vb, mb, p, t_lo);

  const int row[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};
  float L[2], D[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long i = ((long)b * p.H + h) * p.S_q + row[r];
    L[r] = row[r] < p.S_q ? p.lse[i] * kLog2e : 0.f;
    D[r] = row[r] < p.S_q ? p.delta[i] : 0.f;
  }
  float dq[kNB][4];
#pragma unroll
  for (int i = 0; i < kNB; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const uint2 dkey = DROPOUT ? dropout_key(p.drop) : make_uint2(0, 0);

  for (int t = t_lo; t < n_kv; ++t) {
    const int buf = t & 1;
    if (t + 1 < n_kv) {
      load_kv<HD, MASK>(sK, sV, sM, kb, vb, mb, p, t + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const bf16* k = sK + buf * kT;
    const uint8_t* fl = sM + buf * BT;
    float s[8][4], dp[8][4];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) wgmma_m64n64k16_ss(s, desc_k<2 * BT>(sQ, wg * BT, ks), desc_k<BT>(k, 0, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks)                                                    // dP = dO·Vᵀ
      wgmma_m64n64k16_ss(dp, desc_k<2 * BT>(sG, wg * BT, ks), desc_k<BT>(sV + buf * kT, 0, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s);
    fence_acc(dp);
    // dS = P∘(dP∘Z/(1 − p) − δ)
    if constexpr (DROPOUT)
      drop_rows(p.drop, dkey, b, h, row[0], t * BT, dp, [&](float& x, bool keep) { x = keep ? x * p.drop.rscale : 0.f; });
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = t * BT + j * 8 + 2 * (lane & 3) + (e & 1);
        const int r = row[e >> 1];
        const bool vis = kc < p.S_kv && r < p.S_q && sees<WINDOW>(p, r, kc) && (!MASK || fl[j * 8 + 2 * (lane & 3) + (e & 1)]);
        s[j][e] = vis ? exp2f(s[j][e] * p.scale_log2 - L[e >> 1]) : 0.f;
        dp[j][e] = s[j][e] * (dp[j][e] - D[e >> 1]);
      }
    }
    uint32_t pf[4][4];
    to_a_frags(dp, pf);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BT / 16; ++ks) wgmma_m64k16_rs(dq, pf[ks], desc_mn(k, ks));      // dQ += dS·K
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(dq);
    __syncthreads();
  }
  if (WINDOW) cp_async_wait<0>();                    // as in the forward
  store_rows<HD>(dq, p.dq + b * p.dq_sb + h * p.dq_sh, p.dq_ss, r0, p.S_q, p.scale, p.scale);
}

static View view(const void* ptr, const long* s) {
  if (((uintptr_t)ptr % 16) || (s[0] % 8) || (s[1] % 8) || (s[2] % 8))
    nxd_throw("attention: q/k/v/o rows must be 16-byte aligned", __FILE__, __LINE__);
  return View{(const bf16*)ptr, s[0], s[1], s[2]};
}

// f(std::integral_constant<int, HD>, std::integral_constant<bool, MASK>, std::integral_constant<bool, WINDOW>,
// std::integral_constant<bool, DROPOUT>) for the runtime head dimension, mask, window and dropout flags
template <class F>
static void dispatch(int D, bool mask, bool window, bool dropout, F&& f) {
  auto with_dropout = [&](auto hd, auto mk, auto wd) {
    if (dropout) f(hd, mk, wd, std::true_type{});
    else f(hd, mk, wd, std::false_type{});
  };
  auto with_window = [&](auto hd, auto mk) {
    if (window) with_dropout(hd, mk, std::true_type{});
    else with_dropout(hd, mk, std::false_type{});
  };
  auto with_mask = [&](auto hd) {
    if (mask) with_window(hd, std::true_type{});
    else with_window(hd, std::false_type{});
  };
  dispatch_head_dim(D, "attention", with_mask);
}

template <int HD, bool MASK, bool WINDOW, bool DROPOUT>
static void launch_fwd(const FwdParams& p, cudaStream_t st) {
  constexpr int smem = kSmemFwd<HD> + (MASK ? kSmemFlags : 0);
  static bool configured = false;
  if (!configured) {
    NXD_CUDA_CHECK(cudaFuncSetAttribute(fa_fwd_kernel<HD, MASK, WINDOW, DROPOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem));
    configured = true;
  }
  fa_fwd_kernel<HD, MASK, WINDOW, DROPOUT><<<dim3((p.S_q + 2 * BT - 1) / (2 * BT), p.H, p.B), kWgThreads, smem, st>>>(p);
}

template <int HD, bool MASK, bool WINDOW, bool DROPOUT>
static void launch_bwd(const BwdParams& p, cudaStream_t st) {
  constexpr int smem_dkv = kSmemDkv<HD>, smem_dq = kSmemDq<HD> + (MASK ? kSmemFlags : 0);
  static bool configured = false;
  if (!configured) {
    NXD_CUDA_CHECK(cudaFuncSetAttribute(fa_bwd_dkdv_kernel<HD, MASK, WINDOW, DROPOUT>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, smem_dkv));
    NXD_CUDA_CHECK(cudaFuncSetAttribute(fa_bwd_dq_kernel<HD, MASK, WINDOW, DROPOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem_dq));
    configured = true;
  }
  fa_bwd_dkdv_kernel<HD, MASK, WINDOW, DROPOUT><<<dim3((p.S_kv + 2 * BT - 1) / (2 * BT), p.Hkv, p.B), kWgThreads, smem_dkv,
                                                   st>>>(p);
  fa_bwd_dq_kernel<HD, MASK, WINDOW, DROPOUT><<<dim3((p.S_q + 2 * BT - 1) / (2 * BT), p.H, p.B), kWgThreads, smem_dq, st>>>(p);
}

// checks the arguments and fills the fields every kernel reads
static void set_params(Params& p, const void* q, const void* k, const void* v, const long* qs, const long* ks, const long* vs,
                       int B, int S_q, int S_kv, int H, int Hkv, float scale, bool causal, const void* kpm, long kpm_sb,
                       long window, long q_offset) {
  if (causal && S_q != S_kv) nxd_throw("attention: causal needs S_q == S_kv", __FILE__, __LINE__);
  if (window < 0) nxd_throw("attention: window must be >= 0 (0 = none)", __FILE__, __LINE__);
  if (window > 0 && !causal) nxd_throw("attention: a sliding window needs causal attention", __FILE__, __LINE__);
  if (q_offset < 0) nxd_throw("attention: q_offset must be >= 0", __FILE__, __LINE__);
  if (q_offset > 0 && window == 0) nxd_throw("attention: q_offset needs a sliding window", __FILE__, __LINE__);
  // tile bounds reach 2·S + q_offset + 2·64 in 32-bit arithmetic
  if (q_offset > INT32_MAX - 2L * S_kv - 2 * BT) nxd_throw("attention: q_offset too large", __FILE__, __LINE__);
  p.q = view(q, qs); p.k = view(k, ks); p.v = view(v, vs);
  p.B = B; p.H = H; p.Hkv = Hkv; p.S_q = S_q; p.S_kv = S_kv; p.causal = causal ? 1 : 0;
  p.scale_log2 = scale * kLog2e;
  p.mask = (const uint8_t*)kpm; p.mask_sb = kpm_sb;
  // W ≥ S_kv + q_offset sees every causal key; the clamp keeps the tile bounds in range
  p.window = (int)std::min(window, S_kv + q_offset);
  p.q_offset = (int)q_offset;
}

// checks the dropout arguments and fills `Dropout`; returns whether the DROPOUT kernels run (p > 0)
static bool set_dropout(Dropout& d, double dropout_p, const void* seed, bool seed64, long head_offset, int H) {
  if (!(dropout_p >= 0.0 && dropout_p < 1.0)) nxd_throw("attention: dropout_p must be in [0, 1)", __FILE__, __LINE__);
  if (head_offset < 0 || head_offset > INT32_MAX - H) nxd_throw("attention: head_offset out of range", __FILE__, __LINE__);
  d = Dropout{seed, seed64 ? 1 : 0, 0u, 1.f, (int)head_offset};
  if (dropout_p == 0.0) return false;
  if (!seed) nxd_throw("attention: dropout_p > 0 needs a seed", __FILE__, __LINE__);
  // the same double arithmetic as ops.attention.attention_dropout_keep
  const double t = std::floor((1.0 - dropout_p) * 4294967296.0 + 0.5);
  d.keep_threshold = (uint32_t)std::min(t, 4294967295.0);
  d.rscale = (float)(1.0 / (1.0 - dropout_p));
  return true;
}

}  // namespace fa

void flash_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int S_q, int S_kv, int H,
                    int Hkv, int D, const long* qs, const long* ks, const long* vs, const long* os, float scale, bool causal,
                    const void* kpm, long kpm_sb, long window, long q_offset, double dropout_p, const void* seed,
                    bool seed64, long head_offset, cudaStream_t st) {
  using namespace fa;
  FwdParams p;
  set_params(p, q, k, v, qs, ks, vs, B, S_q, S_kv, H, Hkv, scale, causal, kpm, kpm_sb, window, q_offset);
  const bool dropout = set_dropout(p.drop, dropout_p, seed, seed64, head_offset, H);
  p.o = (bf16*)out; p.o_sb = os[0]; p.o_ss = os[1]; p.o_sh = os[2];
  p.lse = lse;
  dispatch(D, kpm != nullptr, window > 0, dropout, [&](auto hd, auto mk, auto wd, auto dr) {
    launch_fwd<decltype(hd)::value, decltype(mk)::value, decltype(wd)::value, decltype(dr)::value>(p, st);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void flash_attn_bwd(const void* go, const void* q, const void* k, const void* v, const void* o, const float* lse,
                    const float* dlse, void* dq, void* dk, void* dv, float* delta, int B, int S_q, int S_kv, int H, int Hkv,
                    int D, const long* gs, const long* qs, const long* ks, const long* vs, const long* os, const long* dqs,
                    const long* dks, const long* dvs, float scale, bool causal, const void* kpm, long kpm_sb, long window,
                    long q_offset, double dropout_p, const void* seed, bool seed64, long head_offset, cudaStream_t st) {
  using namespace fa;
  BwdParams p;
  set_params(p, q, k, v, qs, ks, vs, B, S_q, S_kv, H, Hkv, scale, causal, kpm, kpm_sb, window, q_offset);
  const bool dropout = set_dropout(p.drop, dropout_p, seed, seed64, head_offset, H);
  p.g = view(go, gs);
  p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv;
  p.dq_sb = dqs[0]; p.dq_ss = dqs[1]; p.dq_sh = dqs[2];
  p.dk_sb = dks[0]; p.dk_ss = dks[1]; p.dk_sh = dks[2];
  p.dv_sb = dvs[0]; p.dv_ss = dvs[1]; p.dv_sh = dvs[2];
  p.lse = lse; p.delta = delta;
  p.scale = scale;
  dispatch(D, kpm != nullptr, window > 0, dropout, [&](auto hd, auto mk, auto wd, auto dr) {
    constexpr int HD = decltype(hd)::value;
    const long rows = (long)B * H * S_q;
    fa_bwd_prep_kernel<HD><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(
        (const bf16*)o, (const bf16*)go, dlse, delta, B, S_q, H, os[0], os[1], os[2], gs[0], gs[1], gs[2]);
    launch_bwd<HD, decltype(mk)::value, decltype(wd)::value, decltype(dr)::value>(p, st);
  });
  NXD_CUDA_CHECK(cudaGetLastError());
}

void speculation_attention(const void* q, const void* k, const void* v, const long* positions, const void* mask,
                           const long* depth, void* out, float* part_o, float* part_ml, int B, int W, int H, int Hkv, int D,
                           int L, const long* qs, const long* ks, const long* vs, float scale, int window, int splits, bool kv_e4m3,
                           float k_scale, float v_scale, bool rolling, cudaStream_t st) {
  using namespace fa;
  const int G = H / Hkv;
  SpecParams p;
  p.q = (const bf16*)q; p.q_sb = qs[0]; p.q_ss = qs[1]; p.q_sh = qs[2];
  p.k = k; p.k_sb = ks[0]; p.k_ss = ks[1]; p.k_sh = ks[2];
  p.v = v; p.v_sb = vs[0]; p.v_ss = vs[1]; p.v_sh = vs[2];
  p.positions = positions; p.mask = (const uint8_t*)mask; p.depth = depth;
  p.part_o = part_o; p.part_ml = part_ml;
  p.W = W; p.H = H; p.L = L; p.splits = splits; p.row_tiles = (W * G + BT - 1) / BT; p.window = window;
  p.scale_log2 = scale * kLog2e * k_scale;
  p.v_scale = v_scale;
  const dim3 grid(p.row_tiles * splits, Hkv, B);
  // the shared-memory attribute is set once per (HD, G, E4M3, ROLL) instantiation, before its first launch
  auto launch = [&](auto hd, auto g, auto e4, auto roll) {
    constexpr int HD = decltype(hd)::value, Gv = decltype(g)::value;
    constexpr bool E4 = decltype(e4)::value, R = decltype(roll)::value;
    static bool configured = false;
    if (!configured) {
      NXD_CUDA_CHECK(cudaFuncSetAttribute(spec_attn_kernel<HD, Gv, E4, R>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          kSmemSpec<HD, E4>));
      configured = true;
    }
    spec_attn_kernel<HD, Gv, E4, R><<<grid, kThreads, kSmemSpec<HD, E4>, st>>>(p);
  };
  auto with_roll = [&](auto hd, auto g, auto e4) {
    if (rolling) launch(hd, g, e4, std::true_type{});
    else launch(hd, g, e4, std::false_type{});
  };
  auto with_cache = [&](auto hd, auto g) {
    if (kv_e4m3) with_roll(hd, g, std::true_type{});
    else with_roll(hd, g, std::false_type{});
  };
  dispatch_head_dim(D, "speculation_attention", [&](auto hd) {
    dispatch_gqa_group(G, "speculation_attention", [&](auto g) { with_cache(hd, g); });
  });
  NXD_CUDA_CHECK(cudaGetLastError());
  // row (b·W + w)·H + h of the partials → out [B, W, H, D]
  decode_combine(part_o, part_ml, out, B * W * H, splits, D, (long)H * D, D, H, st);
}

}  // namespace nxd
