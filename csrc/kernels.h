// Launcher declarations shared between the .cu translation units and binding.cpp.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

namespace nxd {

enum DType : int { kF32 = 0, kBF16 = 1, kF16 = 2 };

// ---- elementwise.cu
void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H, float eps, int dt, cudaStream_t st);
int rmsnorm_bwd_num_partials(int rows);
void rmsnorm_bwd(const void* g, const void* x, const void* w, const float* rstd, void* dx, float* partial, float* dw,
                 int rows, int H, int dt, cudaStream_t st);
// residual-add fused with RMSNorm (fused_norm.cu)
void add_rmsnorm_fwd(const void* x, const void* r, const void* w, void* h, void* y, float* rstd, int rows, int H, float eps,
                     int dt, cudaStream_t st);
void add_rmsnorm_bwd(const void* gy, const void* gh, const void* h, const void* w, const float* rstd, void* dh, float* partial,
                     float* dw, int rows, int H, int dt, cudaStream_t st);
void swiglu_fwd(const void* gu, void* out, long rows, int I, int dt, cudaStream_t st);
void swiglu_bwd(const void* go, const void* gu, void* dgu, long rows, int I, int dt, cudaStream_t st);
void rope_apply(const void* x, void* out, const float* cos_t, const float* sin_t, int B, int S, int Hh, int D, long sb,
                long ss, long sh, float sign, int dt, cudaStream_t st);
void ce_stats(const void* logits, const int64_t* target, float* stats, int rows, int V, int vocab_start, int dt,
              cudaStream_t st);
void ce_backward(const void* logits, const int64_t* target, const float* lse, const float* gout, void* grad, int rows,
                 int V, int vocab_start, float smoothing, int vocab, int dt, cudaStream_t st);

// ---- optim.cu
struct TensorRef { void* ptr; long numel; };
void multi_tensor_sq_norm(const std::vector<TensorRef>& ts, int dt, float* out, cudaStream_t st);
void multi_tensor_scale(const std::vector<TensorRef>& ts, int dt, const float* scale, cudaStream_t st);
// p,m,v fp32; g dtype gdt; optional low-precision copy lowp (dtype ldt, may be empty)
void fused_adamw(const std::vector<TensorRef>& p, const std::vector<TensorRef>& g, const std::vector<TensorRef>& m,
                 const std::vector<TensorRef>& v, const std::vector<TensorRef>& lowp, int gdt, int ldt, float lr,
                 float beta1, float beta2, float eps, float wd, float bc1, float bc2, const float* grad_scale,
                 int hf_form, cudaStream_t st);

// ---- gemm_sm90.cu
struct GemmComm {          // in-kernel NVLink communication description (all zero → plain GEMM)
  int mode = 0;            // 0 none, 1 all-gather A rows then GEMM, 2 GEMM then reduce-scatter rows
  int rank = 0, world = 1;
  const int64_t* peer_bufs = nullptr;   // device table [world] of peer payload base addresses
  const int64_t* peer_flags = nullptr;  // device table [world] of peer flag base addresses
  long buf_offset = 0;     // byte offset of this call's payload region inside every peer buffer
  int flag_offset = 0;     // index of this call's first flag
  uint32_t epoch = 0;      // monotonically increasing per (workspace, purpose)
  int comm_sms = 0;        // CTAs dedicated to communication (mode 1)
  const uint32_t* rs_targets = nullptr;  // host array [64]: cumulative per-row-block tile counts (mode 2)
};
void gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, bool trans_a, bool trans_b, int out_dt,
               bool accumulate, const GemmComm& comm, const void* a_local_shard, cudaStream_t st);
bool gemm_self_check_supported();
// NVLS (multicast / in-switch reduce) fused TP GEMMs, gemm_sm90.cu; mode 1 = all-gather → GEMM, 2 = GEMM → reduce-scatter
int gemm_bf16_nvls(int mode, const void* a, const void* b, void* out, void* rs_out, const void* a_local, int M, int N, int K,
                   bool trans_b, int rank, int world, const int64_t* peer_bases, int64_t mc_base, int64_t local_base,
                   long buf_offset, long flag_offset, uint32_t epoch, int comm_ctas, uint32_t* tile_done, uint32_t* claim,
                   uint32_t claim_base, bool wire_fp32, bool gemm_join, cudaStream_t st);

// stand-alone NVLS collectives (nvls_coll.cu); `state` = [2 + 1024] u32 device words (epoch, CTA counter, per-CTA barrier counts)
void nvls_allreduce(const void* x, const void* residual, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base,
                    long flag_off, long data_off, long half_bytes, uint32_t* state, int rank, int world, long numel, int dt,
                    int ctas, cudaStream_t st);
void gemv_allreduce(const void* x, const void* w, const void* residual, void* y, int M, int N, int K, const int64_t* peer_bases,
                    int64_t mc_base, int64_t local_base, long flag_off, long data_off, long half_bytes, uint32_t* state, int rank,
                    int world, int max_ctas, cudaStream_t st);
void nvls_all_gather(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                     long data_off, long half_bytes, uint32_t* state, int rank, int world, long bytes, int ctas, cudaStream_t st);
void nvls_all_to_all(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                     long data_off, long half_bytes, uint32_t* state, int rank, int world, long bytes, int ctas, cudaStream_t st);
void nvls_publish(const void* x, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off, long data_off,
                  long half_bytes, uint32_t* state, int rank, int world, long bytes, int parity, int ctas, cudaStream_t st);
void nvls_embedding_gather(const void* table, const long* ids, void* out, const int64_t* peer_bases, int64_t mc_base,
                           int64_t local_base, long flag_off, long data_off, long half_bytes, uint32_t* state, int rank, int world,
                           long rows_per_rank, long row_bytes, long ntok, int ctas, cudaStream_t st);
void nvls_reduce_scatter(const void* x, void* out, const int64_t* peer_bases, int64_t mc_base, int64_t local_base, long flag_off,
                         long data_off, long half_bytes, uint32_t* state, int rank, int world, long chunk_numel, int dt, int ctas,
                         cudaStream_t st);

// ---- zero1_comm.cu
void zero1_reduce_scatter(const int64_t* peer_bufs, long grad_off_bytes, const int64_t* peer_flags, int flag_off,
                          uint32_t epoch, int rank, int world, long shard_numel, long sub_begin, long sub_len, float scale,
                          float* out, uint32_t* done_ctr, int grad_dt, int max_ctas, cudaStream_t st);
void zero1_all_gather(const float* master, const int64_t* peer_bufs, long param_off_bytes, const int64_t* peer_flags,
                      int flag_off, uint32_t epoch, int rank, int world, long shard_numel, uint32_t* done_ctr, int param_dt,
                      cudaStream_t st);

// out[M,N] (+)= (a_e4m3[M,K] · b_e4m3[N,K]ᵀ) ∘ scale_a[M] ⊗ scale_b[N]; out_dt kBF16, or kF32 (accumulate: add into out)
void gemm_fp8(const void* a, const void* b, void* out, int M, int N, int K, const float* scale_a, const float* scale_b,
              int out_dt, bool accumulate, cudaStream_t st);
// ---- row-wise e4m3 quantisers of fp8 training (fp8_quant.cu), rule of fp8_rule.cuh
// x bf16 [M, K] → q e4m3 [M, K], scale fp32 [M]; K % 8 == 0
void quantize_fp8_rows(const void* x, void* q, float* scale, int M, int K, cudaStream_t st);
// x bf16 [R, C] → q e4m3 [C, R] (= rows of xᵀ), scale fp32 [C]; amax_bits: zeroed u32 scratch [C]; R % 16 == 0, C % 8 == 0
void quantize_fp8_cols_t(const void* x, void* q, float* scale, uint32_t* amax_bits, int R, int C, cudaStream_t st);
// ---- block-scaled fp8 GEMM and its activation quantiser (gemm_fp8_block_sm90.cu); group = 32, 64 or 128 elements of K
// out[M,N] (bf16) = Σ_g (a[:, g] · b[:, g]ᵀ) ∘ scale_a[g, :M] ⊗ scale_b[g, :N];  scale_a [K/group, scale_a_ld], scale_b [K/group, N]
void gemm_fp8_block(const void* a, const void* b, void* out, const float* scale_a, long scale_a_ld, const float* scale_b,
                    int M, int N, int K, int group, cudaStream_t st);
// grouped (MoE) mode: rows [i·block_rows, (i+1)·block_rows) of a use expert e = block_expert[i]: b [E·N, K] (rows e·N ..),
// scale_b [E·K/group, N] (rows e·K/group ..); block_rows % 128 == 0 and M % block_rows == 0
void grouped_gemm_fp8_block(const void* a, const void* b, void* out, const float* scale_a, long scale_a_ld,
                            const float* scale_b, int M, int N, int K, int E, const int* block_expert, int block_rows,
                            int group, cudaStream_t st);
// x bf16 [M, K] → q e4m3 [M, K] and fp32 scale [K/group, scale_ld] (group-major); mx: OCP MX power-of-two scales, else absmax / 448
void quantize_fp8_groups(const void* x, void* q, float* scale, int M, int K, long scale_ld, int group, bool mx, float clamp_bound,
                         cudaStream_t st);
// ---- grouped (MoE blockwise) GEMMs, gemm_sm90.cu
void grouped_gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, int E, bool trans_b,
                       const int* block_expert, int block_rows, int out_dt, cudaStream_t st);
void grouped_wgrad_bf16(const void* a, const void* b, void* out, int rows_total, int Mo, int No, int E,
                        const int* seg_first_block, int block_rows, int out_dt, bool accumulate, cudaStream_t st);

// ---- one-shot all-reduce over peer memory (allreduce.cu)
void oneshot_allreduce(const void* x, void* out, const int64_t* peer_bufs, const int64_t* peer_flags, long slot_bytes,
                       uint32_t* state, int rank, int world, long numel, int dt, int ctas, cudaStream_t st);

// ---- row selection for sampling (select.cu)
void row_argmax(const void* x, float* val, long* idx, int rows, int V, long row_stride, long index_offset, int dt, cudaStream_t st);
bool row_topk_supported(int V, int k);
void row_topk(const void* x, float* vals, long* idxs, int rows, int V, int k, long row_stride, long index_offset, int dt,
              cudaStream_t st);

void moe_block_metadata(const void* expert_index, bool idx64, long n, int k, int E, int B, int nb, long* block_to_expert, long* tp2id,
                        long* counts, cudaStream_t st);

// ---- decode-time MoE block in one cooperative launch (moe_tkg.cu)
bool moe_block_tkg_supported(int T, int H, int E, int I, int K);
void moe_block_tkg(const void* x, const void* gamma, const void* router_w, const float* router_bias, const void* w_gu,
                   const void* w_dn, float* logits, float* gu, float* yacc, void* out, long* topk_idx, float* topk_w,
                   unsigned* barrier, int T, int H, int E, int El, int e0, int I, int K, float eps, int router_act,
                   int act_over_topk, int normalize, int pre_scale, int round_logits, int act, float act_alpha, float act_beta,
                   float gate_lo, float gate_hi, float up_lo, float up_hi, bool cooperative, cudaStream_t st);

// ---- decode GEMV on MX (block-scaled fp4 / fp8) weights (gemv_mx.cu)
void gemv_mx(const void* x, const void* w, const void* scale, const void* residual, void* y, int M, int N, int K, int fmt,
             cudaStream_t st);

void gemv_mx_grouped(const void* x, const void* w, const void* scale, const long* expert, void* y, int S, int N, int K, int E, int fmt,
                     cudaStream_t st);

// ---- decode (decode.cu)
void decode_attention(const void* q, const void* k, const void* v, const long* positions, void* out, float* part_o,
                      float* part_ml, int B, int H, int Hkv, int D, int L, const long* ks, const long* vs, long q_sb,
                      long q_sh, long o_sb, long o_sh, float scale, int splits, int window, cudaStream_t st, float* fin_o,
                      float* fin_ml, bool kv_e4m3, float k_scale, float v_scale, bool rolling = false);
                      // q [B,1,H,D], k/v [B,L,Hkv,D] with D ∈ {64, 80, 96, 128}; part_o [B*H*splits, D]
                      // fin_o/fin_ml: un-normalised [B*H,D] + (max, sum) [B*H,2] instead of ``out`` (nullptr: ``out``)
                      // window: keys positions[b] − window < j ≤ positions[b] visible (0: no window)
                      // kv_e4m3: k/v are fp8 e4m3 caches holding k / k_scale and v / v_scale (bf16: both scales 1)
                      // rolling: the cache is a ring of L rows, position j in row j mod L (needs 0 < window < L)
// q/k/v [B,W,·,D] (strides qs/ks/vs = (b, s, h)); token w is rotated at positions[b] + depth[w] (depth null: + w), clamped to
// [0, n_pos) (n_pos: rows of cos_t / sin_t), and written to slot positions[b] + w, clamped to [0, L) (rolling: mod L)
void decode_rope_kv(const void* q, const void* k, const void* v, const long* positions, const long* depth, const float* cos_t,
                    const float* sin_t, void* q_out, void* kc, void* vc, int B, int W, int H, int Hkv, int D, int L, int n_pos,
                    const long* qs, const long* ks, const long* vs, long c_sb, long c_ss, long c_sh, cudaStream_t st, bool kv_e4m3,
                    float k_inv, float v_inv, bool rolling, int rot);   // kv_e4m3: the cache stores k·k_inv and v·v_inv as e4m3;
                                                                         // rot: rotary width R (even, 2 ≤ R ≤ D; R < D: dims ≥ R copied)
// merge of per-split decode partials [rows·splits, D] + (max, sum) → bf16 row r at out + (r / H)·o_sb + (r % H)·o_sh
void decode_combine(const float* part_o, const float* part_ml, void* out, int rows, int splits, int D, long o_sb, long o_sh,
                    int H, cudaStream_t st);
// bias: optional bf16 [N]; act: 0 none, 1 exact GELU, 2 tanh GELU (csrc/moe_tkg.cu numbering) → y = act(x·Wᵀ + bias) + residual
void gemv_bf16(const void* x, const void* w, const void* residual, void* y, int M, int N, int K, cudaStream_t st,
               const void* bias = nullptr, int act = 0);

// ---- attention (attention_sm90.cu): q [B,S_q,H,D], k/v [B,S_kv,Hkv,D] bf16 views, D ∈ {64, 80, 96, 128}; strides = (b, s, h)
// in elements.  kpm: optional key-padding mask, uint8 [B, S_kv] with row stride kpm_sb (key visible iff nonzero), or null.
// window: sliding window W (causal only; query i sees keys i − W < j ≤ i), or 0 for none.  q_offset ≥ 0 (window only): global
// position of query row 0 minus that of key row 0, so query i sees keys i + q_offset − W < j ≤ i + q_offset.
// dropout_p ∈ [0, 1): attention dropout by the rule in attention_sm90.cu, with the seed read on the device (int64 when
// seed64, else int32; needed when dropout_p > 0) and head h of this call counted as global head head_offset + h.
void flash_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int S_q, int S_kv, int H,
                    int Hkv, int D, const long* qs, const long* ks, const long* vs, const long* os, float scale, bool causal,
                    const void* kpm, long kpm_sb, long window, long q_offset, double dropout_p, const void* seed,
                    bool seed64, long head_offset, cudaStream_t st);

// delta: fp32 scratch [B, H, S_q]; dlse may be null
void flash_attn_bwd(const void* go, const void* q, const void* k, const void* v, const void* o, const float* lse,
                    const float* dlse, void* dq, void* dk, void* dv, float* delta, int B, int S_q, int S_kv, int H, int Hkv,
                    int D, const long* gs, const long* qs, const long* ks, const long* vs, const long* os, const long* dqs,
                    const long* dks, const long* dvs, float scale, bool causal, const void* kpm, long kpm_sb, long window,
                    long q_offset, double dropout_p, const void* seed, bool seed64, long head_offset, cudaStream_t st);

// W ≤ 64 new tokens per sequence against a KV cache (speculation / Medusa verification): q [B,W,H,D] bf16, k/v caches
// [B,L,Hkv,D] bf16 or e4m3 (kv_e4m3), D ∈ {64, 80, 96, 128}, H/Hkv ∈ {1,2,4,8}; mask uint8 [W,W] and depth int64 [W] (both
// null: a chain); window: sliding window (0: none).  part_o [B·W·H·splits, D] / part_ml [B·W·H·splits, 2] fp32 scratch; out
// [B,W,H,D].
// rolling: the cache is a ring of L rows, position j in row j mod L (needs window > 0 and window + W − 1 ≤ L).
void speculation_attention(const void* q, const void* k, const void* v, const long* positions, const void* mask,
                           const long* depth, void* out, float* part_o, float* part_ml, int B, int W, int H, int Hkv, int D,
                           int L, const long* qs, const long* ks, const long* vs, float scale, int window, int splits, bool kv_e4m3,
                           float k_scale, float v_scale, bool rolling, cudaStream_t st);

}  // namespace nxd
