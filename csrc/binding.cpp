// pybind11 bindings: tensor checks + raw-pointer extraction; all math lives in the .cu files.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cmath>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include "kernels.h"
#include "symm.h"

namespace py = pybind11;
using at::Tensor;

static int dt_code(const Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return nxd::kF32;
    case at::kBFloat16: return nxd::kBF16;
    case at::kHalf: return nxd::kF16;
    default: TORCH_CHECK(false, "unsupported dtype ", t.scalar_type());
  }
}
static cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }
static int num_sms() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }
#define CHECK_IN(t) TORCH_CHECK((t).is_cuda() && (t).is_contiguous(), #t " must be a contiguous CUDA tensor")

static std::vector<Tensor> rmsnorm_fwd(const Tensor& x, const Tensor& w, double eps) {
  CHECK_IN(x); CHECK_IN(w);
  TORCH_CHECK(x.dim() == 2 && w.numel() == x.size(1) && w.scalar_type() == x.scalar_type());
  c10::cuda::CUDAGuard g(x.device());
  auto y = at::empty_like(x);
  auto rstd = at::empty({x.size(0), 1}, x.options().dtype(at::kFloat));
  if (x.size(0) > 0)
    nxd::rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr<float>(), (int)x.size(0), (int)x.size(1),
                     (float)eps, dt_code(x), stream());
  return {y, rstd};
}

static std::vector<Tensor> rmsnorm_bwd(const Tensor& g, const Tensor& x, const Tensor& w, const Tensor& rstd) {
  CHECK_IN(g); CHECK_IN(x); CHECK_IN(w); CHECK_IN(rstd);
  c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), H = (int)x.size(1);
  auto dx = at::empty_like(x);
  auto dw = at::zeros({H}, x.options().dtype(at::kFloat));
  if (rows > 0) {
    auto partial = at::empty({nxd::rmsnorm_bwd_num_partials(rows), H}, x.options().dtype(at::kFloat));
    nxd::rmsnorm_bwd(g.data_ptr(), x.data_ptr(), w.data_ptr(), rstd.data_ptr<float>(), dx.data_ptr(),
                     partial.data_ptr<float>(), dw.data_ptr<float>(), rows, H, dt_code(x), stream());
  }
  return {dx, dw};
}

static std::vector<Tensor> add_rmsnorm_fwd(const Tensor& x, const Tensor& r, const Tensor& w, double eps) {
  CHECK_IN(x); CHECK_IN(r); CHECK_IN(w);
  TORCH_CHECK(x.dim() == 2 && r.sizes() == x.sizes() && w.numel() == x.size(1) && w.scalar_type() == x.scalar_type() &&
              r.scalar_type() == x.scalar_type());
  c10::cuda::CUDAGuard g(x.device());
  auto h = at::empty_like(x);
  auto y = at::empty_like(x);
  auto rstd = at::empty({x.size(0), 1}, x.options().dtype(at::kFloat));
  if (x.size(0) > 0)
    nxd::add_rmsnorm_fwd(x.data_ptr(), r.data_ptr(), w.data_ptr(), h.data_ptr(), y.data_ptr(), rstd.data_ptr<float>(),
                         (int)x.size(0), (int)x.size(1), (float)eps, dt_code(x), stream());
  return {y, h, rstd};
}

static std::vector<Tensor> add_rmsnorm_bwd(const Tensor& gy, const Tensor& gh, const Tensor& h, const Tensor& w, const Tensor& rstd) {
  CHECK_IN(gy); CHECK_IN(gh); CHECK_IN(h); CHECK_IN(w); CHECK_IN(rstd);
  c10::cuda::CUDAGuard guard(h.device());
  const int rows = (int)h.size(0), H = (int)h.size(1);
  auto dh = at::empty_like(h);
  auto dw = at::zeros({H}, h.options().dtype(at::kFloat));
  if (rows > 0) {
    auto partial = at::empty({nxd::rmsnorm_bwd_num_partials(rows), H}, h.options().dtype(at::kFloat));
    nxd::add_rmsnorm_bwd(gy.data_ptr(), gh.data_ptr(), h.data_ptr(), w.data_ptr(), rstd.data_ptr<float>(), dh.data_ptr(),
                         partial.data_ptr<float>(), dw.data_ptr<float>(), rows, H, dt_code(h), stream());
  }
  return {dh, dw};
}

static Tensor swiglu_fwd(const Tensor& gu) {
  CHECK_IN(gu);
  c10::cuda::CUDAGuard g(gu.device());
  const int I = (int)gu.size(1) / 2;
  auto out = at::empty({gu.size(0), I}, gu.options());
  if (gu.numel()) nxd::swiglu_fwd(gu.data_ptr(), out.data_ptr(), gu.size(0), I, dt_code(gu), stream());
  return out;
}
static Tensor swiglu_bwd(const Tensor& go, const Tensor& gu) {
  CHECK_IN(go); CHECK_IN(gu);
  c10::cuda::CUDAGuard g(gu.device());
  auto d = at::empty_like(gu);
  if (gu.numel()) nxd::swiglu_bwd(go.data_ptr(), gu.data_ptr(), d.data_ptr(), gu.size(0), (int)gu.size(1) / 2, dt_code(gu), stream());
  return d;
}

static Tensor rope_apply(const Tensor& x, const Tensor& cos_t, const Tensor& sin_t, double sign) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && x.stride(3) == 1, "rope: x must be [B,S,H,D] with contiguous D");
  CHECK_IN(cos_t); CHECK_IN(sin_t);
  TORCH_CHECK(cos_t.scalar_type() == at::kFloat && cos_t.size(0) >= x.size(1) && cos_t.size(1) == x.size(3) / 2);
  c10::cuda::CUDAGuard g(x.device());
  auto out = at::empty(x.sizes(), x.options());
  const int es = (int)x.element_size();
  (void)es;      // unaligned / odd rotary dims take the scalar kernel (csrc/elementwise.cu rope_scalar_kernel)
  if (x.numel())
    nxd::rope_apply(x.data_ptr(), out.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), (int)x.size(0),
                    (int)x.size(1), (int)x.size(2), (int)x.size(3), x.stride(0), x.stride(1), x.stride(2), (float)sign,
                    dt_code(x), stream());
  return out;
}

static Tensor ce_stats(const Tensor& logits, const Tensor& target, int64_t vocab_start) {
  CHECK_IN(logits); CHECK_IN(target);
  TORCH_CHECK(target.scalar_type() == at::kLong && logits.dim() == 2 && target.numel() == logits.size(0));
  c10::cuda::CUDAGuard g(logits.device());
  auto stats = at::empty({logits.size(0), 4}, logits.options().dtype(at::kFloat));
  if (logits.size(0))
    nxd::ce_stats(logits.data_ptr(), target.data_ptr<int64_t>(), stats.data_ptr<float>(), (int)logits.size(0),
                  (int)logits.size(1), (int)vocab_start, dt_code(logits), stream());
  return stats;
}
static Tensor ce_backward(const Tensor& logits, const Tensor& target, const Tensor& lse, const Tensor& gout,
                          int64_t vocab_start, double smoothing, int64_t vocab) {
  CHECK_IN(logits); CHECK_IN(target); CHECK_IN(lse); CHECK_IN(gout);
  c10::cuda::CUDAGuard g(logits.device());
  auto grad = at::empty_like(logits);
  if (logits.size(0))
    nxd::ce_backward(logits.data_ptr(), target.data_ptr<int64_t>(), lse.data_ptr<float>(), gout.data_ptr<float>(),
                     grad.data_ptr(), (int)logits.size(0), (int)logits.size(1), (int)vocab_start, (float)smoothing,
                     (int)vocab, dt_code(logits), stream());
  return grad;
}

static std::vector<nxd::TensorRef> refs(const std::vector<Tensor>& ts) {
  std::vector<nxd::TensorRef> r;
  r.reserve(ts.size());
  for (auto& t : ts) {
    TORCH_CHECK(t.is_cuda() && t.is_contiguous());
    r.push_back({t.data_ptr(), (long)t.numel()});
  }
  return r;
}
static void multi_tensor_sq_norm(const std::vector<Tensor>& ts, Tensor out) {
  if (ts.empty()) return;
  c10::cuda::CUDAGuard g(ts[0].device());
  nxd::multi_tensor_sq_norm(refs(ts), dt_code(ts[0]), out.data_ptr<float>(), stream());
}
static void multi_tensor_scale(const std::vector<Tensor>& ts, const Tensor& scale) {
  if (ts.empty()) return;
  c10::cuda::CUDAGuard g(ts[0].device());
  nxd::multi_tensor_scale(refs(ts), dt_code(ts[0]), scale.data_ptr<float>(), stream());
}
static void fused_adamw(const std::vector<Tensor>& p, const std::vector<Tensor>& g, const std::vector<Tensor>& m,
                        const std::vector<Tensor>& v, const std::vector<Tensor>& lowp, double lr, double b1, double b2,
                        double eps, double wd, double bc1, double bc2, const Tensor& grad_scale, bool hf_form) {
  if (p.empty()) return;
  TORCH_CHECK(p[0].scalar_type() == at::kFloat && m[0].scalar_type() == at::kFloat);
  c10::cuda::CUDAGuard guard(p[0].device());
  nxd::fused_adamw(refs(p), refs(g), refs(m), refs(v), refs(lowp), dt_code(g[0]), lowp.empty() ? 0 : dt_code(lowp[0]),
                   (float)lr, (float)b1, (float)b2, (float)eps, (float)wd, (float)bc1, (float)bc2,
                   grad_scale.data_ptr<float>(), hf_form ? 1 : 0, stream());
}

// out bf16 [M, N], or fp32 [M, N] that `accumulate` adds into (the fp8 weight gradient into an fp32 main_grad)
static void gemm_fp8(const Tensor& a, const Tensor& b, Tensor out, const Tensor& scale_a, const Tensor& scale_b, bool accumulate) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn);
  TORCH_CHECK(a.is_contiguous() && b.is_contiguous() && out.is_contiguous() &&
              (out.scalar_type() == at::kBFloat16 || out.scalar_type() == at::kFloat));
  TORCH_CHECK(!accumulate || out.scalar_type() == at::kFloat, "gemm_fp8: accumulate needs an fp32 out");
  // the register epilogue (out without a 16-byte aligned tensor map) stores element pairs
  TORCH_CHECK(reinterpret_cast<uintptr_t>(out.data_ptr()) % (2 * out.element_size()) == 0,
              "gemm_fp8: out must start aligned to two elements");
  const int M = a.size(0), K = a.size(1), N = b.size(0);
  TORCH_CHECK(b.size(1) == K && out.size(0) == M && out.size(1) == N && K % 16 == 0 && N % 8 == 0);
  TORCH_CHECK(scale_a.scalar_type() == at::kFloat && scale_a.numel() == M && scale_b.scalar_type() == at::kFloat &&
              scale_b.numel() == N && scale_a.is_contiguous() && scale_b.is_contiguous());
  c10::cuda::CUDAGuard guard(a.device());
  nxd::gemm_fp8(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, scale_a.data_ptr<float>(), scale_b.data_ptr<float>(),
                dt_code(out), accumulate, stream());
}

// x bf16 [M, K] → (e4m3 [M, K], fp32 [M]): one absmax scale per row
static std::vector<Tensor> quantize_fp8_rows(const Tensor& x) {
  CHECK_IN(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.size(1) % 8 == 0, "quantize_fp8_rows: bf16 [M, K], K % 8 == 0");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "quantize_fp8_rows: x must start 16-byte aligned");
  const int M = x.size(0), K = x.size(1);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = at::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = at::empty({M}, x.options().dtype(at::kFloat));
  nxd::quantize_fp8_rows(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), M, K, stream());
  return {q, s};
}

// x bf16 [R, C] → (e4m3 [C, R], fp32 [C]): the rows of xᵀ, one absmax scale per column of x
static std::vector<Tensor> quantize_fp8_cols_t(const Tensor& x) {
  CHECK_IN(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.size(0) % 16 == 0 && x.size(1) % 8 == 0,
              "quantize_fp8_cols_t: bf16 [R, C], R % 16 == 0 (the e4m3 rows are a TMA operand) and C % 8 == 0");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "quantize_fp8_cols_t: x must start 16-byte aligned");
  const int R = x.size(0), C = x.size(1);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = at::empty({C, R}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = at::empty({C}, x.options().dtype(at::kFloat));
  Tensor amax = at::zeros({C}, x.options().dtype(at::kInt));
  nxd::quantize_fp8_cols_t(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), reinterpret_cast<uint32_t*>(amax.data_ptr<int>()),
                           R, C, stream());
  return {q, s};
}

// a e4m3 [M, K], b e4m3 [N, K]; scale_a fp32 [K/group, M] with unit column stride (row stride >= M, a multiple of 4);
// scale_b fp32 [K/group, N] contiguous → bf16 [M, N]
static Tensor gemm_fp8_block(const Tensor& a, const Tensor& b, const Tensor& scale_a, const Tensor& scale_b, int64_t group) {
  CHECK_IN(a); CHECK_IN(b); CHECK_IN(scale_b);
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn && a.dim() == 2 && b.dim() == 2 &&
              a.size(1) == b.size(1), "gemm_fp8_block: a [M, K] and b [N, K] must be e4m3");
  const int M = a.size(0), K = a.size(1), N = b.size(0);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(a.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(b.data_ptr()) % 16 == 0,
              "gemm_fp8_block: a and b must start 16-byte aligned (TMA)");
  TORCH_CHECK(group > 0 && K % group == 0, "gemm_fp8_block: K must be a multiple of the group size");
  TORCH_CHECK(scale_a.is_cuda() && scale_a.scalar_type() == at::kFloat && scale_a.dim() == 2 && scale_a.size(0) == K / group &&
              scale_a.size(1) == M && scale_a.stride(1) == 1 && reinterpret_cast<uintptr_t>(scale_a.data_ptr()) % 16 == 0,
              "gemm_fp8_block: scale_a must be fp32 [K/group, M] with unit column stride and a 16-byte aligned start");
  TORCH_CHECK(scale_b.scalar_type() == at::kFloat && scale_b.dim() == 2 && scale_b.size(0) == K / group && scale_b.size(1) == N,
              "gemm_fp8_block: scale_b must be fp32 [K/group, N]");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor out = at::empty({M, N}, a.options().dtype(at::kBFloat16));
  nxd::gemm_fp8_block(a.data_ptr(), b.data_ptr(), out.data_ptr(), scale_a.data_ptr<float>(), scale_a.stride(0),
                      scale_b.data_ptr<float>(), M, N, K, (int)group, stream());
  return out;
}

// grouped (MoE) mode: a e4m3 [M, K] in block_rows-row blocks, block i using expert block_expert[i]; b e4m3 [E, N, K]
// (K-major experts); scale_a as gemm_fp8_block; scale_b fp32 [E, K/group, N] → bf16 [M, N]
static Tensor grouped_gemm_fp8_block(const Tensor& a, const Tensor& b, const Tensor& scale_a, const Tensor& scale_b,
                                     const Tensor& block_expert, int64_t block_rows, int64_t group) {
  CHECK_IN(a); CHECK_IN(b); CHECK_IN(scale_b); CHECK_IN(block_expert);
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn && a.dim() == 2 && b.dim() == 3 &&
              a.size(1) == b.size(2), "grouped_gemm_fp8_block: a [M, K] and b [E, N, K] must be e4m3");
  const int M = a.size(0), K = a.size(1), E = b.size(0), N = b.size(1);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(a.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(b.data_ptr()) % 16 == 0 &&
              reinterpret_cast<uintptr_t>(scale_b.data_ptr()) % 16 == 0,
              "grouped_gemm_fp8_block: a, b and scale_b must start 16-byte aligned (TMA)");
  TORCH_CHECK(group == 32 || group == 64 || group == 128, "grouped_gemm_fp8_block: group size must be 32, 64 or 128");
  TORCH_CHECK(K % 128 == 0 && N % 8 == 0, "grouped_gemm_fp8_block: needs K % 128 == 0 and N % 8 == 0");
  TORCH_CHECK(block_rows > 0 && block_rows % 128 == 0, "grouped_gemm_fp8_block: block_rows must be a positive multiple of 128");
  TORCH_CHECK(block_expert.scalar_type() == at::kInt && block_expert.dim() == 1 && block_expert.numel() * block_rows == M,
              "grouped_gemm_fp8_block: block_expert must be int32 [M / block_rows]");
  TORCH_CHECK(scale_a.is_cuda() && scale_a.scalar_type() == at::kFloat && scale_a.dim() == 2 && scale_a.size(0) == K / group &&
              scale_a.size(1) == M && scale_a.stride(1) == 1 && scale_a.stride(0) >= M && scale_a.stride(0) % 4 == 0 &&
              reinterpret_cast<uintptr_t>(scale_a.data_ptr()) % 16 == 0,
              "grouped_gemm_fp8_block: scale_a must be fp32 [K/group, M] with unit column stride, a row stride >= M that is a "
              "multiple of 4 and a 16-byte aligned start");
  TORCH_CHECK(scale_b.scalar_type() == at::kFloat && scale_b.dim() == 3 && scale_b.size(0) == E && scale_b.size(1) == K / group &&
              scale_b.size(2) == N, "grouped_gemm_fp8_block: scale_b must be fp32 [E, K/group, N]");
  TORCH_CHECK(b.device() == a.device() && scale_a.device() == a.device() && scale_b.device() == a.device() &&
              block_expert.device() == a.device(), "grouped_gemm_fp8_block: all operands must be on one device");
  c10::cuda::CUDAGuard guard(a.device());
  Tensor out = at::empty({M, N}, a.options().dtype(at::kBFloat16));
  nxd::grouped_gemm_fp8_block(a.data_ptr(), b.data_ptr(), out.data_ptr(), scale_a.data_ptr<float>(), scale_a.stride(0),
                              scale_b.data_ptr<float>(), M, N, K, E, block_expert.data_ptr<int>(), (int)block_rows, (int)group,
                              stream());
  return out;
}

// x bf16 [M, K] → (e4m3 [M, K], fp32 scales [K/group, round_up(M, 4)]: group-major, the layout gemm_fp8_block reads)
static std::vector<Tensor> quantize_fp8_groups(const Tensor& x, int64_t group, bool mx, double clamp_bound) {
  CHECK_IN(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.size(1) % group == 0, "quantize_fp8_groups: bf16 [M, K], K % group == 0");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "quantize_fp8_groups: x must start 16-byte aligned");
  const int M = x.size(0), K = x.size(1);
  const long ld = ((long)M + 3) / 4 * 4;
  c10::cuda::CUDAGuard guard(x.device());
  Tensor q = at::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor s = at::empty({K / group, ld}, x.options().dtype(at::kFloat));
  nxd::quantize_fp8_groups(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), M, K, ld, (int)group, mx, (float)clamp_bound, stream());
  return {q, s};
}

static Tensor oneshot_allreduce(const Tensor& x, const Tensor& peer_bufs, const Tensor& peer_flags, int64_t slot_bytes,
                                Tensor state, int64_t rank, int64_t world) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && (x.scalar_type() == at::kBFloat16 || x.scalar_type() == at::kFloat));
  const long nbytes = x.numel() * x.element_size();
  TORCH_CHECK(nbytes % 16 == 0 && nbytes <= slot_bytes && state.scalar_type() == at::kInt && state.numel() >= 2);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty_like(x);
  int ctas = (int)std::max<long>(1, std::min<long>(64, nbytes / 16384));
  nxd::oneshot_allreduce(x.data_ptr(), out.data_ptr(), peer_bufs.data_ptr<int64_t>(), peer_flags.data_ptr<int64_t>(), slot_bytes,
                         (uint32_t*)state.data_ptr(), (int)rank, (int)world, x.numel(), dt_code(x), ctas, stream());
  return out;
}

// ---- row selection (sampling) -------------------------------------------------------------------------
static py::tuple row_argmax(const Tensor& x, int64_t index_offset) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1, "row_argmax: [rows, V] with contiguous last dim");
  c10::cuda::CUDAGuard g(x.device());
  auto val = at::empty({x.size(0)}, x.options().dtype(at::kFloat));
  auto idx = at::empty({x.size(0)}, x.options().dtype(at::kLong));
  nxd::row_argmax(x.data_ptr(), val.data_ptr<float>(), idx.data_ptr<long>(), (int)x.size(0), (int)x.size(1), x.stride(0), index_offset,
                  dt_code(x), stream());
  return py::make_tuple(val, idx);
}
static bool row_topk_supported(int64_t V, int64_t k) { return nxd::row_topk_supported((int)V, (int)k); }
static py::tuple row_topk(const Tensor& x, int64_t k, int64_t index_offset) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1, "row_topk: [rows, V] with contiguous last dim");
  c10::cuda::CUDAGuard g(x.device());
  auto vals = at::empty({x.size(0), k}, x.options().dtype(at::kFloat));
  auto idx = at::empty({x.size(0), k}, x.options().dtype(at::kLong));
  nxd::row_topk(x.data_ptr(), vals.data_ptr<float>(), idx.data_ptr<long>(), (int)x.size(0), (int)x.size(1), (int)k, x.stride(0),
                index_offset, dt_code(x), stream());
  return py::make_tuple(vals, idx);
}

// expert_index [T, k] (int32 / int64) → (block_to_expert [nb], token_position_to_id [nb*B], tokens_per_expert [E]) int64
static py::tuple moe_block_metadata(const Tensor& expert_index, int64_t num_experts, int64_t block_size, int64_t num_blocks) {
  CHECK_IN(expert_index);
  TORCH_CHECK(expert_index.dim() == 2 && (expert_index.scalar_type() == at::kLong || expert_index.scalar_type() == at::kInt));
  c10::cuda::CUDAGuard g(expert_index.device());
  auto o = expert_index.options().dtype(at::kLong);
  auto b2e = at::empty({num_blocks}, o), tp2id = at::empty({num_blocks * block_size}, o), counts = at::empty({num_experts}, o);
  nxd::moe_block_metadata(expert_index.data_ptr(), expert_index.scalar_type() == at::kLong, expert_index.numel(), (int)expert_index.size(1),
                          (int)num_experts, (int)block_size, (int)num_blocks, b2e.data_ptr<long>(), tp2id.data_ptr<long>(),
                          counts.data_ptr<long>(), stream());
  return py::make_tuple(b2e, tp2id, counts);
}

// KV-cache element type of the decode kernels: bf16, or fp8 e4m3 holding k / k_scale and v / v_scale (one fp32 scale per
// tensor, the format of inference/kv_cache.py).  Returns true for e4m3.
static bool kv_cache_e4m3(const char* fn, const Tensor& kc, const Tensor& vc, double k_scale, double v_scale) {
  const auto t = kc.scalar_type();
  TORCH_CHECK(t == at::kBFloat16 || t == at::kFloat8_e4m3fn, fn, ": the KV cache must be bfloat16 or float8_e4m3fn, got ", t);
  TORCH_CHECK(vc.scalar_type() == t, fn, ": k and v caches must have the same dtype");
  TORCH_CHECK(k_scale > 0 && v_scale > 0 && std::isfinite(k_scale) && std::isfinite(v_scale), fn, ": scales must be finite and > 0");
  TORCH_CHECK(t != at::kBFloat16 || (k_scale == 1.0 && v_scale == 1.0), fn, ": k_scale / v_scale apply to an fp8 cache only");
  return t == at::kFloat8_e4m3fn;
}

// q [B,W,H,D], k/v [B,W,Hkv,D] (views of the fused QKV projection output), cache [B,L,Hkv,D]: rotate q → new tensor, rotate
// k and copy v straight into the cache (token w at slot positions[b] + w, rotated at positions[b] + depth[w], or + w without
// depth; an e4m3 cache gets k / k_scale and v / v_scale, rounded as the cache's torch rule rounds them).  rolling: the cache is
// a ring of L rows, token w goes to row (positions[b] + w) mod L, and the rotation position is clamped to the table length
// instead of L.
static Tensor decode_rope_kv(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& positions, const Tensor& cos_t,
                             const Tensor& sin_t, Tensor kc, Tensor vc, double k_scale, double v_scale,
                             const c10::optional<Tensor>& depth, bool rolling) {
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kBFloat16 && q.dim() == 4 && q.size(1) >= 1 && q.stride(3) == 1);
  TORCH_CHECK(k.scalar_type() == at::kBFloat16 && k.dim() == 4 && k.size(1) == q.size(1) && k.stride(3) == 1 && v.stride(3) == 1 && v.sizes() == k.sizes());
  const bool e4m3 = kv_cache_e4m3("decode_rope_kv", kc, vc, k_scale, v_scale);
  TORCH_CHECK(kc.dim() == 4 && kc.stride(3) == 1 && vc.sizes() == kc.sizes() && vc.strides() == kc.strides());
  TORCH_CHECK(positions.scalar_type() == at::kLong && positions.is_contiguous() && positions.numel() == q.size(0));
  CHECK_IN(cos_t); CHECK_IN(sin_t);
  // the tables' width is half the rotary width R: R = D rotates the whole head, R < D (GPT-NeoX rotary_pct) only its first R dims
  TORCH_CHECK(cos_t.scalar_type() == at::kFloat && cos_t.size(0) >= kc.size(1) && sin_t.sizes() == cos_t.sizes(),
              "decode_rope_kv: cos and sin must be fp32 tables of the same shape, at least as long as the cache");
  TORCH_CHECK(cos_t.dim() == 2 && cos_t.size(1) >= 1 && 2 * cos_t.size(1) <= q.size(3),
              "decode_rope_kv: the cos/sin tables must be [n_pos, R/2] with rotary width R even and 2 <= R <= head_dim");
  // rolling: positions run past the ring, up to the table length, which bounds the rotation instead of L (both tables are
  // read, so the shorter one bounds it).  The W slots of one call are distinct rows when W <= L, which the caller keeps
  // (LlamaForInference: W <= 64 < L).
  const long* dp = nullptr;
  if (depth.has_value()) {
    TORCH_CHECK(depth->is_cuda() && depth->scalar_type() == at::kLong && depth->is_contiguous() && depth->numel() == q.size(1),
                "decode_rope_kv: depth must be a contiguous int64 CUDA tensor [W]");
    dp = depth->data_ptr<long>();
  }
  c10::cuda::CUDAGuard g(q.device());
  const int B = (int)q.size(0), W = (int)q.size(1), H = (int)q.size(2), Hkv = (int)k.size(2), D = (int)q.size(3), L = (int)kc.size(1);
  Tensor q_out = at::empty({B, W, H, D}, q.options());
  const long qs[3] = {q.stride(0), q.stride(1), q.stride(2)}, ks[3] = {k.stride(0), k.stride(1), k.stride(2)};
  const long vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  const int n_pos = rolling ? (int)std::min<int64_t>(std::min(cos_t.size(0), sin_t.size(0)), INT32_MAX) : L;
  nxd::decode_rope_kv(q.data_ptr(), k.data_ptr(), v.data_ptr(), positions.data_ptr<long>(), dp, cos_t.data_ptr<float>(),
                      sin_t.data_ptr<float>(), q_out.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, W, H, Hkv, D, L, n_pos, qs, ks,
                      vs, kc.stride(0), kc.stride(1), kc.stride(2), stream(), e4m3, 1.0f / (float)k_scale, 1.0f / (float)v_scale,
                      rolling, 2 * (int)cos_t.size(1));
  return q_out;
}

// ---- decode ---------------------------------------------------------------------------------------
// q [B,1,H,D]; k/v cache [B,L,Hkv,D], D ∈ {64, 80, 96, 128} (any b/s/h strides, head_dim contiguous); positions [B] int64 (attend to ≤ pos);
// window > 0: only the last `window` positions up to pos are visible.  The cache is bf16, or e4m3 with per-tensor scales
// (the kernel then loads 8 bytes per lane: base pointers and strides must be multiples of 8 elements, as on bf16)
static int decode_splits(int B, int Hkv, int L, int64_t window) {
  TORCH_CHECK(window >= 0, "decode_attention: window must be >= 0 (0 = none)");
  const int rows = window > 0 && window < L ? (int)window : L;      // cache rows one sequence reads at most
  // enough CTAs for ~6 per SM (the kernel is latency-bound per CTA: 8 cache rows in flight), at least 64 rows per split
  int splits = (6 * num_sms() + B * Hkv - 1) / (B * Hkv);
  return std::max(1, std::min(std::min(splits, 64), (rows + 63) / 64));
}
// argument checks shared by decode_attention, decode_attention_partial (one token per sequence) and speculation_attention
// (max_tokens = 64); returns true for an e4m3 cache.  The head sizes are those of the flash kernels (check_qkv).
static bool check_decode_args(const char* fn, const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& positions,
                              double k_scale, double v_scale, int64_t max_tokens = 1) {
  const int64_t d = q.dim() == 4 ? q.size(3) : 0;
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kBFloat16 && q.dim() == 4 && q.size(1) >= 1 && q.size(1) <= max_tokens &&
                  (d == 64 || d == 80 || d == 96 || d == 128) && q.stride(3) == 1,
              fn, ": expected a bf16 CUDA q [B,W,H,D] view (W = 1; verification: W <= 64) with D in {64, 80, 96, 128} and "
              "contiguous head_dim");
  const bool e4m3 = kv_cache_e4m3(fn, k, v, k_scale, v_scale);
  TORCH_CHECK(k.dim() == 4 && k.size(3) == d && k.stride(3) == 1 && v.stride(3) == 1 && v.sizes() == k.sizes(),
              fn, ": expected k / v caches [B,L,Hkv,D] of one shape, with q's D and contiguous head_dim");
  TORCH_CHECK(positions.scalar_type() == at::kLong && positions.is_cuda() && positions.is_contiguous() && positions.numel() == q.size(0));
  TORCH_CHECK(q.size(2) % k.size(2) == 0 && k.size(0) == q.size(0));
  TORCH_CHECK(q.stride(2) % 8 == 0 && k.stride(1) % 8 == 0 && k.stride(2) % 8 == 0 && v.stride(1) % 8 == 0 && v.stride(2) % 8 == 0);
  TORCH_CHECK(!e4m3 || ((reinterpret_cast<uintptr_t>(k.data_ptr()) | reinterpret_cast<uintptr_t>(v.data_ptr())) % 8 == 0 &&
                        k.stride(0) % 8 == 0 && v.stride(0) % 8 == 0),
              fn, ": e4m3 caches are read 8 bytes at a time: their base addresses and strides must be multiples of 8");
  return e4m3;
}
// rolling: the cache is a ring of L rows holding position j in row j mod L; only a sliding window shorter than the ring
// keeps every visible position in its own row
static Tensor decode_attention(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& positions, double scale,
                               int64_t window, double k_scale, double v_scale, bool rolling) {
  const bool e4m3 = check_decode_args("decode_attention", q, k, v, positions, k_scale, v_scale);
  const int B = q.size(0), H = q.size(2), D = q.size(3), L = k.size(1), Hkv = k.size(2);
  TORCH_CHECK(!rolling || (window > 0 && window < L), "decode_attention: a rolling cache needs 0 < window < L (",
                    L, " rows), got window ", window);
  c10::cuda::CUDAGuard guard(q.device());
  const int splits = decode_splits(B, Hkv, L, window);
  Tensor out = at::empty({B, 1, H, D}, q.options());
  Tensor part_o = at::empty({B * H * splits, D}, q.options().dtype(at::kFloat));
  Tensor part_ml = at::empty({B * H * splits, 2}, q.options().dtype(at::kFloat));
  const long ks[3] = {k.stride(0), k.stride(1), k.stride(2)}, vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  nxd::decode_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), positions.data_ptr<long>(), out.data_ptr(),
                        part_o.data_ptr<float>(), part_ml.data_ptr<float>(), B, H, Hkv, D, L, ks, vs, q.stride(0), q.stride(2),
                        out.stride(0), out.stride(2), (float)scale, splits, (int)std::min<int64_t>(window, INT32_MAX), stream(),
                        nullptr, nullptr, e4m3, (float)k_scale, (float)v_scale, rolling);
  return out;
}
// This rank's contribution to distributed flash-decoding: un-normalised output (relative to the row maximum) [B,H,D] fp32 and
// (row maximum in natural-log units, row sum) [B,H,2] fp32 over the local cache shard; ``positions`` are LOCAL (may be < 0 or
// >= L: nothing / everything of this shard is visible).
static std::vector<Tensor> decode_attention_partial(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& positions,
                                                    double scale, int64_t window, double k_scale, double v_scale) {
  const bool e4m3 = check_decode_args("decode_attention_partial", q, k, v, positions, k_scale, v_scale);
  const int B = q.size(0), H = q.size(2), D = q.size(3), L = k.size(1), Hkv = k.size(2);
  c10::cuda::CUDAGuard guard(q.device());
  const int splits = decode_splits(B, Hkv, L, window);
  Tensor fin_o = at::empty({B, H, D}, q.options().dtype(at::kFloat));
  Tensor fin_ml = at::empty({B, H, 2}, q.options().dtype(at::kFloat));
  Tensor part_o = at::empty({B * H * splits, D}, q.options().dtype(at::kFloat));
  Tensor part_ml = at::empty({B * H * splits, 2}, q.options().dtype(at::kFloat));
  const long ks[3] = {k.stride(0), k.stride(1), k.stride(2)}, vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  nxd::decode_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), positions.data_ptr<long>(), nullptr, part_o.data_ptr<float>(),
                        part_ml.data_ptr<float>(), B, H, Hkv, D, L, ks, vs, q.stride(0), q.stride(2), 0, 0, (float)scale, splits,
                        (int)std::min<int64_t>(window, INT32_MAX), stream(), fin_o.data_ptr<float>(), fin_ml.data_ptr<float>(),
                        e4m3, (float)k_scale, (float)v_scale);
  return {fin_o, fin_ml};
}
// q [B,W≤64,H,D] (any b/s/h strides, rows 16-byte aligned) verified against the cache as decode_attention reads it; tree_mask
// [W,W] bool / uint8 and tree_depth [W] int64 (both or neither: a chain).  Never reads them on the host.  rolling: a ring of L
// rows, as in decode_attention.
static Tensor speculation_attention(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& positions,
                                    const c10::optional<Tensor>& tree_mask, const c10::optional<Tensor>& tree_depth, double scale,
                                    int64_t window, double k_scale, double v_scale, bool rolling) {
  const char* fn = "speculation_attention";
  const bool e4m3 = check_decode_args(fn, q, k, v, positions, k_scale, v_scale, 64);
  const int B = q.size(0), W = q.size(1), H = q.size(2), D = q.size(3), L = k.size(1), Hkv = k.size(2), G = H / Hkv;
  TORCH_CHECK(reinterpret_cast<uintptr_t>(q.data_ptr()) % 16 == 0 && q.stride(0) % 8 == 0 && q.stride(1) % 8 == 0,
              fn, ": q rows must be 16-byte aligned");
  TORCH_CHECK(e4m3 || ((reinterpret_cast<uintptr_t>(k.data_ptr()) | reinterpret_cast<uintptr_t>(v.data_ptr())) % 16 == 0 &&
                       k.stride(0) % 8 == 0 && v.stride(0) % 8 == 0),
              fn, ": bf16 cache rows must be 16-byte aligned");
  TORCH_CHECK(window >= 0, fn, ": window must be >= 0 (0 = none)");
  // token w writes row (p + w) mod L over position p + w − L, which no token of the window may see: every token sees only
  // positions > p − window, so p + W − 1 − L ≤ p − window
  TORCH_CHECK(!rolling || (window > 0 && window + W - 1 <= L), fn, ": a rolling cache needs window > 0 and window + W - 1 "
                    "<= L, got window ", window, ", W ", W, ", L ", L);
  TORCH_CHECK(tree_mask.has_value() == tree_depth.has_value(), fn, ": tree_mask and tree_depth go together");
  const void* mp = nullptr;
  const long* dp = nullptr;
  if (tree_mask.has_value()) {
    TORCH_CHECK((tree_mask->scalar_type() == at::kBool || tree_mask->scalar_type() == at::kByte) && tree_mask->is_contiguous() &&
                    tree_mask->dim() == 2 && tree_mask->size(0) == W && tree_mask->size(1) == W && tree_mask->device() == q.device(),
                fn, ": tree_mask must be a contiguous bool / uint8 [W, W] tensor on q's device");
    TORCH_CHECK(tree_depth->scalar_type() == at::kLong && tree_depth->is_contiguous() && tree_depth->numel() == W &&
                    tree_depth->device() == q.device(),
                fn, ": tree_depth must be a contiguous int64 [W] tensor on q's device");
    mp = tree_mask->data_ptr();
    dp = tree_depth->data_ptr<long>();
  }
  c10::cuda::CUDAGuard guard(q.device());
  // slots one row tile reads at most; enough CTAs for ~4 per SM, at least 128 slots per split
  const int row_tiles = (W * G + 63) / 64;
  const int64_t rows = window > 0 ? std::min<int64_t>(L, std::min<int64_t>(window, L) + W - 1) : L;
  const int ctas = B * Hkv * row_tiles;
  const int splits = std::max(1, std::min({(4 * num_sms() + ctas - 1) / ctas, 64, (int)((rows + 127) / 128)}));
  Tensor out = at::empty({B, W, H, D}, q.options());
  Tensor part_o = at::empty({(int64_t)B * W * H * splits, D}, q.options().dtype(at::kFloat));
  Tensor part_ml = at::empty({(int64_t)B * W * H * splits, 2}, q.options().dtype(at::kFloat));
  const long qs[3] = {q.stride(0), q.stride(1), q.stride(2)};
  const long ks[3] = {k.stride(0), k.stride(1), k.stride(2)}, vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  nxd::speculation_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), positions.data_ptr<long>(), mp, dp, out.data_ptr(),
                             part_o.data_ptr<float>(), part_ml.data_ptr<float>(), B, W, H, Hkv, D, L, qs, ks, vs, (float)scale,
                             (int)std::min<int64_t>(window, INT32_MAX), splits, e4m3, (float)k_scale, (float)v_scale, rolling,
                             stream());
  return out;
}
// x [T,H] bf16; gamma [H] bf16 or none; router_w [E,H] bf16; router_bias [E] fp32 or none; w_gu [El,H,2I]; w_dn [El,I,H]
// → (out [T,H] bf16 partial over this rank's experts / intermediate shard, router logits [T,E] fp32, top-k idx [T,K], top-k w [T,K])
static std::vector<Tensor> moe_block_tkg(const Tensor& x, const c10::optional<Tensor>& gamma, const Tensor& router_w,
                                         const c10::optional<Tensor>& router_bias, const Tensor& w_gu, const Tensor& w_dn,
                                         int64_t e0, int64_t top_k, double eps, int64_t router_act, bool act_over_topk, bool normalize,
                                         bool pre_scale, bool round_logits, int64_t act, double act_alpha, double act_beta,
                                         double gate_lo, double gate_hi, double up_lo, double up_hi, bool cooperative) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous());
  TORCH_CHECK(router_w.scalar_type() == at::kBFloat16 && router_w.dim() == 2 && router_w.is_contiguous() && router_w.size(1) == x.size(1));
  TORCH_CHECK(w_gu.scalar_type() == at::kBFloat16 && w_gu.dim() == 3 && w_gu.is_contiguous() && w_gu.size(1) == x.size(1) &&
              w_gu.size(2) % 2 == 0);
  TORCH_CHECK(w_dn.scalar_type() == at::kBFloat16 && w_dn.dim() == 3 && w_dn.is_contiguous() && w_dn.size(0) == w_gu.size(0) &&
              w_dn.size(1) * 2 == w_gu.size(2) && w_dn.size(2) == x.size(1));
  const int T = x.size(0), H = x.size(1), E = router_w.size(0), El = w_gu.size(0), I = w_dn.size(1), K = top_k;
  TORCH_CHECK(nxd::moe_block_tkg_supported(T, H, E, I, K), "moe_block_tkg: unsupported shape");
  TORCH_CHECK(e0 >= 0 && e0 + El <= E);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(x.data_ptr()) | reinterpret_cast<uintptr_t>(router_w.data_ptr()) |
               reinterpret_cast<uintptr_t>(w_gu.data_ptr()) | reinterpret_cast<uintptr_t>(w_dn.data_ptr())) % 16 == 0,
              "moe_block_tkg: x, router_w, w_gu and w_dn must start 16-byte aligned (the kernel loads 16-byte vectors)");
  const void* g = nullptr;
  if (gamma.has_value()) {
    TORCH_CHECK(gamma->scalar_type() == at::kBFloat16 && gamma->is_contiguous() && gamma->numel() == H);
    TORCH_CHECK(reinterpret_cast<uintptr_t>(gamma->data_ptr()) % 16 == 0, "moe_block_tkg: gamma must start 16-byte aligned");
    g = gamma->data_ptr();
  }
  const float* rb = nullptr;
  if (router_bias.has_value()) {
    TORCH_CHECK(router_bias->scalar_type() == at::kFloat && router_bias->is_contiguous() && router_bias->numel() == E);
    rb = router_bias->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(x.device());
  auto f32 = x.options().dtype(at::kFloat);
  Tensor out = at::empty({T, H}, x.options());
  Tensor logits = at::empty({T, E}, f32);
  Tensor idx = at::empty({T, K}, x.options().dtype(at::kLong));
  Tensor w = at::empty({T, K}, f32);
  Tensor gu = at::empty({(long)T * K, 2L * I}, f32);
  Tensor yacc = at::empty({T, H}, f32);
  Tensor bar = at::empty({1}, x.options().dtype(at::kInt));
  nxd::moe_block_tkg(x.data_ptr(), g, router_w.data_ptr(), rb, w_gu.data_ptr(), w_dn.data_ptr(), logits.data_ptr<float>(),
                     gu.data_ptr<float>(), yacc.data_ptr<float>(), out.data_ptr(), idx.data_ptr<long>(), w.data_ptr<float>(),
                     (unsigned*)bar.data_ptr<int>(), T, H, E, El, (int)e0, I, K, (float)eps, (int)router_act, act_over_topk, normalize,
                     pre_scale, round_logits, (int)act, (float)act_alpha, (float)act_beta, (float)gate_lo, (float)gate_hi, (float)up_lo,
                     (float)up_hi, cooperative, stream());
  return {out, logits, idx, w};
}
// x [M<=8, K] bf16; w = MX byte stream of [N, K] (fp4: K/2 bytes per row, fp8: K), any integer dtype view; scale [N, K/32] uint8
static Tensor gemv_mx(const Tensor& x, const Tensor& w, const Tensor& scale, int64_t fmt, const c10::optional<Tensor>& residual) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous() && x.size(0) >= 1 && x.size(0) <= 8);
  TORCH_CHECK(w.is_cuda() && w.is_contiguous() && scale.is_cuda() && scale.is_contiguous() && scale.scalar_type() == at::kByte &&
              scale.dim() == 2);
  const int M = x.size(0), K = x.size(1), N = scale.size(0);
  TORCH_CHECK(K % 32 == 0 && scale.size(1) == K / 32, "gemv_mx: scale must be [N, K/32]");
  const long row_bytes = fmt == 0 ? K / 2 : K;
  TORCH_CHECK((long)(w.numel() * w.element_size()) == (long)N * row_bytes, "gemv_mx: weight bytes do not match [N, K] in this format");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(w.data_ptr()) % 16 == 0,
              "gemv_mx: x and w must start 16-byte aligned (the kernel loads 16-byte vectors)");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({M, N}, x.options());
  const void* res = nullptr;
  if (residual.has_value()) {
    TORCH_CHECK(residual->is_contiguous() && residual->sizes() == y.sizes() && residual->scalar_type() == at::kBFloat16);
    res = residual->data_ptr();
  }
  nxd::gemv_mx(x.data_ptr(), w.data_ptr(), scale.data_ptr(), res, y.data_ptr(), M, N, K, (int)fmt, stream());
  return y;
}
// x [S, K] bf16 (one row per (token, slot)); w = MX byte stream of [E, N, K]; scale [E, N, K/32]; expert [S] int64 → [S, N] bf16
static Tensor gemv_mx_grouped(const Tensor& x, const Tensor& w, const Tensor& scale, const Tensor& expert, int64_t fmt) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous());
  TORCH_CHECK(w.is_cuda() && w.is_contiguous() && scale.is_cuda() && scale.is_contiguous() && scale.scalar_type() == at::kByte &&
              scale.dim() == 3);
  TORCH_CHECK(expert.is_cuda() && expert.scalar_type() == at::kLong && expert.is_contiguous() && expert.numel() == x.size(0));
  const int S = x.size(0), K = x.size(1), E = scale.size(0), N = scale.size(1);
  TORCH_CHECK(K % 32 == 0 && scale.size(2) == K / 32, "gemv_mx_grouped: scale must be [E, N, K/32]");
  const long row_bytes = fmt == 0 ? K / 2 : K;
  TORCH_CHECK((long)(w.numel() * w.element_size()) == (long)E * N * row_bytes, "gemv_mx_grouped: weight bytes do not match [E, N, K]");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(w.data_ptr()) % 16 == 0,
              "gemv_mx_grouped: x and w must start 16-byte aligned (the kernel loads 16-byte vectors)");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({S, N}, x.options());
  nxd::gemv_mx_grouped(x.data_ptr(), w.data_ptr(), scale.data_ptr(), expert.data_ptr<long>(), y.data_ptr(), S, N, K, E, (int)fmt, stream());
  return y;
}
// y = act(x · wᵀ + bias) + residual; act: 0 none, 1 exact GELU (erf), 2 tanh GELU
static Tensor gemv(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& residual, const c10::optional<Tensor>& bias,
                   int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && x.dim() == 2 && w.dim() == 2);
  TORCH_CHECK(x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1) && x.size(0) >= 1 && x.size(0) <= 8 && x.size(1) % 8 == 0);
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(w.data_ptr()) % 16 == 0,
              "gemv: x and w must start 16-byte aligned (the kernel loads 16-byte vectors)");
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), w.size(0)}, x.options());
  const void* res = nullptr;
  if (residual.has_value()) {
    TORCH_CHECK(residual->is_contiguous() && residual->sizes() == y.sizes() && residual->scalar_type() == at::kBFloat16);
    res = residual->data_ptr();
  }
  TORCH_CHECK(act >= 0 && act <= 2, "gemv: act must be 0 (none), 1 (exact GELU) or 2 (tanh GELU)");
  const void* bp = nullptr;
  if (bias.has_value()) {
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->dim() == 1 && bias->size(0) == w.size(0) &&
                bias->scalar_type() == at::kBFloat16, "gemv: bias must be a contiguous bf16 CUDA tensor [N]");
    bp = bias->data_ptr();
  }
  nxd::gemv_bf16(x.data_ptr(), w.data_ptr(), res, y.data_ptr(), x.size(0), w.size(0), x.size(1), stream(), bp, (int)act);
  return y;
}

// ---- grouped (MoE) GEMMs -------------------------------------------------------------------------
static Tensor grouped_gemm(const Tensor& a, const Tensor& w, const Tensor& block_expert, int64_t block_rows, bool trans_b) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && a.dim() == 2 && a.is_contiguous());
  TORCH_CHECK(w.scalar_type() == at::kBFloat16 && w.dim() == 3 && w.is_contiguous());
  TORCH_CHECK(block_expert.scalar_type() == at::kInt && block_expert.is_cuda());
  const int M = a.size(0), K = a.size(1), E = w.size(0);
  const int N = trans_b ? w.size(1) : w.size(2);
  TORCH_CHECK((trans_b ? w.size(2) : w.size(1)) == K && M % block_rows == 0 && K % 8 == 0 && N % 8 == 0);
  TORCH_CHECK(block_expert.numel() * block_rows == M);
  c10::cuda::CUDAGuard guard(a.device());
  Tensor out = at::empty({M, N}, a.options());
  nxd::grouped_gemm_bf16(a.data_ptr(), w.data_ptr(), out.data_ptr(), M, N, K, E, trans_b, block_expert.data_ptr<int>(),
                         (int)block_rows, nxd::kBF16, stream());
  return out;
}
// dW[e] = x[rows of e]ᵀ · dy[rows of e]  → out [E, Mo, No] (bf16 or fp32), optionally accumulated
static void grouped_wgrad(const Tensor& x, const Tensor& dy, Tensor out, const Tensor& seg_first_block, int64_t block_rows,
                          bool accumulate) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.is_contiguous() && dy.scalar_type() == at::kBFloat16 &&
              dy.is_contiguous() && out.is_contiguous() && out.dim() == 3);
  TORCH_CHECK(seg_first_block.scalar_type() == at::kInt && seg_first_block.numel() == out.size(0) + 1);
  TORCH_CHECK(x.size(0) == dy.size(0) && out.size(1) == x.size(1) && out.size(2) == dy.size(1));
  TORCH_CHECK(x.size(1) % 8 == 0 && dy.size(1) % 8 == 0);
  c10::cuda::CUDAGuard guard(x.device());
  nxd::grouped_wgrad_bf16(x.data_ptr(), dy.data_ptr(), out.data_ptr(), x.size(0), x.size(1), dy.size(1), out.size(0),
                          seg_first_block.data_ptr<int>(), (int)block_rows, dt_code(out), accumulate, stream());
}

// ---- attention ----------------------------------------------------------------------------------
static void check_qkv(const Tensor& t, const char* name) {
  const int64_t d = t.dim() == 4 ? t.size(3) : 0;
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.dim() == 4 && (d == 64 || d == 80 || d == 96 || d == 128) &&
                  t.stride(3) == 1,
              name, ": expected a bf16 CUDA [B,S,H,D] view with D in {64, 80, 96, 128} and contiguous head_dim");
}
// optional key-padding mask [B, S_kv] (bool / uint8, key visible iff nonzero) → (data, batch stride), or null
static const void* check_kpm(const c10::optional<Tensor>& m, const Tensor& q, int64_t B, int64_t Skv, long* sb) {
  *sb = 0;
  if (!m.has_value()) return nullptr;
  TORCH_CHECK(m->scalar_type() == at::kBool || m->scalar_type() == at::kByte, "key_padding_mask: expected bool or uint8");
  TORCH_CHECK(m->dim() == 2 && m->size(0) == B && m->size(1) == Skv, "key_padding_mask: expected shape [B, S_kv] = [", B, ", ",
              Skv, "], got ", m->sizes());
  TORCH_CHECK(m->size(1) <= 1 || m->stride(1) == 1, "key_padding_mask: the key dimension must be contiguous");
  TORCH_CHECK(m->device() == q.device(), "key_padding_mask: expected it on ", q.device(), ", got ", m->device());
  *sb = m->stride(0);
  return m->data_ptr();
}
// attention dropout arguments: 0 ≤ dropout_p < 1; with dropout_p > 0 a one-element int32 / int64 seed on q's device →
// (data, seed is int64), else (null, false)
static const void* check_dropout(double dropout_p, const c10::optional<Tensor>& seed, const Tensor& q, bool* seed64) {
  TORCH_CHECK(dropout_p >= 0.0 && dropout_p < 1.0, "dropout_p must be in [0, 1), got ", dropout_p);
  *seed64 = false;
  if (dropout_p == 0.0) return nullptr;
  TORCH_CHECK(seed.has_value(), "dropout_p > 0 needs a seed");
  TORCH_CHECK(seed->numel() == 1 && (seed->scalar_type() == at::kInt || seed->scalar_type() == at::kLong),
              "seed: expected a one-element int32 or int64 tensor");
  TORCH_CHECK(seed->device() == q.device(), "seed: expected it on ", q.device(), ", got ", seed->device());
  *seed64 = seed->scalar_type() == at::kLong;
  return seed->data_ptr();
}
// returns (out [B,S,H,D] view — memory laid out [S,B,H,D] when sbhd_out —, lse [B,H,S] fp32)
static std::vector<Tensor> flash_attn_fwd(const Tensor& q, const Tensor& k, const Tensor& v, bool causal, double scale,
                                          bool sbhd_out, const c10::optional<Tensor>& key_padding_mask, int64_t window,
                                          int64_t q_offset, double dropout_p, const c10::optional<Tensor>& seed,
                                          int64_t head_offset) {
  check_qkv(q, "q"); check_qkv(k, "k"); check_qkv(v, "v");
  const int B = q.size(0), S = q.size(1), H = q.size(2), D = q.size(3), Skv = k.size(1), Hkv = k.size(2);
  TORCH_CHECK(k.size(0) == B && v.size(0) == B && v.size(1) == Skv && v.size(2) == Hkv && H % Hkv == 0);
  TORCH_CHECK(k.size(3) == D && v.size(3) == D, "q, k and v must have the same head_dim");
  long kpm_sb;
  const void* kpm = check_kpm(key_padding_mask, q, B, Skv, &kpm_sb);
  bool seed64;
  const void* seed_p = check_dropout(dropout_p, seed, q, &seed64);
  c10::cuda::CUDAGuard guard(q.device());
  Tensor out = sbhd_out ? at::empty({S, B, H, D}, q.options()).transpose(0, 1) : at::empty({B, S, H, D}, q.options());
  Tensor lse = at::empty({B, H, S}, q.options().dtype(at::kFloat));
  const long qs[3] = {q.stride(0), q.stride(1), q.stride(2)}, ks[3] = {k.stride(0), k.stride(1), k.stride(2)};
  const long vs[3] = {v.stride(0), v.stride(1), v.stride(2)}, os[3] = {out.stride(0), out.stride(1), out.stride(2)};
  nxd::flash_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr<float>(), B, S, Skv, H, Hkv, D,
                      qs, ks, vs, os, (float)scale, causal, kpm, kpm_sb, window, q_offset, dropout_p, seed_p, seed64,
                      head_offset, stream());
  return {out, lse};
}

static std::vector<Tensor> flash_attn_bwd(const Tensor& go, const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& o,
                                          const Tensor& lse, bool causal, double scale, bool sbhd_out,
                                          const c10::optional<Tensor>& dlse, const c10::optional<Tensor>& key_padding_mask,
                                          int64_t window, int64_t q_offset, double dropout_p,
                                          const c10::optional<Tensor>& seed, int64_t head_offset) {
  check_qkv(q, "q"); check_qkv(k, "k"); check_qkv(v, "v"); check_qkv(go, "grad_out"); check_qkv(o, "out");
  const int B = q.size(0), S = q.size(1), H = q.size(2), D = q.size(3), Skv = k.size(1), Hkv = k.size(2);
  TORCH_CHECK(k.size(3) == D && v.size(3) == D && go.size(3) == D && o.size(3) == D,
              "q, k, v, out and grad_out must have the same head_dim");
  TORCH_CHECK(lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == (int64_t)B * H * S);
  long kpm_sb;
  const void* kpm = check_kpm(key_padding_mask, q, B, Skv, &kpm_sb);
  bool seed64;
  const void* seed_p = check_dropout(dropout_p, seed, q, &seed64);
  c10::cuda::CUDAGuard guard(q.device());
  auto mk = [&](int s, int h) {
    return sbhd_out ? at::empty({s, B, h, D}, q.options()).transpose(0, 1) : at::empty({B, s, h, D}, q.options());
  };
  Tensor dq = mk(S, H), dk = mk(Skv, Hkv), dv = mk(Skv, Hkv);
  Tensor delta = at::empty({B, H, S}, q.options().dtype(at::kFloat));
  auto st3 = [](const Tensor& t, long* out) { out[0] = t.stride(0); out[1] = t.stride(1); out[2] = t.stride(2); };
  long gs[3], qs[3], ks[3], vs[3], os[3], dqs[3], dks[3], dvs[3];
  st3(go, gs); st3(q, qs); st3(k, ks); st3(v, vs); st3(o, os); st3(dq, dqs); st3(dk, dks); st3(dv, dvs);
  const float* dlse_p = nullptr;
  if (dlse.has_value()) {
    TORCH_CHECK(dlse->scalar_type() == at::kFloat && dlse->is_contiguous() && dlse->numel() == lse.numel());
    dlse_p = dlse->data_ptr<float>();
  }
  nxd::flash_attn_bwd(go.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), dlse_p,
                      dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), delta.data_ptr<float>(), B, S, Skv, H, Hkv, D, gs, qs, ks,
                      vs, os, dqs, dks, dvs, (float)scale, causal, kpm, kpm_sb, window, q_offset, dropout_p, seed_p, seed64,
                      head_offset, stream());
  return {dq, dk, dv};
}

// ---- GEMM ---------------------------------------------------------------------------------------
static void gemm_bf16(const Tensor& a, const Tensor& b, Tensor out, bool trans_a, bool trans_b, bool accumulate) {
  CHECK_IN(a); CHECK_IN(b); CHECK_IN(out);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16 && a.dim() == 2 && b.dim() == 2);
  const int M = (int)(trans_a ? a.size(1) : a.size(0)), K = (int)(trans_a ? a.size(0) : a.size(1));
  const int N = (int)(trans_b ? b.size(0) : b.size(1));
  TORCH_CHECK((trans_b ? b.size(1) : b.size(0)) == K && out.size(0) == M && out.size(1) == N, "gemm shape mismatch");
  c10::cuda::CUDAGuard g(a.device());
  nxd::GemmComm none;
  nxd::gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, trans_a, trans_b, dt_code(out), accumulate, none,
                 nullptr, stream());
}

// all-gather(A shards along rows) → GEMM.  `a_shard` [M/world, K]; gathered A lives in the symmetric payload at
// buf_offset (every rank), out = A_full @ op(B).
static void ag_gemm_bf16(const Tensor& a_shard, const Tensor& b, Tensor out, bool trans_b, int64_t local_buf_ptr,
                         const Tensor& peer_bufs, const Tensor& peer_flags, int64_t buf_offset, int64_t flag_offset,
                         int64_t epoch, int64_t rank, int64_t world, int64_t comm_sms) {
  CHECK_IN(a_shard); CHECK_IN(b); CHECK_IN(out);
  const int Ms = (int)a_shard.size(0), K = (int)a_shard.size(1), M = Ms * (int)world;
  const int N = (int)(trans_b ? b.size(0) : b.size(1));
  TORCH_CHECK(out.size(0) == M && out.size(1) == N);
  c10::cuda::CUDAGuard g(a_shard.device());
  nxd::GemmComm c;
  c.mode = 1; c.rank = (int)rank; c.world = (int)world;
  c.peer_bufs = peer_bufs.data_ptr<int64_t>(); c.peer_flags = peer_flags.data_ptr<int64_t>();
  c.buf_offset = buf_offset; c.flag_offset = (int)flag_offset; c.epoch = (uint32_t)epoch; c.comm_sms = (int)comm_sms;
  // A operand = this rank's gathered buffer
  const void* a_full = (const void*)(local_buf_ptr + buf_offset);
  nxd::gemm_bf16(a_full, b.data_ptr(), out.data_ptr(), M, N, K, false, trans_b, dt_code(out), false, c,
                 a_shard.data_ptr(), stream());
}

// GEMM → reduce-scatter over rows.  a [M, K]; out [M/world, N] bf16 (sum over ranks of rows owned by this rank).
static void gemm_rs_bf16(const Tensor& a, const Tensor& b, Tensor out, bool trans_b, int64_t local_buf_ptr,
                         const Tensor& peer_bufs, const Tensor& peer_flags, int64_t buf_offset, int64_t flag_offset,
                         const std::vector<int64_t>& targets, int64_t rank, int64_t world) {
  CHECK_IN(a); CHECK_IN(b); CHECK_IN(out);
  const int M = (int)a.size(0), K = (int)a.size(1);
  const int N = (int)(trans_b ? b.size(0) : b.size(1));
  TORCH_CHECK(out.size(0) * world == M && out.size(1) == N && out.scalar_type() == at::kBFloat16);
  (void)local_buf_ptr;
  c10::cuda::CUDAGuard g(a.device());
  nxd::GemmComm c;
  c.mode = 2; c.rank = (int)rank; c.world = (int)world;
  c.peer_bufs = peer_bufs.data_ptr<int64_t>(); c.peer_flags = peer_flags.data_ptr<int64_t>();
  c.buf_offset = buf_offset; c.flag_offset = (int)flag_offset; c.epoch = 0;
  uint32_t tg[64] = {0};
  for (size_t i = 0; i < targets.size() && i < 64; ++i) tg[i] = (uint32_t)targets[i];
  c.rs_targets = tg;
  nxd::gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, false, trans_b, nxd::kBF16, false, c, nullptr,
                 stream());
}

// ---- ZeRO-1 collectives over peer memory
static void zero1_reduce_scatter(const Tensor& peer_bufs, int64_t grad_off_bytes, const Tensor& peer_flags, int64_t flag_off,
                                 int64_t epoch, int64_t rank, int64_t world, int64_t shard_numel, double scale, Tensor out,
                                 Tensor done_ctr, bool grads_fp32, int64_t sub_begin, int64_t sub_len, int64_t max_ctas) {
  TORCH_CHECK(sub_begin >= 0 && sub_len >= 0 && sub_begin + sub_len <= shard_numel && sub_begin % 8 == 0 && sub_len % 8 == 0);
  // 16-byte loads of every peer's shard and float4 stores into `out`: misaligned offsets or a short `out` would read or
  // write outside the buffers instead of failing
  TORCH_CHECK(shard_numel >= 0 && shard_numel % 8 == 0, "zero1_reduce_scatter: shard_numel must be a multiple of 8");
  TORCH_CHECK(grad_off_bytes >= 0 && grad_off_bytes % 16 == 0, "zero1_reduce_scatter: grad_off_bytes must be a multiple of 16");
  TORCH_CHECK(out.is_cuda() && out.is_contiguous() && out.scalar_type() == at::kFloat && out.numel() >= shard_numel,
              "zero1_reduce_scatter: out must be a contiguous fp32 CUDA tensor of at least shard_numel elements");
  TORCH_CHECK(world >= 1 && world <= 8 && rank >= 0 && rank < world && peer_bufs.numel() >= world && peer_flags.numel() >= world,
              "zero1_reduce_scatter: 1 <= world <= 8, 0 <= rank < world, one peer pointer per rank");
  c10::cuda::CUDAGuard g(out.device());
  nxd::zero1_reduce_scatter(peer_bufs.data_ptr<int64_t>(), grad_off_bytes, peer_flags.data_ptr<int64_t>(), (int)flag_off,
                            (uint32_t)epoch, (int)rank, (int)world, shard_numel, sub_begin, sub_len, (float)scale,
                            out.data_ptr<float>(), (uint32_t*)done_ctr.data_ptr(), grads_fp32 ? nxd::kF32 : nxd::kBF16,
                            (int)max_ctas, stream());
}
static void zero1_all_gather(const Tensor& master, const Tensor& peer_bufs, int64_t param_off_bytes, const Tensor& peer_flags,
                             int64_t flag_off, int64_t epoch, int64_t rank, int64_t world, int64_t shard_numel,
                             Tensor done_ctr, bool params_bf16) {
  // the kernel moves 8 master elements per thread with 16-byte stores: a shard_numel that is not a multiple of 8 would drop
  // its tail, a short master would be read past its end
  TORCH_CHECK(shard_numel >= 0 && shard_numel % 8 == 0, "zero1_all_gather: shard_numel must be a multiple of 8");
  TORCH_CHECK(master.is_cuda() && master.is_contiguous() && master.scalar_type() == at::kFloat && master.numel() >= shard_numel,
              "zero1_all_gather: master must be a contiguous fp32 CUDA tensor of at least shard_numel elements");
  TORCH_CHECK(param_off_bytes >= 0 && param_off_bytes % 16 == 0, "zero1_all_gather: param_off_bytes must be a multiple of 16");
  TORCH_CHECK(world >= 1 && world <= 8 && rank >= 0 && rank < world && peer_bufs.numel() >= world && peer_flags.numel() >= world,
              "zero1_all_gather: 1 <= world <= 8, 0 <= rank < world, one peer pointer per rank");
  c10::cuda::CUDAGuard g(master.device());
  nxd::zero1_all_gather(master.data_ptr<float>(), peer_bufs.data_ptr<int64_t>(), param_off_bytes,
                        peer_flags.data_ptr<int64_t>(), (int)flag_off, (uint32_t)epoch, (int)rank, (int)world, shard_numel,
                        (uint32_t*)done_ctr.data_ptr(), params_bf16 ? nxd::kBF16 : nxd::kF32, stream());
}

// ---- symmetric memory ---------------------------------------------------------------------------
static py::tuple symm_alloc(int64_t nbytes, int64_t nflags) {
  auto a = nxd::symm_alloc((size_t)nbytes, (size_t)nflags);
  return py::make_tuple(a.id, py::bytes(a.payload_handle), py::bytes(a.flags_handle));
}
static py::tuple symm_open(int64_t id, int64_t rank, const std::vector<py::bytes>& ph, const std::vector<py::bytes>& fh) {
  std::vector<std::string> p, f;
  for (auto& b : ph) p.push_back((std::string)b);
  for (auto& b : fh) f.push_back((std::string)b);
  auto r = nxd::symm_open(id, (int)rank, p, f);
  return py::make_tuple(r.payload, r.flags);
}
static Tensor symm_view(int64_t id, int64_t offset, const std::vector<int64_t>& shape, py::object dtype) {
  size_t nbytes = 0;
  auto* base = (uint8_t*)nxd::symm_local_payload(id, &nbytes);
  auto st = torch::python::detail::py_object_to_dtype(dtype);
  int dev; cudaGetDevice(&dev);
  auto opts = at::TensorOptions().dtype(st).device(at::kCUDA, dev);
  return at::from_blob(base + offset, shape, opts);
}

// ---- NVLS symmetric memory (symm_vmm.cpp) + stand-alone collectives on it (nvls_coll.cu) ----------
static py::tuple vmm_begin(int64_t nbytes, int64_t rank, int64_t world, bool want_multicast) {
  auto b = nxd::vmm_begin((size_t)nbytes, (int)rank, (int)world, want_multicast);
  return py::make_tuple(b.id, b.sock_name, b.multicast_supported, (int64_t)b.size);
}
static py::tuple vmm_ptrs(int64_t id, bool multicast_everywhere) {
  auto p = nxd::vmm_ptrs(id, multicast_everywhere);
  return py::make_tuple(p.peer, p.multicast, (int64_t)p.size);
}
static Tensor vmm_view(int64_t id, int64_t offset, const std::vector<int64_t>& shape, py::object dtype) {
  size_t nbytes = 0;
  auto* base = (uint8_t*)nxd::vmm_local(id, &nbytes);
  auto st = torch::python::detail::py_object_to_dtype(dtype);
  int64_t need = at::elementSize(st);
  for (auto d : shape) need *= d;
  TORCH_CHECK(offset >= 0 && (size_t)(offset + need) <= nbytes, "vmm_view out of range");
  int dev; cudaGetDevice(&dev);
  auto opts = at::TensorOptions().dtype(st).device(at::kCUDA, dev);
  return at::from_blob(base + offset, shape, opts);
}

// mode 1: a = shard [M/world, K] → out [M, N]; gathered A = region payload at buf_offset.
// mode 2: a = [M, K] → out [M/world, N]; partials live in the region payload at buf_offset.  Returns reducer claims used.
static int64_t tp_gemm_nvls(int64_t mode, const Tensor& a, const Tensor& b, Tensor out, bool trans_b, const Tensor& peer_bases,
                            int64_t mc_base, int64_t local_base, int64_t buf_offset, int64_t flag_offset, int64_t epoch,
                            int64_t rank, int64_t world, int64_t comm_ctas, Tensor counters, int64_t claim_base, bool wire_fp32,
                            bool gemm_join) {
  CHECK_IN(a); CHECK_IN(b); CHECK_IN(out);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16);
  TORCH_CHECK(counters.scalar_type() == at::kInt && counters.numel() >= 64 + 8 * 256);
  TORCH_CHECK(peer_bases.scalar_type() == at::kLong && peer_bases.is_cuda() && peer_bases.numel() >= world);
  c10::cuda::CUDAGuard g(a.device());
  const int K = (int)a.size(1);
  const int N = (int)(trans_b ? b.size(0) : b.size(1));
  auto* ctr = (uint32_t*)counters.data_ptr();           // [0] = reducer claim counter, [64..] = tile_done per 128-row block
  if (mode == 1) {
    const int M = (int)a.size(0) * (int)world;
    TORCH_CHECK(out.size(0) == M && out.size(1) == N);
    return nxd::gemm_bf16_nvls(1, nullptr, b.data_ptr(), out.data_ptr(), nullptr, a.data_ptr(), M, N, K, trans_b, (int)rank,
                               (int)world, peer_bases.data_ptr<int64_t>(), mc_base, local_base, buf_offset, flag_offset,
                               (uint32_t)epoch, (int)comm_ctas, ctr + 64, ctr, 0u, false, true, stream());
  }
  TORCH_CHECK(mode == 2, "tp_gemm_nvls: mode 1 or 2");
  const int M = (int)a.size(0);
  TORCH_CHECK(out.size(0) * world == M && out.size(1) == N);
  return nxd::gemm_bf16_nvls(2, a.data_ptr(), b.data_ptr(), nullptr, out.data_ptr(), nullptr, M, N, K, trans_b, (int)rank,
                             (int)world, peer_bases.data_ptr<int64_t>(), mc_base, local_base, buf_offset, flag_offset,
                             (uint32_t)epoch, (int)comm_ctas, ctr + 64, ctr, (uint32_t)claim_base, wire_fp32, gemm_join, stream());
}
static Tensor nvls_allreduce(const Tensor& x, const c10::optional<Tensor>& residual, const Tensor& peer_bases, int64_t mc_base,
                             int64_t local_base, int64_t flag_off, int64_t data_off, int64_t half_bytes, Tensor state,
                             int64_t rank, int64_t world) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && (x.scalar_type() == at::kBFloat16 || x.scalar_type() == at::kFloat));
  TORCH_CHECK(state.scalar_type() == at::kInt && state.numel() >= 2 + 1024);
  if (residual) TORCH_CHECK(residual->is_contiguous() && residual->scalar_type() == x.scalar_type() && residual->numel() == x.numel());
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty_like(x);
  const long nbytes = x.numel() * x.element_size();
  int ctas = (int)std::max<long>(1, std::min<long>(64, nbytes / 16384));
  nxd::nvls_allreduce(x.data_ptr(), residual ? residual->data_ptr() : nullptr, out.data_ptr(), peer_bases.data_ptr<int64_t>(),
                      mc_base, local_base, flag_off, data_off, half_bytes, (uint32_t*)state.data_ptr(), (int)rank, (int)world,
                      x.numel(), dt_code(x), ctas, stream());
  return out;
}
// y[M<=8, N] = sum over ranks of x[M, K] · w[N, K]ᵀ (+ residual): GEMV fused with the in-switch all-reduce
static Tensor gemv_allreduce(const Tensor& x, const Tensor& w, const c10::optional<Tensor>& residual, const Tensor& peer_bases,
                             int64_t mc_base, int64_t local_base, int64_t flag_off, int64_t data_off, int64_t half_bytes, Tensor state,
                             int64_t rank, int64_t world) {
  CHECK_IN(x); CHECK_IN(w);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1));
  TORCH_CHECK(state.scalar_type() == at::kInt && state.numel() >= 2 + 1024);
  const int M = (int)x.size(0), N = (int)w.size(0), K = (int)x.size(1);
  if (residual) TORCH_CHECK(residual->is_contiguous() && residual->scalar_type() == at::kBFloat16 && residual->numel() == (int64_t)M * N);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({M, N}, x.options());
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  nxd::gemv_allreduce(x.data_ptr(), w.data_ptr(), residual ? residual->data_ptr() : nullptr, y.data_ptr(), M, N, K,
                      peer_bases.data_ptr<int64_t>(), mc_base, local_base, flag_off, data_off, half_bytes, (uint32_t*)state.data_ptr(),
                      (int)rank, (int)world, sms * 4, stream());
  return y;
}
static void nvls_all_gather(const Tensor& x, const c10::optional<Tensor>& out, const Tensor& peer_bases, int64_t mc_base,
                            int64_t local_base, int64_t flag_off, int64_t data_off, int64_t half_bytes, Tensor state, int64_t rank,
                            int64_t world, int64_t ctas) {
  CHECK_IN(x);
  c10::cuda::CUDAGuard guard(x.device());
  const long bytes = x.numel() * x.element_size();
  if (out) TORCH_CHECK(out->is_contiguous() && (long)(out->numel() * out->element_size()) == bytes * world);
  nxd::nvls_all_gather(x.data_ptr(), out ? out->data_ptr() : nullptr, peer_bases.data_ptr<int64_t>(), mc_base, local_base, flag_off,
                       data_off, half_bytes, (uint32_t*)state.data_ptr(), (int)rank, (int)world, bytes, (int)ctas, stream());
}
static void nvls_publish(const Tensor& x, const Tensor& peer_bases, int64_t mc_base, int64_t local_base, int64_t flag_off,
                         int64_t data_off, int64_t half_bytes, Tensor state, int64_t rank, int64_t world, int64_t parity, int64_t ctas) {
  CHECK_IN(x);
  c10::cuda::CUDAGuard guard(x.device());
  nxd::nvls_publish(x.data_ptr(), peer_bases.data_ptr<int64_t>(), mc_base, local_base, flag_off, data_off, half_bytes,
                    (uint32_t*)state.data_ptr(), (int)rank, (int)world, x.numel() * x.element_size(), (int)parity, (int)ctas, stream());
}
// A tensor over memory this process has mapped (a peer's symmetric slot): the caller guarantees the mapping outlives the view.
static Tensor ptr_view(int64_t ptr, const std::vector<int64_t>& shape, py::object dtype) {
  auto st = torch::python::detail::py_object_to_dtype(dtype);
  int dev; cudaGetDevice(&dev);
  return at::from_blob(reinterpret_cast<void*>(ptr), shape, at::TensorOptions().dtype(st).device(at::kCUDA, dev));
}
// x = [world, chunk…] contiguous: chunk p goes to rank p; returns [world, chunk…] with chunk p received from rank p
static Tensor nvls_all_to_all(const Tensor& x, const Tensor& peer_bases, int64_t mc_base, int64_t local_base, int64_t flag_off,
                              int64_t data_off, int64_t half_bytes, Tensor state, int64_t rank, int64_t world, int64_t ctas) {
  CHECK_IN(x);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty_like(x);
  nxd::nvls_all_to_all(x.data_ptr(), out.data_ptr(), peer_bases.data_ptr<int64_t>(), mc_base, local_base, flag_off, data_off,
                       half_bytes, (uint32_t*)state.data_ptr(), (int)rank, (int)world, x.numel() * x.element_size(), (int)ctas, stream());
  return out;
}
// table [rows_per_rank, H] (this rank's vocab shard), ids [ntok] int64 GLOBAL vocabulary ids of this rank's tokens → [ntok, H]
static Tensor nvls_embedding_gather(const Tensor& table, const Tensor& ids, const Tensor& peer_bases, int64_t mc_base,
                                    int64_t local_base, int64_t flag_off, int64_t data_off, int64_t half_bytes, Tensor state,
                                    int64_t rank, int64_t world, int64_t ctas) {
  CHECK_IN(table);
  TORCH_CHECK(table.dim() == 2 && ids.is_cuda() && ids.scalar_type() == at::kLong && ids.is_contiguous());
  c10::cuda::CUDAGuard guard(table.device());
  const long row_bytes = table.size(1) * table.element_size();
  Tensor out = at::empty({ids.numel(), table.size(1)}, table.options());
  nxd::nvls_embedding_gather(table.data_ptr(), ids.data_ptr<long>(), out.data_ptr(), peer_bases.data_ptr<int64_t>(), mc_base,
                             local_base, flag_off, data_off, half_bytes, (uint32_t*)state.data_ptr(), (int)rank, (int)world,
                             table.size(0), row_bytes, ids.numel(), (int)ctas, stream());
  return out;
}
static Tensor nvls_reduce_scatter(const Tensor& x, const Tensor& peer_bases, int64_t mc_base, int64_t local_base, int64_t flag_off,
                                  int64_t data_off, int64_t half_bytes, Tensor state, int64_t rank, int64_t world, int64_t ctas) {
  CHECK_IN(x);
  TORCH_CHECK(x.numel() % world == 0);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor out = at::empty({x.numel() / world}, x.options());
  nxd::nvls_reduce_scatter(x.data_ptr(), out.data_ptr(), peer_bases.data_ptr<int64_t>(), mc_base, local_base, flag_off, data_off,
                           half_bytes, (uint32_t*)state.data_ptr(), (int)rank, (int)world, x.numel() / world, dt_code(x), (int)ctas,
                           stream());
  return out;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("rmsnorm_fwd", &rmsnorm_fwd);
  m.def("rmsnorm_bwd", &rmsnorm_bwd);
  m.def("add_rmsnorm_fwd", &add_rmsnorm_fwd);
  m.def("add_rmsnorm_bwd", &add_rmsnorm_bwd);
  m.def("swiglu_fwd", &swiglu_fwd);
  m.def("swiglu_bwd", &swiglu_bwd);
  m.def("rope_apply", &rope_apply);
  m.def("ce_stats", &ce_stats);
  m.def("ce_backward", &ce_backward);
  m.def("multi_tensor_sq_norm", &multi_tensor_sq_norm);
  m.def("multi_tensor_scale", &multi_tensor_scale);
  m.def("fused_adamw", &fused_adamw);
  m.def("gemm_bf16", &gemm_bf16);
  m.def("oneshot_allreduce", &oneshot_allreduce);
  m.def("decode_attention", &decode_attention, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("positions"), py::arg("scale"),
        py::arg("window") = 0, py::kw_only(), py::arg("k_scale") = 1.0, py::arg("v_scale") = 1.0, py::arg("rolling") = false);
  m.def("decode_attention_partial", &decode_attention_partial, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("positions"),
        py::arg("scale"), py::arg("window") = 0, py::kw_only(), py::arg("k_scale") = 1.0, py::arg("v_scale") = 1.0);
  m.def("nvls_embedding_gather", &nvls_embedding_gather);
  m.def("nvls_publish", &nvls_publish);
  m.def("ptr_view", &ptr_view);
  m.def("nvls_all_to_all", &nvls_all_to_all);
  m.def("gemv_mx", &gemv_mx);
  m.def("gemv_mx_grouped", &gemv_mx_grouped);
  m.def("moe_block_tkg", &moe_block_tkg);
  m.def("moe_block_tkg_supported", [](int64_t T, int64_t H, int64_t E, int64_t I, int64_t K) {
    return nxd::moe_block_tkg_supported((int)T, (int)H, (int)E, (int)I, (int)K);
  });
  m.def("decode_rope_kv", &decode_rope_kv, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("positions"), py::arg("cos"),
        py::arg("sin"), py::arg("k_cache"), py::arg("v_cache"), py::kw_only(), py::arg("k_scale") = 1.0, py::arg("v_scale") = 1.0,
        py::arg("depth") = py::none(), py::arg("rolling") = false);
  m.def("speculation_attention", &speculation_attention, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("positions"),
        py::arg("tree_mask") = py::none(), py::arg("tree_depth") = py::none(), py::kw_only(), py::arg("scale"),
        py::arg("window") = 0, py::arg("k_scale") = 1.0, py::arg("v_scale") = 1.0, py::arg("rolling") = false);
  m.def("moe_block_metadata", &moe_block_metadata);
  m.def("row_argmax", &row_argmax);
  m.def("row_topk", &row_topk);
  m.def("row_topk_supported", &row_topk_supported);
  m.def("gemv", &gemv, py::arg("x"), py::arg("w"), py::arg("residual") = py::none(), py::kw_only(), py::arg("bias") = py::none(),
        py::arg("act") = 0);
  m.def("gemm_fp8", &gemm_fp8, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("scale_a"), py::arg("scale_b"),
        py::arg("accumulate") = false);
  m.def("gemm_fp8_block", &gemm_fp8_block);
  m.def("grouped_gemm_fp8_block", &grouped_gemm_fp8_block);
  m.def("quantize_fp8_groups", &quantize_fp8_groups);
  m.def("quantize_fp8_rows", &quantize_fp8_rows);
  m.def("quantize_fp8_cols_t", &quantize_fp8_cols_t);
  m.def("grouped_gemm", &grouped_gemm);
  m.def("grouped_wgrad", &grouped_wgrad);
  m.def("flash_attn_fwd", &flash_attn_fwd, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("causal"), py::arg("scale"),
        py::arg("sbhd_out"), py::arg("key_padding_mask") = py::none(), py::arg("window") = 0, py::arg("q_offset") = 0,
        py::arg("dropout_p") = 0.0, py::arg("seed") = py::none(), py::arg("head_offset") = 0);
  m.def("flash_attn_bwd", &flash_attn_bwd, py::arg("go"), py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"), py::arg("lse"),
        py::arg("causal"), py::arg("scale"), py::arg("sbhd_out"), py::arg("dlse") = py::none(),
        py::arg("key_padding_mask") = py::none(), py::arg("window") = 0, py::arg("q_offset") = 0, py::arg("dropout_p") = 0.0,
        py::arg("seed") = py::none(), py::arg("head_offset") = 0);
  m.def("ag_gemm_bf16", &ag_gemm_bf16);
  m.def("gemm_rs_bf16", &gemm_rs_bf16);
  m.def("zero1_reduce_scatter", &zero1_reduce_scatter);
  m.def("zero1_all_gather", &zero1_all_gather);
  m.def("symm_alloc", &symm_alloc);
  m.def("symm_open", &symm_open);
  m.def("symm_free", &nxd::symm_free);
  m.def("symm_view", &symm_view);
  m.def("vmm_begin", &vmm_begin);
  m.def("vmm_send", &nxd::vmm_send);
  m.def("vmm_recv", &nxd::vmm_recv);
  m.def("vmm_bind", &nxd::vmm_bind);
  m.def("vmm_ptrs", &vmm_ptrs);
  m.def("vmm_free", &nxd::vmm_free);
  m.def("vmm_view", &vmm_view);
  m.def("nvls_allreduce", &nvls_allreduce, py::arg("x"), py::arg("residual"), py::arg("peer_bases"), py::arg("mc_base"),
        py::arg("local_base"), py::arg("flag_off"), py::arg("data_off"), py::arg("half_bytes"), py::arg("state"), py::arg("rank"),
        py::arg("world"));
  m.def("gemv_allreduce", &gemv_allreduce, py::arg("x"), py::arg("w"), py::arg("residual"), py::arg("peer_bases"), py::arg("mc_base"),
        py::arg("local_base"), py::arg("flag_off"), py::arg("data_off"), py::arg("half_bytes"), py::arg("state"), py::arg("rank"),
        py::arg("world"));
  m.def("nvls_all_gather", &nvls_all_gather);
  m.def("tp_gemm_nvls", &tp_gemm_nvls);
  m.def("nvls_reduce_scatter", &nvls_reduce_scatter);
}
