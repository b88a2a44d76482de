"""FP8 (e4m3) linear layers on the Hopper FP8 tensor cores.

* :func:`scaled_linear` — per-token × per-channel scales: ``y = (xq @ wqᵀ) · xs[:, None] · ws[None, :]``.  CUDA: the fp8
  instantiation of the wgmma GEMM (``csrc/gemm_sm90.cu``: ``wgmma m64n256k32.e4m3``, e4m3 operands staged by TMA as 128-byte
  swizzle rows of 128 elements, fp32 accumulation in registers, scales applied in the epilogue).
* :func:`blockscaled_linear` — one scale per group of G ∈ {32, 64, 128} consecutive input features on both operands (block-wise
  FP8 checkpoints, MXFP8): ``y = Σ_g (xq[:, g] @ wq[:, g]ᵀ) · xs[:, g] ⊗ ws[:, g]``.  CUDA: ``csrc/gemm_fp8_block_sm90.cu``,
  one ``wgmma m64n128k32.e4m3`` chain per group into a temporary accumulator that is promoted into the fp32 main accumulator
  with the group's scales, in registers.  Weight scales may be per (row, group) ``[N, K/G]`` or per 2-D block ``[N/bn, K/G]``,
  fp32 or E8M0.
* :func:`grouped_blockscaled_linear` — the same product for MoE experts on the dropless block layout: rows come in
  ``block_size``-row blocks and block i uses the weights of expert ``block_to_expert[i]``.  CUDA: the grouped mode of the same
  kernel, where the block's expert only shifts the TMA rows of the weight tile and of its scales.
* :func:`quantize_groups` — the matching per-token activation quantiser (``absmax`` or OCP ``mx`` scale rule); CUDA: one
  bandwidth-bound kernel that writes the codes and the scales in the layout the GEMM reads.
* :func:`fp8_forward`, :func:`fp8_dgrad`, :func:`fp8_wgrad` — the three products of a row-wise scaled FP8 training linear on
  :func:`scaled_linear`'s kernel, fed by :func:`quantize_rows` / :func:`quantize_cols_t` (``csrc/fp8_quant.cu``).

CPU, and shapes or dtypes the kernels do not take: the fp32 oracle of the same quantised operands.  Reference:
quantization/quantization_layers.py (scaled matmul of the quantised parallel layers)."""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch

from . import _ext

_E4M3_MAX = 448.0
GROUP_SIZES = (32, 64, 128)


def scaled_linear(xq: torch.Tensor, xs: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor,
                  out_dtype: torch.dtype = torch.bfloat16, out: Optional[torch.Tensor] = None,
                  accumulate: bool = False) -> torch.Tensor:
    """``(xq @ wqᵀ) · xs[:, None] · ws[None, :]`` for e4m3 ``xq [..., K]`` and ``wq [N, K]``.  ``out``: an fp32 ``[M, N]``
    tensor to write, or with ``accumulate`` to add into (per element ``old + product`` in fp32, one rounding)."""
    shape = xq.shape
    x2 = xq.reshape(-1, shape[-1])
    s2 = xs.reshape(-1, 1).float()
    if out is not None:
        assert out.dtype == torch.float32 and out.shape == (x2.shape[0], wq.shape[0]), "out must be fp32 [M, N]"
        out_dtype = torch.float32
    assert not accumulate or out is not None, "accumulate needs out"
    e = _ext.ext() if x2.is_cuda else None
    if (e is not None and hasattr(e, "gemm_fp8") and x2.shape[1] % 16 == 0 and wq.shape[0] % 8 == 0
            and xq.dtype == torch.float8_e4m3fn and wq.dtype == torch.float8_e4m3fn
            and (out_dtype == torch.bfloat16 or (out is not None and out.is_contiguous() and out.data_ptr() % 8 == 0))):
        if out is None:
            out = torch.empty(x2.shape[0], wq.shape[0], dtype=out_dtype, device=x2.device)
        _ext.count_launch()
        e.gemm_fp8(x2.contiguous(), wq.contiguous(), out, s2.expand(x2.shape[0], 1).contiguous().view(-1),
                   ws.float().reshape(-1).expand(wq.shape[0]).contiguous(), accumulate)
        return out.view(*shape[:-1], wq.shape[0])
    y = (x2.float() @ wq.float().t()) * s2 * ws.float().reshape(1, -1)
    if out is not None:
        return out.add_(y) if accumulate else out.copy_(y)
    return y.to(out_dtype).view(*shape[:-1], wq.shape[0])


# ---- row-wise scaled FP8 training ------------------------------------------------------------------------------------
# A linear y = x·Wᵀ (x [M, K], W [N, K], g = dL/dy [M, N]) runs three e4m3 GEMMs on operands quantised by one rule,
# rows(t) = one absmax scale per row of t (the group rule with G = the row length) and cols_t(t) = rows(tᵀ):
#
#   forward         rows(x)  [M, K] · rows(W)   [N, K]ᵀ → bf16 y  [M, N]
#   input gradient  rows(g)  [M, N] · cols_t(W) [K, N]ᵀ → bf16 dx [M, K]
#   weight gradient cols_t(g)[N, M] · cols_t(x) [K, M]ᵀ → fp32 dW [N, K]   (or added into an fp32 main_grad)
#
# e4m3 wgmma reads K-major operands only, hence the transposed copies of W, g and x.  CUDA (bf16 operands, M, N, K multiples
# of 16, 16-byte aligned starts): csrc/fp8_quant.cu and the fp8 GEMM of csrc/gemm_sm90.cu.  Otherwise, and with
# NXD_DISABLE_TCGEN05_GEMM=1, the torch oracle quantiser and the fp32 matmul of the dequantised operands.
def _rows_reference(t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    q, s = _quantize_groups_reference(t, t.shape[1], "absmax", None)
    return q, s.reshape(-1)


def quantize_rows(t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``t [R, C]`` → (e4m3 ``[R, C]``, fp32 ``[R]``): ``s_r = max(amax_r / 448, 1e-12)``, codes ``RNE(clamp(t / s, ±448))``; a
    row holding a NaN or ±inf gets a NaN scale and NaN codes.  CUDA kernel for bf16 with ``C % 8 == 0`` and a 16-byte aligned
    start, bit for bit the oracle on the same device (NaN sign excepted); otherwise the oracle."""
    t = t.contiguous()
    if (t.dtype == torch.bfloat16 and t.shape[1] % 8 == 0 and t.numel() > 0 and _ext.use_cuda(t)
            and hasattr(_ext.ext(), "quantize_fp8_rows") and t.data_ptr() % 16 == 0):
        _ext.count_launch()
        q, s = _ext.ext().quantize_fp8_rows(t)
        return q, s
    return _rows_reference(t)


def quantize_cols_t(t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``t [R, C]`` → (e4m3 ``[C, R]``, fp32 ``[C]``) = :func:`quantize_rows` of ``tᵀ``: one scale per column of ``t``, the codes
    transposed so that a GEMM contracting over R reads them K-major.  CUDA kernels for bf16 with ``R % 16 == 0`` (the rows are
    a TMA operand), ``C % 8 == 0`` and a 16-byte aligned start; otherwise the oracle."""
    t = t.contiguous()
    if (t.dtype == torch.bfloat16 and t.shape[0] % 16 == 0 and t.shape[1] % 8 == 0 and t.numel() > 0 and _ext.use_cuda(t)
            and hasattr(_ext.ext(), "quantize_fp8_cols_t") and t.data_ptr() % 16 == 0):
        _ext.count_launch(2)                        # column absmax, then quantise-and-transpose
        q, s = _ext.ext().quantize_fp8_cols_t(t)
        return q, s
    return _rows_reference(t.t())


def _fp8_product(a: torch.Tensor, a_cols_t: bool, b: torch.Tensor, b_cols_t: bool, M: int, N: int, K: int,
                 out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """``Q(a) · Q(b)ᵀ`` with Q = cols_t or rows per operand, for a linear of ``M`` tokens, ``N`` outputs and ``K`` inputs."""
    a, b = a.contiguous(), b.contiguous()
    if (os.environ.get("NXD_DISABLE_TCGEN05_GEMM", "0") != "1" and M > 0 and M % 16 == 0 and N % 16 == 0 and K % 16 == 0
            and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0
            and _ext.use_cuda(a, b) and hasattr(_ext.ext(), "quantize_fp8_cols_t")):
        aq, sa = quantize_cols_t(a) if a_cols_t else quantize_rows(a)
        bq, sb = quantize_cols_t(b) if b_cols_t else quantize_rows(b)
        return scaled_linear(aq, sa, bq, sb, out=out, accumulate=accumulate)
    aq, sa = _rows_reference(a.t() if a_cols_t else a)
    bq, sb = _rows_reference(b.t() if b_cols_t else b)
    y = (aq.float() * sa.reshape(-1, 1)) @ (bq.float() * sb.reshape(-1, 1)).t()
    if out is not None:
        return out.add_(y) if accumulate else out.copy_(y)
    return y.bfloat16()


def fp8_forward(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """bf16 ``y [M, N] = rows(x) · rows(W)ᵀ`` for ``x [M, K]``, ``W [N, K]``."""
    return _fp8_product(x, False, w, False, x.shape[0], w.shape[0], w.shape[1])


def fp8_dgrad(g: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """bf16 ``dx [M, K] = rows(g) · cols_t(W)ᵀ`` for ``g [M, N]``, ``W [N, K]``."""
    return _fp8_product(g, False, w, True, g.shape[0], w.shape[0], w.shape[1])


def fp8_wgrad(g: torch.Tensor, x: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """fp32 ``dW [N, K] = cols_t(g) · cols_t(x)ᵀ`` for ``g [M, N]``, ``x [M, K]``, written into ``out`` or, with
    ``accumulate``, added to it (fp32 ``old + product``, one rounding: the TMA reduce-add on CUDA)."""
    if out is None:
        out = torch.empty(g.shape[1], x.shape[1], dtype=torch.float32, device=g.device)
        accumulate = False
    return _fp8_product(g, True, x, True, g.shape[0], g.shape[1], x.shape[1], out, accumulate)


# ---- block-scaled ----------------------------------------------------------------------------------------------------
def _quantize_groups_reference(x2: torch.Tensor, group_size: int, rule: str, clamp_bound: Optional[float]
                               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Torch oracle of the group quantiser: ``[M, K]`` → (e4m3 ``[M, K]``, fp32 ``[M, K/G]``).  A group whose amax is not
    finite (a NaN, or ±inf with no clamp) gets a NaN scale, so all its codes are NaN."""
    M, K = x2.shape
    xf = x2.float()
    if clamp_bound is not None:
        xf = xf.clamp(-clamp_bound, clamp_bound)
    xb = xf.reshape(M, K // group_size, group_size)
    amax = xb.abs().amax(-1)
    if rule == "mx":
        scale = torch.pow(2.0, torch.floor(torch.log2(amax.clamp(min=2.0 ** -100))) - 8)
    else:
        scale = (amax / _E4M3_MAX).clamp(min=1e-12)
    scale = torch.where(torch.isfinite(amax), scale, float("nan"))
    q = (xb / scale.unsqueeze(-1)).clamp(-_E4M3_MAX, _E4M3_MAX).to(torch.float8_e4m3fn).reshape(M, K)
    return q, scale


def quantize_groups(x: torch.Tensor, group_size: int, rule: str = "absmax", clamp_bound: Optional[float] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-token group quantisation to e4m3: ``x [..., K]`` → (codes ``[..., K]``, fp32 scales ``[..., K/G]``), ``x ≈ codes · scale``
    per group of ``group_size`` consecutive elements.

    ``rule="absmax"``: ``scale = max(amax / 448, 1e-12)`` (per-row ``quantize_activation_dynamic`` when G = K);
    ``rule="mx"``: OCP MX ``scale = 2^(⌊log2 amax⌋ − 8)`` (``mx_torch.quantize_mx``).  Codes are ``clamp(x / scale, ±448)`` rounded
    to nearest-even; ``clamp_bound`` clips ``x`` first.  A group holding a NaN, or ±inf when there is no clamp, gets a NaN
    scale and NaN codes, so every output that reads it is NaN rather than a finite-looking number.  On CUDA (bf16 input,
    16-byte aligned rows) the scales are a transposed view of the group-major buffer :func:`blockscaled_linear` streams.
    Codes and scales equal the torch oracle on the same CUDA tensor bit for bit, except that the sign of a NaN code is not
    defined.  torch computes ``amax / 448`` as a product with the rounded reciprocal on CUDA and as a true division on CPU,
    so an absmax scale can differ in the last bit between devices."""
    assert rule in ("absmax", "mx"), rule
    K = x.shape[-1]
    assert K % group_size == 0, f"K={K} is not a multiple of the group size {group_size}"
    lead = x.shape[:-1]
    x2 = x.reshape(-1, K)
    if (group_size in GROUP_SIZES and x2.dtype == torch.bfloat16 and K % 8 == 0 and _ext.use_cuda(x2)
            and hasattr(_ext.ext(), "quantize_fp8_groups") and x2.contiguous().data_ptr() % 16 == 0):
        _ext.count_launch()                         # the kernel loads 16-byte vectors: an unaligned view takes the oracle
        q, sbuf = _ext.ext().quantize_fp8_groups(x2.contiguous(), group_size, rule == "mx",
                                                 float("inf") if clamp_bound is None else float(clamp_bound))
        xs = sbuf[:, : x2.shape[0]].t()
    else:
        q, xs = _quantize_groups_reference(x2, group_size, rule, clamp_bound)
    return q.view(*lead, K), xs.reshape(*lead, K // group_size)


def weight_scales_kn(ws: torch.Tensor, n: int, k: int, group_size: int) -> torch.Tensor:
    """Weight scales ``[N, K/G]`` or ``[N/bn, K/G]`` (2-D blocks), fp32 or E8M0 ``uint8`` → the fp32 ``[K/G, N]`` layout of the
    block-scaled GEMM.  Depends on the weight only, so compiled inference hoists it out of the per-call plan."""
    s = torch.pow(2.0, ws.float() - 127.0) if ws.dtype == torch.uint8 else ws.float()
    s = s.reshape(-1, k // group_size)
    if s.shape[0] != n:
        assert n % s.shape[0] == 0, f"{s.shape[0]} scale rows do not tile {n} weight rows"
        s = s.repeat_interleave(n // s.shape[0], dim=0)
    return s.t().contiguous()


def _dequant_groups(q: torch.Tensor, s: torch.Tensor, group_size: int) -> torch.Tensor:
    R, K = q.shape
    return (q.float().reshape(R, K // group_size, group_size) * s.float().unsqueeze(-1)).reshape(R, K)


def blockscaled_linear(xq: torch.Tensor, xs: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor, group_size: int,
                       out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``dequant(xq, xs) @ dequant(wq, ws)ᵀ`` for e4m3 codes with one scale per ``group_size`` input features.

    ``xq [..., K]`` / ``xs [..., K/G]`` as :func:`quantize_groups` returns them; ``wq [N, K]``; ``ws`` fp32 or E8M0 ``[N, K/G]`` or
    ``[N/bn, K/G]``.  CUDA with e4m3 operands starting 16-byte aligned, G ∈ {32, 64, 128}, ``K % 128 == 0``, ``N % 8 == 0``
    and bf16 output: the block-scaled wgmma GEMM; otherwise the fp32 oracle."""
    K = xq.shape[-1]
    lead = xq.shape[:-1]
    x2 = xq.reshape(-1, K)
    M, N = x2.shape[0], wq.shape[0]
    xs2 = xs.reshape(M, K // group_size)
    sb = weight_scales_kn(ws, N, K, group_size)
    if (group_size in GROUP_SIZES and K % 128 == 0 and N % 8 == 0 and out_dtype == torch.bfloat16
            and xq.dtype == torch.float8_e4m3fn and wq.dtype == torch.float8_e4m3fn and _ext.use_cuda(x2, wq, xs2, sb)
            and hasattr(_ext.ext(), "gemm_fp8_block")
            and x2.contiguous().data_ptr() % 16 == 0 and wq.contiguous().data_ptr() % 16 == 0):   # TMA needs 16-byte starts
        sa = xs2.t()                                # [K/G, M]: a view of the quantiser's group-major buffer needs no copy
        if not (sa.dtype == torch.float32 and sa.stride(1) == 1 and sa.stride(0) >= M and sa.stride(0) % 4 == 0
                and sa.data_ptr() % 16 == 0):
            buf = torch.zeros(K // group_size, (M + 3) // 4 * 4, dtype=torch.float32, device=x2.device)
            buf[:, :M] = xs2.t()
            sa = buf[:, :M]
        _ext.count_launch()
        y = _ext.ext().gemm_fp8_block(x2.contiguous(), wq.contiguous(), sa, sb, group_size)
        return y.view(*lead, N)
    y = _dequant_groups(x2, xs2, group_size) @ _dequant_groups(wq.reshape(N, K), sb.t(), group_size).t()
    return y.to(out_dtype).view(*lead, N)


def expert_weight_scales_kn(ws: torch.Tensor, n: int, k: int, group_size: int) -> torch.Tensor:
    """Expert weight scales ``[E, K/G, N]`` (block axis 1) or ``[E, K/G, N/bn]`` (2-D blocks), fp32 or E8M0 ``uint8`` → the fp32
    ``[E, K/G, N]`` layout of :func:`grouped_blockscaled_linear`'s kernel, as :func:`weight_scales_kn` does per expert.  A
    contiguous fp32 ``[E, K/G, N]`` is returned as it is."""
    s = torch.pow(2.0, ws.float() - 127.0) if ws.dtype == torch.uint8 else ws.float()
    assert s.dim() == 3 and s.shape[1] == k // group_size, f"expert scales {tuple(ws.shape)} do not have K/G = {k // group_size} rows"
    if s.shape[2] != n:
        assert n % s.shape[2] == 0, f"{s.shape[2]} scale columns do not tile {n} weight columns"
        s = s.repeat_interleave(n // s.shape[2], dim=2)
    return s.contiguous()


def grouped_blockscaled_linear(xq: torch.Tensor, xs: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor,
                               block_to_expert: torch.Tensor, block_size: int, group_size: int,
                               out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``y[i·B:(i+1)·B] = dequant(xq, xs)[i·B:(i+1)·B] @ dequant(wq[e], ws[e])`` with ``e = block_to_expert[i]``.  Inference only.

    ``xq [nb·B, K]`` / ``xs [nb·B, K/G]`` as :func:`quantize_groups` returns them; ``wq`` e4m3 ``[E, K, N]`` (in, out);
    ``ws`` fp32 or E8M0 ``[E, K/G, N]`` or ``[E, K/G, N/bn]``.  CUDA with ``wq`` stored K-major (strides ``(N·K, 1, K)``, as
    ``wq.transpose(1, 2).contiguous().transpose(1, 2)`` leaves it), 16-byte aligned operands, G ∈ {32, 64, 128},
    ``K % 128 == 0``, ``N % 8 == 0``, ``B % 128 == 0`` and bf16 output: one launch of the grouped block-scaled kernel;
    otherwise the fp32 oracle of the same quantised operands."""
    K, M = xq.shape[-1], xq.shape[0]
    E, N = wq.shape[0], wq.shape[2]
    nb = block_to_expert.numel()
    assert xq.dim() == 2 and wq.dim() == 3 and wq.shape[1] == K and M == nb * block_size, \
        f"xq {tuple(xq.shape)}, wq {tuple(wq.shape)}, {nb} blocks of {block_size}"
    xs2 = xs.reshape(M, K // group_size)
    sb = expert_weight_scales_kn(ws, N, K, group_size)
    wt = wq.transpose(1, 2)                                   # [E, N, K]: a view of K-major storage, no copy
    if (group_size in GROUP_SIZES and K % 128 == 0 and N % 8 == 0 and block_size % 128 == 0 and out_dtype == torch.bfloat16
            and xq.dtype == torch.float8_e4m3fn and wq.dtype == torch.float8_e4m3fn and wt.is_contiguous()
            and _ext.use_cuda(xq, wq, xs2, sb, block_to_expert) and hasattr(_ext.ext(), "grouped_gemm_fp8_block")
            and xq.contiguous().data_ptr() % 16 == 0 and wt.data_ptr() % 16 == 0 and sb.data_ptr() % 16 == 0):
        sa = xs2.t()                                          # [K/G, M]: a view of the quantiser's group-major buffer
        if not (sa.dtype == torch.float32 and sa.stride(1) == 1 and sa.stride(0) >= M and sa.stride(0) % 4 == 0
                and sa.data_ptr() % 16 == 0):
            buf = torch.zeros(K // group_size, (M + 3) // 4 * 4, dtype=torch.float32, device=xq.device)
            buf[:, :M] = xs2.t()
            sa = buf[:, :M]
        b2e = block_to_expert if block_to_expert.dtype == torch.int32 else block_to_expert.int()
        _ext.count_launch()
        return _ext.ext().grouped_gemm_fp8_block(xq.contiguous(), wt, sa, sb, b2e, block_size, group_size)
    xd = _dequant_groups(xq, xs2, group_size).view(nb, block_size, K)
    wd = (wq.float().reshape(E, K // group_size, group_size, N) * sb.unsqueeze(2)).reshape(E, K, N)
    return torch.bmm(xd, wd[block_to_expert.long()]).reshape(M, N).to(out_dtype)
