"""Decode-time MoE block: RMSNorm → router → top-k → chosen local experts (gate|up, GLU, down) → weighted sum in ONE launch
(kernel: ``csrc/moe_tkg.cu`` — a persistent cooperative kernel with three grid barriers; role of the reference's
``moe_block_tkg`` NKI kernel, ``modules/moe/moe_fused_tkg.py:274-380``).

``moe_block_tkg`` dispatches to the kernel on CUDA / bf16 / T ≤ 8 and to :func:`moe_block_tkg_reference` (the same
semantics in fp32 torch math, used as the numerics oracle by the tests) otherwise."""
from __future__ import annotations

import math
import os
from typing import Optional, Tuple

import torch

from . import _ext

ACT_IDS = {"silu": 0, "swish": 0, "gelu": 1, "gelu_new": 2, "gelu_pytorch_tanh": 2, "gelu_tanh_approx": 2, "relu": 4}
_INF = float("inf")


def act_id(hidden_act: str, glu_type: str) -> Optional[int]:
    if glu_type == "swiglu":
        return 3
    return ACT_IDS.get(hidden_act)


def _glu(g, u, act, alpha, beta, clamps):
    g = g.clamp(min=clamps[0], max=clamps[1])
    u = u.clamp(min=clamps[2], max=clamps[3])
    if act == 0:
        return torch.nn.functional.silu(g) * u
    if act == 1:
        return torch.nn.functional.gelu(g) * u
    if act == 2:
        return torch.nn.functional.gelu(g, approximate="tanh") * u
    if act == 3:
        return g * torch.sigmoid(alpha * g) * (u + beta)
    return torch.relu(g) * u


def moe_block_tkg_reference(x, gamma, router_w, router_bias, w_gu, w_dn, e0: int, top_k: int, eps: float = 1e-6,
                            router_act: int = 0, act_over_topk: bool = False, normalize: bool = True, pre_scale: bool = False,
                            round_logits: bool = True, act: int = 0, act_alpha: float = 1.0, act_beta: float = 0.0,
                            clamps=(-_INF, _INF, -_INF, _INF)) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """fp32 math with the rounding points of the module path that matter for routing (normalised tokens, logits and
    affinities are rounded to ``x.dtype``).  Returns ``(out [T,H] x.dtype, logits [T,E] fp32, idx [T,K] int64, w [T,K] fp32)``."""
    T, H = x.shape
    dt = x.dtype
    xf = x.float()
    if gamma is not None:
        xf = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * gamma.float()).to(dt).float()
    logits = xf @ router_w.float().t()
    if router_bias is not None:
        logits = logits + router_bias.float()
    if round_logits:
        logits = logits.to(dt).float()
    actf = (lambda v: torch.softmax(v, -1)) if router_act == 0 else torch.sigmoid
    if act_over_topk:
        top, idx = torch.topk(logits, top_k, dim=-1)
        w = actf(top)
    else:
        aff = actf(logits)
        w, idx = torch.topk(aff, top_k, dim=-1)
    w = w.to(dt).float()
    if normalize:
        w = (w / w.sum(-1, keepdim=True).to(dt).float().clamp(min=1e-9)).to(dt).float()
    El, I = w_gu.shape[0], w_dn.shape[1]
    out = torch.zeros(T, H, dtype=torch.float32, device=x.device)
    for t in range(T):
        for kk in range(top_k):
            le = int(idx[t, kk]) - e0
            if not 0 <= le < El:
                continue
            wt = w[t, kk]
            gu = xf[t] @ w_gu[le].float()
            if pre_scale:
                gu = gu * wt
            h = _glu(gu[:I], gu[I:], act, act_alpha, act_beta, clamps)
            y = h @ w_dn[le].float()
            out[t] += y if pre_scale else y * wt
    return out.to(dt), logits, idx, w


def kernel_eligible(x: torch.Tensor, router_w: torch.Tensor, w_gu: torch.Tensor, w_dn: torch.Tensor, top_k: int,
                    gamma: Optional[torch.Tensor] = None) -> bool:
    if not (_ext.use_cuda(x, router_w, w_gu, w_dn) and hasattr(_ext.ext(), "moe_block_tkg")):
        return False
    if os.environ.get("NXD_MOE_TKG_KERNEL", "0") != "1":      # opt-in until a decode timing against the composed path
        return False                                           # (numerics: tests/test_moe_tkg_gpu.py)
    if not all(t.dtype == torch.bfloat16 and t.is_contiguous() for t in (x, router_w, w_gu, w_dn)):
        return False
    # the kernel loads x, gamma and the weights as 16-byte vectors: a view at an odd storage offset takes the reference
    if any(t is not None and t.data_ptr() % 16 for t in (x, gamma, router_w, w_gu, w_dn)):
        return False
    return bool(_ext.ext().moe_block_tkg_supported(x.shape[0], x.shape[1], router_w.shape[0], w_dn.shape[1], int(top_k)))


def moe_block_tkg(x, gamma, router_w, router_bias, w_gu, w_dn, e0: int, top_k: int, eps: float = 1e-6, router_act: int = 0,
                  act_over_topk: bool = False, normalize: bool = True, pre_scale: bool = False, round_logits: bool = True,
                  act: int = 0, act_alpha: float = 1.0, act_beta: float = 0.0, clamps=(-_INF, _INF, -_INF, _INF)):
    g = None if gamma is None else gamma.contiguous()
    if kernel_eligible(x, router_w, w_gu, w_dn, top_k, g):
        _ext.count_launch()
        c = [(-3.0e38 if math.isinf(v) and v < 0 else 3.0e38 if math.isinf(v) else float(v)) for v in clamps]
        coop = os.environ.get("NXD_MOE_TKG_COOP", "1") == "1"
        rb = None if router_bias is None else router_bias.float().contiguous()
        out, logits, idx, w = _ext.ext().moe_block_tkg(
            x, g, router_w, rb, w_gu, w_dn, int(e0), int(top_k), float(eps),
            int(router_act), bool(act_over_topk), bool(normalize), bool(pre_scale), bool(round_logits), int(act), float(act_alpha),
            float(act_beta), c[0], c[1], c[2], c[3], coop)
        return out, logits, idx, w
    return moe_block_tkg_reference(x, gamma, router_w, router_bias, w_gu, w_dn, e0, top_k, eps, router_act, act_over_topk,
                                   normalize, pre_scale, round_logits, act, act_alpha, act_beta, clamps)
