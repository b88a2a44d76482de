"""Llama (2/3) built from the tensor-parallel layers.

Role parity with reference ``examples/training/llama/modeling_llama_nxd.py`` (attention :299-362,
MLP :161-220, decoder :532-550, causal-LM + vocab-parallel loss :712-824).  Written for the H100
kernel set: activations are kept in ``[S, B, H]`` ("SBH") so sequence-parallel shards are
contiguous row blocks that the fused AG→GEMM / GEMM→RS kernels treat as 2-D ``[tokens, H]``
matrices; QKV is one fused GEMM; gate/up is one fused GEMM followed by the SwiGLU kernel;
RoPE, RMSNorm, attention and the loss are the hand-written kernels in ``ops/``.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.fx
from torch import nn
from torch.utils.checkpoint import checkpoint

from ..utils.profiling import nvtx_range
from .. import ops
from ..modules.qkv_linear import GQAQKVColumnParallelLinear
from ..modules.rms_norm import RMSNorm
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layers import ColumnParallelLinear, ParallelEmbedding, RowParallelLinear
from ..parallel_layers.loss_functions import fused_linear_cross_entropy, parallel_cross_entropy


@dataclass
class LlamaConfig:
    vocab_size: int = 32000
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: Optional[int] = None
    max_position_embeddings: int = 4096
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    rope_scaling_factor: float = 1.0
    # Llama-3.1 / 3.2 frequency rescaling: the "llama3" keys of a Hugging Face rope_scaling (factor, low_freq_factor,
    # high_freq_factor, original_max_position_embeddings); None = plain RoPE
    rope_scaling: Optional[dict] = None
    # bias on the q / k / v projections (Qwen2); o_proj has none
    qkv_bias: bool = False
    initializer_range: float = 0.02
    tie_word_embeddings: bool = False
    sequence_parallel_enabled: bool = False
    activation_checkpointing: str = "none"      # "none" | "full" | "selective"
    fuse_qkv: bool = True
    kv_size_multiplier: int = 1
    dtype: torch.dtype = torch.bfloat16
    pad_token_id: Optional[int] = None
    # context parallel: each CP rank holds a contiguous S/cp slice; positions are offset
    context_parallel: bool = False
    cp_layout: str = "contiguous"           # "zigzag": rank r holds sequence chunks (r, 2·cp−1−r); needs the pull attention path
    device: Optional[torch.device] = None       # construct parameters directly here (e.g. cuda)
    # sliding-window attention (Mistral / Mixtral): query i sees keys i − W < j ≤ i; None = full causal attention
    sliding_window: Optional[int] = None
    # row-wise scaled FP8 (e4m3) GEMMs in the decoder's qkv, o, gate_up and down projections (tp_linear(fp8=True));
    # lm_head, the embedding and MoE experts stay bf16, and parameters and checkpoints are those of a bf16 model
    fp8_training: bool = False

    def __post_init__(self):
        if self.num_key_value_heads is None:
            self.num_key_value_heads = self.num_attention_heads

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


def llama2_7b_config(**kw) -> LlamaConfig:
    return LlamaConfig(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_hidden_layers=32,
                       num_attention_heads=32, num_key_value_heads=32, **kw)


def llama2_13b_config(**kw) -> LlamaConfig:
    return LlamaConfig(vocab_size=32016, hidden_size=5120, intermediate_size=13824, num_hidden_layers=40,
                       num_attention_heads=40, num_key_value_heads=40, **kw)


def llama2_70b_config(**kw) -> LlamaConfig:
    return LlamaConfig(vocab_size=32000, hidden_size=8192, intermediate_size=28672, num_hidden_layers=80,
                       num_attention_heads=64, num_key_value_heads=8, **kw)


def _normal_init(std: float):
    def f(w):
        return nn.init.normal_(w, mean=0.0, std=std)

    return f


class LlamaMLP(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        init = _normal_init(cfg.initializer_range)
        sp = cfg.sequence_parallel_enabled
        # stride=2 interleaves [gate; up] so each rank's shard is [gate_r ; up_r]
        self.gate_up_proj = ColumnParallelLinear(
            cfg.hidden_size, 2 * cfg.intermediate_size, bias=False, gather_output=False, stride=2,
            init_method=init, sequence_parallel_enabled=sp, sequence_dimension=0, dtype=cfg.dtype, device=cfg.device,
        )
        self.down_proj = RowParallelLinear(
            cfg.intermediate_size, cfg.hidden_size, bias=False, input_is_parallel=True, init_method=init,
            sequence_parallel_enabled=sp, sequence_dimension=0, dtype=cfg.dtype, device=cfg.device,
        )
        self.gate_up_proj.fp8_training = self.down_proj.fp8_training = cfg.fp8_training

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.down_proj(ops.act.swiglu(self.gate_up_proj(x)))


class LlamaAttention(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.cfg = cfg
        tp = ps.get_tensor_model_parallel_size()
        init = _normal_init(cfg.initializer_range)
        sp = cfg.sequence_parallel_enabled
        self.head_dim = cfg.head_dim
        kv_mult = cfg.kv_size_multiplier
        if (cfg.num_key_value_heads * kv_mult) % tp != 0:
            # smallest replication that makes kv heads divisible by tp
            kv_mult = tp // math.gcd(tp, cfg.num_key_value_heads)
        self.num_heads_local = cfg.num_attention_heads // tp
        self.num_kv_heads_local = cfg.num_key_value_heads * kv_mult // tp
        self.qkv_proj = GQAQKVColumnParallelLinear(
            cfg.hidden_size,
            [cfg.num_attention_heads * self.head_dim, cfg.num_key_value_heads * self.head_dim],
            bias=cfg.qkv_bias, gather_output=False, init_method=init, sequence_parallel_enabled=sp,
            kv_size_multiplier=kv_mult, fuse_qkv=cfg.fuse_qkv, dtype=cfg.dtype, sequence_dimension=0,
            head_dim=self.head_dim, device=cfg.device,
        )
        self.o_proj = RowParallelLinear(
            cfg.num_attention_heads * self.head_dim, cfg.hidden_size, bias=False, input_is_parallel=True,
            init_method=init, sequence_parallel_enabled=sp, sequence_dimension=0, dtype=cfg.dtype, device=cfg.device,
        )
        self.qkv_proj.fp8_training = self.o_proj.fp8_training = cfg.fp8_training

    def forward(self, x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
        # x: [S(/tp), B, H]  →  q/k/v: [S, B, h_local*D]
        q, k, v = self.qkv_proj(x)
        clip = getattr(self.cfg, "clip_qkv", None)
        if clip is not None:                      # DBRX: clamp the projections (HF DbrxAttention clip_qkv)
            q, k, v = q.clamp(-clip, clip), k.clamp(-clip, clip), v.clamp(-clip, clip)
        S, B = q.shape[0], q.shape[1]
        # [S,B,h,D] → [B,S,h,D] views (free when B == 1)
        q = q.reshape(S, B, self.num_heads_local, self.head_dim).transpose(0, 1)
        k = k.reshape(S, B, self.num_kv_heads_local, self.head_dim).transpose(0, 1)
        v = v.reshape(S, B, self.num_kv_heads_local, self.head_dim).transpose(0, 1)
        q = ops.rope.apply_rotary(q, cos, sin)
        k = ops.rope.apply_rotary(k, cos, sin)
        if self.cfg.context_parallel and ps.get_context_model_parallel_size() > 1:
            from ..modules.attention.ring import pull_attention, ring_attention

            w = self.cfg.sliding_window
            if w is not None and not _CP_WINDOW:
                raise NotImplementedError("sliding_window with context parallelism is opt-in until the windowed ring has run on "
                                          "several GPUs: set NXD_CP_WINDOW=1")
            if self.cfg.cp_layout != "contiguous":
                # the ring keeps the contiguous split
                o = pull_attention(q, k, v, causal=True, layout=self.cfg.cp_layout, sliding_window=w)
            else:
                o = (pull_attention if _CP_PULL else ring_attention)(q, k, v, causal=True, sliding_window=w)
        else:
            o = ops.attention.flash_attention(q, k, v, causal=True, sliding_window=self.cfg.sliding_window)
        o = o.transpose(0, 1).reshape(S, B, self.num_heads_local * self.head_dim)
        return self.o_proj(o)


# Residual adds fused with the RMSNorm that follows them (csrc/fused_norm.cu; GPU numerics:
# tests/test_kernels_gpu.py::test_fused_add_rmsnorm_vs_fp32_reference, measured +0.8 % on the TP=1 step with the
# post-attention norm alone).  NXD_FUSED_ADD_NORM=0 restores the separate add + norm kernels.
_FUSED_ADD_NORM = os.environ.get("NXD_FUSED_ADD_NORM", "1") == "1"
# lm_head + vocab-parallel CE in row chunks without materialising the logits (parallel_layers/loss_functions.py
# ``fused_linear_cross_entropy``).  Opt-in: CPU-verified against the unfused path, not yet timed on hardware.
_FUSED_LMHEAD_CE = os.environ.get("NXD_FUSED_LMHEAD_CE", "0") == "1"
_LMHEAD_CE_CHUNK = int(os.environ.get("NXD_LMHEAD_CE_CHUNK", "2048"))
# context parallelism without a ring: K/V published in symmetric memory, peers' slices read inside the attention kernel
# (modules/attention/ring.py ``pull_attention``).  Opt-in: CPU-verified against the ring and dense attention only.
_CP_PULL = os.environ.get("NXD_CP_PULL", "0") == "1"
# sliding window under context parallelism (ring / pull attention with the windowed block plan).  Opt-in: CPU-verified
# multi-process and emulated in one process on an H100 (tests/test_cp_sliding_window_*.py); the NCCL ring with a window has
# not yet run on more than one GPU.  Without it a windowed model raises NotImplementedError at CP > 1, as before.
_CP_WINDOW = os.environ.get("NXD_CP_WINDOW", "0") == "1"


class LlamaDecoderLayer(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        sp = cfg.sequence_parallel_enabled
        self.input_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps, sequence_parallel_enabled=sp, dtype=cfg.dtype, device=cfg.device)
        self.self_attn = LlamaAttention(cfg)
        self.post_attention_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps, sequence_parallel_enabled=sp,
                                                dtype=cfg.dtype, device=cfg.device)
        self.mlp = LlamaMLP(cfg)

    def forward(self, x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
        with nvtx_range("attn"):
            a = self.self_attn(self.input_layernorm(x), cos, sin)
        with nvtx_range("mlp"):
            if _FUSED_ADD_NORM:                    # residual add + post-attention norm in one pass over the rows
                n = self.post_attention_layernorm
                y, x = ops.norm.add_rms_norm(a, x, n.weight, n.variance_epsilon)
                x = x + self.mlp(y)
            else:
                x = x + a
                x = x + self.mlp(self.post_attention_layernorm(x))
        return x

    def forward_deferred(self, x: torch.Tensor, d: Optional[torch.Tensor], cos: torch.Tensor, sin: torch.Tensor):
        """Same block with the residual stream kept as ``x + d``: the MLP output ``d`` of the previous block is added inside
        THIS block's input norm (one fused add+norm pass instead of an add pass and a norm pass, forward and backward).
        Returns ``(x, d)`` for the next block; ``LlamaModel`` folds the last ``d`` into the final norm."""
        n1, n2 = self.input_layernorm, self.post_attention_layernorm
        with nvtx_range("attn"):
            if d is None:
                y = n1(x)
            else:
                y, x = ops.norm.add_rms_norm(d, x, n1.weight, n1.variance_epsilon)
            a = self.self_attn(y, cos, sin)
        with nvtx_range("mlp"):
            y, x = ops.norm.add_rms_norm(a, x, n2.weight, n2.variance_epsilon)
            d = self.mlp(y)
        return x, d


class LlamaModel(nn.Module):
    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.cfg = cfg
        self.embed_tokens = ParallelEmbedding(
            cfg.vocab_size, cfg.hidden_size, init_method=_normal_init(cfg.initializer_range), dtype=cfg.dtype,
            sequence_parallel_enabled=cfg.sequence_parallel_enabled, device=cfg.device,
        )
        self.layers = nn.ModuleList([LlamaDecoderLayer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.norm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps, sequence_parallel_enabled=cfg.sequence_parallel_enabled,
                            dtype=cfg.dtype, device=cfg.device)
        self._rope_cache: Optional[Tuple[int, int, torch.device, torch.Tensor, torch.Tensor]] = None

    def rope(self, seq_len: int, device, offset: int = 0):
        c = self._rope_cache
        if c is None or c[0] != seq_len or c[1] != offset or c[2] != device:
            cos, sin = ops.rope.rope_tables(seq_len, self.cfg.head_dim, self.cfg.rope_theta, device, offset,
                                            self.cfg.rope_scaling_factor, self.cfg.rope_scaling)
            self._rope_cache = (seq_len, offset, device, cos, sin)
            c = self._rope_cache
        return c[3], c[4]

    def forward(self, input_ids: torch.Tensor) -> torch.Tensor:
        """``input_ids`` [B, S] → hidden [S(/tp), B, H]."""
        B, S = input_ids.shape
        x = self.embed_tokens(input_ids)  # SP: [S/tp, B, H]; else [B, S, H]
        if not self.cfg.sequence_parallel_enabled:
            x = x.transpose(0, 1).contiguous()
        offset = 0
        cp = ps.get_context_model_parallel_size() if self.cfg.context_parallel else 1
        if cp > 1 and self.cfg.cp_layout == "zigzag":
            # local tokens = sequence chunks (r, 2·cp−1−r): two position ranges
            r, c = ps.get_context_model_parallel_rank(), S // 2
            zz = self.__dict__.get("_rope_cache_zz")
            if zz is None or zz[0] != (S, r, cp, input_ids.device):
                tabs = [ops.rope.rope_tables(c, self.cfg.head_dim, self.cfg.rope_theta, input_ids.device, off,
                                             self.cfg.rope_scaling_factor, self.cfg.rope_scaling)
                        for off in (r * c, (2 * cp - 1 - r) * c)]
                zz = ((S, r, cp, input_ids.device), torch.cat([tabs[0][0], tabs[1][0]]), torch.cat([tabs[0][1], tabs[1][1]]))
                self.__dict__["_rope_cache_zz"] = zz
            cos, sin = zz[1], zz[2]
        else:
            if cp > 1:
                offset = ps.get_context_model_parallel_rank() * S
            cos, sin = self.rope(S, input_ids.device, offset)
        ckpt = self.cfg.activation_checkpointing == "full" and self.training
        if _FUSED_ADD_NORM and not ckpt and type(self.layers[0]).forward is LlamaDecoderLayer.forward \
                and not torch.jit.is_tracing() and not isinstance(x, torch.fx.Proxy):
            d = None
            for layer in self.layers:
                x, d = layer.forward_deferred(x, d, cos, sin)
            y, _ = ops.norm.add_rms_norm(d, x, self.norm.weight, self.norm.variance_epsilon)
            return y
        for layer in self.layers:
            if ckpt:
                x = checkpoint(layer, x, cos, sin, use_reentrant=False)
            else:
                x = layer(x, cos, sin)
        return self.norm(x)


class LlamaForCausalLM(nn.Module):
    _no_split_modules = ["LlamaDecoderLayer"]      # unit of activation checkpointing / pipeline partitioning (HF convention)

    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.config = cfg
        self.model = LlamaModel(cfg)
        self.lm_head = ColumnParallelLinear(
            cfg.hidden_size, cfg.vocab_size, bias=False, gather_output=False,
            init_method=_normal_init(cfg.initializer_range), sequence_parallel_enabled=cfg.sequence_parallel_enabled,
            sequence_dimension=0, dtype=cfg.dtype, device=cfg.device,
        )
        if cfg.tie_word_embeddings:
            self.lm_head.weight = self.model.embed_tokens.weight
            self.lm_head.weight._nxd_multi_use = True      # two gradient contributions per backward (ZeRO-1 overlap defers it)

    def forward(self, input_ids: torch.Tensor, labels: Optional[torch.Tensor] = None, shift_labels: bool = True):
        """Returns ``(loss, logits)``; ``logits`` are vocab-parallel ``[S, B, V/tp]`` and are only
        returned when ``labels`` is None (so training never holds two copies)."""
        h = self.model(input_ids)
        if labels is None:
            return None, self.lm_head(h)  # [S, B, V/tp]
        # next-token objective: position s predicts labels[s+1]
        tgt = labels.transpose(0, 1)  # [S, B]
        if shift_labels:
            tgt = torch.cat([tgt[1:], torch.full_like(tgt[:1], -100)], dim=0)
        if _FUSED_LMHEAD_CE:
            # lm_head GEMM, CE statistics, CE gradient, dgrad and wgrad per row chunk: the [S·B, V/tp] logits never exist
            loss = fused_linear_cross_entropy(h, self.lm_head.weight, tgt, sequence_parallel=self.config.sequence_parallel_enabled,
                                              chunk_rows=_LMHEAD_CE_CHUNK)
            return loss, None
        logits = self.lm_head(h)  # [S, B, V/tp]
        mask = tgt != -100
        safe_tgt = torch.where(mask, tgt, torch.zeros_like(tgt))
        per_tok = parallel_cross_entropy(logits, safe_tgt)
        loss = (per_tok * mask).sum() / mask.sum().clamp(min=1)
        return loss, None

    def num_parameters_global(self) -> int:
        c = self.config
        hd = c.head_dim
        per_layer = (c.hidden_size * (c.num_attention_heads * hd + 2 * c.num_key_value_heads * hd)
                     + c.num_attention_heads * hd * c.hidden_size + 3 * c.hidden_size * c.intermediate_size
                     + 2 * c.hidden_size)
        return per_layer * c.num_hidden_layers + 2 * c.vocab_size * c.hidden_size + c.hidden_size
