"""GPT-NeoX built from the tensor-parallel layers (role of reference
``examples/training/tp_dp_gpt_neox_hf_pretrain/.../modeling_gpt_neox_nxd.py:73-95,228-290,454-460``):
fused QKV column-parallel projection (per-head [q|k|v] interleave as in HF), partial rotary (``rotary_pct``),
parallel residual, GELU MLP, LayerNorm with sequence-parallel tagged affine parameters.  ``[S, B, H]`` layout."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn
from torch.utils.checkpoint import checkpoint

from .. import ops
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layer_norm import LayerNorm
from ..parallel_layers.layers import ColumnParallelLinear, ParallelEmbedding, RowParallelLinear
from ..parallel_layers.loss_functions import parallel_cross_entropy


@dataclass
class GPTNeoXConfig:
    vocab_size: int = 50432
    hidden_size: int = 6144
    num_hidden_layers: int = 44
    num_attention_heads: int = 64
    intermediate_size: int = 24576
    rotary_pct: float = 0.25
    rotary_emb_base: float = 10000.0
    max_position_embeddings: int = 2048
    layer_norm_eps: float = 1e-5
    use_parallel_residual: bool = True
    hidden_act: str = "gelu"                 # HF name: "gelu" (erf), or "gelu_fast" / "gelu_new" / "gelu_pytorch_tanh" (tanh)
    attention_dropout: float = 0.0           # dropout on the attention probabilities (training only)
    initializer_range: float = 0.02
    sequence_parallel_enabled: bool = False
    activation_checkpointing: str = "none"
    dtype: torch.dtype = torch.bfloat16
    device: Optional[torch.device] = None

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


def gpt_neox_20b_config(**kw) -> GPTNeoXConfig:
    return GPTNeoXConfig(**kw)


def _init(std):
    return lambda w: nn.init.normal_(w, mean=0.0, std=std)


class GPTNeoXAttention(nn.Module):
    def __init__(self, cfg: GPTNeoXConfig):
        super().__init__()
        tp = ps.get_tensor_model_parallel_size()
        self.cfg = cfg
        self.heads_local = cfg.num_attention_heads // tp
        self.head_dim = cfg.head_dim
        self.head_offset = ps.get_tensor_model_parallel_rank() * self.heads_local     # global index of the first local head
        self.rot = int(self.head_dim * cfg.rotary_pct)
        sp = cfg.sequence_parallel_enabled
        # HF layout: output rows ordered head-major [h0:(q,k,v), h1:(q,k,v), …] → plain dim-0 sharding keeps whole heads
        self.query_key_value = ColumnParallelLinear(cfg.hidden_size, 3 * cfg.hidden_size, bias=True, gather_output=False,
                                                    init_method=_init(cfg.initializer_range), sequence_parallel_enabled=sp,
                                                    sequence_dimension=0, dtype=cfg.dtype, device=cfg.device)
        self.dense = RowParallelLinear(cfg.hidden_size, cfg.hidden_size, bias=True, input_is_parallel=True,
                                       init_method=_init(cfg.initializer_range), sequence_parallel_enabled=sp,
                                       sequence_dimension=0, dtype=cfg.dtype, device=cfg.device)

    def forward(self, x, cos, sin):
        qkv = self.query_key_value(x)                                  # [S, B, 3·h_l·D]
        S, B = qkv.shape[:2]
        qkv = qkv.view(S, B, self.heads_local, 3 * self.head_dim)
        q, k, v = (t.transpose(0, 1) for t in qkv.split(self.head_dim, dim=-1))   # [B, S, h, D]
        if self.rot > 0:
            q = torch.cat([ops.rope.apply_rotary(q[..., : self.rot].contiguous(), cos, sin), q[..., self.rot:]], dim=-1)
            k = torch.cat([ops.rope.apply_rotary(k[..., : self.rot].contiguous(), cos, sin), k[..., self.rot:]], dim=-1)
        p = self.cfg.attention_dropout
        drop = dict(dropout_p=p, head_offset=self.head_offset) if self.training and p > 0 else {}
        o = ops.attention.flash_attention(q.contiguous(), k.contiguous(), v.contiguous(), causal=True, **drop)
        return self.dense(o.transpose(0, 1).reshape(S, B, self.heads_local * self.head_dim))


_GELU_APPROX = {"gelu": "none", "gelu_fast": "tanh", "gelu_new": "tanh", "gelu_pytorch_tanh": "tanh"}


class GPTNeoXMLP(nn.Module):
    def __init__(self, cfg: GPTNeoXConfig):
        super().__init__()
        sp = cfg.sequence_parallel_enabled
        if cfg.hidden_act not in _GELU_APPROX:
            raise ValueError(f"hidden_act {cfg.hidden_act!r} is not supported (one of {sorted(_GELU_APPROX)})")
        self.gelu_approximate = _GELU_APPROX[cfg.hidden_act]
        self.dense_h_to_4h = ColumnParallelLinear(cfg.hidden_size, cfg.intermediate_size, bias=True, gather_output=False,
                                                  init_method=_init(cfg.initializer_range), sequence_parallel_enabled=sp,
                                                  sequence_dimension=0, dtype=cfg.dtype, device=cfg.device)
        self.dense_4h_to_h = RowParallelLinear(cfg.intermediate_size, cfg.hidden_size, bias=True, input_is_parallel=True,
                                               init_method=_init(cfg.initializer_range), sequence_parallel_enabled=sp,
                                               sequence_dimension=0, dtype=cfg.dtype, device=cfg.device)

    def forward(self, x):
        return self.dense_4h_to_h(torch.nn.functional.gelu(self.dense_h_to_4h(x), approximate=self.gelu_approximate))


class GPTNeoXLayer(nn.Module):
    def __init__(self, cfg: GPTNeoXConfig):
        super().__init__()
        sp = cfg.sequence_parallel_enabled
        self.use_parallel_residual = cfg.use_parallel_residual
        self.input_layernorm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, sequence_parallel_enabled=sp, dtype=cfg.dtype, device=cfg.device)
        self.post_attention_layernorm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, sequence_parallel_enabled=sp, dtype=cfg.dtype, device=cfg.device)
        self.attention = GPTNeoXAttention(cfg)
        self.mlp = GPTNeoXMLP(cfg)

    def forward(self, x, cos, sin):
        a = self.attention(self.input_layernorm(x), cos, sin)
        if self.use_parallel_residual:
            return x + a + self.mlp(self.post_attention_layernorm(x))
        x = x + a
        return x + self.mlp(self.post_attention_layernorm(x))


class GPTNeoXModel(nn.Module):
    def __init__(self, cfg: GPTNeoXConfig):
        super().__init__()
        self.cfg = cfg
        self.embed_in = ParallelEmbedding(cfg.vocab_size, cfg.hidden_size, init_method=_init(cfg.initializer_range),
                                          dtype=cfg.dtype, sequence_parallel_enabled=cfg.sequence_parallel_enabled, device=cfg.device)
        self.layers = nn.ModuleList([GPTNeoXLayer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.final_layer_norm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps,
                                          sequence_parallel_enabled=cfg.sequence_parallel_enabled, dtype=cfg.dtype, device=cfg.device)

    def forward(self, input_ids):
        B, S = input_ids.shape
        x = self.embed_in(input_ids)
        if not self.cfg.sequence_parallel_enabled:
            x = x.transpose(0, 1).contiguous()
        rot = int(self.cfg.head_dim * self.cfg.rotary_pct)
        cos, sin = ops.rope.rope_tables(S, max(rot, 2), self.cfg.rotary_emb_base, input_ids.device)
        for layer in self.layers:
            if self.cfg.activation_checkpointing == "full" and self.training:
                x = checkpoint(layer, x, cos, sin, use_reentrant=False)
            else:
                x = layer(x, cos, sin)
        return self.final_layer_norm(x)


class GPTNeoXForCausalLM(nn.Module):
    _no_split_modules = ["GPTNeoXLayer"]

    def __init__(self, cfg: GPTNeoXConfig):
        super().__init__()
        self.config = cfg
        self.gpt_neox = GPTNeoXModel(cfg)
        self.embed_out = ColumnParallelLinear(cfg.hidden_size, cfg.vocab_size, bias=False, gather_output=False,
                                              init_method=_init(cfg.initializer_range),
                                              sequence_parallel_enabled=cfg.sequence_parallel_enabled, sequence_dimension=0,
                                              dtype=cfg.dtype, device=cfg.device)

    def forward(self, input_ids, labels=None):
        logits = self.embed_out(self.gpt_neox(input_ids))           # [S, B, V/tp]
        if labels is None:
            return None, logits
        tgt = labels.transpose(0, 1)
        tgt = torch.cat([tgt[1:], torch.full_like(tgt[:1], -100)], dim=0)
        mask = tgt != -100
        per_tok = parallel_cross_entropy(logits, torch.where(mask, tgt, torch.zeros_like(tgt)))
        return (per_tok * mask).sum() / mask.sum().clamp(min=1), None
