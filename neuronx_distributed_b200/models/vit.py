"""Vision Transformer (image classification) on the tensor-parallel layers — role of the reference's
``examples/inference/vit`` (HF ``ViTForImageClassification`` with the patch projection as an output-channel-parallel
convolution and the encoder linears as Column/RowParallelLinear).  Pre-LN encoder, ``[B, N, H]`` layout."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from .. import ops
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layer_norm import LayerNorm
from ..parallel_layers.layers import ColumnParallelLinear, OutputChannelParallelConv2d, RowParallelLinear


@dataclass
class ViTConfig:
    image_size: int = 224
    patch_size: int = 16
    num_channels: int = 3
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    intermediate_size: int = 3072
    num_labels: int = 1000
    layer_norm_eps: float = 1e-12
    dtype: torch.dtype = torch.bfloat16
    device: Optional[torch.device] = None

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2


class ViTEmbeddings(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        # patch projection: conv with stride = patch, output channels sharded over TP then gathered
        self.projection = OutputChannelParallelConv2d(cfg.num_channels, cfg.hidden_size, cfg.patch_size, stride=cfg.patch_size,
                                                      gather_output=True, dtype=cfg.dtype, device=cfg.device)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device))
        self.position_embeddings = nn.Parameter(torch.zeros(1, cfg.num_patches + 1, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device))
        nn.init.trunc_normal_(self.position_embeddings, std=0.02)

    def forward(self, pixel_values):
        x = self.projection(pixel_values).flatten(2).transpose(1, 2)            # [B, N, H]
        x = torch.cat([self.cls_token.expand(x.shape[0], -1, -1), x], dim=1)
        return x + self.position_embeddings


class ViTLayer(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        tp = ps.get_tensor_model_parallel_size()
        self.heads_local = cfg.num_attention_heads // tp
        self.head_dim = cfg.hidden_size // cfg.num_attention_heads
        kw = dict(dtype=cfg.dtype, device=cfg.device)
        self.layernorm_before = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, **kw)
        self.qkv = ColumnParallelLinear(cfg.hidden_size, 3 * cfg.hidden_size, bias=True, gather_output=False, stride=3, **kw)
        self.out = RowParallelLinear(cfg.hidden_size, cfg.hidden_size, bias=True, input_is_parallel=True, **kw)
        self.layernorm_after = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, **kw)
        self.fc1 = ColumnParallelLinear(cfg.hidden_size, cfg.intermediate_size, bias=True, gather_output=False, **kw)
        self.fc2 = RowParallelLinear(cfg.intermediate_size, cfg.hidden_size, bias=True, input_is_parallel=True, **kw)

    def forward(self, x):
        B, N, _ = x.shape
        q, k, v = self.qkv(self.layernorm_before(x)).chunk(3, dim=-1)
        q, k, v = (t.reshape(B, N, self.heads_local, self.head_dim) for t in (q, k, v))
        a = ops.attention.flash_attention(q, k, v, causal=False).reshape(B, N, self.heads_local * self.head_dim)
        x = x + self.out(a)
        return x + self.fc2(F.gelu(self.fc1(self.layernorm_after(x))))


class ViTForImageClassification(nn.Module):
    _no_split_modules = ["ViTLayer"]

    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.config = cfg
        self.embeddings = ViTEmbeddings(cfg)
        self.layers = nn.ModuleList([ViTLayer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.layernorm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, dtype=cfg.dtype, device=cfg.device)
        self.classifier = ColumnParallelLinear(cfg.hidden_size, cfg.num_labels, bias=True, gather_output=True,
                                               dtype=cfg.dtype, device=cfg.device)

    def forward(self, pixel_values, labels=None):
        x = self.embeddings(pixel_values)
        for layer in self.layers:
            x = layer(x)
        logits = self.classifier(self.layernorm(x)[:, 0])
        if labels is None:
            return logits
        return F.cross_entropy(logits.float(), labels), logits
