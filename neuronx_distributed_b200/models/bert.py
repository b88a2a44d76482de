"""BERT (encoder, MLM + NSP pre-training heads) built from the tensor-parallel layers — role of the reference's
``examples/training/tp_dp_bert_hf_pretrain/tp_dp_bert_large_hf_pretrain_hdf5.py`` (HF ``BertForPreTraining`` with the
self-attention / intermediate / output linears swapped for Column/RowParallelLinear and a vocab-parallel decoder).
``[B, S, H]`` layout (no sequence parallelism in the reference's BERT recipe), bidirectional attention with a padding mask."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from .. import ops
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layer_norm import LayerNorm
from ..parallel_layers.layers import ColumnParallelLinear, ParallelEmbedding, RowParallelLinear
from ..parallel_layers.loss_functions import parallel_cross_entropy


@dataclass
class BertConfig:
    vocab_size: int = 30528            # padded to a multiple of 64 like the reference recipe
    hidden_size: int = 1024
    num_hidden_layers: int = 24
    num_attention_heads: int = 16
    intermediate_size: int = 4096
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    layer_norm_eps: float = 1e-12
    hidden_dropout_prob: float = 0.0
    attention_probs_dropout_prob: float = 0.0    # dropout on the attention probabilities (training only)
    initializer_range: float = 0.02
    dtype: torch.dtype = torch.bfloat16
    device: Optional[torch.device] = None


def bert_large_config(**kw) -> BertConfig:
    return BertConfig(**kw)


def _init(std):
    return lambda w: nn.init.normal_(w, mean=0.0, std=std)


class BertEmbeddings(nn.Module):
    def __init__(self, cfg: BertConfig):
        super().__init__()
        self.word_embeddings = ParallelEmbedding(cfg.vocab_size, cfg.hidden_size, init_method=_init(cfg.initializer_range),
                                                 dtype=cfg.dtype, device=cfg.device)
        self.position_embeddings = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device)
        self.token_type_embeddings = nn.Embedding(cfg.type_vocab_size, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device)
        self.LayerNorm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, dtype=cfg.dtype, device=cfg.device)
        self.dropout = nn.Dropout(cfg.hidden_dropout_prob)

    def forward(self, input_ids, token_type_ids=None):
        B, S = input_ids.shape
        pos = torch.arange(S, device=input_ids.device).unsqueeze(0)
        tt = token_type_ids if token_type_ids is not None else torch.zeros_like(input_ids)
        x = self.word_embeddings(input_ids) + self.position_embeddings(pos) + self.token_type_embeddings(tt)
        return self.dropout(self.LayerNorm(x))


class BertSelfAttention(nn.Module):
    def __init__(self, cfg: BertConfig):
        super().__init__()
        tp = ps.get_tensor_model_parallel_size()
        self.heads_local = cfg.num_attention_heads // tp
        self.head_dim = cfg.hidden_size // cfg.num_attention_heads
        self.dropout_p = cfg.attention_probs_dropout_prob
        self.head_offset = ps.get_tensor_model_parallel_rank() * self.heads_local     # global index of the first local head
        mk = dict(bias=True, gather_output=False, init_method=_init(cfg.initializer_range), dtype=cfg.dtype, device=cfg.device)
        self.query = ColumnParallelLinear(cfg.hidden_size, cfg.hidden_size, **mk)
        self.key = ColumnParallelLinear(cfg.hidden_size, cfg.hidden_size, **mk)
        self.value = ColumnParallelLinear(cfg.hidden_size, cfg.hidden_size, **mk)
        self.dense = RowParallelLinear(cfg.hidden_size, cfg.hidden_size, bias=True, input_is_parallel=True,
                                       init_method=_init(cfg.initializer_range), dtype=cfg.dtype, device=cfg.device)

    def forward(self, x, key_padding_mask):
        B, S, _ = x.shape
        q, k, v = (lin(x).view(B, S, self.heads_local, self.head_dim) for lin in (self.query, self.key, self.value))
        drop = dict(dropout_p=self.dropout_p, head_offset=self.head_offset) if self.training and self.dropout_p > 0 else {}
        o = ops.attention.flash_attention(q, k, v, causal=False, key_padding_mask=key_padding_mask, **drop)   # bidirectional
        return self.dense(o.reshape(B, S, self.heads_local * self.head_dim))


class BertLayer(nn.Module):
    def __init__(self, cfg: BertConfig):
        super().__init__()
        self.attention = BertSelfAttention(cfg)
        self.attention_norm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, dtype=cfg.dtype, device=cfg.device)
        self.intermediate = ColumnParallelLinear(cfg.hidden_size, cfg.intermediate_size, bias=True, gather_output=False,
                                                 init_method=_init(cfg.initializer_range), dtype=cfg.dtype, device=cfg.device)
        self.output = RowParallelLinear(cfg.intermediate_size, cfg.hidden_size, bias=True, input_is_parallel=True,
                                        init_method=_init(cfg.initializer_range), dtype=cfg.dtype, device=cfg.device)
        self.output_norm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, dtype=cfg.dtype, device=cfg.device)
        self.dropout = nn.Dropout(cfg.hidden_dropout_prob)

    def forward(self, x, key_padding_mask):
        x = self.attention_norm(x + self.dropout(self.attention(x, key_padding_mask)))   # post-LN, as in BERT
        return self.output_norm(x + self.dropout(self.output(F.gelu(self.intermediate(x)))))


class BertModel(nn.Module):
    def __init__(self, cfg: BertConfig):
        super().__init__()
        self.cfg = cfg
        self.embeddings = BertEmbeddings(cfg)
        self.layers = nn.ModuleList([BertLayer(cfg) for _ in range(cfg.num_hidden_layers)])
        self.pooler = nn.Linear(cfg.hidden_size, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None):
        x = self.embeddings(input_ids, token_type_ids)
        key_padding_mask = attention_mask != 0 if attention_mask is not None else None     # [B, S], True = real token
        for layer in self.layers:
            x = layer(x, key_padding_mask)
        return x, torch.tanh(self.pooler(x[:, 0]))


class BertForPreTraining(nn.Module):
    """MLM (vocab-parallel decoder tied to the word embeddings, as in HF) + next-sentence head; returns the summed loss."""
    _no_split_modules = ["BertLayer"]

    def __init__(self, cfg: BertConfig):
        super().__init__()
        self.config = cfg
        self.bert = BertModel(cfg)
        self.transform = nn.Linear(cfg.hidden_size, cfg.hidden_size, dtype=cfg.dtype, device=cfg.device)
        self.transform_norm = LayerNorm(cfg.hidden_size, cfg.layer_norm_eps, dtype=cfg.dtype, device=cfg.device)
        self.decoder = ColumnParallelLinear(cfg.hidden_size, cfg.vocab_size, bias=True, gather_output=False,
                                            init_method=_init(cfg.initializer_range), dtype=cfg.dtype, device=cfg.device)
        self.decoder.weight = self.bert.embeddings.word_embeddings.weight            # tied (same vocab sharding)
        self.seq_relationship = nn.Linear(cfg.hidden_size, 2, dtype=cfg.dtype, device=cfg.device)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None, next_sentence_label=None):
        seq, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        h = self.transform_norm(F.gelu(self.transform(seq)))
        logits = self.decoder(h)                                                     # [B, S, V/tp]
        nsp_logits = self.seq_relationship(pooled)
        if labels is None:
            return None, (logits, nsp_logits)
        mask = labels != -100
        per_tok = parallel_cross_entropy(logits, torch.where(mask, labels, torch.zeros_like(labels)))
        loss = (per_tok * mask).sum() / mask.sum().clamp(min=1)
        if next_sentence_label is not None:
            loss = loss + F.cross_entropy(nsp_logits.float(), next_sentence_label)
        return loss, None
