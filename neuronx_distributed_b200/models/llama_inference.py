"""Llama inference model: context encoding (prefill) + token generation (decode) over a persistent KV cache, with
on-device sampling — role of reference ``examples/inference`` (``NeuronBaseModel`` / ``ModelWrapper`` /
``KVCacheManager`` / ``hf_adapter``), re-using the training model's parameter names so the same checkpoints load.
No sequence parallelism at inference: Row-parallel outputs are all-reduced."""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from .. import ops
from ..inference.kv_cache import KVCacheManager, per_tensor
from ..quantization.quantization_config import KVQuantizationConfig
from ..utils.sampling import Sampler
from .llama import LlamaConfig, LlamaForCausalLM


class LlamaForInference(nn.Module):
    def __init__(self, cfg: LlamaConfig, batch_size: int = 1, max_seq_len: int = 2048, on_device_sampling: bool = True,
                 sampler: Optional[Sampler] = None, lm_cls=None, flash_decoding: bool = False,
                 kv_quant: Optional[KVQuantizationConfig] = None, rolling_kv_cache: bool = False):
        """``lm_cls``: any decoder built from Llama attention blocks (``LlamaForCausalLM`` default; ``MixtralForCausalLM`` for
        the MoE families — its layers' ``mlp`` returns ``(y, router_logits)``, handled in ``_body``).
        ``kv_quant``: store the KV cache quantised, with one scale per tensor (fp8 e4m3 is read by the decode kernels
        directly).  Prefill attention runs on the un-quantised k/v it computes; only the cache write is quantised.
        ``rolling_kv_cache`` (needs ``cfg.sliding_window``): keep only the last ``sliding_window + 64`` positions of each
        sequence in a ring (``inference.kv_cache``), so cache memory no longer grows with ``max_seq_len``.  The model then
        computes what it computes on the full cache; ``kv_len`` must be None."""
        super().__init__()
        if rolling_kv_cache and cfg.sliding_window is None:
            raise ValueError("rolling_kv_cache needs a model with a sliding window (cfg.sliding_window)")
        if rolling_kv_cache and flash_decoding:
            raise ValueError("rolling_kv_cache does not combine with flash_decoding")
        cfg.sequence_parallel_enabled = False
        cfg.activation_checkpointing = "none"
        self.cfg = cfg
        self.lm = (lm_cls or LlamaForCausalLM)(cfg)
        self.batch_size, self.max_seq_len = batch_size, max_seq_len
        # flash decoding (reference examples/inference ``flash_decoding_enabled``): TP ranks that hold replicas of the same KV
        # heads shard the cache along the SEQUENCE inside that replica group instead of storing it ``m`` times
        self.flash_decoding, self.kv_group, self.kv_rank, shards = bool(flash_decoding), None, 0, 1
        if flash_decoding:
            import torch.distributed as dist

            attn0 = self._core.layers[0].self_attn
            self.kv_group = getattr(attn0.qkv_proj, "kv_group", None)
            assert self.kv_group is not None and dist.get_world_size(self.kv_group) > 1, \
                "flash decoding needs replicated KV heads (tensor-parallel size > number of KV heads)"
            shards, self.kv_rank = dist.get_world_size(self.kv_group), dist.get_rank(self.kv_group)
            assert max_seq_len % shards == 0, f"max_seq_len {max_seq_len} must divide by the KV replication factor {shards}"
        if kv_quant is not None and not per_tensor(kv_quant):
            raise ValueError("kv_quant: the KV cache implements one scale per tensor; per-key and per-channel methods are "
                             "not supported")
        if kv_quant is not None and kv_quant.dequant_dtype != cfg.dtype:
            raise ValueError(f"kv_quant.dequant_dtype ({kv_quant.dequant_dtype}) must be the model dtype ({cfg.dtype}): "
                             "attention off the kernels reads the de-quantised cache next to the model's queries")
        self.kv = KVCacheManager(cfg.num_hidden_layers, batch_size, max_seq_len, self._kv_heads_local(), cfg.head_dim,
                                 dtype=cfg.dtype, device=cfg.device, kv_quant=kv_quant, num_cores_per_group=shards,
                                 rolling_window=cfg.sliding_window if rolling_kv_cache else None)
        self.sampler = sampler or Sampler(top_k=1, vocab_parallel=True)
        self.on_device_sampling = on_device_sampling
        cos, sin = self._rope_tables(max_seq_len)
        self.register_buffer("rope_cos", cos, persistent=False)
        self.register_buffer("rope_sin", sin, persistent=False)

    # ------------------------------------------------------------------ what another decoder family overrides
    @property
    def _core(self):
        return getattr(self.lm, "model", self.lm)        # Llama nests the decoder under .model, Mixtral/DBRX do not

    def _kv_heads_local(self) -> int:
        return self._core.layers[0].self_attn.num_kv_heads_local

    def _rope_tables(self, max_seq_len: int):
        """``(cos, sin) [max_seq_len, R/2]``: the rotary width R is twice the tables' width (R = head_dim here)."""
        c = self.cfg
        return ops.rope.rope_tables(max_seq_len, c.head_dim, c.rope_theta, c.device, 0, c.rope_scaling_factor, c.rope_scaling)

    def _logits(self, h: torch.Tensor) -> torch.Tensor:
        return self.lm.lm_head(h)

    def load_state_dict(self, sd, strict: bool = True):
        return self.lm.load_state_dict(sd, strict=strict)

    def state_dict(self, *a, **k):
        return self.lm.state_dict(*a, **k)

    # ------------------------------------------------------------------ shared pieces
    def _attn_block(self, layer_idx: int, layer, x: torch.Tensor, positions: Optional[torch.Tensor], prefill: bool,
                    kv_len: Optional[int], tree=None, prompt_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        att = layer.self_attn
        h = layer.input_layernorm(x)
        q, k, v = att.qkv_proj(h)                          # [S, B, h*D]
        S, B = q.shape[0], q.shape[1]
        D = att.head_dim
        q = q.reshape(S, B, att.num_heads_local, D).transpose(0, 1)
        k = k.reshape(S, B, att.num_kv_heads_local, D).transpose(0, 1)
        v = v.reshape(S, B, att.num_kv_heads_local, D).transpose(0, 1).contiguous()
        o = self._attention(layer_idx, q, k, v, positions, prefill, kv_len, tree, prompt_lens)
        o = o.transpose(0, 1).reshape(S, B, att.num_heads_local * D)
        return _row_linear_plus_residual(att.o_proj, o, x)

    def _attention(self, layer_idx: int, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, positions: Optional[torch.Tensor],
                   prefill: bool, kv_len: Optional[int], tree=None, prompt_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """RoPE, the cache write and attention of one layer: q ``[B, S, H, D]``, k / v ``[B, S, Hkv, D]`` (any b / s / h
        strides) → o ``[B, S, H, D]``.  The rotary width R is twice the tables' width: R < D (GPT-NeoX ``rotary_pct``)
        rotates dims [0, R) and passes the rest through, on the kernel and on the torch paths alike."""
        S = q.shape[1]
        sw = getattr(self.cfg, "sliding_window", None)     # Mistral / Mixtral window (None: full causal attention)
        roll = {"rolling": True} if self.kv.rolling else {}   # ring cache: the kernels and torch paths map positions to rows
        # (k_scale, v_scale) when the decode kernels read the cache as stored; the defaults (1.0) are not passed on, so a bf16
        # cache makes the calls it makes without quantisation
        scales = self.kv.kernel_scales()
        scale_kw = {} if scales in (None, (1.0, 1.0)) else {"k_scale": scales[0], "v_scale": scales[1]}
        if prefill:
            cos, sin = self.rope_cos[:S], self.rope_sin[:S]
            q, k = _rotary(ops.rope.apply_rotary, q, cos, sin), _rotary(ops.rope.apply_rotary, k, cos, sin)
            if self.flash_decoding:
                self.kv.write_prefill_sharded(layer_idx, k, v, self.kv_rank)
            else:
                self.kv.write_prefill(layer_idx, k, v, lengths=prompt_lens)
            o = ops.attention.flash_attention(q, k, v, causal=True, sliding_window=sw)
        elif self.flash_decoding:
            assert S == 1 and tree is None, "flash decoding serves plain token generation (no speculation window)"
            from ..modules.attention.flash_decode import flash_decode_attention

            cos = self.rope_cos[positions].unsqueeze(1)     # [B, 1, R/2]
            sin = self.rope_sin[positions].unsqueeze(1)
            q, k = _rotary(ops.rope.rotate, q, cos, sin), _rotary(ops.rope.rotate, k, cos, sin)
            self.kv.write_decode_sharded(layer_idx, k, v, positions, self.kv_rank)                  # owner-only write
            kc, vc = self.kv.stored(layer_idx) if scales is not None else self.kv.get(layer_idx)
            o = flash_decode_attention(q, kc, vc, positions, self.kv_group, sliding_window=sw, **scale_kw)
        else:
            # generation: W = S new tokens per sequence in cache slots p..p+W-1.  A chain puts token w at sequence position
            # p+w; a Medusa tree puts node w at p+depth[w], seeing only its ancestors inside the window
            # (ops.attention.speculation_attention).  One token (W = 1) is plain decode, whatever tree comes with it.
            tree_mask, depth = (None, None) if tree is None or S == 1 else tree
            fused = (q.is_cuda and q.dtype == torch.bfloat16 and scales is not None and self.kv.seq_shards == 1
                     and ops._ext.ext() is not None and hasattr(ops._ext.ext(), "decode_rope_kv"))
            if fused:
                # RoPE + cache append in one launch (csrc/decode.cu), then attention on the cache as stored
                ops._ext.count_launch()
                q = ops._ext.ext().decode_rope_kv(q, k, v, positions.to(torch.long).contiguous(), self.rope_cos, self.rope_sin,
                                                  self.kv.k[layer_idx], self.kv.v[layer_idx], depth=depth, **scale_kw, **roll)
                kc, vc = self.kv.stored(layer_idx, kv_len)
            else:
                d = torch.arange(S, device=q.device) if depth is None else depth
                idx = (positions.unsqueeze(1) + d.unsqueeze(0)).clamp(max=self.max_seq_len - 1)
                cos, sin = self.rope_cos[idx], self.rope_sin[idx]                 # [B, W, R/2]
                q, k = _rotary(ops.rope.rotate, q, cos, sin), _rotary(ops.rope.rotate, k, cos, sin)
                self.kv.write_window(layer_idx, k, v, positions)
                kc, vc = self.kv.get(layer_idx, kv_len)
                scale_kw = {}                                                     # kv.get de-quantised the cache
            if S == 1:
                o = ops.attention.decode_attention(q, kc, vc, positions, sliding_window=sw, **scale_kw, **roll)
            elif fused:
                o = ops.attention.speculation_attention(q, kc, vc, positions, tree_mask, depth, sw, **scale_kw, **roll)
            else:
                o = ops.attention.speculation_attention_torch(q, kc, vc, positions, tree_mask, depth, sw, **roll)
        return o

    def _tkg_block(self, layer_idx: int, layer):
        """Decode-time fused view of a MoE layer (shares its router / experts / norm; owns no parameters).  Kept outside the
        module tree so that state dicts and ``named_modules`` of the served model do not change."""
        blocks = self.__dict__.setdefault("_tkg_blocks", {})
        if layer_idx not in blocks:
            from ..modules.moe.moe_fused_tkg import MoEFusedTKG

            mlp = layer.mlp
            blocks[layer_idx] = MoEFusedTKG(mlp.router, mlp.expert_mlps, getattr(mlp, "shared_experts", None),
                                            layer.post_attention_layernorm, sequence_dimension=0,
                                            tensor_model_parallel_group=getattr(mlp, "tensor_parallel_group", None)).eval()
        return blocks[layer_idx]

    def _body(self, input_ids: torch.Tensor, positions: Optional[torch.Tensor], prefill: bool, kv_len: Optional[int], tree=None,
              prompt_lens: Optional[torch.Tensor] = None):
        if kv_len is not None and self.kv.rolling:
            raise ValueError("kv_len must be None with a rolling KV cache: a prefix of a ring holds no prefix of positions")
        core = self._core
        x = core.embed_tokens(input_ids).transpose(0, 1).contiguous()               # [S, B, H]
        for i, layer in enumerate(core.layers):
            x = self._attn_block(i, layer, x, positions, prefill, kv_len, tree, prompt_lens)
            mlp = layer.mlp
            if hasattr(mlp, "gate_up_proj") and hasattr(mlp, "down_proj") and not prefill and x.shape[0] * x.shape[1] <= 8:
                # dense decode MLP: the residual add rides in the down-projection's GEMV(+all-reduce) epilogue
                hmid = ops.act.swiglu(mlp.gate_up_proj(layer.post_attention_layernorm(x)))
                x = _row_linear_plus_residual(mlp.down_proj, hmid, x)
                continue
            if not prefill and x.shape[0] * x.shape[1] <= 8 and hasattr(mlp, "expert_mlps") and hasattr(mlp, "router"):
                # MoE decode: norm → router → top-k → chosen experts → weighted sum as ONE launch when the kernel applies
                # (modules/moe/moe_fused_tkg.py, csrc/moe_tkg.cu); otherwise the MoE layer's own dispatch below
                fused = self._tkg_block(i, layer)
                if fused._can_use_kernel(x):
                    x = x + fused(x)[0]
                    continue
            y = mlp(layer.post_attention_layernorm(x))
            x = x + (y[0] if isinstance(y, tuple) else y)                           # MoE blocks also return router logits
        return core.norm(x)

    # ------------------------------------------------------------------ entry points
    @torch.no_grad()
    def context_encoding(self, input_ids: torch.Tensor, last_token_index: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``input_ids`` [B, S_bucket] (right-padded) → next token ids [B] (or vocab-parallel logits)."""
        lens = None if last_token_index is None else last_token_index + 1        # a rolling cache keeps no right-padding
        h = self._body(input_ids, None, True, None, prompt_lens=lens)            # [S, B, H]
        B = input_ids.shape[0]
        if last_token_index is None:
            last = h[-1]
        else:
            last = h[last_token_index, torch.arange(B, device=h.device)]
        logits = self._logits(last.unsqueeze(0))[0].float()                   # [B, V/tp]
        return self.sampler.sample(logits) if self.on_device_sampling else logits

    @torch.no_grad()
    def token_generation(self, input_ids: torch.Tensor, positions: torch.Tensor, kv_len: Optional[int] = None) -> torch.Tensor:
        """``input_ids`` [B, 1], ``positions`` [B] → next token ids [B]."""
        h = self._body(input_ids, positions, False, kv_len)
        logits = self._logits(h)[0].float()
        return self.sampler.sample(logits) if self.on_device_sampling else logits

    @torch.no_grad()
    def speculation_forward(self, input_ids: torch.Tensor, positions: torch.Tensor, kv_len: Optional[int] = None,
                            tree_mask: Optional[torch.Tensor] = None, tree_depth: Optional[torch.Tensor] = None,
                            return_hidden: bool = False):
        """Verify a window: ``input_ids`` [B, W] placed at ``positions[b] .. positions[b]+W-1`` → greedy next token after
        each of the W positions, ``[B, W]`` (reference ``examples/inference`` speculation model, ``speculation_length``).
        With ``tree_mask [W, W]`` (True = node row sees node column) and ``tree_depth [W]`` the window is a Medusa candidate
        tree instead of a chain.  ``return_hidden`` also returns the final hidden states ``[B, W, H]`` (Medusa heads input)."""
        dev = input_ids.device
        tree = None if tree_mask is None else (tree_mask.to(dev, torch.bool).contiguous(), tree_depth.to(dev, torch.long).contiguous())
        h = self._body(input_ids, positions, False, kv_len, tree)                # [W, B, H]
        logits = self._logits(h).float()                                          # [W, B, V/tp]
        W, B = logits.shape[:2]
        out = self.sampler.sample(logits.reshape(W * B, -1)).view(W, B).t() if self.on_device_sampling else logits.transpose(0, 1)
        return (out, h.transpose(0, 1)) if return_hidden else out

    @torch.no_grad()
    def generate(self, prompt_ids: torch.Tensor, max_new_tokens: int, prompt_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        B, S = prompt_ids.shape
        lens = prompt_lens if prompt_lens is not None else torch.full((B,), S, device=prompt_ids.device, dtype=torch.long)
        tok = self.context_encoding(prompt_ids, lens - 1)
        out = [tok]
        pos = lens.clone()
        for _ in range(max_new_tokens - 1):
            tok = self.token_generation(tok.view(B, 1), pos)
            out.append(tok)
            pos = pos + 1
        return torch.stack(out, dim=1)


def _rotary(rot, x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """``rot`` (``ops.rope.apply_rotary`` / ``ops.rope.rotate``) on the first R = 2·cos.shape[-1] dims of x; the rest pass."""
    R = 2 * cos.shape[-1]
    if R == x.shape[-1]:
        return rot(x, cos, sin)
    return torch.cat([rot(x[..., :R].contiguous(), cos, sin), x[..., R:]], dim=-1)


def _row_linear_plus_residual(lin, inp: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
    """``residual + RowParallelLinear(inp)``.  At decode (<= 8 rows, bf16) this is ONE kernel: the GEMV with the bias and the
    residual in its epilogue (tp = 1) or, without a bias, the fused GEMV + in-switch all-reduce + residual (tp > 1,
    csrc/nvls_coll.cu)."""
    M = inp.numel() // inp.shape[-1]
    w = lin.weight
    bias = getattr(lin, "bias", None)
    e = ops._ext.ext() if inp.is_cuda else None
    if (e is not None and M <= 8 and inp.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
            and (bias is None or bias.dtype == torch.bfloat16) and not torch.is_grad_enabled() and getattr(lin, "reduce_output", True) and w.shape[1] % 8 == 0 and w.shape[0] % 8 == 0
            and not getattr(lin, "sequence_parallel_enabled", False)):
        x2 = inp.reshape(M, inp.shape[-1]).contiguous()
        r2 = residual.reshape(M, residual.shape[-1]).contiguous()
        tp = lin.tensor_model_parallel_size
        if tp == 1 and hasattr(e, "gemv") and x2.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0:   # 16-byte vector loads
            ops._ext.count_launch()
            return (e.gemv(x2, w, r2) if bias is None else e.gemv(x2, w, r2, bias=bias)).view_as(residual)
        if tp > 1 and bias is None and ops.tp_fused.get_backend() == "fused" and ops.nvls.gemv_all_reduce_eligible(x2, w):
            return ops.nvls.gemv_all_reduce(x2, w, lin.tensor_parallel_group, residual=r2).view_as(residual)
    return residual + lin(inp)
