"""GPT-NeoX / Pythia inference model: the serving entry points of :class:`LlamaForInference` (context encoding, token
generation, speculation windows and Medusa trees, ``generate``, an fp8 KV cache) on :class:`GPTNeoXForCausalLM`, so training
checkpoints and HF checkpoints (``hf_compat.load_hf_checkpoint``) load unchanged.

What differs from Llama is the layer: LayerNorm, the per-head ``[q|k|v]`` fused QKV projection with a bias, partial rotary
(``rotary_pct``: only the first R = head_dim · rotary_pct dims of q and k rotate), biased dense / MLP projections with a GELU,
and the parallel residual.  RoPE, the cache write and attention are :meth:`LlamaForInference._attention`, which learns R from
the width of the rotary tables.  At decode (≤ 8 rows, bf16, CUDA) every projection is one GEMV launch with its bias, GELU
and residual in the epilogue (``csrc/decode.cu``); at tensor-parallel size > 1 the row-parallel layers add their bias after
the fused GEMV + all-reduce."""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops
from ..quantization.quantization_config import KVQuantizationConfig
from ..utils.sampling import Sampler
from .gpt_neox import GPTNeoXConfig, GPTNeoXForCausalLM
from .llama_inference import LlamaForInference, _row_linear_plus_residual


class GPTNeoXForInference(LlamaForInference):
    def __init__(self, cfg: GPTNeoXConfig, batch_size: int = 1, max_seq_len: int = 2048, on_device_sampling: bool = True,
                 sampler: Optional[Sampler] = None, flash_decoding: bool = False, kv_quant: Optional[KVQuantizationConfig] = None,
                 rolling_kv_cache: bool = False):
        """Arguments as :class:`LlamaForInference`.  ``rolling_kv_cache`` and ``flash_decoding`` raise ``ValueError``: GPT-NeoX
        has no sliding window, and its attention is multi-head, so no tensor-parallel rank holds a replicated KV head."""
        if rolling_kv_cache:
            raise ValueError("GPTNeoXForInference: rolling_kv_cache needs a sliding window, which GPT-NeoX does not have")
        if flash_decoding:
            raise ValueError("GPTNeoXForInference: flash_decoding needs replicated KV heads; GPT-NeoX attention is multi-head")
        rot = int(cfg.head_dim * cfg.rotary_pct)
        if rot < 2 or rot % 2:
            raise ValueError(f"GPTNeoXForInference: the rotary width head_dim · rotary_pct = {rot} must be even and >= 2")
        if cfg.hidden_act not in ops.gemm.GEMV_ACT:
            raise ValueError(f"GPTNeoXForInference: hidden_act {cfg.hidden_act!r} is not supported ({sorted(ops.gemm.GEMV_ACT)})")
        self.rotary_dim, self.act = rot, ops.gemm.GEMV_ACT[cfg.hidden_act]
        super().__init__(cfg, batch_size, max_seq_len, on_device_sampling, sampler, lm_cls=GPTNeoXForCausalLM, kv_quant=kv_quant)

    @property
    def _core(self):
        return self.lm.gpt_neox

    def _kv_heads_local(self) -> int:
        return self._core.layers[0].attention.heads_local

    def _rope_tables(self, max_seq_len: int):
        return ops.rope.rope_tables(max_seq_len, self.rotary_dim, self.cfg.rotary_emb_base, self.cfg.device)

    def _logits(self, h: torch.Tensor) -> torch.Tensor:
        return self.lm.embed_out(h)

    def _body(self, input_ids: torch.Tensor, positions: Optional[torch.Tensor], prefill: bool, kv_len: Optional[int], tree=None,
              prompt_lens: Optional[torch.Tensor] = None):
        core = self._core
        x = core.embed_in(input_ids).transpose(0, 1).contiguous()                    # [S, B, hidden]
        S, B = x.shape[:2]
        for i, layer in enumerate(core.layers):
            att, mlp = layer.attention, layer.mlp
            H, D = att.heads_local, att.head_dim
            # the fused output is head-major [h: (q, k, v)]; q / k / v are strided views of [B, S, H, 3D], no copies
            qkv = ops.gemm.linear_nt(layer.input_layernorm(x), att.query_key_value.weight, att.query_key_value.bias)
            q, k, v = qkv.view(S, B, H, 3 * D).transpose(0, 1).split(D, dim=-1)
            if prefill:                                                               # flash attention reads dense rows
                q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
            o = self._attention(i, q, k, v, positions, prefill, kv_len, tree, prompt_lens)
            a = _row_linear_plus_residual(att.dense, o.transpose(0, 1).reshape(S, B, H * D), x)              # x + attn
            # parallel residual: the MLP reads LayerNorm(x); sequential: LayerNorm(x + attn)
            hmid = ops.gemm.linear_nt(layer.post_attention_layernorm(x if layer.use_parallel_residual else a),
                                      mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.bias, self.act)
            x = _row_linear_plus_residual(mlp.dense_4h_to_h, hmid, a)
        return core.final_layer_norm(x)
