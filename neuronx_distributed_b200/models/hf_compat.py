"""HuggingFace interoperability for the built-in model families: build a config from an HF ``config.json``, translate
checkpoints between the HF parameter naming / layout and this package's, and load / save HF checkpoints directly into / from
a (TP, EP)-sharded model without an intermediate conversion run.

This is the in-process form of what the reference does with ``examples/training/*/convert_checkpoints.py`` +
``scripts/checkpoint_converter.py`` (HF full state → per-rank files → ``load_checkpoint``) and of the inference examples'
``modules/checkpoint.py`` + ``hf_adapter.py`` (``from_pretrained``): each rank reads the HF files (memory-mapped safetensors),
renames, and keeps only its own shard.

Layout differences handled here:

* decoder prefix: HF ``model.layers.N.…`` / ``lm_head`` ↔ ``layers.N.…`` / ``lm_head``;
* attention: HF ``q_proj / k_proj / v_proj`` ↔ ``qkv_proj.weight_{q,k,v}`` (the module's ``preshard_hook`` then replicates
  K/V ``kv_size_multiplier`` times and fuses per rank); with replicated KV heads in the *tile* layout the Q heads (and the
  ``o_proj`` columns) are permuted so each rank's Q heads sit next to the KV head they attend to
  (``scripts.checkpoint_converter.gqa_q_head_permutation``);
* dense MLP: HF ``gate_proj`` + ``up_proj`` ↔ one ``gate_up_proj`` ``[2I, H]`` (sharded with stride 2);
* Mixtral experts: HF ``block_sparse_moe.experts.E.{w1,w3,w2}`` ``[I,H] / [I,H] / [H,I]`` ↔ stacked, transposed
  ``expert_mlps.mlp_op.gate_up_proj [E, H, 2I]`` and ``down_proj [E, I, H]``; ``block_sparse_moe.gate`` ↔ ``router.linear_router``;
* DBRX: HF ``transformer.blocks.N.norm_attn_norm.{norm_1, attn.Wqkv, attn.out_proj, norm_2}``, ``ffn.router.layer`` and
  ``ffn.experts.mlp.{w1, v1, w2}`` (all experts concatenated along dim 0, ``w2`` stored ``[E·I, H]``) ↔ the same targets.
"""
from __future__ import annotations

import glob
import json
import os
import re
from typing import Any, Dict, Iterable, List, Optional

import torch
import torch.distributed as dist

from ..parallel_layers import parallel_state as ps
from ..scripts.checkpoint_converter import gqa_q_head_permutation

__all__ = ["config_from_hf", "hf_to_nxd_state_dict", "nxd_to_hf_state_dict", "hf_to_nxd_bert_state_dict", "nxd_to_hf_bert_state_dict",
           "hf_to_nxd_vit_state_dict", "nxd_to_hf_vit_state_dict", "read_hf_state_dict", "load_hf_checkpoint",
           "gather_full_state_dict", "save_hf_checkpoint"]


# ---------------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------------
def _as_dict(hf_config: Any) -> Dict[str, Any]:
    if isinstance(hf_config, (str, os.PathLike)):
        path = os.fspath(hf_config)
        if os.path.isdir(path):
            path = os.path.join(path, "config.json")
        with open(path) as f:
            return json.load(f)
    if isinstance(hf_config, dict):
        return dict(hf_config)
    return hf_config.to_dict() if hasattr(hf_config, "to_dict") else dict(vars(hf_config))


def _family(d: Dict[str, Any]) -> str:
    mt = str(d.get("model_type", "")).lower()
    if mt in ("mixtral", "dbrx", "gpt_neox"):
        return mt
    if mt in ("llama", "mistral", "qwen2", ""):
        return "llama"
    raise ValueError(f"unsupported HF model_type {mt!r} (llama / mistral / mixtral / dbrx / gpt_neox)")


def config_from_hf(hf_config: Any, **overrides):
    """``LlamaConfig`` / ``MixtralConfig`` / ``DbrxConfig`` / ``GPTNeoXConfig`` from an HF config object, dict, ``config.json``
    or model directory.  ``overrides`` (``dtype=…, device=…, sequence_parallel_enabled=…``) are applied last."""
    from .gpt_neox import GPTNeoXConfig
    from .llama import LlamaConfig
    from .mixtral import DbrxConfig, MixtralConfig

    d = _as_dict(hf_config)
    fam = _family(d)
    if fam == "gpt_neox":
        if d.get("tie_word_embeddings", False):
            raise ValueError("gpt_neox: tied word embeddings are not supported (embed_out is a separate weight)")
        # the rotary settings: rotary_pct / rotary_emb_base in Pythia / NeoX config.json files, rope_parameters
        # {partial_rotary_factor, rope_theta} in transformers >= 5
        rp = d.get("rope_parameters") or {}
        pct = next((v for v in (d.get("rotary_pct"), rp.get("partial_rotary_factor"), d.get("partial_rotary_factor")) if v is not None), None)
        base = next((v for v in (d.get("rotary_emb_base"), rp.get("rope_theta"), d.get("rope_theta")) if v is not None), None)
        kw = dict(vocab_size=d["vocab_size"], hidden_size=d["hidden_size"], intermediate_size=d["intermediate_size"],
                  num_hidden_layers=d["num_hidden_layers"], num_attention_heads=d["num_attention_heads"],
                  max_position_embeddings=d.get("max_position_embeddings"), layer_norm_eps=d.get("layer_norm_eps"),
                  use_parallel_residual=d.get("use_parallel_residual"), hidden_act=d.get("hidden_act"),
                  rotary_pct=None if pct is None else float(pct), rotary_emb_base=None if base is None else float(base))
        cls = GPTNeoXConfig
    elif fam == "dbrx":
        attn, ffn = d.get("attn_config", {}), d.get("ffn_config", {})
        kw = dict(vocab_size=d["vocab_size"], hidden_size=d["d_model"], intermediate_size=ffn["ffn_hidden_size"],
                  num_hidden_layers=d["n_layers"], num_attention_heads=d["n_heads"], num_key_value_heads=attn.get("kv_n_heads", d["n_heads"]),
                  max_position_embeddings=d.get("max_seq_len", 2048), rope_theta=float(attn.get("rope_theta", 10000.0)),
                  num_local_experts=ffn["moe_num_experts"], num_experts_per_tok=ffn["moe_top_k"], clip_qkv=attn.get("clip_qkv"))
        cls = DbrxConfig
    else:
        kw = dict(vocab_size=d["vocab_size"], hidden_size=d["hidden_size"], intermediate_size=d["intermediate_size"],
                  num_hidden_layers=d["num_hidden_layers"], num_attention_heads=d["num_attention_heads"],
                  num_key_value_heads=d.get("num_key_value_heads") or d["num_attention_heads"],
                  max_position_embeddings=d.get("max_position_embeddings", 4096), rms_norm_eps=d.get("rms_norm_eps", 1e-5),
                  tie_word_embeddings=bool(d.get("tie_word_embeddings", False)), pad_token_id=d.get("pad_token_id"))
        scaling = d.get("rope_parameters") or d.get("rope_scaling") or {}       # transformers>=5 keeps theta + scaling together
        kw["rope_theta"] = float(d.get("rope_theta") or scaling.get("rope_theta") or 10000.0)
        rope_type = scaling.get("type", scaling.get("rope_type"))
        if rope_type == "linear":
            kw["rope_scaling_factor"] = float(scaling["factor"])
        elif rope_type == "llama3":                  # Llama-3.1 / 3.2 frequency rescaling
            kw["rope_scaling"] = {k: scaling[k] for k in ("factor", "low_freq_factor", "high_freq_factor",
                                                          "original_max_position_embeddings")}
        # Qwen2 biases q / k / v (not o_proj)
        kw["qkv_bias"] = str(d.get("model_type", "")).lower() == "qwen2"
        cls = LlamaConfig
        if str(d.get("model_type", "")).lower() in ("mistral", "mixtral"):
            # Mistral / Mixtral attend within a sliding window (None: full attention).  Qwen2 carries the field too but
            # gates it with ``use_sliding_window`` and per-layer limits, so it is read for these two families only.
            kw["sliding_window"] = d.get("sliding_window")
        if fam == "mixtral":
            kw.update(num_local_experts=d["num_local_experts"], num_experts_per_tok=d["num_experts_per_tok"],
                      router_aux_loss_coef=d.get("router_aux_loss_coef", 0.02))
            cls = MixtralConfig
    dt = d.get("torch_dtype")
    if isinstance(dt, str) and hasattr(torch, dt):
        kw["dtype"] = getattr(torch, dt)
    fields = getattr(cls, "__dataclass_fields__", {})
    kw = {k: v for k, v in kw.items() if k in fields and v is not None}
    kw.update(overrides)
    return cls(**kw)


# ---------------------------------------------------------------------------------------------------------------------
# name / layout translation on FULL (unsharded) state dicts
# ---------------------------------------------------------------------------------------------------------------------
def _permute_heads(w: torch.Tensor, order: Iterable[int], head_dim: int, dim: int) -> torch.Tensor:
    shape = list(w.shape)
    v = w.reshape(*shape[:dim], shape[dim] // head_dim, head_dim, *shape[dim + 1:])
    return v.index_select(dim, torch.as_tensor(list(order))).reshape(shape)


def _q_order(cfg, kv_size_multiplier: int, layout: str) -> Optional[List[int]]:
    if kv_size_multiplier <= 1 or layout != "tile":
        return None
    order = gqa_q_head_permutation(cfg.num_attention_heads, cfg.num_key_value_heads, kv_size_multiplier, layout)
    return None if list(order) == list(range(len(order))) else list(order)


def _is_moe(cfg) -> bool:
    return hasattr(cfg, "num_local_experts")


def _dbrx_to_common(sd: Dict[str, torch.Tensor], cfg) -> Dict[str, torch.Tensor]:
    """HF DBRX names → the HF-Mixtral-like intermediate spelling used below."""
    E, inter, hid = cfg.num_local_experts, cfg.intermediate_size, cfg.hidden_size
    kv = cfg.num_key_value_heads * cfg.head_dim
    out: Dict[str, torch.Tensor] = {}
    for k, v in sd.items():
        m = re.match(r"^transformer\.blocks\.(\d+)\.(.*)$", k)
        if m is None:
            out[{"transformer.wte.weight": "model.embed_tokens.weight", "transformer.norm_f.weight": "model.norm.weight"}.get(k, k)] = v
            continue
        base, rest = f"model.layers.{m.group(1)}.", m.group(2)
        if rest == "norm_attn_norm.norm_1.weight":
            out[base + "input_layernorm.weight"] = v
        elif rest == "norm_attn_norm.norm_2.weight":
            out[base + "post_attention_layernorm.weight"] = v
        elif rest == "norm_attn_norm.attn.Wqkv.weight":
            q, kk, vv = torch.split(v, [hid, kv, kv], 0)
            out[base + "self_attn.q_proj.weight"], out[base + "self_attn.k_proj.weight"], out[base + "self_attn.v_proj.weight"] = q, kk, vv
        elif rest == "norm_attn_norm.attn.out_proj.weight":
            out[base + "self_attn.o_proj.weight"] = v
        elif rest == "ffn.router.layer.weight":
            out[base + "block_sparse_moe.gate.weight"] = v
        elif rest in ("ffn.experts.mlp.w1", "ffn.experts.mlp.v1", "ffn.experts.mlp.w2"):
            per = v.reshape(E, inter, hid)
            name = {"w1": "w1", "v1": "w3", "w2": "w2"}[rest.rsplit(".", 1)[1]]
            for e in range(E):                       # DBRX stores w2 as [I, H] per expert; HF-Mixtral w2 is [H, I]
                out[base + f"block_sparse_moe.experts.{e}.{name}.weight"] = per[e].t() if name == "w2" else per[e]
        else:
            out[base + rest] = v
    return out


def _common_to_dbrx(sd: Dict[str, torch.Tensor], cfg) -> Dict[str, torch.Tensor]:
    E = cfg.num_local_experts
    out: Dict[str, torch.Tensor] = {}
    layers: Dict[str, Dict[str, torch.Tensor]] = {}
    for k, v in sd.items():
        m = re.match(r"^model\.layers\.(\d+)\.(.*)$", k)
        if m is None:
            out[{"model.embed_tokens.weight": "transformer.wte.weight", "model.norm.weight": "transformer.norm_f.weight"}.get(k, k)] = v
        else:
            layers.setdefault(m.group(1), {})[m.group(2)] = v
    for i, t in layers.items():
        b = f"transformer.blocks.{i}."
        out[b + "norm_attn_norm.norm_1.weight"] = t.pop("input_layernorm.weight")
        out[b + "norm_attn_norm.norm_2.weight"] = t.pop("post_attention_layernorm.weight")
        out[b + "norm_attn_norm.attn.Wqkv.weight"] = torch.cat([t.pop("self_attn.q_proj.weight"), t.pop("self_attn.k_proj.weight"),
                                                               t.pop("self_attn.v_proj.weight")], 0)
        out[b + "norm_attn_norm.attn.out_proj.weight"] = t.pop("self_attn.o_proj.weight")
        out[b + "ffn.router.layer.weight"] = t.pop("block_sparse_moe.gate.weight")
        for src, dst in (("w1", "w1"), ("w3", "v1"), ("w2", "w2")):
            per = [t.pop(f"block_sparse_moe.experts.{e}.{src}.weight") for e in range(E)]
            out[b + f"ffn.experts.mlp.{dst}"] = torch.cat([p.t() if src == "w2" else p for p in per], 0).contiguous()
        for rest, v in t.items():
            out[b + rest] = v
    return out


def hf_to_nxd_state_dict(hf_sd: Dict[str, torch.Tensor], cfg, kv_size_multiplier: int = 1, kv_replication_layout: str = "tile",
                         prefix: str = "") -> Dict[str, torch.Tensor]:
    """Full HF state → full state in this package's names (``qkv_proj.weight_{q,k,v}`` un-replicated: the module's preshard
    hook replicates / fuses; everything else is exactly what ``inference.sharding.shard_state_dict_for_rank`` slices).
    ``prefix`` is prepended to every key (``"lm."`` for the serving wrappers)."""
    sd = _dbrx_to_common(hf_sd, cfg) if any(k.startswith("transformer.blocks.") for k in hf_sd) else hf_sd
    order = _q_order(cfg, kv_size_multiplier, kv_replication_layout)
    hd = cfg.head_dim
    out: Dict[str, torch.Tensor] = {}
    experts: Dict[str, Dict[int, Dict[str, torch.Tensor]]] = {}
    for k, v in sd.items():
        if k.endswith("rotary_emb.inv_freq"):
            continue
        name = k[len("model."):] if k.startswith("model.") else k
        m = re.match(r"^(layers\.\d+\.)block_sparse_moe\.experts\.(\d+)\.(w1|w2|w3)\.weight$", name)
        if m is not None:
            experts.setdefault(m.group(1), {}).setdefault(int(m.group(2)), {})[m.group(3)] = v
            continue
        name = name.replace("block_sparse_moe.gate.weight", "mlp.router.linear_router.weight")
        if _is_moe(cfg):                              # transformers>=5 in-memory spelling: fused 3-D expert parameters
            if name.endswith("mlp.gate.weight"):
                name = name[: -len("gate.weight")] + "router.linear_router.weight"
            elif name.endswith("mlp.experts.gate_up_proj"):          # [E, 2I, H] → [E, H, 2I]
                name, v = name[: -len("experts.gate_up_proj")] + "expert_mlps.mlp_op.gate_up_proj.weight", v.transpose(1, 2).contiguous()
            elif name.endswith("mlp.experts.down_proj"):             # [E, H, I] → [E, I, H]
                name, v = name[: -len("experts.down_proj")] + "expert_mlps.mlp_op.down_proj.weight", v.transpose(1, 2).contiguous()
        for p in ("q", "k", "v"):
            for kind in ("weight", "bias"):
                name = name.replace(f"self_attn.{p}_proj.{kind}", f"self_attn.qkv_proj.{kind}_{p}")
        if order is not None:
            if name.endswith(("qkv_proj.weight_q", "qkv_proj.bias_q")):
                v = _permute_heads(v, order, hd, 0)
            elif name.endswith("self_attn.o_proj.weight"):
                v = _permute_heads(v, order, hd, 1)
        out[name] = v
    for k in [k for k in out if k.endswith("mlp.gate_proj.weight")]:          # dense MLP: [gate; up] fused along dim 0
        base = k[: -len("gate_proj.weight")]
        out[base + "gate_up_proj.weight"] = torch.cat([out.pop(k), out.pop(base + "up_proj.weight")], 0)
    for base, per in experts.items():                                         # experts: stacked, input-major
        ids = sorted(per)
        out[base + "mlp.expert_mlps.mlp_op.gate_up_proj.weight"] = torch.stack(
            [torch.cat([per[e]["w1"].t(), per[e]["w3"].t()], 1) for e in ids]).contiguous()
        out[base + "mlp.expert_mlps.mlp_op.down_proj.weight"] = torch.stack([per[e]["w2"].t() for e in ids]).contiguous()
    if getattr(cfg, "tie_word_embeddings", False) and "lm_head.weight" not in out and "embed_tokens.weight" in out:
        out["lm_head.weight"] = out["embed_tokens.weight"]
    return {prefix + k: v for k, v in out.items()} if prefix else out


def nxd_to_hf_state_dict(full_sd: Dict[str, torch.Tensor], cfg, kv_size_multiplier: int = 1, kv_replication_layout: str = "tile",
                         style: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """Inverse of :func:`hf_to_nxd_state_dict` on a gathered full state (``weight_qkv`` fused tensors are accepted in the
    *un-replicated* ``[Q; K; V]`` order :func:`gather_full_state_dict` produces).  ``style``: ``None`` — the on-disk HF
    spelling (per-expert ``block_sparse_moe.experts.E.w{1,2,3}``); ``"fused_experts"`` — the 3-D ``mlp.experts.*`` parameters
    transformers ≥ 5 keeps in memory; ``"dbrx"`` — DBRX names."""
    fused_experts = (style or "").lower() == "fused_experts"
    order = _q_order(cfg, kv_size_multiplier, kv_replication_layout)
    inv = sorted(range(len(order)), key=order.__getitem__) if order is not None else None
    hd, qs, kvs = cfg.head_dim, cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
    out: Dict[str, torch.Tensor] = {}
    for k, v in full_sd.items():
        name = k if k.startswith("lm_head.") else "model." + k
        if k.endswith("qkv_proj.weight_qkv") or k.endswith("qkv_proj.bias_qkv"):
            kind = "weight" if k.endswith("weight_qkv") else "bias"
            base = name[: -len(f"qkv_proj.{kind}_qkv")]
            q, kk, vv = torch.split(v, [qs, kvs, kvs], 0)
            if inv is not None:
                q = _permute_heads(q, inv, hd, 0)
            out[base + f"q_proj.{kind}"], out[base + f"k_proj.{kind}"], out[base + f"v_proj.{kind}"] = q, kk, vv
        elif re.search(r"qkv_proj\.(weight|bias)_(q|k|v)$", k):
            kind, p = re.search(r"qkv_proj\.(weight|bias)_(q|k|v)$", k).groups()
            if p == "q" and inv is not None:
                v = _permute_heads(v, inv, hd, 0)
            out[name[: name.rfind("qkv_proj.")] + f"{p}_proj.{kind}"] = v
        elif k.endswith("self_attn.o_proj.weight"):
            out[name] = _permute_heads(v, inv, hd, 1) if inv is not None else v
        elif fused_experts and k.endswith(("mlp.expert_mlps.mlp_op.gate_up_proj.weight", "mlp.expert_mlps.mlp_op.down_proj.weight")):
            which = "gate_up_proj" if k.endswith("gate_up_proj.weight") else "down_proj"
            out[name[: name.rfind("expert_mlps.")] + f"experts.{which}"] = v.transpose(1, 2).contiguous()
        elif fused_experts and k.endswith("mlp.router.linear_router.weight"):
            out[name.replace("mlp.router.linear_router.weight", "mlp.gate.weight")] = v
        elif k.endswith("mlp.expert_mlps.mlp_op.gate_up_proj.weight"):
            base = name[: -len("mlp.expert_mlps.mlp_op.gate_up_proj.weight")] + "block_sparse_moe.experts."
            for e in range(v.shape[0]):
                g, u = v[e].chunk(2, dim=1)
                out[f"{base}{e}.w1.weight"], out[f"{base}{e}.w3.weight"] = g.t().contiguous(), u.t().contiguous()
        elif k.endswith("mlp.expert_mlps.mlp_op.down_proj.weight"):
            base = name[: -len("mlp.expert_mlps.mlp_op.down_proj.weight")] + "block_sparse_moe.experts."
            for e in range(v.shape[0]):
                out[f"{base}{e}.w2.weight"] = v[e].t().contiguous()
        elif k.endswith("mlp.router.linear_router.weight"):
            out[name.replace("mlp.router.linear_router.weight", "block_sparse_moe.gate.weight")] = v
        elif k.endswith("mlp.gate_up_proj.weight"):
            g, u = v.chunk(2, dim=0)
            base = name[: -len("gate_up_proj.weight")]
            out[base + "gate_proj.weight"], out[base + "up_proj.weight"] = g, u
        else:
            out[name] = v
    if getattr(cfg, "tie_word_embeddings", False):
        out.pop("lm_head.weight", None)
    if (style or "").lower() == "dbrx":
        out = _common_to_dbrx(out, cfg)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# encoder families (BERT, ViT) and GPT-NeoX: pure renames + QKV fusion; GPT-NeoX already uses the HF names and layout
# ---------------------------------------------------------------------------------------------------------------------
_BERT_RENAMES = [
    (r"^bert\.encoder\.layer\.(\d+)\.attention\.self\.(query|key|value)\.", r"bert.layers.\1.attention.\2."),
    (r"^bert\.encoder\.layer\.(\d+)\.attention\.output\.dense\.", r"bert.layers.\1.attention.dense."),
    (r"^bert\.encoder\.layer\.(\d+)\.attention\.output\.LayerNorm\.", r"bert.layers.\1.attention_norm."),
    (r"^bert\.encoder\.layer\.(\d+)\.intermediate\.dense\.", r"bert.layers.\1.intermediate."),
    (r"^bert\.encoder\.layer\.(\d+)\.output\.dense\.", r"bert.layers.\1.output."),
    (r"^bert\.encoder\.layer\.(\d+)\.output\.LayerNorm\.", r"bert.layers.\1.output_norm."),
    (r"^bert\.pooler\.dense\.", "bert.pooler."),
    (r"^cls\.predictions\.transform\.dense\.", "transform."),
    (r"^cls\.predictions\.transform\.LayerNorm\.", "transform_norm."),
    (r"^cls\.predictions\.decoder\.", "decoder."),
    (r"^cls\.seq_relationship\.", "seq_relationship."),
]
_BERT_INVERSE = [
    (r"^bert\.layers\.(\d+)\.attention\.(query|key|value)\.", r"bert.encoder.layer.\1.attention.self.\2."),
    (r"^bert\.layers\.(\d+)\.attention\.dense\.", r"bert.encoder.layer.\1.attention.output.dense."),
    (r"^bert\.layers\.(\d+)\.attention_norm\.", r"bert.encoder.layer.\1.attention.output.LayerNorm."),
    (r"^bert\.layers\.(\d+)\.intermediate\.", r"bert.encoder.layer.\1.intermediate.dense."),
    (r"^bert\.layers\.(\d+)\.output\.", r"bert.encoder.layer.\1.output.dense."),
    (r"^bert\.layers\.(\d+)\.output_norm\.", r"bert.encoder.layer.\1.output.LayerNorm."),
    (r"^bert\.pooler\.", "bert.pooler.dense."),
    (r"^transform\.", "cls.predictions.transform.dense."),
    (r"^transform_norm\.", "cls.predictions.transform.LayerNorm."),
    (r"^decoder\.", "cls.predictions.decoder."),
    (r"^seq_relationship\.", "cls.seq_relationship."),
]


def _rename(sd: Dict[str, torch.Tensor], rules) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in sd.items():
        for pat, rep in rules:
            k2, n = re.subn(pat, rep, k)
            if n:
                k = k2
                break
        out[k] = v
    return out


def hf_to_nxd_bert_state_dict(hf_sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """HF ``BertForPreTraining`` names → ``models.bert.BertForPreTraining`` (same tensors; ``cls.predictions.bias`` is the
    decoder bias; ``position_ids`` buffers are dropped)."""
    out = _rename({k: v for k, v in hf_sd.items() if not k.endswith("position_ids")}, _BERT_RENAMES)
    if "cls.predictions.bias" in out:
        out.setdefault("decoder.bias", out["cls.predictions.bias"])
        del out["cls.predictions.bias"]
    out.setdefault("decoder.weight", out.get("bert.embeddings.word_embeddings.weight"))
    return out


def nxd_to_hf_bert_state_dict(full_sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    out = _rename(full_sd, _BERT_INVERSE)
    if "cls.predictions.decoder.bias" in out:
        out["cls.predictions.bias"] = out["cls.predictions.decoder.bias"]
    return out


def hf_to_nxd_vit_state_dict(hf_sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """HF ``ViTForImageClassification`` names → ``models.vit`` (query / key / value fused to one ``qkv`` ``[q; k; v]``,
    sharded with stride 3)."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in hf_sd.items():
        k = k[len("vit."):] if k.startswith("vit.") else k
        k = k.replace("embeddings.patch_embeddings.projection.", "embeddings.projection.")
        k = re.sub(r"^encoder\.layer\.(\d+)\.", r"layers.\1.", k)
        k = k.replace("attention.output.dense.", "out.").replace("intermediate.dense.", "fc1.").replace("output.dense.", "fc2.")
        out[k] = v
    for k in [k for k in out if k.endswith("attention.attention.query.weight")]:
        base = k[: -len("attention.attention.query.weight")]
        for kind in ("weight", "bias"):
            parts = [out.pop(f"{base}attention.attention.{p}.{kind}", None) for p in ("query", "key", "value")]
            if parts[0] is not None:
                out[f"{base}qkv.{kind}"] = torch.cat(parts, 0)
    return out


def nxd_to_hf_vit_state_dict(full_sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    out: Dict[str, torch.Tensor] = {}
    for k, v in full_sd.items():
        m = re.match(r"^layers\.(\d+)\.(.*)$", k)
        if m is None:
            k2 = k if k.startswith("classifier.") else "vit." + k.replace("embeddings.projection.", "embeddings.patch_embeddings.projection.")
            out[k2] = v
            continue
        base, rest = f"vit.encoder.layer.{m.group(1)}.", m.group(2)
        if rest.startswith("qkv."):
            kind = rest.split(".", 1)[1]
            for p, t in zip(("query", "key", "value"), v.chunk(3, 0)):
                out[f"{base}attention.attention.{p}.{kind}"] = t
        else:
            rest = rest.replace("out.", "attention.output.dense.", 1) if rest.startswith("out.") else rest
            rest = rest.replace("fc1.", "intermediate.dense.", 1) if rest.startswith("fc1.") else rest
            rest = rest.replace("fc2.", "output.dense.", 1) if rest.startswith("fc2.") else rest
            out[base + rest] = v
    return out


def _encoder_family(model) -> Optional[str]:
    name = type(model).__name__.lower()
    for fam in ("bert", "vit", "gptneox"):
        if fam in name.replace("_", ""):
            return fam
    return None


# ---------------------------------------------------------------------------------------------------------------------
# files
# ---------------------------------------------------------------------------------------------------------------------
def read_hf_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """All tensors of an HF checkpoint directory (``*.safetensors`` — memory-mapped, sharded or not — else
    ``pytorch_model*.bin``) or of a single file."""
    files: List[str]
    if os.path.isdir(path):
        files = sorted(glob.glob(os.path.join(path, "*.safetensors"))) or sorted(glob.glob(os.path.join(path, "pytorch_model*.bin")))
        if not files:
            raise FileNotFoundError(f"no *.safetensors / pytorch_model*.bin under {path}")
    else:
        files = [path]
    sd: Dict[str, torch.Tensor] = {}
    for f in files:
        if f.endswith(".safetensors"):
            from safetensors import safe_open

            with safe_open(f, framework="pt", device="cpu") as h:
                for k in h.keys():
                    sd[k] = h.get_tensor(k)
        else:
            sd.update(torch.load(f, map_location="cpu", weights_only=True, mmap=True))
    return sd


def _kv_args(model) -> Dict[str, Any]:
    from ..modules.qkv_linear import GQAQKVColumnParallelLinear

    for m in model.modules():
        if isinstance(m, GQAQKVColumnParallelLinear):
            return {"kv_size_multiplier": m.kv_size_multiplier, "kv_replication_layout": m.kv_replication_layout}
    return {"kv_size_multiplier": 1, "kv_replication_layout": "tile"}


def _layout(model):
    """``(root, decoder_prefix, head_prefix)``: the module to load into (serving wrappers keep the LM under ``.lm``), the
    state-dict prefix of its decoder stack (the module owning ``embed_tokens`` and ``layers``) and of its ``lm_head``."""
    root = model.lm if isinstance(getattr(model, "lm", None), torch.nn.Module) else model
    dec = head = None
    for prefix, m in root.named_modules():
        if dec is None and hasattr(m, "embed_tokens") and hasattr(m, "layers"):
            dec = prefix + "." if prefix else ""
        if head is None and (prefix == "lm_head" or prefix.endswith(".lm_head")):
            head = prefix + "."
    if dec is None:
        raise ValueError("model has no decoder with embed_tokens / layers")
    return root, dec, head


def _config_of(model, root):
    for m in (root, model, *root.children()):
        for attr in ("config", "cfg"):
            c = getattr(m, attr, None)
            if c is not None and hasattr(c, "num_attention_heads"):
                return c
    raise ValueError("pass cfg= (the model does not expose its config)")


def _to_model_keys(canon: Dict[str, torch.Tensor], dec: str, head: Optional[str]) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in canon.items():
        if k.startswith("lm_head."):
            if head is not None:
                out[head + k[len("lm_head."):]] = v
        else:
            out[dec + k] = v
    return out


def _to_canonical_key(k: str, dec: str, head: Optional[str]) -> Optional[str]:
    if head is not None and k.startswith(head):
        return "lm_head." + k[len(head):]
    return k[len(dec):] if k.startswith(dec) else None


def _unwrap(model):
    """``(module, pipeline_model)``: strips the trainer's ``NxDModel`` wrapper; for a pipeline-partitioned model returns the
    original (un-partitioned) module — whose local layers share their Parameters with the stage modules — and the
    ``NxDPPModel`` that owns the partition."""
    from ..pipeline.model import NxDPPModel
    from ..trainer.model import NxDModel

    if isinstance(model, NxDModel):
        model = model.module
    if isinstance(model, NxDPPModel):
        return model.original_torch_module, model
    return model, None


def _load_into_pipeline_stage(pp, original, hf_sd, cfg, strict: bool):
    """Each (tp, pp) rank keeps the tensors of ITS stage only: the translated full state is filtered to the modules that own
    a local parameter before any slicing happens."""
    from ..inference.sharding import shard_state_dict_for_rank

    root, dec, head = _layout(original)
    cfg = cfg or _config_of(original, root)
    full = _to_model_keys(hf_to_nxd_state_dict(hf_sd, cfg, **_kv_args(root)), dec, head)
    local_names = set(pp.original_name_to_local_name)
    local_mods = {n.rpartition(".")[0] for n in local_names}
    full = {k: v for k, v in full.items() if k in local_names or k.rpartition(".")[0] in local_mods}
    local = shard_state_dict_for_rank(root, full, ps.get_tensor_model_parallel_rank(), ps.get_tensor_model_parallel_size())
    want = pp.local_state_dict()
    missing = [k for k in want if k not in local]
    if strict and missing:
        raise RuntimeError(f"HF checkpoint lacks tensors for local parameters: {missing[:8]}")
    local = {k: (v.to(want[k].dtype) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in local.items() if k in want}
    pp.load_state_dict(local, strict=False)
    return torch.nn.modules.module._IncompatibleKeys(missing, [])


def load_hf_checkpoint(model, path_or_state, cfg=None, strict: bool = True):
    """Load an HF checkpoint (directory, file or state dict) into ``model`` — a ``LlamaForCausalLM`` / ``MixtralForCausalLM`` /
    serving wrapper built under the current TP (and EP) groups; every rank slices its own shard.  Returns the
    ``load_state_dict`` result."""
    from ..inference.sharding import shard_state_dict_for_rank

    hf_sd = path_or_state if isinstance(path_or_state, dict) else read_hf_state_dict(os.fspath(path_or_state))
    model, pp = _unwrap(model)
    if pp is not None:
        return _load_into_pipeline_stage(pp, model, hf_sd, cfg, strict)
    fam = _encoder_family(model)
    if fam is not None:                               # BERT / ViT: renames (+ QKV fusion); GPT-NeoX: HF names as they are
        model = model.lm if isinstance(getattr(model, "lm", None), torch.nn.Module) else model   # serving wrapper
        full = {"bert": hf_to_nxd_bert_state_dict, "vit": hf_to_nxd_vit_state_dict, "gptneox": dict}[fam](hf_sd)
        full = {k: v for k, v in full.items() if not k.endswith(("rotary_emb.inv_freq", "attention.bias", "attention.masked_bias"))}
        want = model.state_dict()
        local = shard_state_dict_for_rank(model, full, ps.get_tensor_model_parallel_rank(), ps.get_tensor_model_parallel_size())
        local = {k: (v.to(want[k].dtype) if k in want and isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in local.items()}
        return model.load_state_dict(local, strict=strict)
    root, dec, head = _layout(model)
    cfg = cfg or _config_of(model, root)
    full = _to_model_keys(hf_to_nxd_state_dict(hf_sd, cfg, **_kv_args(root)), dec, head)
    rank, world = ps.get_tensor_model_parallel_rank(), ps.get_tensor_model_parallel_size()
    local = shard_state_dict_for_rank(root, full, rank, world)
    want = root.state_dict()
    local = {k: (v.to(want[k].dtype) if k in want and isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in local.items()}
    return root.load_state_dict(local, strict=strict)


def gather_full_state_dict(model, group=None) -> Dict[str, torch.Tensor]:
    """All-gather every TP-sharded parameter of ``model`` over the TP group into its full, *un-replicated* tensor (fused
    ``weight_qkv`` → ``[Q; K; V]`` with the KV replicas dropped; strided ``gate_up`` → ``[gate; up]``).  Collective: call on
    all TP ranks; every rank returns the full CPU state (EP-sharded experts are gathered over the EP group as well)."""
    from ..parallel_layers.utils import gather_full_weight

    root, dec, head = _layout(model)
    group = group if group is not None else ps.get_tensor_model_parallel_group()
    tp = dist.get_world_size(group)
    out: Dict[str, torch.Tensor] = {}
    for key, p in root.state_dict(keep_vars=True).items():
        name = _to_canonical_key(key, dec, head)
        if name is None:
            continue
        t = p.detach()
        if not getattr(p, "tensor_model_parallel", False) or tp == 1:
            full = t
        else:
            shards = [torch.empty_like(t) for _ in range(tp)]
            dist.all_gather(shards, t.contiguous(), group=group)
            if getattr(p, "fused_qkv", False):
                qs, ks, _ = p.qkv_sections                              # full sizes incl. replication
                qp, kp = qs // tp, ks // tp
                q = torch.cat([s[:qp] for s in shards], 0)
                k = torch.cat([s[qp:qp + kp] for s in shards], 0)
                v = torch.cat([s[qp + kp:] for s in shards], 0)
                mult = getattr(p, "kv_size_multiplier", None)
                full = (q, k, v, mult)
            else:
                full = gather_full_weight(shards, p.partition_dim, getattr(p, "partition_stride", 1))
        if getattr(p, "expert_model_parallel", False) and ps.get_expert_model_parallel_size() > 1 and not isinstance(full, tuple):
            eg = ps.get_expert_model_parallel_group()
            parts = [torch.empty_like(full) for _ in range(dist.get_world_size(eg))]
            dist.all_gather(parts, full.contiguous(), group=eg)
            full = torch.cat(parts, 0)
        out[name] = full
    kv = _kv_args(root)
    mult, layout = kv["kv_size_multiplier"], kv["kv_replication_layout"]
    hd = _config_of(model, root).head_dim
    for name, full in list(out.items()):
        if isinstance(full, tuple):
            q, k, v, _ = full
            if mult > 1:
                if layout == "tile":
                    k, v = k[: k.shape[0] // mult], v[: v.shape[0] // mult]
                else:
                    sel = torch.arange(0, k.shape[0] // hd, mult, device=k.device)
                    k, v = (t.reshape(-1, hd, *t.shape[1:])[sel].reshape(-1, *t.shape[1:]) for t in (k, v))
            out[name] = torch.cat([q, k, v], 0)
        elif mult > 1 and re.search(r"qkv_proj\.(weight|bias)_(k|v)$", name):
            t = full
            if layout == "tile":
                out[name] = t[: t.shape[0] // mult]
            else:
                sel = torch.arange(0, t.shape[0] // hd, mult, device=t.device)
                out[name] = t.reshape(-1, hd, *t.shape[1:])[sel].reshape(-1, *t.shape[1:])
    return {k: v.cpu() for k, v in out.items()}


def save_hf_checkpoint(model, path: str, cfg=None, hf_config: Optional[Dict[str, Any]] = None, style: Optional[str] = None,
                       max_shard_bytes: int = 5 << 30) -> None:
    """Write ``model`` as an HF checkpoint directory (``model-0000x-of-0000y.safetensors`` + index, and ``config.json`` when
    ``hf_config`` is given).  Collective over the TP group; the global rank-0 process writes."""
    root, _, _ = _layout(model)
    cfg = cfg or _config_of(model, root)
    full = gather_full_state_dict(model)
    if dist.is_initialized() and dist.get_rank() != 0:
        dist.barrier()
        return
    hf = nxd_to_hf_state_dict(full, cfg, style=style, **_kv_args(root))
    os.makedirs(path, exist_ok=True)
    from safetensors.torch import save_file

    shards: List[Dict[str, torch.Tensor]] = [{}]
    size = 0
    for k, v in hf.items():
        n = v.numel() * v.element_size()
        if size + n > max_shard_bytes and shards[-1]:
            shards.append({})
            size = 0
        shards[-1][k] = v.contiguous().clone()
        size += n
    index = {"metadata": {"total_size": sum(v.numel() * v.element_size() for v in hf.values())}, "weight_map": {}}
    for i, shard in enumerate(shards):
        fname = "model.safetensors" if len(shards) == 1 else f"model-{i + 1:05d}-of-{len(shards):05d}.safetensors"
        save_file(shard, os.path.join(path, fname), metadata={"format": "pt"})
        index["weight_map"].update({k: fname for k in shard})
    if len(shards) > 1:
        with open(os.path.join(path, "model.safetensors.index.json"), "w") as f:
            json.dump(index, f, indent=1)
    if hf_config is not None:
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(_as_dict(hf_config), f, indent=1, default=str)
    if dist.is_initialized():
        dist.barrier()
