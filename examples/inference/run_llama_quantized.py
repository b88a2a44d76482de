#!/usr/bin/env python
"""Weight-quantised Llama inference (int8 / fp8 per-tensor or per-channel, optional dynamic fp8 activations → the fp8 wgmma
GEMM) — counterpart of the reference's ``examples/inference/run_llama_quantized.py``.

  python examples/inference/run_llama_quantized.py --quantized_dtype f8e4m3 --quantization_type per_channel_symmetric --dynamic_activations
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "training"))

from neuronx_distributed_b200.models.llama import LlamaConfig, llama2_7b_config  # noqa: E402
from neuronx_distributed_b200.models.llama_inference import LlamaForInference  # noqa: E402
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, convert  # noqa: E402
from neuronx_distributed_b200.quantization.quantization_config import (  # noqa: E402
    get_default_per_channel_custom_qconfig_dict, get_default_per_tensor_custom_qconfig_dict)
from training_utils import init_distributed  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="tiny", choices=["tiny", "7b"])
    p.add_argument("--tp_degree", type=int, default=1)
    p.add_argument("--quantized_dtype", default="int8", choices=["int8", "f8e4m3"])
    p.add_argument("--quantization_type", default="per_channel_symmetric", choices=["per_tensor_symmetric", "per_channel_symmetric"])
    p.add_argument("--dynamic_activations", action="store_true")
    p.add_argument("--prompt_length", type=int, default=32)
    p.add_argument("--max_new_tokens", type=int, default=16)
    a = p.parse_args()
    dev = init_distributed()
    ps.initialize_model_parallel(tensor_model_parallel_size=a.tp_degree)
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    L = a.prompt_length + a.max_new_tokens
    kw = dict(dtype=dtype, device=dev, max_position_embeddings=L)
    cfg = llama2_7b_config(**kw) if a.model == "7b" else LlamaConfig(vocab_size=4096, hidden_size=256, intermediate_size=704,
                                                                    num_hidden_layers=4, num_attention_heads=8, **kw)
    torch.manual_seed(0)
    model = LlamaForInference(cfg, batch_size=1, max_seq_len=L).eval()
    prompt = torch.randint(0, cfg.vocab_size, (1, a.prompt_length), device=dev)
    ref = model.generate(prompt, a.max_new_tokens)
    q = (get_default_per_channel_custom_qconfig_dict() if a.quantization_type == "per_channel_symmetric"
         else get_default_per_tensor_custom_qconfig_dict())
    q["quantized_dtype"] = QuantizedDtype.F8E4M3 if a.quantized_dtype == "f8e4m3" else QuantizedDtype.INT8
    if a.dynamic_activations:
        q["activation_quantization_type"] = ActivationQuantizationType.DYNAMIC
    model.kv.reset()
    model.lm = convert(model.lm, q, inplace=True, modules_to_not_convert=["lm_head"])
    out = model.generate(prompt, a.max_new_tokens)
    nq = sum(1 for m in model.lm.modules() if type(m).__name__.startswith("Quantized"))
    if dist.get_rank() == 0:
        agree = (out == ref).float().mean().item()
        print(f"{nq} layers quantised to {a.quantized_dtype} ({a.quantization_type}); greedy tokens equal to bf16 run: {100 * agree:.0f} %",
              flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
