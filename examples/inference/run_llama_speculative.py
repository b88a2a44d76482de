#!/usr/bin/env python
"""Speculative decoding: a small draft Llama proposes ``--speculation_length`` tokens, the target verifies the window in one
forward — counterpart of the reference's ``examples/inference/run_llama_speculative.py``.

  python examples/inference/run_llama_speculative.py --model tiny --speculation_length 4
  python examples/inference/run_llama_speculative.py --model 7b --kv_cache_quant fp8
  torchrun --nproc-per-node 8 examples/inference/run_llama_speculative.py --model 13b --draft_layers 4 --tp_degree 8
"""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "training"))

from neuronx_distributed_b200.models.llama import LlamaConfig, llama2_13b_config, llama2_7b_config  # noqa: E402
from neuronx_distributed_b200.models.llama_inference import LlamaForInference  # noqa: E402
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from neuronx_distributed_b200.quantization import KVQuantizationConfig  # noqa: E402
from neuronx_distributed_b200.utils.speculative import speculative_generate  # noqa: E402
from training_utils import init_distributed  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="tiny", choices=["tiny", "7b", "13b"])
    p.add_argument("--draft_layers", type=int, default=1, help="the draft is the same architecture with this many layers")
    p.add_argument("--tp_degree", type=int, default=1)
    p.add_argument("--prompt_length", type=int, default=32)
    p.add_argument("--max_new_tokens", type=int, default=32)
    p.add_argument("--speculation_length", type=int, default=4)
    p.add_argument("--kv_cache_quant", default="none", choices=["none", "fp8"],
                   help="fp8: store both models' KV caches in float8 e4m3 with one scale per tensor (--kv_cache_scale)")
    p.add_argument("--kv_cache_scale", type=float, default=1.0, help="the cache stores k / scale and v / scale")
    a = p.parse_args()
    dev = init_distributed()
    ps.initialize_model_parallel(tensor_model_parallel_size=a.tp_degree)
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    L = a.prompt_length + a.max_new_tokens + a.speculation_length + 1
    kw = dict(dtype=dtype, device=dev, max_position_embeddings=L)
    mk = {"7b": llama2_7b_config, "13b": llama2_13b_config}.get(a.model, lambda **k: LlamaConfig(
        vocab_size=4096, hidden_size=256, intermediate_size=704, num_hidden_layers=4, num_attention_heads=8, **k))
    kv_quant = None
    if a.kv_cache_quant == "fp8":
        kv_quant = KVQuantizationConfig(quant_dtype=torch.float8_e4m3fn, dequant_dtype=dtype, scale=a.kv_cache_scale)
    torch.manual_seed(0)
    target = LlamaForInference(mk(**kw), batch_size=1, max_seq_len=L, kv_quant=kv_quant).eval()
    dcfg = mk(**kw)
    dcfg.num_hidden_layers = a.draft_layers
    torch.manual_seed(0)        # same seed: the draft's layers start as a prefix of the target's (a crude "distilled" draft)
    draft = LlamaForInference(dcfg, batch_size=1, max_seq_len=L, kv_quant=kv_quant).eval()
    prompt = torch.randint(0, target.cfg.vocab_size, (1, a.prompt_length), device=dev)
    t0 = time.perf_counter()
    ref = target.generate(prompt, a.max_new_tokens)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    t1 = time.perf_counter()
    target.kv.reset()
    verify_s = []                 # wall time of each target verification forward (one per round), device work included
    forward = target.speculation_forward

    def timed_forward(*args, **kwargs):
        if dev.type == "cuda":
            torch.cuda.synchronize()
        t = time.perf_counter()
        out = forward(*args, **kwargs)
        if dev.type == "cuda":
            torch.cuda.synchronize()
        verify_s.append(time.perf_counter() - t)
        return out

    target.speculation_forward = timed_forward
    out, acc = speculative_generate(target, draft, prompt, a.max_new_tokens, a.speculation_length)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    t2 = time.perf_counter()
    if dist.get_rank() == 0:
        per_round = 1e3 * sum(verify_s) / max(len(verify_s), 1)
        print(f"identical to greedy: {bool(torch.equal(out, ref))}; accepted draft tokens / target forward: {acc:.2f}; "
              f"greedy {1e3 * (t1 - t0):.1f} ms, speculative {1e3 * (t2 - t1):.1f} ms; target verification "
              f"{per_round:.2f} ms / round over {len(verify_s)} rounds (KV cache: {a.kv_cache_quant})", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
