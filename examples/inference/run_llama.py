#!/usr/bin/env python
"""Llama inference sample + latency benchmark (BASELINE config 5: Llama-2-13B, TP=8, batch 1, seq 2048) — counterpart of the
reference's ``examples/inference/run_llama.py`` / ``runner.py`` (trace → load → generate → benchmark → report).

  torchrun --nproc-per-node 8 examples/inference/run_llama.py --model 13b --tp_degree 8 --batch_size 1 \
      --max_prompt_length 1024 --sequence_length 2048 --benchmark
  # GQA with fewer KV heads than ranks: replicas of a KV head shard its cache along the sequence (flash decoding)
  torchrun --nproc-per-node 8 examples/inference/run_llama.py --model 7b --num_kv_heads 4 --tp_degree 8 --flash_decoding
  # KV cache stored in fp8 e4m3 (one scale per tensor): half the cache bytes, read directly by the decode kernels
  torchrun --nproc-per-node 1 examples/inference/run_llama.py --model 7b --batch_size 16 --max_prompt_length 2048 \
      --sequence_length 4096 --benchmark --kv_cache_quant fp8
  # Mistral-7B geometry (sliding window 4096): a rolling KV cache keeps 4096 + 64 rows per sequence instead of 8192
  torchrun --nproc-per-node 1 examples/inference/run_llama.py --model mistral-7b --batch_size 16 --max_prompt_length 2048 \
      --sequence_length 8192 --benchmark --num_runs 1 --rolling_kv_cache
  # Llama-3.2-1B geometry (head_dim 64, 4 query heads per KV head, Llama-3 RoPE scaling) with random weights
  torchrun --nproc-per-node 1 examples/inference/run_llama.py --model llama3.2-1b --batch_size 16 --max_prompt_length 2048 \
      --sequence_length 4096 --benchmark
  # Llama-3.2-3B (3 query heads per KV head) and Qwen2.5-7B (7 per KV head, q / k / v bias) geometries
  torchrun --nproc-per-node 1 examples/inference/run_llama.py --model qwen2.5-7b --batch_size 8 --max_prompt_length 2048 \
      --sequence_length 4096 --benchmark
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "training"))

from neuronx_distributed_b200.inference.autobucketing import generate_buckets  # noqa: E402
from neuronx_distributed_b200.inference.benchmark import Benchmark, generate_report  # noqa: E402
from neuronx_distributed_b200.trace.model_builder import ModelBuilder  # noqa: E402
from neuronx_distributed_b200.models.llama import LlamaConfig, llama2_7b_config, llama2_13b_config  # noqa: E402
from neuronx_distributed_b200.models.llama_inference import LlamaForInference  # noqa: E402
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from neuronx_distributed_b200.quantization import KVQuantizationConfig  # noqa: E402
from training_utils import init_distributed  # noqa: E402


def mistral_7b_config(**kw) -> LlamaConfig:
    """Mistral-7B geometry: GQA with 8 KV heads and a 4096-token sliding window."""
    return LlamaConfig(vocab_size=32000, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                       num_key_value_heads=8, sliding_window=4096, **kw)


# the rope_scaling of the Llama-3.2 config.json files
LLAMA3_2_ROPE_SCALING = {"factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}


def llama3_2_1b_config(**kw) -> LlamaConfig:
    """Llama-3.2-1B geometry: head_dim 2048 / 32 = 64, 8 KV heads (GQA group 4), rope_theta 500000, Llama-3 RoPE scaling."""
    return LlamaConfig(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32,
                       num_key_value_heads=8, rope_theta=500000.0, rope_scaling=dict(LLAMA3_2_ROPE_SCALING), **kw)


def llama3_2_3b_config(**kw) -> LlamaConfig:
    """Llama-3.2-3B geometry: head_dim 128, 24 / 8 heads (GQA group 3), rope_theta 500000, Llama-3 RoPE scaling."""
    return LlamaConfig(vocab_size=128256, hidden_size=3072, intermediate_size=8192, num_hidden_layers=28, num_attention_heads=24,
                       num_key_value_heads=8, rope_theta=500000.0, rope_scaling=dict(LLAMA3_2_ROPE_SCALING), **kw)


def qwen2_5_7b_config(**kw) -> LlamaConfig:
    """Qwen2.5-7B geometry: head_dim 128, 28 / 4 heads (GQA group 7), q / k / v bias, rope_theta 10⁶."""
    return LlamaConfig(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28, num_attention_heads=28,
                       num_key_value_heads=4, rope_theta=1e6, rms_norm_eps=1e-6, qkv_bias=True, **kw)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="tiny", choices=["tiny", "7b", "13b", "mistral-7b", "llama3.2-1b", "llama3.2-3b", "qwen2.5-7b"],
                   help="model geometry, random weights; the Llama-3.2 geometries carry Llama-3 RoPE scaling, qwen2.5-7b q / k / v bias")
    p.add_argument("--tp_degree", type=int, default=1)
    p.add_argument("--batch_size", type=int, default=1)
    p.add_argument("--max_prompt_length", type=int, default=128)
    p.add_argument("--sequence_length", type=int, default=256)
    p.add_argument("--num_layers", type=int, default=-1)
    p.add_argument("--benchmark", action="store_true")
    p.add_argument("--num_runs", type=int, default=20)
    p.add_argument("--no_cuda_graphs", action="store_true")
    p.add_argument("--flash_decoding", action="store_true",
                   help="shard the KV cache along the sequence inside each KV-replica group (needs tp_degree > number of KV heads)")
    p.add_argument("--num_kv_heads", type=int, default=0, help="override the number of KV heads (GQA experiments)")
    p.add_argument("--kv_cache_quant", default="none", choices=["none", "fp8"],
                   help="fp8: store the KV cache in float8 e4m3 with one scale per tensor (--kv_cache_scale)")
    p.add_argument("--kv_cache_scale", type=float, default=1.0, help="the cache stores k / scale and v / scale")
    p.add_argument("--rolling_kv_cache", action="store_true",
                   help="sliding-window models: keep only the last window + 64 positions of each sequence in a ring")
    p.add_argument("--max_new_tokens", type=int, default=0,
                   help="tokens generated per sequence (default: fill the sequence); the cache size is set by --sequence_length")
    a = p.parse_args()
    dev = init_distributed()
    ps.initialize_model_parallel(tensor_model_parallel_size=a.tp_degree)
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    kw = dict(dtype=dtype, device=dev, max_position_embeddings=a.sequence_length)
    cfg = {"7b": llama2_7b_config, "13b": llama2_13b_config, "mistral-7b": mistral_7b_config,
           "llama3.2-1b": llama3_2_1b_config, "llama3.2-3b": llama3_2_3b_config, "qwen2.5-7b": qwen2_5_7b_config}.get(a.model, lambda **k: LlamaConfig(
        vocab_size=4096, hidden_size=512, intermediate_size=1408, num_hidden_layers=4, num_attention_heads=8, **k))(**kw)
    if a.num_layers > 0:
        cfg.num_hidden_layers = a.num_layers
    if a.num_kv_heads > 0:
        cfg.num_key_value_heads = a.num_kv_heads
    torch.manual_seed(0)
    kv_quant = None
    if a.kv_cache_quant == "fp8":
        kv_quant = KVQuantizationConfig(quant_dtype=torch.float8_e4m3fn, dequant_dtype=dtype, scale=a.kv_cache_scale)
    model = LlamaForInference(cfg, batch_size=a.batch_size, max_seq_len=a.sequence_length,
                              flash_decoding=a.flash_decoding, kv_quant=kv_quant, rolling_kv_cache=a.rolling_kv_cache).eval()
    B, P = a.batch_size, a.max_prompt_length
    mb = ModelBuilder(tp_degree=a.tp_degree, use_cuda_graphs=(dev.type == "cuda" and not a.no_cuda_graphs))
    for bucket in generate_buckets(min(128, P), P):
        mb.add("context_encoding_model", model, [(torch.zeros(B, bucket, dtype=torch.long, device=dev),
                                                  torch.full((B,), bucket - 1, dtype=torch.long, device=dev))],
               step_fn=lambda m, i, l: m.context_encoding(i, l))
    mb.add("token_generation_model", model, [(torch.zeros(B, 1, dtype=torch.long, device=dev),
                                              torch.full((B,), P, dtype=torch.long, device=dev))],
           step_fn=lambda m, i, pos: m.token_generation(i, pos))
    nxd_model = mb.trace()
    prompt = torch.randint(0, cfg.vocab_size, (B, P), device=dev)
    new_tokens = min(a.max_new_tokens, a.sequence_length - P) if a.max_new_tokens > 0 else a.sequence_length - P

    def generate():
        tok = nxd_model(prompt, torch.full((B,), P - 1, dtype=torch.long, device=dev)).clone()
        pos = torch.full((B,), P, dtype=torch.long, device=dev)
        out = [tok]
        for _ in range(new_tokens - 1):
            tok = nxd_model(tok.view(B, 1), pos).clone()
            pos = pos + 1
            out.append(tok)
        return torch.stack(out, 1)

    toks = generate()
    if dist.get_rank() == 0:
        print("generated", tuple(toks.shape), toks[0, :8].tolist(), flush=True)
    if a.benchmark:
        lat = Benchmark(generate, num_runs=a.num_runs).run()
        rep = generate_report(lat, a.sequence_length, B)
        rep["generated_tokens_per_s"] = B * new_tokens / (sum(lat) / len(lat))
        if dev.type == "cuda":
            rep["peak_allocated_GiB"] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
            rep["kv_cache_GiB"] = sum(t.nbytes for t in model.kv.k + model.kv.v) / 2 ** 30
            rep["kv_cache_rows"], rep["kv_cache_rolling"] = model.kv.rows, model.kv.rolling
        if dist.get_rank() == 0:
            print(json.dumps({"e2e_model": rep, "config": vars(a)}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
