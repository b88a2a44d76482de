#!/usr/bin/env python
"""Row-wise scaled FP8 training against bf16 on one GPU; prints one JSON line.

    python tools/bench_fp8_train.py [--iters 20] [--steps 4] [--warmup 2] [--layers 12]

1. GEMMs at the Llama-2-7B TP=1 shapes (M = 4096 tokens): forward x·Wᵀ, input gradient g·W and weight gradient gᵀ·x added into
   an fp32 main_grad, each as the bf16 wgmma GEMM and as the quantisers + fp8 GEMM of ``ops.gemm_fp8`` (quantiser time also
   reported on its own).  CUDA events around ``--iters`` calls after a warm-up.
2. ``bench.py``'s training-step geometry (12 Llama-2-7B layers, seq 4096, global batch 4 in micro-batches of 1, ZeRO-1 with
   fp32 gradient accumulation).  Both arms share one model: ``fp8_training`` only changes the arithmetic of the decoder's
   linears, so the arms alternate step by step on the same parameters (bf16, fp8, bf16, …) and the host clock around each
   synchronised step times it.  The two loss traces therefore come from one interleaved trajectory.

The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"qkv": (4096, 12288), "o": (4096, 4096), "gate_up": (4096, 22016), "down": (11008, 4096)}   # (K, N)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def time_ms(fn, iters):
    import torch

    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gemms(iters):
    import torch

    from neuronx_distributed_b200.ops import gemm, gemm_fp8

    M, dev, out = 4096, torch.device("cuda"), {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (K, N) in SHAPES.items():
        x = torch.randn(M, K, device=dev, generator=g).bfloat16()
        w = (torch.randn(N, K, device=dev, generator=g) * 0.02).bfloat16()
        gy = (torch.randn(M, N, device=dev, generator=g) * 1e-3).bfloat16()
        mg = torch.zeros(N, K, device=dev)
        flop = 2.0 * M * N * K
        r = {}
        for which, bf16, quant, fp8 in (
            ("fwd", lambda: gemm.matmul(x, w, False, True),
             lambda: (gemm_fp8.quantize_rows(x), gemm_fp8.quantize_rows(w)),
             lambda: gemm_fp8.fp8_forward(x, w)),
            ("dgrad", lambda: gemm.matmul(gy, w, False, False),
             lambda: (gemm_fp8.quantize_rows(gy), gemm_fp8.quantize_cols_t(w)),
             lambda: gemm_fp8.fp8_dgrad(gy, w)),
            ("wgrad", lambda: gemm.matmul(gy, x, True, False, out=mg, accumulate=True),
             lambda: (gemm_fp8.quantize_cols_t(gy), gemm_fp8.quantize_cols_t(x)),
             lambda: gemm_fp8.fp8_wgrad(gy, x, out=mg, accumulate=True)),
        ):
            t_bf16, t_q, t_fp8 = time_ms(bf16, iters), time_ms(quant, iters), time_ms(fp8, iters)
            r[which] = {"bf16_ms": round(t_bf16, 4), "fp8_total_ms": round(t_fp8, 4), "fp8_quantise_ms": round(t_q, 4),
                        "fp8_gemm_ms": round(t_fp8 - t_q, 4), "bf16_tflops": round(flop / t_bf16 / 1e9, 1),
                        "fp8_gemm_tflops": round(flop / max(t_fp8 - t_q, 1e-6) / 1e9, 1)}
        out[name] = r
    return out


def steps(n_steps, warmup, layers):
    import time

    import torch
    import torch.distributed as dist

    import neuronx_distributed_b200 as nxd
    from neuronx_distributed_b200.models.llama import LlamaForCausalLM, llama2_7b_config
    from neuronx_distributed_b200.modules.qkv_linear import GQAQKVColumnParallelLinear
    from neuronx_distributed_b200.parallel_layers.layers import BaseParallelLinear
    from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams

    dev = torch.device("cuda", 0)
    cfg = nxd.neuronx_distributed_config(
        tensor_parallel_size=1, optimizer_config={"zero_one_enabled": True, "grad_clipping": True, "max_grad_norm": 1.0},
        mixed_precision_config={"use_master_weights": True, "use_fp32_grad_acc": True, "use_master_weights_in_ckpt": False})
    S, gbs = 4096, 4
    mcfg = llama2_7b_config(dtype=torch.bfloat16, device=dev, max_position_embeddings=S)
    mcfg.num_hidden_layers = layers

    def model_fn():
        torch.manual_seed(1234)
        torch.cuda.manual_seed(1234)
        return LlamaForCausalLM(mcfg)

    model = nxd.initialize_parallel_model(cfg, model_fn)
    opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=3e-4, betas=(0.9, 0.95),
                                            weight_decay=0.1)
    decoder = [m for n, m in model.named_modules() if ".layers." in n
               and isinstance(m, (BaseParallelLinear, GQAQKVColumnParallelLinear))]
    assert len(decoder) == 4 * layers, len(decoder)
    gen = torch.Generator().manual_seed(7)
    batches = [torch.randint(0, mcfg.vocab_size, (gbs, S), generator=gen).to(dev) for _ in range(2 * (n_steps + warmup))]

    def step(ids, fp8):
        for m in decoder:
            m.fp8_training = fp8
        opt.zero_grad()
        total = 0.0
        for i in range(gbs):
            total = total + model.run_train(input_ids=ids[i:i + 1], labels=ids[i:i + 1])
        opt.step()
        return total / gbs

    times, losses = {False: [], True: []}, {False: [], True: []}
    for i, ids in enumerate(batches):
        fp8 = bool(i % 2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss = float(step(ids, fp8))
        torch.cuda.synchronize()
        losses[fp8].append(round(loss, 4))
        if i >= 2 * warmup:
            times[fp8].append(time.perf_counter() - t0)
    tok = gbs * S
    res = {}
    for fp8, key in ((False, "bf16"), (True, "fp8")):
        med = statistics.median(times[fp8])
        res[key] = {"step_s_median": round(med, 4), "step_s_all": [round(t, 4) for t in times[fp8]],
                    "tokens_per_s": round(tok / med, 1), "loss_trace": losses[fp8]}
    res["fp8_over_bf16_tokens_per_s"] = round(res["fp8"]["tokens_per_s"] / res["bf16"]["tokens_per_s"], 4)
    dist.barrier()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=4, help="timed steps per arm")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps per arm")
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--skip-steps", action="store_true")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist

    from neuronx_distributed_b200 import ops

    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    assert ops.extension_available(), ops._ext.load_error()
    torch.cuda.set_device(0)
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29571")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    out = {"metric": "fp8_training_vs_bf16", **card(), "gemms_M4096": gemms(a.iters)}
    if not a.skip_steps:
        out["step_seq4096_gbs4"] = {"layers": a.layers, **steps(a.steps, a.warmup, a.layers)}
    out.update(card())                       # read again after the run: the limit the numbers ran under
    print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
