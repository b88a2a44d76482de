"""Time the dropless MoE expert MLP (gate|up projection, SwiGLU, down projection, combine) at prefill with three kinds of
expert weights, at real per-rank shapes:

* ``w8a8``: block-wise e4m3 experts with dynamic activations: per projection the group quantiser and the grouped
  block-scaled FP8 GEMM;
* ``dequant``: the same weights weight-only: de-quantise every local expert to bf16, then the bf16 grouped GEMM;
* ``bf16``: the bf16 grouped GEMM on bf16 weights.

CUDA events around ``iters`` calls after ``warmup`` calls of every arm; arms alternate within one run.  ``TFLOP/s`` counts
the two projections on the routed rows (T·k tokens), not the padded block rows.  Prints one JSON line per (model, T) and
the card's name and power limit from the same run.  ``python tools/bench_moe_fp8.py [--iters 20] [--warmup 5]``"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# name: (hidden, intermediate per rank, experts, top-k, block_axis, block_size)
MODELS = {"mixtral-8x7b-tp8": (4096, 1792, 8, 2, [1], [128]), "qwen3-30b-a3b": (2048, 768, 128, 8, [1], [128]),
          "deepseek-v3-slice": (7168, 2048, 32, 8, [1, 2], [128, 128])}
TOKENS = (512, 4096)


def _card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def _time(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, RoutedExpertsMLPOpsConfig
    from neuronx_distributed_b200.modules.moe.blockwise import blockwise_expert_mlp
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import get_default_blockwise_custom_qconfig_dict

    assert ops.extension_available(), ops._ext.load_error()
    print(json.dumps({"card": _card()}), flush=True)
    dev = torch.device("cuda")
    for name, (H, I, E, k, axis, size) in MODELS.items():
        torch.manual_seed(0)
        cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=k, hidden_size=H,
                                        intermediate_size=I)
        em = ExpertMLPsV2(cfg, dtype=torch.bfloat16, device=dev).eval()
        with torch.no_grad():
            for p in em.parameters():
                if p.dim() == 3:
                    p.normal_(0, p.shape[1] ** -0.5)
        q = {**get_default_blockwise_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3, "block_axis": axis,
             "block_size": size}
        arms = {"w8a8": convert(em, {**q, "activation_quantization_type": ActivationQuantizationType.DYNAMIC},
                                inplace=False).get_mlp_op(),
                "dequant": convert(em, q, inplace=False).get_mlp_op(),
                "bf16": em.get_mlp_op()}
        for T in TOKENS:
            x = torch.randn(T, H, device=dev).to(torch.bfloat16)
            aff = torch.softmax(torch.randn(T, E, device=dev), -1)
            idx = aff.topk(k, -1).indices
            a = em._topk_affinities(aff, idx)
            B = min(em.bw.block_size, max(16, T))
            fns = {arm: (lambda ex=ex: blockwise_expert_mlp(x, a, idx, ex, B)) for arm, ex in arms.items()}
            with torch.no_grad():
                outs = {arm: fn() for arm, fn in fns.items()}
                for _ in range(args.warmup):
                    for fn in fns.values():
                        fn()
                torch.cuda.synchronize()
                ms = {arm: [] for arm in fns}
                for _ in range(3):                                   # alternate the arms, three rounds
                    for arm, fn in fns.items():
                        ms[arm].append(_time(fn, args.iters))
            flops = 2.0 * T * k * H * (2 * I) + 2.0 * T * k * I * H
            ref = outs["bf16"].float()
            res = {"model": name, "T": T, "block": B}
            for arm in fns:
                best = min(ms[arm])
                res[arm] = {"ms": round(best, 4), "spread_pct": round(100 * (max(ms[arm]) - best) / best, 2),
                            "tflops": round(flops / best / 1e9, 1),
                            "rel_err_vs_bf16": round(float((outs[arm].float() - ref).norm() / ref.norm()), 5)}
            print(json.dumps(res), flush=True)
        del arms, em
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
