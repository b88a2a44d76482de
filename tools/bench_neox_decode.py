#!/usr/bin/env python
"""Decode throughput of ``GPTNeoXForInference`` at Pythia-2.8B (32 layers, hidden 2560, 32 heads of 80, rotary width 20,
random bf16 weights): prompt 2048, 128 new tokens, batch 1 / 8 / 32, bf16 and e4m3 KV caches, every decode step replayed
from a CUDA graph.  Two arms in the same process on the same inputs, alternated:

  fused     what the model runs: ``decode_rope_kv`` (partial-rotary RoPE + cache append in one launch), the decode
            attention kernel on the cache as stored, and GEMVs with the bias / GELU / residual in their epilogue;
  composed  the same model with those extension entry points replaced here: torch RoPE + ``KVCacheManager.write_window``
            + torch attention over ``kv.get`` (which de-quantises an e4m3 cache), and the plain GEMV followed by separate
            bias, GELU and residual kernels.

Reported per arm: ms per decode step (one token per sequence), tokens/s, and the share of the HBM floor: (weight bytes + KV
bytes read in the step) / 3.35 TB/s over the step time.  The card's name and power limit are read in the same run.

  python tools/bench_neox_decode.py [--batch 1 8 32] [--kv bf16 e4m3] [--repeats 3] [--out results.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + " (nvidia-smi unavailable)"


class _Composed:
    """Replace the fused extension entry points with the composed path for the duration of a ``with`` block."""

    def __init__(self, e):
        self.e, self.saved = e, {}

    def __enter__(self):
        e = self.e
        gemv = e.gemv
        self.saved = {n: getattr(e, n) for n in ("decode_rope_kv", "decode_attention", "gemv")}

        def composed_gemv(x, w, residual=None, *, bias=None, act=0):
            from neuronx_distributed_b200.ops.gemm import _act_torch

            y = gemv(x, w, None)
            if bias is not None:
                y = y + bias
            y = _act_torch(y, act)
            return y if residual is None else y + residual

        delattr(e, "decode_rope_kv")          # the model then rotates in torch and writes through write_window
        delattr(e, "decode_attention")        # ops.attention.decode_attention then takes the torch path
        e.gemv = composed_gemv
        return self

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(self.e, n, f)


def _bytes_per_step(m, B, prompt, new, kv_elem):
    """Weight bytes every step reads (all parameters but the input embedding, of which B rows are read) + the KV bytes read,
    averaged over the ``new`` steps (step i attends to prompt + i + 1 positions)."""
    w = sum(p.numel() * p.element_size() for n, p in m.lm.named_parameters() if "embed_in" not in n)
    c = m.cfg
    kv_rows = prompt + (new + 1) / 2
    kv = 2 * c.num_hidden_layers * B * kv_rows * c.hidden_size * kv_elem
    return w, kv


def run_config(B, kv, prompt, new, repeats, e):
    from neuronx_distributed_b200.models.gpt_neox import GPTNeoXConfig
    from neuronx_distributed_b200.models.gpt_neox_inference import GPTNeoXForInference
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = GPTNeoXConfig(vocab_size=50304, hidden_size=2560, intermediate_size=10240, num_hidden_layers=32, num_attention_heads=32,
                        rotary_pct=0.25, max_position_embeddings=2048, hidden_act="gelu", initializer_range=0.02,
                        dtype=torch.bfloat16, device=dev)
    torch.manual_seed(0)
    m = GPTNeoXForInference(cfg, batch_size=B, max_seq_len=prompt + new, on_device_sampling=False,
                            kv_quant=KVQuantizationConfig(scale=0.05) if kv == "e4m3" else None).eval()
    ids = torch.randint(0, cfg.vocab_size, (B, prompt), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    last = torch.full((B,), prompt - 1, device=dev)
    first = m.context_encoding(ids, last).argmax(-1)
    tok = first.view(B, 1).clone()
    pos = torch.full((B,), prompt, device=dev, dtype=torch.long)

    def capture():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                m.token_generation(tok, pos)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m.token_generation(tok, pos).argmax(-1)          # greedy
        return g, out

    graphs = {"fused": capture()}
    with _Composed(e):
        graphs["composed"] = capture()

    def decode(arm):
        """``new`` decode steps from the prompt's end: the same tokens and cache rows for both arms."""
        g, out = graphs[arm]
        tok.copy_(first.view(B, 1))
        pos.fill_(prompt)
        toks = []
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(new):
            g.replay()
            toks.append(out.clone())
            tok.copy_(out.view(B, 1))
            pos.add_(1)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / new, torch.stack(toks, 1)

    for arm in graphs:                                         # warm-up
        decode(arm)
    times = {"fused": [], "composed": []}
    toks = {}
    for _ in range(repeats):
        for arm in ("fused", "composed"):
            ms, toks[arm] = decode(arm)
            times[arm].append(ms)
    w_bytes, kv_bytes = _bytes_per_step(m, B, prompt, new, 1 if kv == "e4m3" else 2)
    floor_ms = (w_bytes + kv_bytes) / HBM_BYTES_PER_S * 1e3
    res = {"batch": B, "kv_cache": kv, "prompt": prompt, "new_tokens": new, "weight_bytes": w_bytes, "kv_bytes_per_step": kv_bytes,
           "hbm_floor_ms": floor_ms, "same_tokens": bool(torch.equal(toks["fused"], toks["composed"])),
           "token_agreement": float((toks["fused"] == toks["composed"]).float().mean())}
    for arm, ts in times.items():
        ms = statistics.median(ts)
        res[arm] = {"ms_per_step": ms, "tokens_per_s": B / ms * 1e3, "hbm_floor_share": floor_ms / ms, "all_ms": ts}
    res["speedup"] = res["composed"]["ms_per_step"] / res["fused"]["ms_per_step"]
    del graphs, m
    torch.cuda.empty_cache()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, nargs="+", default=[1, 8, 32])
    p.add_argument("--kv", nargs="+", default=["bf16", "e4m3"], choices=["bf16", "e4m3"])
    p.add_argument("--prompt", type=int, default=2048)
    p.add_argument("--new", type=int, default=128)
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_neox_decode: needs a CUDA device")
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    import torch.distributed as dist

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29561")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(1)
    card = _card()
    print(json.dumps({"card": card}), flush=True)
    results = []
    for kv in a.kv:
        for B in a.batch:
            r = run_config(B, kv, a.prompt, a.new, a.repeats, ops._ext.ext())
            r["card"] = card
            print(json.dumps(r), flush=True)
            results.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": card, "results": results}, f, indent=1)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
