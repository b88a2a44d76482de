"""Numerics + timing of the flash-attention kernels against a plain fp32 PyTorch reference and SDPA (cuDNN).
usage: python tools/fa_check.py [--head-dim 64|80|96|128] [--perf] [--bwd] [--window [--cp N]] [--kv-fp8] [--spec] [--rolling]
                                [--decode-dims] [--decode-groups] [--dropout]

--perf times forward and forward+backward of the own kernels and of SDPA in the same process, alternating, at the shapes
the models run (BERT-large with right padding, ViT-B/16, GPT-NeoX-20B per rank at TP=8, Pythia-2.8B, Llama-2-7B).  FLOPs
come from the shapes: 4·D per visible (query, key) pair forward, 2.5× that backward; causal counts only the lower
triangle and a key-padding mask only the visible keys.

--window (with --perf) times sliding-window attention instead, at the Mistral-7B per-GPU shape (B = 1, H = 32, Hkv = 8,
D = 128, W = 4096) for S = 4k … 32k: the windowed kernels, the same kernels causal without a window, and SDPA with the windowed
mask, all counted over the pairs the window leaves visible; then the decode kernel on a 32k cache with and without the
window.

--window --cp N (with --perf) emulates one layer's context-parallel attention at the same shape for S = 32k, 64k and 128k on
one GPU: the blocks the rank with the most work computes under the windowed block plan (``modules/attention/ring.py``
``_visible_pairs``), run through ``block_attention`` and the LSE merge as ring attention runs them, against the causal plan
(what CP computes if the window is dropped).  It reports the time, the TFLOP/s over the visible pairs and the K/V bytes each
rank sends per layer (hops × 2·c·Hkv·D·2 B).  All ranks' blocks come from one process, so no NCCL time is measured.  Pair and
byte counts come from shapes and are printed without a GPU too; times need one.

--kv-fp8 (with --perf) times ``decode_attention`` on a bf16 and on an fp8 e4m3 KV cache of the same shape, alternating in one
process: the Mistral-7B per-GPU shape (H 32, Hkv 8, D 128) on a full 32k cache at B = 1, 8 and 32, and the Llama-2-13B
MHA shape (H = Hkv = 40) at B = 8, L = 4096.  Bytes read come from the shapes (the K and V rows and q; the fp32 split
partials, which stay in L2, are left out); GB/s is those bytes over the time of the call (both kernels).  Both caches hold the same values (the bf16 one
is the de-quantised e4m3 one), and the two outputs are compared.

--spec (with --perf) times ``speculation_attention`` (the verification kernel and its combine) against the path it replaces
(de-quantise the whole fp8 cache, then SDPA with a [B, 1, W, L] mask on K / V repeated over the GQA group), alternating in
one process: Llama-2-7B (H = Hkv = 32) at L = 4096, B = 1, and Mistral-7B (H 32, Hkv 8) at L = 32768, B = 1 and 8, with and
without a 4096 sliding window; a 5-token chain, the Medusa example's 10-node tree and a random 64-node tree; bf16 and e4m3
caches holding the same values.  Bytes come from the shapes: the K and V rows some token can see, read once, plus q and the
output.

--rolling (with --perf) times ``decode_attention`` and ``speculation_attention`` on a rolling KV cache (SW + 64 = 4160 rows,
position t in row t mod 4160) against the linear 32k cache holding the same history, alternating in one process: Mistral-7B
(H 32, Hkv 8, SW 4096) at B = 1, 8 and 32, position 32767 − W, decode and the chain5 / tree10 / tree64 windows, bf16 and
e4m3.  Both read the same rows, so the times should match; the outputs are checked bit for bit.

--decode-dims (with --perf) times token generation at head_dim 64, 80 and 96 on the kernels against the path those head
sizes took before the kernels took them (``speculation_attention_torch`` on the de-quantised cache for decode and
verification, ``_local_partial``'s fp32 torch math for flash decoding's partial), alternating in one process: Llama-3.2-1B
attention (H 32, Hkv 8, D 64), Phi-3-mini (H = Hkv = 32, D 96) and Pythia-2.8B heads (H = Hkv = 32, D 80), with the D = 128
kernel on a Mistral-7B head geometry (H 32, Hkv 8) as the control; B = 1, 8, 32, L = 4096 and 32768 (pairs that fit the
card), bf16 and e4m3 caches holding the same values, one-token decode, a 5-token chain and a random 64-node tree.  GB/s is
the K and V bytes of the visible cache rows (from the shapes) over the time of the call.  The D = 128 control's torch path
is timed only at B = 1 (it is the one the kernels have replaced since they exist).  The partial at B = 8, L = 4096.

--decode-groups (with --perf) times the same table at the GQA groups 3, 5, 6 and 7 the kernels took from the torch path:
Llama-3.2-3B (H 24, Hkv 8), Qwen2.5-14B (H 40, Hkv 8), Qwen2.5-1.5B (H 12, Hkv 2), Qwen2.5-7B (H 28, Hkv 4) and its TP = 4
shard (H 7, Hkv 1) at D = 128, and Qwen2.5-0.5B (H 14, Hkv 2, D 64); the torch path is timed at every shape.

--dropout (with --perf) times attention dropout: the own kernels at p = 0.1 against the same kernels at p = 0 and against
SDPA with dropout_p = 0.1, forward and (with --bwd) forward + backward, alternating in one process, at the BERT-large
(right-padded, D = 64) and GPT-NeoX-20B per TP = 8 rank (D = 96) shapes of --perf."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuronx_distributed_b200.ops import _ext, attention  # noqa: E402


def ref_attn(q, k, v, causal, scale, mask=None):
    # q [B,S,H,D] fp32 math; mask: optional key-padding mask [B, S_kv] (True = visible, no fully masked row)
    B, S, H, D = q.shape
    Hkv = k.shape[2]
    qf, kf, vf = q.float().transpose(1, 2), k.float().transpose(1, 2), v.float().transpose(1, 2)
    if H != Hkv:
        kf = kf.repeat_interleave(H // Hkv, 1)
        vf = vf.repeat_interleave(H // Hkv, 1)
    s = qf @ kf.transpose(-1, -2) * scale
    if causal:
        m = torch.ones(S, k.shape[1], device=q.device, dtype=torch.bool).tril()
        s = s.masked_fill(~m, float("-inf"))
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    p = s.softmax(-1)
    return (p @ vf).transpose(1, 2), torch.logsumexp(s, -1)


def gpu_info():
    """Name, power limit and max SM clock of the GPU the numbers are measured on (read in the same run)."""
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        info["power_limit"], info["max_sm_clock"] = (x.strip() for x in out.strip().split(","))
    except Exception as ex:  # noqa: BLE001 - the record still has the device name
        info["power_limit"] = f"unavailable ({type(ex).__name__})"
    return info


# name, B, S, H, D, causal, padded fraction of the keys (right padding, per-sequence lengths drawn around it)
PERF_SHAPES = [
    ("bert_large", 32, 512, 16, 64, False, 0.15),
    ("vit_b16", 64, 197, 12, 64, False, 0.0),
    ("neox20b_tp8", 1, 2048, 8, 96, True, 0.0),
    ("pythia2.8b", 4, 2048, 32, 80, True, 0.0),
    ("llama2_7b", 4, 4096, 32, 128, True, 0.0),
]


def perf(e, bwd: bool):
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    for (name, B, S, H, D, causal, pad) in PERF_SHAPES:
        q, k, v, go = (torch.randn(B, S, H, D, device=dev, generator=g).bfloat16() for _ in range(4))
        scale = 1.0 / math.sqrt(D)
        mask = None
        if pad > 0:
            lens = (S * (1.0 - 2 * pad * torch.rand(B, device=dev, generator=g))).long().clamp(1, S)
            mask = torch.arange(S, device=dev)[None, :] < lens[:, None]
        vis_keys = mask.sum(1).double() if mask is not None else torch.full((B,), float(S), device=dev, dtype=torch.float64)
        pairs = float((vis_keys * ((S + 1) / 2 if causal else S)).sum()) * H      # visible (query, key) pairs
        fl = 4 * D * pairs
        qt, kt, vt, gt = (t.transpose(1, 2) for t in (q, k, v, go))
        bias = None
        if mask is not None:                        # the additive bias the models pass to SDPA
            bias = torch.zeros(B, 1, 1, S, device=dev, dtype=q.dtype).masked_fill(~mask[:, None, None, :], float("-inf"))

        def own_f():
            return e.flash_attn_fwd(q, k, v, causal, scale, True, mask)

        def sdpa_f(qq=qt, kk=kt, vv=vt):
            if bias is None:
                return torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, is_causal=causal)
            return torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, attn_mask=bias)

        qr, kr, vr = (t.detach().requires_grad_(True) for t in (qt, kt, vt))

        def own_fb():
            o, lse = own_f()
            e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True, None, mask)

        def sdpa_fb():
            torch.autograd.grad(sdpa_f(qr, kr, vr), (qr, kr, vr), gt)

        # alternate own / SDPA three times and keep each one's best, so drift of the shared clock hits both alike
        t = {"own_fwd": [], "sdpa_fwd": [], "own_fwd_bwd": [], "sdpa_fwd_bwd": []}
        for _ in range(3):
            t["own_fwd"].append(time_fn(own_f))
            t["sdpa_fwd"].append(time_fn(sdpa_f))
            if bwd:
                t["own_fwd_bwd"].append(time_fn(own_fb))
                t["sdpa_fwd_bwd"].append(time_fn(sdpa_fb))
        rec = {"bench": name, "B": B, "S": S, "H": H, "D": D, "causal": causal, "visible_key_frac": round(float(vis_keys.sum()) / (B * S), 3)}
        for key, vals in t.items():
            if not vals:
                continue
            ms = min(vals)
            tf = (3.5 if "bwd" in key else 1.0) * fl / ms / 1e9
            rec[key + "_ms"], rec[key + "_tflops"] = round(ms, 4), round(tf, 1)
        rec["own_vs_sdpa_fwd"] = round(rec["sdpa_fwd_ms"] / rec["own_fwd_ms"], 2)
        if bwd:
            rec["own_vs_sdpa_fwd_bwd"] = round(rec["sdpa_fwd_bwd_ms"] / rec["own_fwd_bwd_ms"], 2)
        print(json.dumps(rec), flush=True)


DROPOUT_SHAPES = ("bert_large", "neox20b_tp8")


def dropout_perf(e, bwd: bool, p: float = 0.1):
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    seed = torch.tensor([1234], dtype=torch.int64, device=dev)
    for (name, B, S, H, D, causal, pad) in PERF_SHAPES:
        if name not in DROPOUT_SHAPES:
            continue
        q, k, v, go = (torch.randn(B, S, H, D, device=dev, generator=g).bfloat16() for _ in range(4))
        scale = 1.0 / math.sqrt(D)
        mask = bias = None
        if pad > 0:
            lens = (S * (1.0 - 2 * pad * torch.rand(B, device=dev, generator=g))).long().clamp(1, S)
            mask = torch.arange(S, device=dev)[None, :] < lens[:, None]
            bias = torch.zeros(B, 1, 1, S, device=dev, dtype=q.dtype).masked_fill(~mask[:, None, None, :], float("-inf"))
        qt, kt, vt, gt = (t.transpose(1, 2) for t in (q, k, v, go))
        qr, kr, vr = (t.detach().requires_grad_(True) for t in (qt, kt, vt))

        def own(pp):
            def f():
                return e.flash_attn_fwd(q, k, v, causal, scale, True, mask, 0, 0, pp, seed)

            def fb():
                o, lse = f()
                e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True, None, mask, 0, 0, pp, seed)
            return f, fb

        def sdpa_f(qq=qt, kk=kt, vv=vt):
            return torch.nn.functional.scaled_dot_product_attention(qq, kk, vv, attn_mask=bias, dropout_p=p,
                                                                    is_causal=causal and bias is None)

        def sdpa_fb():
            torch.autograd.grad(sdpa_f(qr, kr, vr), (qr, kr, vr), gt)

        fns = {"own_p0_fwd": own(0.0)[0], f"own_p{p}_fwd": own(p)[0], f"sdpa_p{p}_fwd": sdpa_f}
        if bwd:
            fns.update({"own_p0_fwd_bwd": own(0.0)[1], f"own_p{p}_fwd_bwd": own(p)[1], f"sdpa_p{p}_fwd_bwd": sdpa_fb})
        t = {key: [] for key in fns}
        for _ in range(3):                          # alternate, keep each one's best
            for key, fn in fns.items():
                t[key].append(time_fn(fn))
        rec = {"bench": name + "_dropout", "B": B, "S": S, "H": H, "D": D, "causal": causal, "p": p}
        rec.update({key + "_ms": round(min(vals), 4) for key, vals in t.items()})
        for step in ("fwd", "fwd_bwd") if bwd else ("fwd",):
            rec[f"dropout_overhead_{step}"] = round(rec[f"own_p{p}_{step}_ms"] / rec[f"own_p0_{step}_ms"], 3)
            rec[f"own_vs_sdpa_dropout_{step}"] = round(rec[f"sdpa_p{p}_{step}_ms"] / rec[f"own_p{p}_{step}_ms"], 2)
        print(json.dumps(rec), flush=True)


def visible_pairs(S: int, W: int) -> int:
    """(query, key) pairs with i − W < j ≤ i: Σ_i min(i + 1, W)."""
    w = min(W, S)
    return w * (w + 1) // 2 + (S - w) * w


def window_perf(e, bwd: bool, W: int = 4096):
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    B, H, Hkv, D = 1, 32, 8, 128
    scale = 1.0 / math.sqrt(D)
    g = torch.Generator(device=dev).manual_seed(0)
    for S in (4096, 8192, 16384, 32768):
        q, go = (torch.randn(B, S, H, D, device=dev, generator=g).bfloat16() for _ in range(2))
        k, v = (torch.randn(B, S, Hkv, D, device=dev, generator=g).bfloat16() for _ in range(2))
        fl = 4 * D * H * B * visible_pairs(S, W)                  # forward FLOPs over the pairs the window keeps

        def own(window):
            def f():
                return e.flash_attn_fwd(q, k, v, True, scale, True, None, window)

            def fb():
                o, lse = f()
                e.flash_attn_bwd(go, q, k, v, o, lse, True, scale, True, None, None, window)
            return f, fb

        qt, gt = q.transpose(1, 2), go.transpose(1, 2)
        kt, vt = (t.transpose(1, 2).repeat_interleave(H // Hkv, 1) for t in (k, v))
        bias = torch.zeros(S, S, device=dev, dtype=q.dtype).masked_fill(
            ~attention.window_visibility(S, S, W, dev), float("-inf"))[None, None]
        qr, kr, vr = (t.detach().requires_grad_(True) for t in (qt, kt, vt))

        def sdpa_f():
            return torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=bias)

        def sdpa_fb():
            o = torch.nn.functional.scaled_dot_product_attention(qr, kr, vr, attn_mask=bias)
            torch.autograd.grad(o, (qr, kr, vr), gt)

        fns = {"window": own(W), "causal": own(0), "sdpa_mask": (sdpa_f, sdpa_fb)}
        # the windowed result against the masked SDPA one, at the shape that is timed
        ow, _ = fns["window"][0]()
        err = ((ow.float() - sdpa_f().transpose(1, 2).float()).abs().max() / ow.float().abs().max()).item()
        t = {}
        iters = max(3, 20 * 4096 // S)
        for _ in range(2):                                        # alternate, keep each one's best
            for name, (f, fb) in fns.items():
                for key, fn in ((name + "_fwd", f), (name + "_fwd_bwd", fb if bwd else None)):
                    if fn is None:
                        continue
                    try:
                        t.setdefault(key, []).append(time_fn(fn, iters))
                    except torch.OutOfMemoryError:
                        t.setdefault(key, []).append(float("nan"))
                        torch.cuda.empty_cache()
        rec = {"bench": "mistral7b_window", "B": B, "S": S, "H": H, "Hkv": Hkv, "D": D, "W": W,
               "visible_pairs_frac_of_causal": round(visible_pairs(S, W) / visible_pairs(S, S), 4),
               "window_vs_sdpa_mask_rel_err": round(err, 5)}
        for key, vals in t.items():
            ms = min(vals)
            rec[key + "_ms"] = round(ms, 4) if ms == ms else None
            # TFLOP/s over the window's visible pairs for every column, so the causal column shows the cost of ignoring W
            rec[key + "_tflops"] = round((3.5 if "bwd" in key else 1.0) * fl / ms / 1e9, 1) if ms == ms else None
        for key in ("fwd", "fwd_bwd"):
            if rec.get(f"window_{key}_ms") and rec.get(f"causal_{key}_ms"):
                rec[f"causal_over_window_{key}"] = round(rec[f"causal_{key}_ms"] / rec[f"window_{key}_ms"], 2)
            if rec.get(f"window_{key}_ms") and rec.get(f"sdpa_mask_{key}_ms"):
                rec[f"sdpa_mask_over_window_{key}"] = round(rec[f"sdpa_mask_{key}_ms"] / rec[f"window_{key}_ms"], 2)
        print(json.dumps(rec), flush=True)
        del bias, q, k, v, go, qt, kt, vt, qr, kr, vr, fns, ow
        torch.cuda.empty_cache()
    # decode: one token per sequence against a 32k cache, newest position at the end of the cache
    L = 32768
    for Bd in (1, 8):
        qd = torch.randn(Bd, 1, H, D, device=dev, generator=g).bfloat16()
        kc, vc = (torch.randn(Bd, L, Hkv, D, device=dev, generator=g).bfloat16() for _ in range(2))
        pos = torch.full((Bd,), L - 1, device=dev, dtype=torch.long)
        t = {"full": [], "window": []}
        for _ in range(3):
            t["full"].append(time_fn(lambda: e.decode_attention(qd, kc, vc, pos, scale, 0)))
            t["window"].append(time_fn(lambda: e.decode_attention(qd, kc, vc, pos, scale, W)))
        rec = {"bench": "mistral7b_decode", "B": Bd, "L": L, "H": H, "Hkv": Hkv, "D": D, "W": W}
        for name, rows in (("full", L), ("window", W)):
            ms = min(t[name])
            rec[name + "_us"] = round(ms * 1e3, 2)
            rec[name + "_kv_GBps"] = round(2 * Bd * rows * Hkv * D * 2 / ms / 1e6, 1)   # K and V rows read, bf16
        rec["full_over_window"] = round(rec["full_us"] / rec["window_us"], 2)
        print(json.dumps(rec), flush=True)


KV_FP8_SHAPES = [  # name, B, L, H, Hkv
    ("mistral7b", 1, 32768, 32, 8), ("mistral7b", 8, 32768, 32, 8), ("mistral7b", 32, 32768, 32, 8),
    ("llama2_13b", 8, 4096, 40, 40),
]


def kv_fp8_perf():
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    D, ks, vs = 128, 0.05, 0.05
    g = torch.Generator(device=dev).manual_seed(0)
    for name, B, L, H, Hkv in KV_FP8_SHAPES:
        q = torch.randn(B, 1, H, D, device=dev, generator=g).bfloat16()
        k8, v8 = ((torch.randn(B, L, Hkv, D, device=dev, generator=g) / s).to(torch.float8_e4m3fn) for s in (ks, vs))
        k16, v16 = (k8.float() * ks).bfloat16(), (v8.float() * vs).bfloat16()
        pos = torch.full((B,), L - 1, device=dev, dtype=torch.long)
        scale = 1.0 / math.sqrt(D)
        o16 = attention.decode_attention(q, k16, v16, pos, scale)
        o8 = attention.decode_attention(q, k8, v8, pos, scale, k_scale=ks, v_scale=vs)
        err = ((o8.float() - o16.float()).abs().max() / o16.float().abs().max()).item()
        t = {"bf16": [], "e4m3": []}
        iters = max(20, 2000 // B)
        for _ in range(3):                                     # alternate, keep each one's best
            t["bf16"].append(time_fn(lambda: attention.decode_attention(q, k16, v16, pos, scale), iters))
            t["e4m3"].append(time_fn(lambda: attention.decode_attention(q, k8, v8, pos, scale, k_scale=ks, v_scale=vs), iters))
        rec = {"bench": f"{name}_decode_kv_fp8", "B": B, "L": L, "H": H, "Hkv": Hkv, "D": D, "e4m3_vs_bf16_rel_err": round(err, 5)}
        for dt, elt in (("bf16", 2), ("e4m3", 1)):
            ms = min(t[dt])
            nbytes = 2 * B * L * Hkv * D * elt + B * H * D * 2   # K and V rows, q
            rec[f"{dt}_us"] = round(ms * 1e3, 2)
            rec[f"{dt}_bytes"] = nbytes
            rec[f"{dt}_GBps"] = round(nbytes / ms / 1e6, 1)
        rec["bf16_over_e4m3"] = round(rec["bf16_us"] / rec["e4m3_us"], 2)
        print(json.dumps(rec), flush=True)
        del q, k8, v8, k16, v16
        torch.cuda.empty_cache()


# name, B, L, H, Hkv, sliding window
SPEC_SHAPES = [
    ("llama2_7b", 1, 4096, 32, 32, None),
    ("mistral7b", 1, 32768, 32, 8, None),
    ("mistral7b", 1, 32768, 32, 8, 4096),
    ("mistral7b", 8, 32768, 32, 8, None),
    ("mistral7b", 8, 32768, 32, 8, 4096),
]
# the candidate tree of examples/inference/run_llama_medusa.py (10 nodes)
MEDUSA_CHOICES = [[0], [1], [2], [0, 0], [0, 1], [1, 0], [0, 0, 0], [0, 0, 1], [0, 1, 0]]


def spec_windows(dev):
    """(name, tree_mask, tree_depth, W): a 5-token chain, the example's 10-node Medusa tree and a random 64-node tree."""
    from neuronx_distributed_b200.utils.medusa_utils import generate_medusa_buffers

    buf = generate_medusa_buffers(MEDUSA_CHOICES, device=dev, topk=10)
    g = torch.Generator().manual_seed(0)
    mask, depth = torch.eye(64, dtype=torch.bool), torch.zeros(64, dtype=torch.long)
    for i in range(1, 64):
        par = int(torch.randint(0, i, (1,), generator=g))
        mask[i] |= mask[par]
        depth[i] = depth[par] + 1
    return [("chain5", None, None, 5), ("tree10", buf["medusa_attn_mask"][0, 0].bool(), buf["medusa_position_ids"].long(), 10),
            ("tree64", mask.to(dev), depth.to(dev), 64)]


def spec_perf():
    """``speculation_attention`` (kernel) against the path it replaces (de-quantise the whole cache, then the torch path),
    alternating in one process, on a full cache (p = L − W)."""
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    D, ks, vs = 128, 0.05, 0.05
    for name, B, L, H, Hkv, sw in SPEC_SHAPES:
        g = torch.Generator(device=dev).manual_seed(L + B)
        k8, v8 = ((torch.randn(B, L, Hkv, D, device=dev, generator=g) / s).to(torch.float8_e4m3fn) for s in (ks, vs))
        k16, v16 = (k8.float() * ks).bfloat16(), (v8.float() * vs).bfloat16()
        for wname, mask, depth, W in spec_windows(dev):
            q = torch.randn(B, W, H, D, device=dev, generator=g).bfloat16()
            pos = torch.full((B,), L - W, device=dev, dtype=torch.long)
            rows = L if sw is None else min(L, W + sw - 1)             # cache rows one sequence's tokens can see
            for cache in ("bf16", "e4m3"):
                kc, vc = (k16, v16) if cache == "bf16" else (k8, v8)
                kw = {} if cache == "bf16" else {"k_scale": ks, "v_scale": vs}

                def new():
                    return attention.speculation_attention(q, kc, vc, pos, mask, depth, sw, **kw)

                def old():
                    kd, vd = (kc, vc) if cache == "bf16" else ((kc.float() * ks).bfloat16(), (vc.float() * vs).bfloat16())
                    return attention.speculation_attention_torch(q, kd, vd, pos, mask, depth, sw)

                n0 = _ext.launches()
                o_new = new()
                assert _ext.launches() == n0 + 2, "the kernel did not run"
                o_old = old()
                err = ((o_new.float() - o_old.float()).abs().max() / o_old.float().abs().max()).item()
                t = {"new": [], "old": []}
                iters = 20 if B * L <= 32768 else 5
                for _ in range(3):                             # alternate, keep each one's best
                    t["new"].append(time_fn(new, iters))
                    t["old"].append(time_fn(old, iters))
                elt = 2 if cache == "bf16" else 1
                nbytes = 2 * B * rows * Hkv * D * elt + 2 * B * W * H * D * 2       # K and V rows read once, q and out
                rec = {"bench": f"{name}_spec_{wname}", "cache": cache, "B": B, "L": L, "H": H, "Hkv": Hkv, "W": W,
                       "sliding_window": sw, "bytes": nbytes, "rel_err_vs_old": round(err, 5)}
                for key in ("new", "old"):
                    ms = min(t[key])
                    rec[f"{key}_us"] = round(ms * 1e3, 1)
                    rec[f"{key}_GBps"] = round(nbytes / ms / 1e6, 1)
                rec["speedup"] = round(rec["old_us"] / rec["new_us"], 2)
                print(json.dumps(rec), flush=True)
            del q
        del k8, v8, k16, v16
        torch.cuda.empty_cache()


# name, H, Hkv, D
DECODE_DIM_SHAPES = [
    ("llama3.2_1b", 32, 8, 64),
    ("phi3_mini", 32, 32, 96),
    ("pythia2.8b", 32, 32, 80),
    ("mistral7b_control", 32, 8, 128),
]


# name, H, Hkv, D: the GQA groups 3, 5, 6 and 7 of --decode-groups
DECODE_GROUP_SHAPES = [
    ("llama3.2_3b", 24, 8, 128),
    ("qwen2.5_14b", 40, 8, 128),
    ("qwen2.5_1.5b", 12, 2, 128),
    ("qwen2.5_7b", 28, 4, 128),
    ("qwen2.5_7b_tp4", 7, 1, 128),
    ("qwen2.5_0.5b", 14, 2, 64),
]


def decode_dims_perf(shapes=DECODE_DIM_SHAPES, time_old=lambda D, B: D != 128 or B == 1):
    """Decode, verification and flash decoding's partial at head_dim 64 / 80 / 96 (and the D = 128 control) on the kernels
    against the torch paths those head sizes took before, alternating in one process, on a full cache (p = L − W).
    ``shapes`` / ``time_old(D, B)``: the geometries, and where the torch path is timed (--decode-groups: all of them)."""
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    ks, vs = 0.05, 0.05
    windows = [(n, m, d, W) for n, m, d, W in spec_windows(dev) if n != "tree10"]
    for name, H, Hkv, D in shapes:
        for L in (4096, 32768):
            for B in (1, 8, 32):
                if 2 * B * L * Hkv * D * 2 > 24 * 2 ** 30:                 # bf16 + e4m3 + de-quantised copies must fit
                    continue
                g = torch.Generator(device=dev).manual_seed(L + B + D)
                k8, v8 = ((torch.randn(B, L, Hkv, D, device=dev, generator=g) / s).to(torch.float8_e4m3fn) for s in (ks, vs))
                k16, v16 = (k8.float() * ks).bfloat16(), (v8.float() * vs).bfloat16()
                for wname, mask, depth, W in [("decode", None, None, 1)] + windows:
                    q = torch.randn(B, W, H, D, device=dev, generator=g).bfloat16()
                    pos = torch.full((B,), L - W, device=dev, dtype=torch.long)
                    for cache in ("bf16", "e4m3"):
                        kc, vc = (k16, v16) if cache == "bf16" else (k8, v8)
                        kw = {} if cache == "bf16" else {"k_scale": ks, "v_scale": vs}
                        if W == 1:
                            def new():
                                return attention.decode_attention(q, kc, vc, pos, **kw)
                        else:
                            def new():
                                return attention.speculation_attention(q, kc, vc, pos, mask, depth, **kw)

                        def old():
                            kd, vd = (kc, vc) if cache == "bf16" else ((kc.float() * ks).bfloat16(), (vc.float() * vs).bfloat16())
                            return attention.speculation_attention_torch(q, kd, vd, pos, mask, depth)

                        n0 = _ext.launches()
                        o_new = new()
                        assert _ext.launches() == n0 + 2, "the kernel did not run"
                        timed_old = time_old(D, B)
                        t = {"new": [], "old": []}
                        iters = 20 if B * L <= 32768 else 5
                        rec = {"bench": f"{name}_{wname}", "cache": cache, "B": B, "L": L, "H": H, "Hkv": Hkv, "D": D, "W": W}
                        if timed_old:
                            o_old = old()
                            rec["rel_err_vs_old"] = round(((o_new.float() - o_old.float()).abs().max()
                                                           / o_old.float().abs().max()).item(), 5)
                            del o_old
                        for _ in range(3):                         # alternate, keep each one's best
                            t["new"].append(time_fn(new, iters))
                            if timed_old:
                                t["old"].append(time_fn(old, iters))
                        elt = 2 if cache == "bf16" else 1
                        rec["kv_bytes"] = nbytes = 2 * B * L * Hkv * D * elt        # K and V rows, each read once
                        for key in ("new", "old"):
                            if not t[key]:
                                rec[f"{key}_us"] = "not measured"
                                continue
                            ms = min(t[key])
                            rec[f"{key}_us"] = round(ms * 1e3, 1)
                            rec[f"{key}_GBps"] = round(nbytes / ms / 1e6, 1)
                        if t["old"]:
                            rec["speedup"] = round(rec["old_us"] / rec["new_us"], 2)
                        print(json.dumps(rec), flush=True)
                    del q
                if L == 4096 and B == 8:                           # flash decoding's local partial: kernel vs fp32 torch math
                    q = torch.randn(B, 1, H, D, device=dev, generator=g).bfloat16()
                    local = torch.full((B,), L - 1, device=dev, dtype=torch.long)
                    for cache in ("bf16", "e4m3"):
                        kc, vc = (k16, v16) if cache == "bf16" else (k8, v8)
                        sc = (1.0, 1.0) if cache == "bf16" else (ks, vs)
                        new = lambda: _local_partial(q, kc, vc, local, 1.0 / math.sqrt(D), None, *sc)  # noqa: E731
                        old = lambda: _local_partial(q.float(), kc, vc, local, 1.0 / math.sqrt(D), None, *sc)  # noqa: E731
                        n0 = _ext.launches()
                        new()
                        assert _ext.launches() == n0 + 2, "the kernel did not run"
                        t = {"new": [], "old": []}
                        for _ in range(3):
                            t["new"].append(time_fn(new, 20))
                            t["old"].append(time_fn(old, 20))
                        nbytes = 2 * B * L * Hkv * D * (2 if cache == "bf16" else 1)
                        rec = {"bench": f"{name}_flash_decode_partial", "cache": cache, "B": B, "L": L, "H": H, "Hkv": Hkv, "D": D,
                               "kv_bytes": nbytes}
                        for key in ("new", "old"):
                            ms = min(t[key])
                            rec[f"{key}_us"] = round(ms * 1e3, 1)
                            rec[f"{key}_GBps"] = round(nbytes / ms / 1e6, 1)
                        rec["speedup"] = round(rec["old_us"] / rec["new_us"], 2)
                        print(json.dumps(rec), flush=True)
                    del q
                del k8, v8, k16, v16
                torch.cuda.empty_cache()


def _ring_of(lin: torch.Tensor, rows: int, end: int) -> torch.Tensor:
    """The rolling cache (``inference.kv_cache``) of ``rows`` rows holding positions < ``end`` of the linear cache ``lin``."""
    j = torch.arange(rows, device=lin.device)
    t = (end - 1 - (end - 1 - j) % rows).clamp(min=0)
    return lin[:, t].contiguous()


def rolling_perf(sw: int = 4096):
    """``decode_attention`` and ``speculation_attention`` on a rolling cache of SW + 64 rows against the linear 32k cache
    holding the same history, alternating in one process; outputs must be bit-identical."""
    dev = torch.device("cuda")
    print(json.dumps(gpu_info()), flush=True)
    D, H, Hkv, L, ks, vs = 128, 32, 8, 32768, 0.05, 0.05
    R = sw + attention.SPEC_MAX_TOKENS
    for B in (1, 8, 32):
        g = torch.Generator(device=dev).manual_seed(B)
        k8, v8 = ((torch.randn(B, L, Hkv, D, device=dev, generator=g) / s).to(torch.float8_e4m3fn) for s in (ks, vs))
        for cache in ("bf16", "e4m3"):
            kl, vl = (k8, v8) if cache == "e4m3" else ((k8.float() * ks).bfloat16(), (v8.float() * vs).bfloat16())
            kw = {} if cache == "bf16" else {"k_scale": ks, "v_scale": vs}
            elt = 2 if cache == "bf16" else 1
            for wname, mask, depth, W in [("decode", None, None, 1)] + spec_windows(dev):
                pos = torch.full((B,), L - W, device=dev, dtype=torch.long)
                kr, vr = _ring_of(kl, R, L), _ring_of(vl, R, L)
                q = torch.randn(B, W, H, D, device=dev, generator=g).bfloat16()
                if W == 1:
                    def call(kc, vc, roll):
                        return attention.decode_attention(q, kc, vc, pos, sliding_window=sw, rolling=roll, **kw)
                else:
                    def call(kc, vc, roll):
                        return attention.speculation_attention(q, kc, vc, pos, mask, depth, sw, rolling=roll, **kw)
                n0 = _ext.launches()
                equal = torch.equal(call(kl, vl, False), call(kr, vr, True))
                assert _ext.launches() == n0 + 4, "a kernel did not run"
                t = {"linear": [], "rolling": []}
                iters = max(20, 2000 // B)
                for _ in range(3):                             # alternate, keep each one's best
                    t["linear"].append(time_fn(lambda: call(kl, vl, False), iters))
                    t["rolling"].append(time_fn(lambda: call(kr, vr, True), iters))
                nbytes = 2 * B * (sw + W - 1) * Hkv * D * elt + 2 * B * W * H * D * 2    # visible K / V rows, q and out
                rec = {"bench": f"mistral7b_rolling_{wname}", "cache": cache, "B": B, "position": L - W, "W": W,
                       "sliding_window": sw, "linear_rows": L, "rolling_rows": R, "bit_equal": equal, "bytes": nbytes}
                for key in ("linear", "rolling"):
                    ms = min(t[key])
                    rec[f"{key}_us"] = round(ms * 1e3, 2)
                    rec[f"{key}_GBps"] = round(nbytes / ms / 1e6, 1)
                rec["rolling_over_linear"] = round(rec["rolling_us"] / rec["linear_us"], 3)
                print(json.dumps(rec), flush=True)
                del kr, vr
            del kl, vl
        del k8, v8
        torch.cuda.empty_cache()


def block_pairs(c: int, causal: bool, off: int, W) -> int:
    """Visible (query, key) pairs of one c × c CP block: all c² when dense, else i + off − W < j ≤ i + off (W None: no lower
    bound)."""
    if not causal:
        return c * c
    i = torch.arange(c, dtype=torch.int64)
    hi = torch.clamp(i + off, max=c - 1)
    lo = torch.zeros_like(i) if W is None else torch.clamp(i + off - W + 1, min=0)
    return int(torch.clamp(hi - lo + 1, min=0).sum())


def cp_window_perf(bwd: bool, cp: int, W: int = 4096):
    """Per-rank CP attention work of the windowed and the causal block plan (contiguous split), timed on one GPU when present."""
    from neuronx_distributed_b200.modules.attention.ring import _merge_block, _visible_pairs, block_attention, ring_hops

    B, H, Hkv, D = 1, 32, 8, 128
    scale = 1.0 / math.sqrt(D)
    gpu = torch.cuda.is_available()
    if gpu:
        print(json.dumps(gpu_info()), flush=True)
    for S in (32768, 65536, 131072):
        c = S // cp
        if gpu:
            g = torch.Generator(device="cuda").manual_seed(S)
            q, go = (torch.randn(B, c, H, D, device="cuda", generator=g).bfloat16() for _ in range(2))
            k, v = (torch.randn(B, S, Hkv, D, device="cuda", generator=g).bfloat16() for _ in range(2))
        for plan_name, window in (("window", W), ("causal", None)):
            plans = [_visible_pairs(r, cp, "contiguous", True, window, c) for r in range(cp)]
            work = [sum(block_pairs(c, bc, off, window) for _, _, _, bc, off in p) for p in plans]
            r = max(range(cp), key=lambda i: (work[i], i))
            hops = ring_hops(cp, c, window)
            rec = {"bench": "mistral7b_cp_window", "plan": plan_name, "cp": cp, "S": S, "chunk": c, "B": B, "H": H, "Hkv": Hkv,
                   "D": D, "W": W, "rank": r, "blocks": len(plans[r]), "visible_pairs": work[r] * H * B, "hops": hops,
                   "kv_bytes_sent_per_layer": hops * 2 * B * c * Hkv * D * 2, "nccl": "not measured (one-process emulation)"}
            fl = 4 * D * H * B * work[r]
            if gpu:
                qr = q.detach().requires_grad_(True)
                kv = [(k[:, src * c:(src + 1) * c], v[:, src * c:(src + 1) * c]) for _, src, _, _, _ in plans[r]]

                def fwd(plan=plans[r], kv=kv, window=window):
                    out = lse = None
                    for (_, _, _, bc, off), (kb, vb) in zip(plan, kv):
                        out, lse = _merge_block(out, lse, *block_attention(qr, kb, vb, bc, scale, window, off))
                    return out.to(q.dtype)

                def fwd_only():
                    with torch.no_grad():
                        fwd()

                def fwd_bwd():
                    fwd().backward(go)

                runs = {"fwd": fwd_only, "fwd_bwd": fwd_bwd if bwd else None}
                for key, fn in runs.items():
                    if fn is None:
                        continue
                    ms = min(time_fn(fn, 5) for _ in range(2))
                    rec[key + "_ms"] = round(ms, 3)
                    rec[key + "_tflops"] = round((3.5 if key == "fwd_bwd" else 1.0) * fl / ms / 1e9, 1)
            else:
                rec["fwd_ms"] = rec["fwd_bwd_ms"] = "not measured"
            print(json.dumps(rec), flush=True)
        if gpu:
            del q, go, k, v
            torch.cuda.empty_cache()


def time_fn(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--perf", action="store_true")
    ap.add_argument("--bwd", action="store_true")
    ap.add_argument("--window", action="store_true", help="with --perf: the sliding-window table instead of the model shapes")
    ap.add_argument("--cp", type=int, default=0, help="with --perf --window: the context-parallel block schedule at this CP size")
    ap.add_argument("--kv-fp8", action="store_true", help="with --perf: decode attention on bf16 vs fp8 e4m3 KV caches")
    ap.add_argument("--spec", action="store_true", help="with --perf: speculation / Medusa verification attention")
    ap.add_argument("--rolling", action="store_true", help="with --perf: decode / verification on rolling vs linear KV caches")
    ap.add_argument("--decode-dims", action="store_true",
                    help="with --perf: decode / verification / flash-decoding partial at head_dim 64, 80, 96 vs the torch path")
    ap.add_argument("--decode-groups", action="store_true",
                    help="with --perf: decode / verification / flash-decoding partial at GQA groups 3, 5, 6, 7 vs the torch path")
    ap.add_argument("--dropout", action="store_true", help="with --perf: attention dropout p = 0.1 vs p = 0 and SDPA")
    ap.add_argument("--head-dim", type=int, default=128, choices=attention.FLASH_HEAD_DIMS)
    a = ap.parse_args()
    if a.perf and a.window and a.cp > 1 and not torch.cuda.is_available():
        cp_window_perf(a.bwd, a.cp)                   # shapes only: pair and byte counts, times "not measured"
        return
    dev = torch.device("cuda")
    e = _ext.ext()
    ok_all = True
    torch.manual_seed(0)
    cases = [  # B, S, H, Hkv, causal, layout, masked (right padding)
        (1, 128, 1, 1, False, "bshd", False), (1, 256, 2, 2, True, "bshd", False), (2, 512, 4, 2, True, "sbhd", False),
        (2, 384, 4, 4, False, "bhsd", False), (1, 1024, 8, 8, True, "fused", False), (2, 200, 2, 1, True, "bshd", False),
        (3, 300, 4, 2, False, "bshd", True), (3, 300, 4, 2, True, "sbhd", True),
    ]
    for (B, S, H, Hkv, causal, layout, masked) in cases:
        D = a.head_dim
        if layout == "bshd":
            q = torch.randn(B, S, H, D, device=dev).bfloat16(); k = torch.randn(B, S, Hkv, D, device=dev).bfloat16()
            v = torch.randn(B, S, Hkv, D, device=dev).bfloat16()
        elif layout == "sbhd":
            q = torch.randn(S, B, H, D, device=dev).bfloat16().transpose(0, 1)
            k = torch.randn(S, B, Hkv, D, device=dev).bfloat16().transpose(0, 1)
            v = torch.randn(S, B, Hkv, D, device=dev).bfloat16().transpose(0, 1)
        elif layout == "bhsd":
            q = torch.randn(B, H, S, D, device=dev).bfloat16().transpose(1, 2)
            k = torch.randn(B, Hkv, S, D, device=dev).bfloat16().transpose(1, 2)
            v = torch.randn(B, Hkv, S, D, device=dev).bfloat16().transpose(1, 2)
        else:  # slices of one fused [S, B, (H+2Hkv)*D] projection output
            f = torch.randn(S, B, (H + 2 * Hkv) * D, device=dev).bfloat16()
            q = f[..., : H * D].view(S, B, H, D).transpose(0, 1)
            k = f[..., H * D:(H + Hkv) * D].view(S, B, Hkv, D).transpose(0, 1)
            v = f[..., (H + Hkv) * D:].view(S, B, Hkv, D).transpose(0, 1)
        q = q * 2.0      # larger logits → exercises the lazy rescale
        scale = 1.0 / math.sqrt(D)
        mask = None
        if masked:   # right padding; each row keeps at least its first key, so causal rows are never empty
            lens = torch.tensor([S, S - 77, 1][:B], device=dev)
            mask = torch.arange(S, device=dev)[None, :] < lens[:, None]
        o, lse = e.flash_attn_fwd(q, k, v, causal, scale, True, mask)
        ro, rl = ref_attn(q, k, v, causal, scale, mask)
        err = (o.float() - ro).abs().max().item() / ro.abs().max().item()
        lerr = (lse - rl).abs().max().item()
        ok = err < 2e-2 and lerr < 2e-2 and bool(torch.isfinite(o.float()).all())
        ok_all &= ok
        tag = f"D{D}_B{B}_S{S}_H{H}_{Hkv}_{'c' if causal else 'f'}_{layout}{'_masked' if masked else ''}"
        print(json.dumps({"check": f"fa_fwd_{tag}", "ok": ok,
                          "err": round(err, 5), "lse_err": round(lerr, 5)}), flush=True)
        if a.bwd and hasattr(e, "flash_attn_bwd"):
            go = torch.randn_like(o)
            qq, kk, vv = (t.detach().float().requires_grad_(True) for t in (q, k, v))
            r2, _ = ref_attn(qq, kk, vv, causal, scale, mask)
            r2.backward(go.float())
            dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True, None, mask)
            res = {}
            for n, g, r in (("dq", dq, qq.grad), ("dk", dk, kk.grad), ("dv", dv, vv.grad)):
                res[n] = round((g.float() - r).abs().max().item() / r.abs().max().item(), 5)
            ok = all(x < 3e-2 for x in res.values())
            ok_all &= ok
            print(json.dumps({"check": f"fa_bwd_{tag}", "ok": ok, **res}), flush=True)
    if a.perf:
        if a.kv_fp8:
            kv_fp8_perf()
        elif a.spec:
            spec_perf()
        elif a.rolling:
            rolling_perf()
        elif a.decode_dims:
            decode_dims_perf()
        elif a.decode_groups:
            decode_dims_perf(DECODE_GROUP_SHAPES, lambda D, B: True)
        elif a.dropout:
            dropout_perf(e, a.bwd)
        elif a.window and a.cp > 1:
            cp_window_perf(a.bwd, a.cp)
        else:
            (window_perf if a.window else perf)(e, a.bwd)
    print(json.dumps({"all_ok": ok_all}))
    sys.exit(0 if ok_all else 1)


if __name__ == "__main__":
    main()
