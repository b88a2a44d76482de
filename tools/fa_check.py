"""Numerics + timing of the flash-attention kernels against a plain fp32 PyTorch reference and SDPA (cuDNN).
usage: python tools/fa_check.py [--perf] [--bwd]"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuronx_distributed_b200.ops import _ext, attention  # noqa: E402


def ref_attn(q, k, v, causal, scale):
    # q [B,S,H,D] fp32 math
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
    p = s.softmax(-1)
    return (p @ vf).transpose(1, 2), torch.logsumexp(s, -1)


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
    a = ap.parse_args()
    dev = torch.device("cuda")
    e = _ext.ext()
    ok_all = True
    torch.manual_seed(0)
    cases = [  # B, S, H, Hkv, causal, layout
        (1, 128, 1, 1, False, "bshd"), (1, 256, 2, 2, True, "bshd"), (2, 512, 4, 2, True, "sbhd"),
        (2, 384, 4, 4, False, "bhsd"), (1, 1024, 8, 8, True, "fused"), (2, 200, 2, 1, True, "bshd"),
    ]
    for (B, S, H, Hkv, causal, layout) in cases:
        D = 128
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
        o, lse = e.flash_attn_fwd(q, k, v, causal, scale, True)
        ro, rl = ref_attn(q, k, v, causal, scale)
        err = (o.float() - ro).abs().max().item() / ro.abs().max().item()
        lerr = (lse - rl).abs().max().item()
        ok = err < 2e-2 and lerr < 2e-2 and bool(torch.isfinite(o.float()).all())
        ok_all &= ok
        print(json.dumps({"check": f"fa_fwd_B{B}_S{S}_H{H}_{Hkv}_{'c' if causal else 'f'}_{layout}", "ok": ok,
                          "err": round(err, 5), "lse_err": round(lerr, 5)}), flush=True)
        if a.bwd and hasattr(e, "flash_attn_bwd"):
            go = torch.randn_like(o)
            qq, kk, vv = (t.detach().float().requires_grad_(True) for t in (q, k, v))
            r2, _ = ref_attn(qq, kk, vv, causal, scale)
            r2.backward(go.float())
            dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True)
            res = {}
            for n, g, r in (("dq", dq, qq.grad), ("dk", dk, kk.grad), ("dv", dv, vv.grad)):
                res[n] = round((g.float() - r).abs().max().item() / r.abs().max().item(), 5)
            ok = all(x < 3e-2 for x in res.values())
            ok_all &= ok
            print(json.dumps({"check": f"fa_bwd_B{B}_S{S}_H{H}_{Hkv}_{'c' if causal else 'f'}_{layout}", "ok": ok, **res}), flush=True)
    if a.perf:
        for (B, S, H) in ((4, 4096, 32), (1, 8192, 32), (8, 2048, 32)):
            D = 128
            q, k, v = (torch.randn(B, S, H, D, device=dev).bfloat16() for _ in range(3))
            scale = 1.0 / math.sqrt(D)
            fl = 4 * B * H * S * S * D / 2
            t_own = time_fn(lambda: e.flash_attn_fwd(q, k, v, True, scale, True))
            qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
            t_lib = time_fn(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=True))
            rec = {"bench": f"fa_fwd_B{B}_S{S}_H{H}", "own_ms": round(t_own, 4), "own_tflops": round(fl / t_own / 1e9, 1),
                   "sdpa_ms": round(t_lib, 4), "sdpa_tflops": round(fl / t_lib / 1e9, 1)}
            if a.bwd and hasattr(e, "flash_attn_bwd"):
                o, lse = e.flash_attn_fwd(q, k, v, True, scale, True)
                go = torch.randn_like(o)
                t_b = time_fn(lambda: e.flash_attn_bwd(go, q, k, v, o, lse, True, scale, True))
                qr, kr, vr = (t.detach().requires_grad_(True) for t in (qt, kt, vt))
                oo = torch.nn.functional.scaled_dot_product_attention(qr, kr, vr, is_causal=True)
                got = go.transpose(1, 2)
                t_lb = time_fn(lambda: torch.autograd.grad(oo, (qr, kr, vr), got, retain_graph=True))
                rec.update({"own_bwd_ms": round(t_b, 4), "own_bwd_tflops": round(2.5 * fl / t_b / 1e9, 1),
                            "sdpa_bwd_ms": round(t_lb, 4), "sdpa_bwd_tflops": round(2.5 * fl / t_lb / 1e9, 1)})
            print(json.dumps(rec), flush=True)
    print(json.dumps({"all_ok": ok_all}))
    sys.exit(0 if ok_all else 1)


if __name__ == "__main__":
    main()
