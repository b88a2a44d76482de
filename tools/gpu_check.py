"""On-GPU numerics + timing smoke for every hand-written kernel (run under gpurun).

usage: python tools/gpu_check.py [elementwise|gemm|gemm_perf|decode|fp8|fp8_block|grouped|all]
(gemm / decode / fp8 / grouped given by name also run their timing entries; fp8_block is timing only, its numerics are
in tests/test_fp8_blockscaled_gpu.py)
Each check prints one line `CHECK name PASS/FAIL max_err=…`; results are also appended to
gpurun_out/gpu_check.jsonl.  Comparison target is always a plain PyTorch fp32 reference."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuronx_distributed_b200 import ops  # noqa: E402

OUT = os.path.join(os.environ.get("GRAFT_REPO_ROOT", "."), "gpurun_out")
os.makedirs(OUT, exist_ok=True)
dev = torch.device("cuda")
RESULTS = []


def report(name, ok, **kw):
    rec = {"name": name, "ok": bool(ok), **{k: (float(v) if isinstance(v, (int, float)) else v) for k, v in kw.items()}}
    RESULTS.append(rec)
    print("CHECK", name, "PASS" if ok else "FAIL", " ".join(f"{k}={v}" for k, v in kw.items()), flush=True)
    with open(os.path.join(OUT, "gpu_check.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")


def relerr(a, b):
    a, b = a.float(), b.float()
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def timeit(fn, iters=20, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    times = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2]


def check_elementwise():
    torch.manual_seed(0)
    T, H = 1024, 4096
    for dt in (torch.bfloat16, torch.float32):
        x = torch.randn(T, H, device=dev, dtype=dt)
        w = (torch.rand(H, device=dev) + 0.5).to(dt)
        xr, wr = x.detach().float().clone().requires_grad_(True), w.detach().float().clone().requires_grad_(True)
        ref = (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5) * wr)
        g = torch.randn_like(ref)
        ref.backward(g)
        xx, ww = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
        y = ops.norm.rms_norm(xx, ww, 1e-5)
        y.backward(g.to(dt))
        tol = 2e-2 if dt == torch.bfloat16 else 1e-5
        report(f"rmsnorm_fwd_{dt}", relerr(y, ref) < tol, err=relerr(y, ref))
        report(f"rmsnorm_dx_{dt}", relerr(xx.grad, xr.grad) < tol, err=relerr(xx.grad, xr.grad))
        report(f"rmsnorm_dw_{dt}", relerr(ww.grad, wr.grad) < tol, err=relerr(ww.grad, wr.grad))
    # swiglu
    gu = torch.randn(T, 2 * 2752, device=dev, dtype=torch.bfloat16)
    gur = gu.float().requires_grad_(True)
    a, b = gur.chunk(2, -1)
    ref = torch.nn.functional.silu(a) * b
    g = torch.randn_like(ref)
    ref.backward(g)
    gg = gu.clone().requires_grad_(True)
    y = ops.act.swiglu(gg)
    y.backward(g.bfloat16())
    report("swiglu_fwd", relerr(y, ref) < 2e-2, err=relerr(y, ref))
    report("swiglu_bwd", relerr(gg.grad, gur.grad) < 2e-2, err=relerr(gg.grad, gur.grad))
    # rope on a transposed [S,B,h,D] view
    S, B, Hh, D = 512, 2, 4, 128
    base = torch.randn(S, B, Hh * D, device=dev, dtype=torch.bfloat16)
    q = base.view(S, B, Hh, D).transpose(0, 1)
    cos, sin = ops.rope.rope_tables(S, D, device=dev)
    from neuronx_distributed_b200.ops.rope import rotate
    qq = q.detach().clone().requires_grad_(True)
    out = ops.rope.apply_rotary(qq, cos, sin)
    ref = rotate(q.float(), cos, sin)
    report("rope_fwd", relerr(out, ref) < 2e-2, err=relerr(out, ref))
    g = torch.randn_like(out)
    out.backward(g)
    refb = rotate(g.float(), cos, sin, -1.0)
    report("rope_bwd", relerr(qq.grad, refb) < 2e-2, err=relerr(qq.grad, refb))
    # cross entropy
    for V, dt in ((4000, torch.bfloat16), (32000, torch.float32)):
        Tt = 512
        logits = torch.randn(Tt, V, device=dev, dtype=dt) * 3
        tgt = torch.randint(0, V, (Tt,), device=dev)
        lr = logits.float().requires_grad_(True)
        ref = torch.nn.functional.cross_entropy(lr, tgt, reduction="none")
        ref.sum().backward()
        st = ops.cross_entropy.ce_stats(logits, tgt, 0)
        lse = st[:, 0] + torch.log(st[:, 1])
        loss = lse - st[:, 2]
        report(f"ce_stats_V{V}", relerr(loss, ref) < (2e-2 if dt == torch.bfloat16 else 1e-4), err=relerr(loss, ref))
        gr = ops.cross_entropy.ce_backward(logits, tgt, lse, torch.ones(Tt, device=dev), 0, 0.0, V)
        report(f"ce_bwd_V{V}", relerr(gr, lr.grad) < (2e-2 if dt == torch.bfloat16 else 1e-4), err=relerr(gr, lr.grad))
    # multi tensor ops + adamw
    ts = [torch.randn(n, device=dev, dtype=torch.bfloat16) for n in (5, 1000, 65536 * 3 + 17, 4096 * 4096)]
    ref = sum(t.float().pow(2).sum() for t in ts)
    got = ops.optim.multi_tensor_sq_norm(ts)
    report("multi_sq_norm", abs(float(got) - float(ref)) / float(ref) < 1e-3, got=float(got), ref=float(ref))
    ts2 = [t.clone() for t in ts]
    ops.optim.multi_tensor_scale_(ts2, torch.tensor(0.5, device=dev))
    report("multi_scale", all(relerr(a, b.float() * 0.5) < 1e-2 for a, b in zip(ts2, ts)))
    n = 65536 * 2 + 33
    p = torch.randn(n, device=dev); g = torch.randn(n, device=dev, dtype=torch.bfloat16)
    m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev); low = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    pr, mr, vr = p.clone(), m.clone(), v.clone()
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    ops.optim.fused_adamw_([p], [g], [m], [v], 1e-2, 0.9, 0.95, 1e-8, 0.1, 1, torch.tensor(0.7, device=dev), [low],
                           hf_form=False)
    g32 = g.float() * 0.7
    pr.mul_(1 - 1e-2 * 0.1); mr.mul_(0.9).add_(g32, alpha=0.1); vr.mul_(0.95).addcmul_(g32, g32, value=0.05)
    pr.addcdiv_(mr / (1 - 0.9), (vr / (1 - 0.95)).sqrt() + 1e-8, value=-1e-2)
    report("fused_adamw", relerr(p, pr) < 1e-5 and relerr(low, pr) < 1e-2, perr=relerr(p, pr), lowerr=relerr(low, pr))
    # HF form (the reference optimizer's update): eps before bias correction, decay last; 3 steps
    ph = p2.clone()
    for step in (1, 2, 3):
        ops.optim.fused_adamw_([p2], [g], [m2], [v2], 1e-2, 0.9, 0.95, 1e-3, 0.1, step, None, None, hf_form=True)
    mh = torch.zeros_like(ph); vh = torch.zeros_like(ph); gf = g.float()
    for step in (1, 2, 3):
        mh.mul_(0.9).add_(gf, alpha=0.1); vh.mul_(0.95).addcmul_(gf, gf, value=0.05)
        ph.addcdiv_(mh, vh.sqrt() + 1e-3, value=-1e-2 * (1 - 0.95 ** step) ** 0.5 / (1 - 0.9 ** step))
        ph.add_(ph, alpha=-1e-2 * 0.1)
    report("fused_adamw_hf", relerr(p2, ph) < 1e-5, perr=relerr(p2, ph))


def check_gemm(perf=False):
    torch.manual_seed(0)
    shapes = [(128, 256, 64), (256, 512, 256), (384, 768, 192), (4096, 1536, 4096), (512, 4096, 1376), (1000, 264, 72)]
    for (M, N, K) in shapes:
        for ta, tb in ((False, True), (False, False), (True, False)):
            a = torch.randn((K, M) if ta else (M, K), device=dev, dtype=torch.bfloat16)
            b = torch.randn((N, K) if tb else (K, N), device=dev, dtype=torch.bfloat16)
            ref = (a.float().t() if ta else a.float()) @ (b.float().t() if tb else b.float())
            try:
                out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                ops._ext.ext().gemm_bf16(a, b, out, ta, tb, False)
                torch.cuda.synchronize()
                err = relerr(out, ref)
                report(f"gemm_{M}x{N}x{K}_ta{int(ta)}_tb{int(tb)}", err < 1e-2, err=err)
            except Exception as e:  # noqa: BLE001
                report(f"gemm_{M}x{N}x{K}_ta{int(ta)}_tb{int(tb)}", False, exc=repr(e)[:200])
    # fp32 out + accumulate
    M, N, K = 256, 512, 128
    a = torch.randn(M, K, device=dev, dtype=torch.bfloat16); b = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
    out = torch.ones(M, N, device=dev, dtype=torch.float32)
    ops._ext.ext().gemm_bf16(a, b, out, False, True, True)
    ref = a.float() @ b.float().t() + 1
    report("gemm_f32_accumulate", relerr(out, ref) < 1e-3, err=relerr(out, ref))


def _gpu_info(query="name,power.limit,clocks.sm,clocks.max.sm"):
    import subprocess

    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True)
    lines = r.stdout.strip().splitlines()
    return lines[0] if lines else torch.cuda.get_device_name()


def check_gemm_perf():
    """The bf16 GEMM at the Llama-2-7B training step's shapes (4096 tokens) in its three layouts: `nt` forward
    x[M, K]·W[N, K]ᵀ, `nn` the same product with W stored [K, N], and `tn` weight gradient gᵀ·x into an fp32 [N, K] out, once
    storing and once accumulating (as into ZeRO-1's main_grad).  cuBLAS through torch where it has the same product."""
    report("gpu_info", True, gpu=_gpu_info())
    e = ops._ext.ext()
    M = 4096
    bf = dict(device=dev, dtype=torch.bfloat16)
    for (N, K) in [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008), (32000, 4096)]:
        fl = 2.0 * M * N * K
        x = torch.randn(M, K, **bf)
        w = torch.randn(N, K, **bf)
        y = torch.empty(M, N, **bf)
        rows = {"nt": (timeit(lambda: e.gemm_bf16(x, w, y, False, True, False)), timeit(lambda: torch.matmul(x, w.t())))}
        wkn = w.t().contiguous()
        rows["nn"] = (timeit(lambda: e.gemm_bf16(x, wkn, y, False, False, False)), timeit(lambda: torch.matmul(x, wkn)))
        del wkn, y
        g = torch.randn(M, N, **bf)
        dw = torch.zeros(N, K, device=dev, dtype=torch.float32)
        try:
            lib = timeit(lambda: torch.mm(g.t(), x, out_dtype=torch.float32))
        except (RuntimeError, TypeError):
            lib = None
        rows["tn_store"] = (timeit(lambda: e.gemm_bf16(g, x, dw, True, False, False)), lib)
        rows["tn_accumulate"] = (timeit(lambda: e.gemm_bf16(g, x, dw, True, False, True)), None)
        clk = _gpu_info("clocks.sm")
        for layout, (t_own, t_lib) in rows.items():
            extra = {} if t_lib is None else {"cublas_ms": t_lib, "cublas_tflops": fl / t_lib / 1e9}
            report(f"gemm_perf_{layout}_M{M}_N{N}_K{K}", True, own_ms=t_own, own_tflops=fl / t_own / 1e9, sm_clock=clk, **extra)
        del g, dw, x, w


def check_decode(perf=False):
    """Decode kernels: flash-decoding attention vs fp32 softmax over the valid cache prefix; GEMV vs fp32 matmul."""
    import math
    e = ops._ext.ext()
    torch.manual_seed(0)
    for (B, L, H, Hkv) in [(1, 300, 8, 8), (3, 2048, 8, 2), (2, 1000, 16, 2), (4, 129, 4, 4)]:
        D = 128
        q = torch.randn(B, 1, H, D, device=dev).bfloat16()
        k = torch.randn(B, L, Hkv, D, device=dev).bfloat16(); v = torch.randn(B, L, Hkv, D, device=dev).bfloat16()
        pos = torch.randint(0, L, (B,), device=dev)
        o = e.decode_attention(q, k, v, pos, 1.0 / math.sqrt(D))
        G = H // Hkv
        kf, vf = k.float().repeat_interleave(G, 2), v.float().repeat_interleave(G, 2)
        sc = torch.einsum("bhd,blhd->bhl", q.float()[:, 0], kf) / math.sqrt(D)
        mask = torch.arange(L, device=dev)[None, None, :] <= pos[:, None, None]
        ref = torch.einsum("bhl,blhd->bhd", sc.masked_fill(~mask, float("-inf")).softmax(-1), vf)
        report(f"decode_attn_B{B}_L{L}_H{H}_{Hkv}", relerr(o[:, 0], ref) < 1e-2, err=relerr(o[:, 0], ref))
    for (M, N, K) in [(1, 4096, 4096), (4, 11008, 4096), (8, 1000, 264), (2, 32000, 5120)]:
        x = torch.randn(M, K, device=dev).bfloat16(); w = (torch.randn(N, K, device=dev) / K ** 0.5).bfloat16()
        r = torch.randn(M, N, device=dev).bfloat16()
        y = e.gemv(x, w, r)
        ref = x.float() @ w.float().t() + r.float()
        report(f"gemv_{M}x{N}x{K}", relerr(y, ref) < 1e-2, err=relerr(y, ref))
    if perf:
        N, K = 13824, 5120
        x = torch.randn(1, K, device=dev).bfloat16(); w = torch.randn(N, K, device=dev).bfloat16()
        t = timeit(lambda: e.gemv(x, w, None)); t2 = timeit(lambda: torch.matmul(x, w.t()))
        report("gemv_perf_13b_mlp", True, own_us=t * 1e3, own_gbs=N * K * 2 / t / 1e6, cublas_us=t2 * 1e3)
        B, L, H, Hkv = 1, 2048, 40, 40
        q = torch.randn(B, 1, H, 128, device=dev).bfloat16(); k = torch.randn(B, L, Hkv, 128, device=dev).bfloat16(); v = torch.randn_like(k)
        pos = torch.full((B,), L - 1, device=dev)
        t = timeit(lambda: e.decode_attention(q, k, v, pos, 0.088))
        report("decode_attn_perf_13b", True, own_us=t * 1e3, gbs=2 * L * Hkv * 256 / t / 1e6)


def check_fp8(perf=False):
    """fp8 (e4m3) wgmma GEMM with row/column scales vs the fp32 product of the same quantised operands."""
    from neuronx_distributed_b200.ops import gemm_fp8

    torch.manual_seed(0)
    for (M, N, K) in [(128, 256, 128), (200, 264, 208), (1024, 4096, 4096), (8, 512, 1024)]:
        xq = torch.randn(M, K, device=dev).to(torch.float8_e4m3fn)
        wq = torch.randn(N, K, device=dev).to(torch.float8_e4m3fn)
        xs = torch.rand(M, device=dev) + 0.5
        ws = torch.rand(N, device=dev) + 0.5
        y = gemm_fp8.scaled_linear(xq, xs, wq, ws)
        ref = (xq.float() @ wq.float().t()) * xs[:, None] * ws[None, :]
        report(f"gemm_fp8_{M}x{N}x{K}", relerr(y, ref) < 1e-2, err=relerr(y, ref))
    if perf:
        M, N, K = 8192, 8192, 8192
        xq = torch.randn(M, K, device=dev).to(torch.float8_e4m3fn); wq = torch.randn(N, K, device=dev).to(torch.float8_e4m3fn)
        xs = torch.ones(M, device=dev); ws = torch.ones(N, device=dev)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        t = timeit(lambda: ops._ext.ext().gemm_fp8(xq, wq, out, xs, ws))
        report("gemm_fp8_perf_8192", True, ms=t, tflops=2.0 * M * N * K / t / 1e9)


def _fp8_codes(*shape):
    return (torch.randn(*shape, device=dev) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)


def check_fp8_block_perf():
    """Block-scaled fp8 GEMM at G = 128 / 32 vs the per-row fp8 GEMM, the bf16 GEMM and today's block-wise path
    (de-quantise the weight to bf16 + dense GEMM), at 8192³ and Llama-2-7B prefill shapes (4096 tokens)."""
    import subprocess

    from neuronx_distributed_b200.ops import gemm_fp8
    from neuronx_distributed_b200.quantization.dequantize import blockwise_scale_dequantize

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    report("gpu_info", True, gpu=gpu[0] if gpu else torch.cuda.get_device_name())
    e = ops._ext.ext()
    torch.manual_seed(0)
    for (M, N, K) in [(8192, 8192, 8192), (4096, 4096, 4096), (4096, 12288, 4096), (4096, 22016, 4096), (4096, 4096, 11008)]:
        x = torch.randn(M, K, device=dev).bfloat16()
        wq = _fp8_codes(N, K)
        fl = 2.0 * M * N * K
        res = {}
        for G in (128, 32):
            xq, xs = gemm_fp8.quantize_groups(x, G)
            sa = xs.t()
            sb = gemm_fp8.weight_scales_kn(torch.rand(N, K // G, device=dev), N, K, G)
            res[f"block_g{G}"] = timeit(lambda: e.gemm_fp8_block(xq, wq, sa, sb, G))
        res["quant_g128"] = timeit(lambda: e.quantize_fp8_groups(x, 128, False, float("inf")))
        xq1 = x.to(torch.float8_e4m3fn)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        ones_m, ones_n = torch.ones(M, device=dev), torch.ones(N, device=dev)
        res["fp8_rowscale"] = timeit(lambda: e.gemm_fp8(xq1, wq, out, ones_m, ones_n))
        wb = wq.bfloat16()
        res["bf16"] = timeit(lambda: e.gemm_bf16(x, wb, out, False, True, False))
        ws128 = torch.rand(N, K // 128, device=dev)
        res["dequant_bf16"] = timeit(lambda: torch.nn.functional.linear(x, blockwise_scale_dequantize(wq, ws128, torch.bfloat16)))
        report(f"fp8_block_perf_{M}x{N}x{K}", True, **{f"{k}_ms": v for k, v in res.items()},
               **{f"{k}_tflops": fl / v / 1e9 for k, v in res.items() if k != "quant_g128"})


def check_grouped(perf=False):
    """Grouped (MoE blockwise) GEMMs: forward, dgrad and segmented wgrad vs fp32 einsum, through the autograd front-end."""
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata

    torch.manual_seed(0)
    for (T, k, E, H, I, bs) in [(300, 2, 4, 256, 512, 128), (1000, 2, 8, 512, 1024, 256), (64, 1, 8, 128, 192, 128)]:
        idx = torch.stack([torch.randperm(E, device=dev)[:k] for _ in range(T)])
        b2e, tp2id, counts = build_block_metadata(idx, E, bs)
        bpe = (counts + bs - 1) // bs
        seg = torch.cat([bpe.new_zeros(1), torch.cumsum(bpe, 0)])
        nb = b2e.numel()
        valid = (tp2id >= 0).unsqueeze(-1)
        x = (torch.randn(nb * bs, H, device=dev) * valid).bfloat16().requires_grad_(True)
        w = (torch.randn(E, H, I, device=dev) / H ** 0.5).bfloat16().requires_grad_(True)
        y = ops.gemm.grouped_matmul(x, w, b2e, seg, bs)
        gy = (torch.randn_like(y) * valid).bfloat16()
        y.backward(gy)
        xf, wf = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
        yr = torch.einsum("bth,bhi->bti", xf.view(nb, bs, H), wf[b2e.long()]).reshape(nb * bs, I)
        yr.backward(gy.float())
        e = (relerr(y, yr), relerr(x.grad, xf.grad), relerr(w.grad, wf.grad))
        report(f"grouped_gemm_T{T}_E{E}_H{H}_I{I}_b{bs}", max(e) < 2e-2, y=e[0], dx=e[1], dw=e[2])
    if perf:
        T, k, E, H, I, bs = 16384, 2, 8, 4096, 14336 * 2, 256          # Mixtral-8x7B gate_up, one 16k-token micro-batch
        idx = torch.stack([torch.randperm(E, device=dev)[:k] for _ in range(T)])
        b2e, tp2id, counts = build_block_metadata(idx, E, bs)
        bpe = (counts + bs - 1) // bs
        seg = torch.cat([bpe.new_zeros(1), torch.cumsum(bpe, 0)]).int()
        nb = b2e.numel()
        x = torch.randn(nb * bs, H, device=dev).bfloat16()
        w = torch.randn(E, H, I, device=dev).bfloat16()
        t = timeit(lambda: ops._ext.ext().grouped_gemm(x, w, b2e.int(), bs, False))
        report("grouped_gemm_perf_mixtral_gate_up", True, ms=t, tflops=2.0 * nb * bs * H * I / t / 1e9)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    assert ops.extension_available(), ops._ext.load_error()
    if what in ("elementwise", "all"):
        check_elementwise()
    if what in ("gemm", "all"):
        check_gemm()
    if what in ("decode", "all"):
        check_decode(perf=what == "decode")
    if what in ("fp8", "all"):
        check_fp8(perf=what == "fp8")
    if what == "fp8_block":                       # numerics: tests/test_fp8_blockscaled_gpu.py
        check_fp8_block_perf()
    if what in ("grouped", "all"):
        check_grouped(perf=what == "grouped")
    if what in ("gemm", "gemm_perf", "all"):
        check_gemm_perf()
    bad = [r["name"] for r in RESULTS if not r["ok"]]
    print("SUMMARY", len(RESULTS) - len(bad), "passed,", len(bad), "failed", bad, flush=True)
