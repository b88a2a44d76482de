"""Single-GPU loopback: TWO processes on cuda:0 run the cross-rank kernels against each other (the driver's 1-GPU `pytest -m gpu`
then exercises the flag / epoch protocols of the fused TP kernels, the NVLS-layout collectives and the symmetric-memory
exchange instead of skipping them).  No multicast mapping exists between two contexts of one device, so the NVLS kernels run
their unicast fallback (same protocol, peer pointers instead of the multicast address); the references are plain fp32 matmuls
computed locally — every rank can rebuild all ranks' inputs from the seeds, no library collective is involved."""
import pytest
import torch

from dist_utils import run_distributed

pytestmark = pytest.mark.gpu


def _inputs(rank_like, shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed * 97 + rank_like)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _relerr(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6))


def _symm_and_collectives(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import nvls, symm

    g = dist.group.WORLD
    ws = symm.get_vmm_workspace(g, "loopback_probe", 8 << 20)
    assert not ws.has_multicast and len(ws.ptr_list) == world and ws.ptr_list[rank] == ws.local_ptr
    for it in range(3):                                   # epochs / parity halves
        xs = [_inputs(r, (1 << 16,), 10 + it) for r in range(world)]
        ref = sum(x.float() for x in xs)
        y = nvls.all_reduce_sum(xs[rank], g)
        assert _relerr(y, ref) < 1e-2
        yg = nvls.all_gather(xs[rank], g)
        assert torch.equal(yg, torch.cat(xs))
        big = [_inputs(r, (world * 4096,), 20 + it) for r in range(world)]
        yr = nvls.reduce_scatter_sum(big[rank], g)
        refr = sum(b.float() for b in big)[rank * 4096:(rank + 1) * 4096]
        assert _relerr(yr, refr) < 1e-2
    # fused decode GEMV + all-reduce
    w = [_inputs(r, (512, 256), 31, 0.05) for r in range(world)]
    x = [_inputs(r, (2, 256), 32) for r in range(world)]
    y = nvls.gemv_all_reduce(x[rank], w[rank], g)
    ref = sum(xx.float() @ ww.float().t() for xx, ww in zip(x, w))
    assert _relerr(y, ref) < 1e-2


def test_loopback_symmetric_memory_and_collectives():
    run_distributed(_symm_and_collectives, 2, use_cuda="loopback", timeout=240)


def _fused_tp(rank, world):
    import os

    os.environ["NXD_TP_NVLS"] = "force"
    os.environ["NXD_SYMM_MIN_MB"] = "1"                    # small floor: the shapes below force re-layouts of the region
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import _fused_impl

    _fused_impl._NVLS_MODE = "force"
    ws = _fused_impl.workspace(dist.group.WORLD)
    assert ws.nvls_enabled() and not ws.nv.has_multicast
    for wire in ("bf16", "fp32"):
        os.environ["NXD_TP_WIRE"] = wire
        # (rows per rank, N, K, trans_b): trans_b=False is the [K, N] MN-major weight operand of the backward (dgrad)
        cases = [(256, 512, 256, True), (512, 1000, 512, True), (256, 512, 256, True), (128, 384, 256, True),
                 (128, 256, 384, False), (256, 512, 256, False)]
        for it, (ms, N, K, tb) in enumerate(cases):
            xs = [_inputs(r, (ms, K), 40 + it) for r in range(world)]
            w = _inputs(0, (N, K) if tb else (K, N), 50 + it, 0.05)
            wt = w.float().t() if tb else w.float()
            out, gathered = ws.ag_gemm(xs[rank], w, tb)
            full = torch.cat(xs)
            assert torch.equal(gathered, full)
            assert _relerr(out, full.float() @ wt) < 2e-2, (wire, it)
            # GEMM → reduce-scatter: every rank has its own [world*ms, K] operand
            a = [_inputs(r, (world * ms, K), 60 + it) for r in range(world)]
            o = ws.gemm_rs(a[rank], w, tb)
            ref = sum(x.float() @ wt for x in a)[rank * ms:(rank + 1) * ms]
            assert _relerr(o, ref) < 2e-2, (wire, it)
    os.environ["NXD_TP_WIRE"] = "bf16"
    # a larger shape mid-stream re-lays the region out (barrier, epochs keep counting) and must keep working, first call included
    xs = [_inputs(r, (2048, 1024), 70) for r in range(world)]
    w = _inputs(0, (512, 1024), 71, 0.05)
    out, _ = ws.ag_gemm(xs[rank], w, True)
    assert _relerr(out, torch.cat(xs).float() @ w.float().t()) < 2e-2


def test_loopback_fused_tp_kernels_vs_fp32_reference():
    run_distributed(_fused_tp, 2, use_cuda="loopback", timeout=300)
