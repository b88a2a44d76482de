"""Single-GPU loopback: TWO processes on cuda:0 run the cross-rank kernels against each other (a one-GPU `pytest -m gpu`
then exercises the flag / epoch protocols of the NVLS-layout collectives and the symmetric-memory exchange instead of
skipping them; the fused TP GEMMs have their own file, test_tp_gemm_collectives_gpu.py).  No multicast mapping exists
between two contexts of one device, so the NVLS kernels run their unicast fallback (same protocol, peer pointers instead of
the multicast address); the references are plain fp32 matmuls computed locally — every rank can rebuild all ranks' inputs from the seeds, no library collective is involved."""
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
