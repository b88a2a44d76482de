"""Run a function on N local processes (gloo on CPU / nccl on GPUs) — the analogue of the
reference's ``NXD_CPU_MODE=1 torchrun --nproc-per-node=N`` integration tier (SURVEY §4)."""
from __future__ import annotations

import os
import socket
import sys
import traceback

import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MIN = 2.0 ** -126                           # smallest normal fp32 (and bf16)


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, fn, args, use_cuda, errq):
    try:
        if ROOT not in sys.path:
            sys.path.insert(0, ROOT)
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
        import torch.distributed as dist

        if use_cuda == "loopback":
            # every rank on cuda:0 — NCCL refuses two ranks on one device, so the control plane is gloo; the peer-memory
            # kernels (VMM fd exchange / cudaIpc both work intra-device) run their real flag / epoch protocols between the
            # two processes' contexts, which the GPU time-slices
            torch.cuda.set_device(0)
            os.environ["NXD_LOOPBACK"] = "1"
            dist.init_process_group("gloo", rank=rank, world_size=world)
        elif use_cuda:
            torch.cuda.set_device(rank)
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        else:
            os.environ["NXD_CPU_MODE"] = "1"
            torch.set_num_threads(1)
            dist.init_process_group("gloo", rank=rank, world_size=world)
        try:
            fn(rank, world, *args)
        finally:
            from neuronx_distributed_b200.parallel_layers import parallel_state as ps

            if ps.model_parallel_is_initialized():
                ps.destroy_model_parallel()
            dist.destroy_process_group()
    except Exception:
        errq.put((rank, traceback.format_exc()))
        raise


def run_distributed(fn, world: int, *args, use_cuda: bool = False, timeout: float = 300.0):
    if not use_cuda:
        # CPU workers re-import torch in every spawned process (slow on a cold or busy box): callers' tighter limits are floors
        timeout = max(float(timeout), 300.0)
    ctx = mp.get_context("spawn")
    errq = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, fn, args, use_cuda, errq)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout)
    alive = [p for p in procs if p.is_alive()]
    for p in alive:
        p.terminate()
    errs = []
    while not errq.empty():
        errs.append(errq.get())
    if errs:
        raise AssertionError("worker failure:\n" + "\n".join(f"[rank {r}]\n{tb}" for r, tb in errs))
    assert not alive, "distributed test timed out"
    for p in procs:
        assert p.exitcode == 0, f"worker exit code {p.exitcode}"


# ---------------------------------------------------------------------------------------------------------------------
# Bit-exact checks of the peer-memory kernels run by loopback workers: inputs from seeds, fp32 emulation in a given order,
# bit comparison, failures collected until every rank has made its whole call sequence
# ---------------------------------------------------------------------------------------------------------------------
def _randn(n, seed, dtype, spread=12):
    """``n`` normal numbers of ``dtype``: Gaussian times 2^k, k uniform in [-spread, spread], so that fp32 sums of a few of
    them round and the summation order shows in the last bit."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, device="cuda", generator=g)
    if spread:
        x = x * torch.exp2(torch.randint(-spread, spread + 1, (n,), device="cuda", generator=g).float())
    x = x.to(dtype)
    return torch.where(x.float().abs() < FLT_MIN, torch.ones_like(x), x)


def _emulate(parts, order):
    """fp32 sum of ``parts[p]`` for p in ``order``, starting from +0, inputs flushed to zero below FLT_MIN as the kernels'
    FTZ adds do."""
    acc = torch.zeros(parts[0].shape, dtype=torch.float32, device=parts[0].device)
    for p in order:
        x = parts[p].float()
        acc = acc + torch.where(x.abs() < FLT_MIN, torch.zeros_like(x), x)
    return acc


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _same(a, b):
    """Bit for bit, except that any NaN equals any NaN (the payload is not compared)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    an, bn = torch.isnan(a), torch.isnan(b)
    return torch.equal(an, bn) and torch.equal(_bits(a)[~an], _bits(b)[~bn])


def _first_diff(a, b):
    a, b = a.reshape(-1), b.reshape(-1)
    d = (_bits(a) != _bits(b)).nonzero().reshape(-1)
    if d.numel() == 0:
        return "NaN positions differ"
    i = int(d[0])
    return f"{d.numel()} elements differ, first at {i}: {a[i].item()!r} vs {b[i].item()!r}"


class _Checks:
    """Collects failures instead of raising, so that no rank leaves the call sequence early (its peers would wait on its
    flags); ``settle`` compares the failures of all ranks over gloo and raises on every rank if there is one."""

    def __init__(self):
        self.errs = []

    def same(self, got, want, what):
        if not _same(got, want):
            self.errs.append(f"{what}: {_first_diff(got, want) if got.shape == want.shape else 'shape/dtype'}")

    def true(self, ok, what):
        if not ok:
            self.errs.append(what)

    def settle(self):
        import torch.distributed as dist

        torch.cuda.synchronize()
        every = [None] * dist.get_world_size()
        dist.all_gather_object(every, self.errs)
        bad = [f"rank {r}: {e}" for r, es in enumerate(every) for e in es]
        assert not bad, "\n".join(bad[:40])
