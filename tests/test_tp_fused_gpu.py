"""Fused GEMM+collective kernels over NVLink peer memory vs the NCCL + matmul path (>= 2 GPUs)."""
import pytest
import torch

from dist_utils import run_distributed

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _fused_vs_nccl(rank, world):
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.parallel_layers import ColumnParallelLinear, RowParallelLinear
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    dev = torch.device("cuda", rank)
    torch.manual_seed(5)
    S, B, H, I = 256 * world, 1, 1024, 2048
    col = ColumnParallelLinear(H, I, bias=False, gather_output=False, sequence_parallel_enabled=True, dtype=torch.bfloat16,
                               device=dev)
    row = RowParallelLinear(I, H, bias=False, input_is_parallel=True, sequence_parallel_enabled=True,
                            dtype=torch.bfloat16, device=dev)
    torch.manual_seed(100 + rank)
    x0 = torch.randn(S // world, B, H, device=dev, dtype=torch.bfloat16)
    res = {}
    for backend in ("nccl", "fused"):
        ops.tp_fused.set_backend(backend)
        for it in range(3):  # several calls exercise the double-buffer / epoch protocol
            x = x0.clone().requires_grad_(True)
            col.weight.grad = row.weight.grad = None
            y = row(torch.nn.functional.gelu(col(x)))
            y.float().pow(2).sum().backward()
        torch.cuda.synchronize()
        res[backend] = [t.detach().float().clone() for t in (y, x.grad, col.weight.grad, row.weight.grad)]
    for a, b, name in zip(res["fused"], res["nccl"], ("y", "dx", "dW_col", "dW_row")):
        err = float((a - b).abs().max() / (b.abs().max() + 1e-6))
        assert err < 3e-2, (name, err)
    assert ops._ext.launches() > 0


def test_fused_tp_matches_nccl():
    n = min(torch.cuda.device_count(), 8)
    run_distributed(_fused_vs_nccl, 2 if n < 4 else n if n in (2, 4, 8) else 2, use_cuda=True, timeout=240)


def _zero1_fused(rank, world):
    """DP=2 ZeRO-1: NVLink pull reduce-scatter + push all-gather kernels vs the NCCL path."""
    import neuronx_distributed_b200 as nxd
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.ops import zero1_comm
    from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams

    dev = torch.device("cuda", rank)
    losses = {}
    for fused in (False, True):
        zero1_comm._ENABLED = fused
        from neuronx_distributed_b200.parallel_layers import parallel_state as ps
        if ps.model_parallel_is_initialized():
            ps.destroy_model_parallel()
        cfg = nxd.neuronx_distributed_config(tensor_parallel_size=1, optimizer_config={"zero_one_enabled": True, "grad_clipping": True, "max_grad_norm": 1.0})
        mcfg = LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                           dtype=torch.bfloat16, device=dev, max_position_embeddings=128)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        model = nxd.initialize_parallel_model(cfg, lambda: LlamaForCausalLM(mcfg))
        opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=1e-2)
        assert (opt.optimizer.arena is not None) == fused
        out = []
        for step in range(4):
            ids = torch.randint(0, 512, (2, 128), generator=torch.Generator().manual_seed(10 * step + rank)).to(dev)
            opt.zero_grad()
            loss = model.run_train(input_ids=ids, labels=ids)
            opt.step()
            out.append(float(loss))
        # parameters must be identical on both DP ranks after the all-gather
        flat = opt.optimizer.flat_groups[0].param_flat.float()
        other = flat.clone()
        import torch.distributed as dist
        dist.all_reduce(other)
        assert torch.allclose(other, flat * world, rtol=0, atol=0)
        losses[fused] = out
    for a, b in zip(losses[True], losses[False]):
        assert abs(a - b) < 5e-2, losses


def test_zero1_fused_comm_matches_nccl():
    run_distributed(_zero1_fused, 2, use_cuda=True, timeout=240)


def _zero1_overlap(rank, world):
    """DP=2 ZeRO-1 with the bucketed reduce-scatter launched under the backward pass: same parameters as the single
    reduce-scatter at step() (up to the run-to-run noise of the attention backward), with gradient accumulation
    (no_sync on the first micro-batch)."""
    import contextlib

    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.optimizer import NeuronZero1Optimizer
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams

    dev = torch.device("cuda", rank)
    results = {}
    for overlap in (False, True):
        if ps.model_parallel_is_initialized():
            ps.destroy_model_parallel()
        ps.initialize_model_parallel(tensor_model_parallel_size=1)
        mcfg = LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=2,
                           dtype=torch.bfloat16, device=dev, max_position_embeddings=128, tie_word_embeddings=False)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        model = LlamaForCausalLM(mcfg)
        opt = NeuronZero1Optimizer(model.parameters(), AdamW_FP32OptimParams, lr=1e-2, use_grad_acc_hook=True,
                                   bucket_cap_mb_reduce_scatter=1, overlap_grad_reduce=overlap, grad_clipping=True, max_norm=1.0)
        assert opt.arena is not None and opt._overlap_active == overlap
        if overlap:
            assert len(opt._buckets) > 2
        for step in range(3):
            opt.zero_grad()
            for mb in range(2):
                ids = torch.randint(0, 512, (1, 128), generator=torch.Generator().manual_seed(100 * step + 10 * mb + rank)).to(dev)
                ctx = opt.no_sync() if mb == 0 else contextlib.nullcontext()
                with ctx:
                    loss, _ = model(input_ids=ids, labels=ids)
                    (loss / 2).backward()
            if overlap:
                assert any(opt._bucket_launched), "no bucket was reduced during backward"
            opt.step()
        results[overlap] = opt.flat_groups[0].param_flat.float().clone()
    # The reduce-scatter itself is order-exact (fixed rank order, fp32), but the own attention backward accumulates dQ with
    # bulk fp32 reductions whose arrival order differs between runs, so two runs of the SAME configuration already differ in
    # the last bits.  A bucket reduced too early (a missed contribution) or twice would be off by O(lr) = 1e-2, not 1e-5.
    # AdamW turns a last-bit gradient difference into a +-lr step where the gradient is ~0, so single elements may differ by
    # O(lr); a bucket reduced too early (a missed contribution) or twice would move a large FRACTION of the elements.
    frac = ((results[True] - results[False]).abs() > 1e-3).float().mean().item()
    assert frac < 0.02, frac


def test_zero1_overlapped_reduce_scatter_is_exact():
    run_distributed(_zero1_overlap, 2, use_cuda=True, timeout=240)


def _oneshot_ar(rank, world):
    """One-shot peer-memory all-reduce vs NCCL: eager, repeated back-to-back (epoch / parity protocol) and under CUDA-graph
    replay (device-side epoch)."""
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import allreduce
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    allreduce._MODE = "1"
    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    g = ps.get_tensor_model_parallel_group()
    dev = torch.device("cuda", rank)
    torch.manual_seed(rank)
    for dtype, n in ((torch.bfloat16, 5120), (torch.float32, 4096 * 33), (torch.bfloat16, 8 * 16384)):
        for it in range(5):
            x = torch.randn(n, device=dev).to(dtype)
            ref = x.clone().float()
            dist.all_reduce(ref, group=g)
            out = allreduce.all_reduce_sum(x, g)
            assert out is not None
            tol = 2e-2 if dtype == torch.bfloat16 else 1e-5
            assert (out.float() - ref).abs().max() <= tol * ref.abs().max() + 1e-6
    # graph replay: the same captured launch must stay correct over several replays with new inputs
    x = torch.zeros(5120, device=dev, dtype=torch.bfloat16)
    allreduce.all_reduce_sum(x, g)
    torch.cuda.synchronize(); dist.barrier()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = allreduce.all_reduce_sum(x, g)
    for it in range(4):
        x.copy_(torch.full((5120,), float(it + rank), device=dev))
        graph.replay()
        torch.cuda.synchronize()
        want = sum(it + r for r in range(world))
        assert torch.allclose(y.float(), torch.full_like(y.float(), want)), (it, y[:4])
    assert allreduce.all_reduce_sum(torch.randn(3, device=dev), g) is None      # not 16-byte sized → NCCL path


def test_oneshot_allreduce_matches_nccl_and_replays_in_graphs():
    run_distributed(_oneshot_ar, 2, use_cuda=True, timeout=240)
