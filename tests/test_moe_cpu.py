"""MoE correctness vs a dense per-token reference (role of reference test_impl_correctness.py)."""
import os
import tempfile

import torch

from dist_utils import run_distributed


def _ref_moe(x, aff, idx, experts, normalize=True):
    T, H = x.shape
    out = torch.zeros(T, H)
    proj = experts.gate_up_proj.weight
    down = experts.down_proj.weight
    for t in range(T):
        a = aff[t, idx[t]]
        if normalize:
            a = a / a.sum()
        for j, e in enumerate(idx[t].tolist()):
            h = x[t] @ proj[e]
            g, u = h.chunk(2)
            out[t] += a[j] * ((torch.nn.functional.silu(g) * u) @ down[e])
    return out


def _moe_worker(rank, world):
    from neuronx_distributed_b200.modules.moe import (ExpertMLPsV2, MoE, RoutedExpertsMLPOpsConfig, RouterTopK,
                                                     load_balancing_loss_func)
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata, get_num_blocks
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    E, k, H, I, T = 4, 2, 16, 32, 24
    router = RouterTopK(E, k, H)
    x = torch.randn(T, H)
    logits, aff, idx = router(x)
    assert idx.shape == (T, k) and aff.shape == (T, E)
    if world == 1:
        cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=k, hidden_size=H, intermediate_size=I)
        em = ExpertMLPsV2(cfg)
        ref = _ref_moe(x, aff.detach(), idx, em.mlp_op)
        torch.testing.assert_close(em.forward_all_experts(x, aff, idx), ref, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(em.forward_blockwise(x, aff, idx), ref, rtol=1e-4, atol=1e-5)
        em.capacity_factor = float(E)      # capacity large enough that nothing is dropped
        torch.testing.assert_close(em.forward_capacity_factor(x, aff, idx), ref, rtol=1e-4, atol=1e-5)
        b2e, tp2id, counts = build_block_metadata(idx, E, 8)
        assert b2e.numel() == get_num_blocks(T, k, E, 8) and int(counts.sum()) == T * k
        assert (tp2id >= 0).sum() == T * k
    # full layer with TP (+SP): output must equal the tp=1 computation
    torch.manual_seed(1)
    cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=k, hidden_size=H, intermediate_size=I)
    torch.manual_seed(2)
    layer = MoE(RouterTopK(E, k, H, sequence_parallel_enabled=world > 1), ExpertMLPsV2(cfg),
                sequence_parallel_enabled=world > 1, return_router_logits=True)
    torch.manual_seed(3)
    xs = torch.randn(16, 2, H)
    xin = xs.chunk(world, 0)[rank] if world > 1 else xs
    y, rl = layer(xin)
    assert y.shape == xin.shape
    loss = y.pow(2).mean() + 0.01 * load_balancing_loss_func(rl, E, k)
    loss.backward()
    assert layer.expert_mlps.mlp_op.down_proj.weight.grad is not None
    torch.save(y.detach(), _out_path(world, rank))


def _out_path(world, rank):
    # per user: the worker processes of one test run hand their outputs over through the temp directory
    return os.path.join(tempfile.gettempdir(), f"moe_y_u{os.getuid()}_w{world}_r{rank}.pt")


def test_moe_modes_match_reference():
    run_distributed(_moe_worker, 1, timeout=90)


def test_moe_tensor_parallel_matches_single():
    run_distributed(_moe_worker, 1, timeout=90)
    run_distributed(_moe_worker, 2, timeout=90)
    full = torch.load(_out_path(1, 0))
    got = torch.cat([torch.load(_out_path(2, r)) for r in range(2)], 0)
    torch.testing.assert_close(got, full, rtol=1e-4, atol=1e-5)
