"""GPU checks of opt-in and less-used paths.  Each check runs
in its own process with a timeout (a hang or a CUDA fault cannot take the rest of the suite down) and is marked
``xfail(strict=False)``: a run records XPASS (works on this GPU) or XFAIL (does not) without hiding either.  The
paths they exercise are opt-in (environment flags / explicit API calls), not defaults of the training or serving step."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.xfail(strict=False, reason="written after the GPU budget of the round was spent; "
                                                 "first execution on hardware is this run")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# A kernel that has never run may hang: every check is bounded (subprocess timeout) and the whole file has a time budget, after
# which the remaining checks are skipped — the validated part of the GPU suite (all files before this one) is never at risk.
_BUDGET_S = float(os.environ.get("NXD_LATE_GPU_BUDGET_S", "600"))
_PER_TEST_S = 150
_spent = [0.0]


@pytest.fixture(autouse=True)
def _time_budget():
    import time

    if _spent[0] > _BUDGET_S:
        pytest.skip(f"time budget of the late GPU checks ({_BUDGET_S:.0f} s) is used up")
    t0 = time.time()
    yield
    _spent[0] += time.time() - t0


def _run(code: str, timeout: int = _PER_TEST_S, env=None) -> None:
    timeout = min(timeout, _PER_TEST_S)
    e = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    e.update(env or {})
    # own session = own process group: on a timeout the whole group is killed, so worker processes spawned by the check (the
    # two-rank loopback checks) cannot stay behind with a spinning kernel and occupy the GPU for whatever runs after this file
    import signal

    proc = subprocess.Popen([sys.executable, "-c", textwrap.dedent(code)], cwd=ROOT, env=e, stdout=subprocess.PIPE,
                            stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        try:
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
        out, _ = proc.communicate()
        raise AssertionError(f"timed out after {timeout} s\n{(out or '')[-4000:]}")
    finally:
        try:                                            # stragglers of a check that returned (failed or not)
            os.killpg(proc.pid, signal.SIGKILL)
        except (ProcessLookupError, PermissionError):
            pass
    assert proc.returncode == 0, (out or "")[-4000:]


def test_fused_lmhead_ce_on_device():
    """bf16 chunked lm_head + CE on the wgmma GEMM / ce kernels vs an fp32 PyTorch reference of the same op."""
    _run("""
        import torch, torch.distributed as dist
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29631", rank=0, world_size=1)
        torch.cuda.set_device(0)
        from neuronx_distributed_b200.parallel_layers import parallel_state as ps
        from neuronx_distributed_b200.parallel_layers.loss_functions import fused_linear_cross_entropy
        from neuronx_distributed_b200.ops import _ext
        ps.initialize_model_parallel(1)
        T, H, V = 4096, 1024, 8192
        g = torch.Generator(device="cuda").manual_seed(0)
        h = (torch.randn(T, 1, H, device="cuda", generator=g)).bfloat16().requires_grad_(True)
        w = (torch.randn(V, H, device="cuda", generator=g) * 0.03).bfloat16().requires_grad_(True)
        tgt = torch.randint(0, V, (T, 1), device="cuda", generator=g)
        tgt[-7:] = -100
        _ext.reset_launches()
        loss = fused_linear_cross_entropy(h, w, tgt, chunk_rows=1024)
        loss.backward()
        assert _ext.launches() >= 4 * 5, _ext.launches()        # GEMM + stats + backward + dgrad + wgrad per chunk
        hf, wf = h.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
        ref = torch.nn.functional.cross_entropy(hf.view(T, H) @ wf.t(), tgt.view(-1), ignore_index=-100)
        ref.backward()
        def rel(a, b): return ((a.float() - b).norm() / b.norm()).item()
        print("loss", loss.item(), ref.item(), "dH", rel(h.grad, hf.grad), "dW", rel(w.grad, wf.grad))
        assert abs(loss.item() - ref.item()) < 2e-2 and rel(h.grad, hf.grad) < 2e-2 and rel(w.grad, wf.grad) < 2e-2
    """)


def test_llama_step_with_fused_lmhead_ce_follows_the_default_path():
    """Model level: three optimizer steps of a small bf16 Llama with the chunked lm_head + CE switched on give the loss curve of
    the default (materialised-logits) path within bf16 tolerance."""
    code = """
        import os, json, torch, torch.distributed as dist
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d", rank=0, world_size=1)
        torch.cuda.set_device(0)
        import neuronx_distributed_b200 as nxd
        from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
        from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams
        dev = torch.device("cuda", 0)
        cfg = nxd.neuronx_distributed_config(tensor_parallel_size=1, optimizer_config={"zero_one_enabled": True, "grad_clipping": True,
                                                                                    "max_grad_norm": 1.0})
        mcfg = LlamaConfig(vocab_size=8192, hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8,
                           num_key_value_heads=8, dtype=torch.bfloat16, device=dev, max_position_embeddings=1024)
        torch.manual_seed(0)
        model = nxd.initialize_parallel_model(cfg, lambda: LlamaForCausalLM(mcfg))
        opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=1e-3)
        ids = torch.randint(0, 8192, (2, 1024), device=dev, generator=torch.Generator(device="cuda").manual_seed(1))
        out = []
        for _ in range(3):
            opt.zero_grad(); loss = model.run_train(input_ids=ids, labels=ids); opt.step(); out.append(float(loss))
        print("LOSSES", json.dumps(out))
    """
    import json
    import re

    def losses(flag, port):
        e = dict(os.environ, PYTHONPATH=ROOT, NXD_FUSED_LMHEAD_CE=flag, NXD_LMHEAD_CE_CHUNK="512")
        p = subprocess.run([sys.executable, "-c", textwrap.dedent(code % port)], cwd=ROOT, env=e, timeout=_PER_TEST_S,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
        assert p.returncode == 0, p.stdout[-3000:]
        return json.loads(re.search(r"LOSSES (.*)", p.stdout).group(1))

    a, b = losses("0", 29641), losses("1", 29642)
    print(a, b)
    assert all(abs(x - y) < 3e-2 * max(1.0, abs(x)) for x, y in zip(a, b)) and b[-1] < b[0], (a, b)


def test_quantized_layers_and_moe_training_on_device():
    """Subsystems that so far only ran on the host, now on the GPU against their own CPU results: quantised Column / Row
    parallel layers (int8 per-channel, blockwise, fp8 with dynamic activation scaling) and a Mixtral-style MoE layer trained
    for three steps through the grouped wgmma GEMMs and the device-side block-metadata build."""
    _run("""
        import copy, torch, torch.distributed as dist
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29651", rank=0, world_size=1)
        torch.cuda.set_device(0)
        from neuronx_distributed_b200.parallel_layers import ColumnParallelLinear, RowParallelLinear, parallel_state as ps
        from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, convert
        from neuronx_distributed_b200.quantization.quantization_config import (get_default_blockwise_custom_qconfig_dict,
                                                                            get_default_per_channel_custom_qconfig_dict)
        ps.initialize_model_parallel(1)
        torch.manual_seed(0)
        m = torch.nn.Sequential(ColumnParallelLinear(256, 512, bias=False, gather_output=False),
                                RowParallelLinear(512, 256, bias=False, input_is_parallel=True)).eval()
        x = torch.randn(64, 256)
        for cfg in (get_default_per_channel_custom_qconfig_dict(), get_default_blockwise_custom_qconfig_dict(),
                    {**get_default_per_channel_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3,
                     "activation_quantization_type": ActivationQuantizationType.DYNAMIC}):
            q = convert(copy.deepcopy(m), cfg)
            want = q(x)
            got = q.cuda()(x.cuda()).cpu()
            err = ((got - want).norm() / want.norm()).item()
            print(str(cfg["quantization_type"]), str(cfg.get("quantized_dtype")), "device vs host rel err", err)
            assert err < 2e-2, err
        # MoE layer: same initial weights and data on host (fp32) and device (bf16); loss curves agree, loss falls
        from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, MoE, RoutedExpertsMLPOpsConfig, RouterTopK
        from neuronx_distributed_b200.ops import _ext
        def build():
            torch.manual_seed(1)
            cfg = RoutedExpertsMLPOpsConfig(num_experts=8, top_k=2, hidden_size=256, intermediate_size=512, hidden_act="silu",
                                            glu_mlp=True, normalize_top_k_affinities=True)
            return MoE(RouterTopK(8, 2, 256), ExpertMLPsV2(cfg), return_router_logits=True)
        data = [torch.randn(512, 1, 256, generator=torch.Generator().manual_seed(10))] * 3          # same batch: the loss must fall
        def run(layer, dev, dtype):
            layer = layer.to(dev).to(dtype)
            opt = torch.optim.SGD(layer.parameters(), lr=1.0)
            out = []
            for xb in data:
                xb = xb.to(dev, dtype)
                y, logits = layer(xb)
                loss = (y.float() - torch.tanh(xb.float())).pow(2).mean()
                opt.zero_grad(); loss.backward(); opt.step(); out.append(float(loss))
            return out
        host = run(build(), "cpu", torch.float32)
        _ext.reset_launches()
        dev = run(build(), "cuda", torch.bfloat16)
        print("host", host, "device", dev, "own-kernel launches", _ext.launches())
        assert _ext.launches() > 0, "the MoE layer did not reach the extension kernels"
        assert all(abs(a - b) < 0.05 * max(1.0, abs(a)) for a, b in zip(host, dev)) and dev[-1] < dev[0]
    """, timeout=150)


def test_deterministic_attention_backward_is_bit_reproducible():
    """The attention backward owns every gradient element in one thread (no atomics; ``NXD_FA_DETERMINISTIC`` is accepted and changes nothing) — two
    backward passes give bit-identical dQ / dK / dV, equal to the default kernel within its own run-to-run tolerance; causal and
    not, MHA and GQA."""
    _run("""
        import os, torch
        from neuronx_distributed_b200.ops import attention
        torch.manual_seed(0)
        for (B, S, H, Hkv, causal) in ((2, 1024, 8, 8, True), (1, 2048, 8, 2, True), (2, 512, 4, 4, False)):
            q, k, v = (torch.randn(B, S, h, 128, device="cuda", dtype=torch.bfloat16).requires_grad_(True) for h in (H, Hkv, Hkv))
            go = torch.randn(B, S, H, 128, device="cuda", dtype=torch.bfloat16)
            def grads():
                for t in (q, k, v): t.grad = None
                attention.flash_attention(q, k, v, causal=causal).backward(go)
                torch.cuda.synchronize()
                return [t.grad.clone() for t in (q, k, v)]
            os.environ["NXD_FA_DETERMINISTIC"] = "1"
            a, b = grads(), grads()
            assert all(torch.equal(x, y) for x, y in zip(a, b)), "deterministic mode is not reproducible"
            os.environ["NXD_FA_DETERMINISTIC"] = "0"
            c = grads()
            for x, y in zip(a, c):
                err = ((x.float() - y.float()).norm() / y.float().norm()).item()
                assert err < 1e-2, err
            print(B, S, H, Hkv, causal, "ok")
    """, timeout=150)


def test_decode_attention_partial_shards_merge_to_full_attention():
    """``decode_attention_partial`` (per-rank piece of distributed flash-decoding) on two sequence shards of one cache, merged
    with the log-sum-exp rule, vs fp32 attention over the whole cache — including a shard with nothing visible yet."""
    _run("""
        import math, torch
        from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial
        torch.manual_seed(0)
        B, H, Hkv, D, L = 3, 8, 2, 128, 512
        q = torch.randn(B, 1, H, D, device="cuda").bfloat16()
        k = torch.randn(B, L, Hkv, D, device="cuda").bfloat16()
        v = torch.randn(B, L, Hkv, D, device="cuda").bfloat16()
        pos = torch.tensor([40, 300, 511], device="cuda")            # row 0: the second shard has nothing visible
        scale = 1 / math.sqrt(D)
        parts = []
        for r in range(2):
            sl = slice(r * 256, (r + 1) * 256)
            parts.append(_local_partial(q, k[:, sl], v[:, sl], pos - r * 256, scale))
        m = torch.maximum(parts[0][1], parts[1][1])
        w = [torch.where(torch.isinf(p[1]), torch.zeros_like(m), torch.exp(p[1] - m)) for p in parts]
        o = sum(p[0] * wi.unsqueeze(-1) for p, wi in zip(parts, w)) / sum(p[2] * wi for p, wi in zip(parts, w)).unsqueeze(-1)
        kf, vf = k.float().repeat_interleave(H // Hkv, 2), v.float().repeat_interleave(H // Hkv, 2)
        s = torch.einsum("bhd,blhd->bhl", q[:, 0].float(), kf) * scale
        s = s.masked_fill(torch.arange(L, device="cuda")[None, None, :] > pos[:, None, None], float("-inf"))
        ref = torch.einsum("bhl,blhd->bhd", s.softmax(-1), vf)
        err = ((o - ref).norm() / ref.norm()).item()
        print("rel err", err, "m[0] shard1", parts[1][1][0, 0].item())
        assert err < 5e-3 and torch.isinf(parts[1][1][0]).all() and (parts[1][2][0] == 0).all()
    """)


def test_launch_plan_replays_extension_kernels_and_captures():
    """A bf16 Llama decode + prefill bucket recorded on the GPU (dispatcher ops + ``nxd_b200_C`` kernels as ``ext`` nodes), saved,
    loaded without the model object, re-captured into CUDA graphs: tokens must equal the module's."""
    _run("""
        import torch, torch.distributed as dist, tempfile
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29633", rank=0, world_size=1)
        torch.cuda.set_device(0)
        from neuronx_distributed_b200.parallel_layers import parallel_state as ps
        ps.initialize_model_parallel(1)
        from neuronx_distributed_b200.models.llama import LlamaConfig
        from neuronx_distributed_b200.models.llama_inference import LlamaForInference
        from neuronx_distributed_b200.trace.functions import trace, compile as ncompile, compile_wlo
        from neuronx_distributed_b200.trace.nxd_model import NxDModel
        from torch import nn
        class Wrap(nn.Module):
            def __init__(s, m, which): super().__init__(); s.m, s.which = m, which
            def forward(s, input_ids, aux):
                return s.m.context_encoding(input_ids, aux) if s.which == "cte" else s.m.token_generation(input_ids, aux)
        cfg = LlamaConfig(vocab_size=4096, hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8,
                          num_key_value_heads=2, dtype=torch.bfloat16, device=torch.device("cuda"), max_position_embeddings=256)
        torch.manual_seed(0)
        m = LlamaForInference(cfg, batch_size=2, max_seq_len=256).eval()
        ids = torch.randint(0, 4096, (2, 128), device="cuda"); last = torch.tensor([127, 90], device="cuda")
        want = m.generate(ids, 6, prompt_lens=last + 1)
        ta_c = trace(Wrap(m, "cte"), (ids, last))
        ta_t = trace(Wrap(m, "tkg"), (torch.zeros(2, 1, dtype=torch.long, device="cuda"), torch.tensor([128, 91], device="cuda")))
        nxd = NxDModel(world_size=1)
        wlo = compile_wlo(ta_t, None, None, None, "tkg")
        nxd.add("cte", ta_c, ncompile(ta_c, None, None, "--plan", "cte")).add("tkg", ta_t, wlo)
        nxd.to_neuron()
        print("tkg plan", wlo.plan.summary()); assert wlo.plan.calls_extension() and wlo.captured
        def gen(model, n):
            tok = model(ids, last, model_name="cte"); out, pos = [tok.clone()], last + 1
            for _ in range(n - 1):
                tok = model(tok.view(2, 1), pos, model_name="tkg"); out.append(tok.clone()); pos = pos + 1
            return torch.stack(out, 1)
        assert torch.equal(gen(nxd, 6), want), (gen(nxd, 6), want)
        d = tempfile.mkdtemp()
        nxd.save(d, save_weights=True, portable=True)
        del nxd, wlo, ta_c, ta_t
        loaded = NxDModel.load(d); loaded.to_neuron()
        assert torch.equal(gen(loaded, 6), want)
    """, timeout=420)


def _embedding_gather_loopback(rank, world):
    import torch
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import nvls

    g = dist.group.WORLD
    V, H = 4096, 1024
    tables = [(torch.randn(V // world, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(50 + r))).bfloat16()
              for r in range(world)]
    full = torch.cat(tables)
    for it in range(3):                                    # parity halves / call counter
        ids = torch.randint(-2, V + 2, (257,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(60 + it * 7 + rank))
        got = nvls.embedding_gather(ids, tables[rank], g)
        ok = (ids >= 0) & (ids < V)
        want = full[ids.clamp(0, V - 1)] * ok.unsqueeze(-1)
        assert torch.equal(got, want), (it, (got.float() - want.float()).abs().max())


def test_embedding_gather_over_peer_memory_loopback():
    """``embedding_rs``: two processes on cuda:0 publish their vocabulary shards and pull rows from each other."""
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dist_utils import run_distributed

    run_distributed(_embedding_gather_loopback, 2, use_cuda="loopback", timeout=_PER_TEST_S)


def _all_to_all_loopback(rank, world):
    import os

    os.environ["NXD_NVLS_A2A"] = "1"
    import torch
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import nvls
    from neuronx_distributed_b200.parallel_layers import comm

    g = dist.group.WORLD
    for it in range(3):
        xs = [torch.randn(world * 64, 4, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(70 + it * 5 + r)).bfloat16()
              for r in range(world)]
        assert nvls.all_to_all_eligible(xs[rank], g)
        got = nvls.all_to_all(xs[rank], g)
        want = torch.cat([xs[p].chunk(world, 0)[rank] for p in range(world)], 0)
        assert torch.equal(got, want), it
        # through the comm wrapper with a split dim that is not the leading one (EP dispatch layout)
        got2 = comm.all_to_all(xs[rank], split_dim=1, concat_dim=0, group=g)
        want2 = torch.cat([xs[p].chunk(world, 1)[rank] for p in range(world)], 0)
        assert torch.equal(got2, want2), it


def test_all_to_all_over_peer_memory_loopback():
    """EP dispatch / combine without NCCL: publish + pull kernels between two processes on cuda:0."""
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dist_utils import run_distributed

    run_distributed(_all_to_all_loopback, 2, use_cuda="loopback", timeout=_PER_TEST_S)


def _pull_attention_loopback(rank, world):
    import math

    import torch
    import torch.distributed as dist

    from neuronx_distributed_b200.modules.attention.ring import pull_attention
    from neuronx_distributed_b200.ops import _ext

    g = dist.group.WORLD
    B, S, H, Hkv, D = 1, 512, 4, 2, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(B, S, h, D, device="cuda", generator=gen).bfloat16() for h in (H, Hkv, Hkv))
    go = torch.randn(B, S, H, D, device="cuda", generator=gen).bfloat16()
    from neuronx_distributed_b200.utils.batch_utils import context_parallel_slice

    for it, layout in enumerate(("contiguous", "zigzag")):  # two calls = both halves of the publish slot
        def cut(t, layout=layout):
            return context_parallel_slice(t, rank, world, 1, layout)

        ql, kl, vl = (cut(t).clone().requires_grad_(True) for t in (q, k, v))
        n0 = _ext.launches()
        out = pull_attention(ql, kl, vl, causal=True, group=g, layout=layout)
        assert _ext.launches() > n0                         # publish + own attention kernels, not the SDPA fallback
        out.backward(cut(go))
        qf, kf, vf = (t.float().clone().requires_grad_(True) for t in (q, k, v))
        s = torch.einsum("bqhd,bkhd->bhqk", qf, kf.repeat_interleave(H // Hkv, 2)) / math.sqrt(D)
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device="cuda").tril(), float("-inf"))
        ref = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), vf.repeat_interleave(H // Hkv, 2))
        ref.backward(go.float())

        def rel(a, b):
            return float((a.float() - b).norm() / b.norm())

        errs = (rel(out, cut(ref)), rel(ql.grad, cut(qf.grad)), rel(kl.grad, cut(kf.grad)), rel(vl.grad, cut(vf.grad)))
        assert max(errs) < 2e-2, (layout, errs)


def test_pull_attention_reads_peer_kv_inside_the_kernel_loopback():
    """Context parallelism without a ring: K/V published in symmetric memory, the flash-attention kernels' TMA loads read the
    other process's slice in place; dK/dV return through one reduce-scatter."""
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dist_utils import run_distributed

    run_distributed(_pull_attention_loopback, 2, use_cuda="loopback", timeout=_PER_TEST_S)
