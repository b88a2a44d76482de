"""Quantised expert layers, fp8 KV cache, decode-time fused MoE block, and the Lightning integration driven without Lightning
(its base classes are import-gated stand-ins in this image)."""
import torch

from dist_utils import run_distributed


def _quant_moe(rank, world):
    from neuronx_distributed_b200.inference.kv_cache import KVCacheManager
    from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, MoE, RoutedExpertsMLPOpsConfig, RouterTopK, SharedExperts
    from neuronx_distributed_b200.modules.moe.moe_fused_tkg import MoEFusedTKG
    from neuronx_distributed_b200.modules.rms_norm import RMSNorm
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import QuantizedDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import (KVQuantizationConfig,
                                                                           get_default_expert_wise_per_channel_custom_qconfig_dict)

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    E, k, H, I, T = 4, 2, 32, 64, 6
    cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=k, hidden_size=H, intermediate_size=I)
    router, experts = RouterTopK(E, k, H), ExpertMLPsV2(cfg)
    shared = SharedExperts(H, 16, fused_gate_up_projection=True)
    norm = RMSNorm(H)
    layer = MoE(router, experts, shared_experts=shared).eval()
    x = torch.randn(T, 1, H, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = layer(norm(x))[0]
        # decode-time fused block = same math in one pass (norm → router → all local experts → shared → one reduction)
        fused = MoEFusedTKG(router, experts, shared, norm).eval()
        got = fused(x)[0]
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
        y_res, x_res = fused(x, residual=torch.ones_like(x))
        torch.testing.assert_close(x_res, x + 1)
        # expert-wise per-channel int8 / fp8 weights stay close to the float layer
        for qd, tol in ((QuantizedDtype.INT8, 0.03), (QuantizedDtype.F8E4M3, 0.08)):
            q = {**get_default_expert_wise_per_channel_custom_qconfig_dict(), "quantized_dtype": qd}
            qlayer = convert(layer, q, inplace=False)
            names = [type(m).__name__ for m in qlayer.modules()]
            assert any(n.startswith("QuantizedExpertFused") for n in names)
            err = (qlayer(norm(x))[0] - want).abs().max() / want.abs().max()
            assert err < tol, (qd, float(err))
    # fp8 KV cache: write/read round trip within fp8 precision, decode scatter hits the right slots
    kvq = KVQuantizationConfig(quant_dtype=torch.float8_e4m3fn, dequant_dtype=torch.float32, scale=0.05)
    kv = KVCacheManager(2, 2, 8, 2, 4, dtype=torch.float32, kv_quant=kvq)
    kk = torch.randn(2, 5, 2, 4, generator=torch.Generator().manual_seed(2)); vv = torch.randn(2, 5, 2, 4, generator=torch.Generator().manual_seed(3))
    kv.write_prefill(1, kk, vv)
    k_new = torch.randn(2, 1, 2, 4, generator=torch.Generator().manual_seed(4))
    kv.write_window(1, k_new, k_new, torch.tensor([5, 6]))
    kc, vc = kv.get(1, 8)
    assert kv.k[1].dtype == torch.float8_e4m3fn and kc.dtype == torch.float32
    assert (kc[:, :5] - kk).abs().max() < 0.25 and (vc[:, :5] - vv).abs().max() < 0.25
    assert (kc[0, 5] - k_new[0, 0]).abs().max() < 0.25 and (kc[1, 6] - k_new[1, 0]).abs().max() < 0.25 and kc[0, 6].abs().max() == 0


def test_quantized_experts_fused_tkg_and_fp8_kv_cache_tp2():
    run_distributed(_quant_moe, 2, timeout=120)


def _lightning(rank, world):
    """NeuronLTModule's manual-optimisation loop (setup → configure_optimizers → training_step with gradient accumulation)
    works with the stand-in base classes and trains a tiny Llama."""
    import neuronx_distributed_b200 as nxd
    from neuronx_distributed_b200.lightning import NeuronLTModule
    from neuronx_distributed_b200.lightning._compat import HAVE_LIGHTNING
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM

    cfg = nxd.neuronx_distributed_config(tensor_parallel_size=world, optimizer_config={"zero_one_enabled": True, "grad_clipping": True,
                                                                                       "max_grad_norm": 1.0})
    mcfg = LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4,
                       dtype=torch.float32, max_position_embeddings=16)

    def model_fn():
        torch.manual_seed(3)
        return LlamaForCausalLM(mcfg)

    mod = NeuronLTModule(cfg, model_fn, torch.optim.AdamW, opt_kwargs={"lr": 1e-2}, grad_accum_steps=2)
    mod.setup("fit")
    mod.configure_optimizers()
    ids = torch.randint(0, 64, (2, 16), generator=torch.Generator().manual_seed(9))
    first = None
    for i in range(8):
        mod.training_step({"input_ids": ids, "labels": ids}, i)
        if i == 1:
            first = float(mod.model.run_eval(input_ids=ids, labels=ids))
    last = float(mod.model.run_eval(input_ids=ids, labels=ids))
    assert last < first, (first, last)
    assert isinstance(HAVE_LIGHTNING, bool)


def _lightning_fit(rank, world, tmp):
    """The package's own fit loop drives strategy → module → callbacks → logger → checkpoint IO in Lightning's call order,
    and resumes from the checkpoint it wrote."""
    import os

    from neuronx_distributed_b200.lightning import (NeuronCheckpointIO, NeuronLTModule, NeuronTensorBoardLogger, NxDStrategy, Trainer)
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.trainer import neuronx_distributed_config

    cfg = neuronx_distributed_config(tensor_parallel_size=world, optimizer_config={"zero_one_enabled": True, "grad_clipping": True})
    mcfg = LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4,
                       dtype=torch.float32, max_position_embeddings=16)

    def model_fn():
        torch.manual_seed(3)
        return LlamaForCausalLM(mcfg)

    ids = torch.randint(0, 64, (2, 16), generator=torch.Generator().manual_seed(9))
    batches = [{"input_ids": ids, "labels": ids}] * 8
    events = []

    class Cb:
        def on_train_start(self, trainer, module):
            events.append("start")

        def on_train_batch_end(self, trainer, module, *a):
            events.append("batch")

        def on_train_end(self, trainer, module):
            events.append("end")

    def run(max_steps, resume=None):
        mod = NeuronLTModule(cfg, model_fn, torch.optim.AdamW, opt_kwargs={"lr": 1e-2}, grad_accum_steps=2)
        tr = Trainer(strategy=NxDStrategy(nxd_config=cfg), callbacks=[Cb()], logger=NeuronTensorBoardLogger(tmp, "fit"),
                     max_steps=max_steps, default_root_dir=os.path.join(tmp, "ck"), every_n_train_steps=2,
                     plugins=[NeuronCheckpointIO(save_load_xser=True)])
        tr.fit(mod, train_dataloaders=batches, ckpt_path=resume)
        return tr, mod

    tr, mod = run(4)
    assert tr.global_step == 4 and events[0] == "start" and events[-1] == "end" and events.count("batch") == 8
    assert "loss" in tr.callback_metrics and os.path.isfile(os.path.join(tmp, "ck", "step_4", "done"))
    loss4 = float(mod.model.run_eval(input_ids=ids, labels=ids))
    events.clear()
    tr2, mod2 = run(5, resume=os.path.join(tmp, "ck", "step_4"))
    assert tr2.global_step == 5 and events.count("batch") == 2            # resumed at 4 → one more optimizer step (2 micro-batches)
    assert float(mod2.model.run_eval(input_ids=ids, labels=ids)) < loss4


def test_lightning_fit_loop_checkpoint_resume(tmp_path):
    run_distributed(_lightning_fit, 2, str(tmp_path), timeout=180)


def test_lightning_module_trains_without_lightning_installed():
    run_distributed(_lightning, 2, timeout=120)


def test_add_rms_norm_matches_unfused_composition(monkeypatch):
    """``ops.norm.add_rms_norm`` (residual add fused with RMSNorm): values and all three gradients equal the two-op form; the
    Llama block gives the same loss and gradients with the fusion switched on."""
    from neuronx_distributed_b200.ops import norm

    g = torch.Generator().manual_seed(0)
    x, r = torch.randn(3, 5, 32, generator=g, requires_grad=True), torch.randn(3, 5, 32, generator=g, requires_grad=True)
    w = torch.randn(32, generator=g).abs().requires_grad_(True)
    y, h = norm.add_rms_norm(x, r, w, 1e-5)
    cot_y, cot_h = torch.randn(3, 5, 32, generator=g), torch.randn(3, 5, 32, generator=g)
    (y * cot_y).sum().backward(retain_graph=True)
    (h * cot_h).sum().backward()
    got = [t.grad.clone() for t in (x, r, w)]
    for t in (x, r, w):
        t.grad = None
    h2 = x + r
    y2 = norm.rms_norm(h2, w, 1e-5)
    ((y2 * cot_y).sum() + (h2 * cot_h).sum()).backward()
    torch.testing.assert_close(y, y2)
    torch.testing.assert_close(h, h2)
    for a, b in zip(got, (x.grad, r.grad, w.grad)):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)


def _fused_block(rank, world):
    from neuronx_distributed_b200.models import llama
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(world)
    cfg = llama.LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                            dtype=torch.float32, max_position_embeddings=16, sequence_parallel_enabled=True)
    ids = torch.randint(0, 64, (2, 16), generator=torch.Generator().manual_seed(1))
    out = []
    for fused in (False, True):
        llama._FUSED_ADD_NORM = fused
        torch.manual_seed(0)
        m = llama.LlamaForCausalLM(cfg)
        loss, _ = m(ids, labels=ids)
        loss.backward()
        out.append((loss.detach(), [p.grad.clone() for p in m.parameters()]))
    llama._FUSED_ADD_NORM = False
    torch.testing.assert_close(out[0][0], out[1][0])
    for a, b in zip(out[0][1], out[1][1]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_llama_block_with_fused_add_norm():
    run_distributed(_fused_block, 2, timeout=120)


def _lightning_strategy(rank, world, tmp):
    """Strategy surface of the reference (``lightning/strategy.py:84-238``): DP-only metric reduction, batch / dataloader
    placement, checkpoint routing; ``NeuronLTModule.log`` validation and rank filtering; the device prefetch loader."""
    import os

    import pytest

    from neuronx_distributed_b200.lightning import NeuronCheckpointIO, NeuronLTModule, NeuronXLAStrategy, NxDStrategy
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.trainer import neuronx_distributed_config
    from neuronx_distributed_b200.utils.device_loader import DevicePrefetchLoader, MpDeviceLoader

    assert NeuronXLAStrategy is NxDStrategy and MpDeviceLoader is DevicePrefetchLoader
    cfg = neuronx_distributed_config(tensor_parallel_size=2)
    st = NxDStrategy(nxd_config=cfg)
    st.setup_distributed()                                            # world 4 = TP 2 × DP 2
    assert ps.get_data_parallel_size() == 2 and st.distributed_sampler_kwargs == {"num_replicas": 2, "rank": ps.get_data_parallel_rank()}
    v = torch.tensor(float(ps.get_data_parallel_rank() + 1))
    torch.testing.assert_close(st.reduce(v, reduce_op="mean"), torch.tensor(1.5))       # over DP replicas only
    torch.testing.assert_close(st.reduce(v, reduce_op="sum"), torch.tensor(3.0))
    assert st.reduce("text") == "text"
    with pytest.raises(ValueError):
        st.reduce(v, reduce_op="max")
    b = st.batch_to_device({"a": torch.ones(2), "b": [torch.zeros(1), 3]})
    assert b["a"].device == st.root_device and b["b"][1] == 3
    data = [{"x": torch.full((2,), float(i))} for i in range(5)]
    dl = st.process_dataloader(data)
    assert isinstance(dl, DevicePrefetchLoader) and st.process_dataloader(dl) is dl and len(dl) == 5
    assert [float(d["x"][0]) for d in dl] == [0.0, 1.0, 2.0, 3.0, 4.0]                    # order kept, nothing dropped
    st.model_to_device()
    st._configure_launcher()
    assert st._launcher.launch(lambda a: a + 1, 1) == 2
    # checkpoint routing: strategy → NeuronCheckpointIO → nxd.save_checkpoint layout
    lin = torch.nn.Linear(4, 4)
    st.save_checkpoint({"state_dict": lin, "global_step": 7}, f"{tmp}/ck/step_7")
    user = st.load_checkpoint(f"{tmp}/ck/step_7", model=lin)
    assert int(user["global_step"]) == 7
    # the reference plugin's layout: the whole Lightning dict through the legacy per-rank files, per-DP-rank on request
    legacy = NeuronCheckpointIO(save_load_xser=False, weights_only=False, layout="legacy")
    legacy.save_checkpoint({"state_dict": lin.state_dict(), "global_step": 9}, f"{tmp}/legacy/step_9")
    assert os.path.isfile(f"{tmp}/legacy/step_9/tp_rank_00_pp_rank_00/checkpoint.pt")
    assert int(legacy.load_checkpoint(checkpoint_path=f"{tmp}/legacy/step_9")["global_step"]) == 9
    legacy.save_checkpoint({"r": rank}, f"{tmp}/legacy/per_dp", master_dp_only=False)
    assert legacy.load_checkpoint(f"{tmp}/legacy/per_dp", master_dp_only=False)["r"] == rank
    with pytest.raises(TypeError):
        legacy.save_checkpoint({}, f"{tmp}/legacy/x", storage_options={"a": 1})
    # log(): scalar tensors / numbers only, rank filtering, DP sync through the strategy
    mod = NeuronLTModule(cfg, lambda: lin, torch.optim.SGD, log_rank0=True)

    class T:
        strategy = st

    mod.trainer = T()
    mod.log("m", v, sync_dist=True, prog_bar=True)
    if rank == 0:
        torch.testing.assert_close(mod._logged["m"], torch.tensor(1.5))
        assert "m" in mod._progress_bar_metrics
    else:
        assert "m" not in mod._logged                                  # log_rank0
    for bad in (torch.ones(2), "s", True, None):
        with pytest.raises(ValueError):
            mod.log("bad", bad)
    with pytest.raises(ValueError):
        mod.log("nested", {"a": 1})
    with pytest.raises(TypeError):
        mod.log(3, 1.0)
    st.teardown()


def test_lightning_strategy_surface_and_logging(tmp_path):
    run_distributed(_lightning_strategy, 4, str(tmp_path), timeout=180)


def _launched(x):
    import os

    import torch.distributed as dist

    dist.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
    t = torch.tensor(float(int(os.environ["RANK"]) + x))
    dist.all_reduce(t)
    dist.destroy_process_group()
    if x < 0:
        raise ValueError("boom")
    return float(t)


def test_lightning_launcher_spawns_ranks_and_returns_rank0_value(monkeypatch):
    """``_NeuronXLALauncher`` (reference ``lightning/launcher.py``): outside torchrun it spawns the workers itself, sets their rank
    environment, joins them and hands back worker 0's result; worker failures surface in the parent; under torchrun it runs
    in-process."""
    import pytest

    from neuronx_distributed_b200.lightning.launcher import _NeuronXLALauncher

    for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE"):
        monkeypatch.delenv(k, raising=False)
    assert _NeuronXLALauncher(num_processes=3).launch(_launched, 10) == 33.0          # (0+10) + (1+10) + (2+10)
    with pytest.raises(RuntimeError, match="boom"):
        _NeuronXLALauncher(num_processes=2).launch(_launched, -1)
    monkeypatch.setenv("RANK", "0")
    assert _NeuronXLALauncher(num_processes=4).launch(lambda a: a + 1, 1) == 2         # torchrun: this process is the rank
