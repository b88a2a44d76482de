#!/usr/bin/env python
"""Llama pre-training with TP (+SP) + ZeRO-1 — the H100 counterpart of the reference's
``examples/training/llama/tp_zero1_llama_hf_pretrain/tp_zero1_llama_hf_pretrain.py`` (flags keep its names where they apply).

  torchrun --nproc-per-node 8 examples/training/llama/tp_zero1_llama_pretrain.py --model 7b --tensor_parallel_size 8 \
      --seq_len 4096 --batch_size 1 --grad_accum_usteps 8 --max_steps 100 --output_dir out --use_sequence_parallel 1
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "training"))

import neuronx_distributed_b200 as nxd  # noqa: E402
from neuronx_distributed_b200.models.llama import (LlamaConfig, LlamaForCausalLM, llama2_7b_config, llama2_13b_config,  # noqa: E402
                                                   llama2_70b_config)
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams  # noqa: E402
from training_utils import (Throughput, TrainingMetrics, init_distributed, linear_warmup_cosine, memmap_batches,  # noqa: E402
                            synthetic_batches)


def get_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="7b", choices=["tiny", "7b", "13b", "70b"])
    p.add_argument("--pretrained_hf", "--pretrained_weight", dest="pretrained_hf", default=None,
                   help="HF Llama directory (config.json + safetensors): continue pre-training / fine-tune from it")
    p.add_argument("--num_layers", "--num_layer", dest="num_layers", type=int, default=-1)
    p.add_argument("--hidden_size", type=int, default=-1, help="override the hidden size of the chosen model (shape experiments)")
    p.add_argument("--fuse_qkv", type=int, default=1, help="one fused QKV weight per layer (1) or separate q / k / v weights (0)")
    p.add_argument("--fp8_training", type=int, default=0,
                   help="row-wise scaled FP8 (e4m3) GEMMs in the decoder's qkv / o / gate_up / down projections (1) or bf16 (0)")
    p.add_argument("--tensor_parallel_size", type=int, default=8)
    p.add_argument("--context_parallel_size", type=int, default=1)
    p.add_argument("--cp_layout", default="contiguous", choices=["contiguous", "zigzag"],
                   help="zigzag: rank r holds sequence chunks (r, 2cp-1-r) so causal attention work is balanced (pull attention path)")
    p.add_argument("--use_sequence_parallel", type=int, default=1)
    p.add_argument("--use_zero_1", type=int, default=1)
    p.add_argument("--use_mix_precision", type=int, default=1)
    p.add_argument("--selective_checkpoint_enabled", action="store_true")
    p.add_argument("--seq_len", type=int, default=4096)
    p.add_argument("--batch_size", type=int, default=1)
    p.add_argument("--grad_accum_usteps", type=int, default=8)
    p.add_argument("--max_steps", type=int, default=20)
    p.add_argument("--warmup_steps", type=int, default=5)
    p.add_argument("--lr", type=float, default=3e-4)
    p.add_argument("--weight_decay", type=float, default=0.1)
    p.add_argument("--beta1", type=float, default=0.9)
    p.add_argument("--beta2", type=float, default=0.95)
    p.add_argument("--data_path", default=None, help="flat uint16 token file; synthetic tokens if omitted")
    p.add_argument("--output_dir", default="./output")
    p.add_argument("--metrics_file", default="results.json")
    p.add_argument("--checkpoint_freq", type=int, default=0)
    p.add_argument("--checkpoint_dir", default=None)
    p.add_argument("--loading_step", default="latest_if_exists")
    p.add_argument("--num_kept_checkpoint", type=int, default=2)
    p.add_argument("--save_load_xser", type=int, default=1)
    p.add_argument("--async_checkpoint_saving", type=int, default=0)
    p.add_argument("--logging_interval", type=int, default=1)
    p.add_argument("--seed", type=int, default=1234)
    # pipeline parallelism (the TP x PP script of the reference, run_llama_nxd.py, is this driver with these set)
    p.add_argument("--pipeline_parallel_size", type=int, default=1)
    p.add_argument("--virtual_pipeline_size", type=int, default=1)
    p.add_argument("--num_microbatches", type=int, default=4)
    p.add_argument("--trace_file_path", default=None, help="Chrome trace of the pipeline tasks (CUDA-event times)")
    p.add_argument("--deallocate_pipeline_outputs", type=int, default=0)
    p.add_argument("--fuse_microbatches", type=int, default=0)
    # flags of the reference's scripts (tp_zero1_llama_hf_pretrain.py:528-673, run_llama_nxd.py) under their own names
    p.add_argument("--data_dir", "--training_dir", dest="data_dir", default=None,
                   help="directory holding the token file written by get_dataset.py (tokens.bin / *.bin)")
    p.add_argument("--model_path", "--training_config", dest="model_path", default=None,
                   help="directory with a Hugging Face config.json: architecture only, weights stay random")
    p.add_argument("--kv_replicator", type=int, default=1, help="replicate the KV heads this many times (GQA with tp > kv heads)")
    p.add_argument("--qkv_linear", type=int, default=1, help="accepted: the GQA QKV linear is always used")
    p.add_argument("--sequence_parallel_enabled", action="store_true", help="same as --use_sequence_parallel 1")
    p.add_argument("--use_zero1_optimizer", type=int, default=None, help="same as --use_zero_1")
    p.add_argument("--steps_this_run", type=int, default=-1, help="stop after this many steps of THIS run (resume continues)")
    p.add_argument("--train_batch_size", type=int, default=None, help="global batch in sequences; sets the micro-batch count")
    p.add_argument("--print_grad_norm", action="store_true", help="accepted: the gradient norm is always logged")
    p.add_argument("--use_flash_attention", type=int, default=1, help="accepted: attention is always the flash kernel")
    p.add_argument("--transpose_nki_inputs", type=int, default=1, help="accepted (layout detail of the reference's kernel)")
    p.add_argument("--use_gpu_compatible_precision", type=int, default=1, help="accepted (fp32 softmax / norms are the only mode)")
    p.add_argument("--use_amp", type=int, default=0, help="accepted: parameters are bf16, statistics fp32")
    p.add_argument("--use_meta_device_init", "--use_deferred_init", dest="use_meta_device_init", type=int, default=0,
                   help="build the model on the meta device and materialise only this rank's partition")
    p.add_argument("--use_fp32_optimizer", type=int, default=None, help="fp32 master weights + fp32 gradient accumulation")
    p.add_argument("--use_master_weight_in_ckpt", type=int, default=0)
    p.add_argument("--avoid_saving_lower_precision_weights", type=int, default=0)
    p.add_argument("--use_selective_checkpoint", type=int, default=0, help="same as --selective_checkpoint_enabled")
    p.add_argument("--min_lr", type=float, default=None, help="floor of the cosine schedule (default: lr / 10)")
    p.add_argument("--constant_steps", type=int, default=0, help="steps at the peak learning rate between warm-up and decay")
    p.add_argument("--tb_dir", default=None, help="write the logged scalars here (TensorBoard when available, JSON lines otherwise)")
    return p.parse_args(argv)


def main(argv=None):
    a = get_args(argv)
    if a.sequence_parallel_enabled:
        a.use_sequence_parallel = 1
    if a.use_zero1_optimizer is not None:
        a.use_zero_1 = a.use_zero1_optimizer
    if a.use_selective_checkpoint:
        a.selective_checkpoint_enabled = True
    if a.data_dir and not a.data_path:
        import glob

        cands = [os.path.join(a.data_dir, "tokens.bin")] + sorted(glob.glob(os.path.join(a.data_dir, "*.bin")))
        a.data_path = next((c for c in cands if os.path.isfile(c)), None)
        assert a.data_path, f"no token file (*.bin) under {a.data_dir}"
    pp = a.pipeline_parallel_size
    if a.train_batch_size:                                        # global batch -> micro-batches per step on every DP replica
        world = int(os.environ.get("WORLD_SIZE", "1"))
        dp_guess = max(1, world // (a.tensor_parallel_size * pp * a.context_parallel_size))
        per_replica = max(1, a.train_batch_size // (dp_guess * a.batch_size))
        if pp > 1:
            a.num_microbatches = per_replica
        else:
            a.grad_accum_usteps = per_replica
    dev = init_distributed()
    sp = bool(a.use_sequence_parallel) and a.tensor_parallel_size > 1
    mp = None
    if not a.use_mix_precision:
        mp = {"use_master_weights": False, "use_fp32_grad_acc": False, "use_master_weights_in_ckpt": False}
    elif a.use_fp32_optimizer is not None or a.use_master_weight_in_ckpt:
        on = bool(a.use_fp32_optimizer) if a.use_fp32_optimizer is not None else bool(a.use_zero_1)
        mp = {"use_master_weights": on, "use_fp32_grad_acc": on,
              "use_master_weights_in_ckpt": bool(a.use_master_weight_in_ckpt) and on}
    pipeline_config = None
    if pp > 1:
        from neuronx_distributed_b200.models.llama import LlamaDecoderLayer

        pipeline_config = {"transformer_layer_cls": LlamaDecoderLayer, "num_microbatches": a.num_microbatches,
                           "virtual_pipeline_size": a.virtual_pipeline_size, "output_loss_value_spec": (True, False),
                           "input_names": ["input_ids", "labels"], "broadcast_and_average_loss": True,
                           "trace_file_path": a.trace_file_path, "deallocate_pipeline_outputs": bool(a.deallocate_pipeline_outputs),
                           "fuse_microbatches": bool(a.fuse_microbatches)}
    cfg = nxd.neuronx_distributed_config(
        tensor_parallel_size=a.tensor_parallel_size, pipeline_parallel_size=pp, context_parallel_size=a.context_parallel_size,
        sequence_parallel=sp, pipeline_config=pipeline_config,
        optimizer_config={"zero_one_enabled": bool(a.use_zero_1), "grad_clipping": True, "max_grad_norm": 1.0},
        mixed_precision_config=mp,
        activation_checkpoint_config="full" if a.selective_checkpoint_enabled else None,
        model_init_config={"meta_device_init": True, "param_init_fn": None, "sequential_move_factor": 11} if a.use_meta_device_init else None,
    )
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    kw = dict(sequence_parallel_enabled=sp, dtype=dtype, device=None if (a.use_meta_device_init or pp > 1) else dev,
              max_position_embeddings=a.seq_len,
              context_parallel=a.context_parallel_size > 1, cp_layout=a.cp_layout)
    mcfg = {"7b": llama2_7b_config, "13b": llama2_13b_config, "70b": llama2_70b_config}.get(a.model, lambda **k: LlamaConfig(
        vocab_size=4096, hidden_size=512, intermediate_size=1408, num_hidden_layers=4, num_attention_heads=8, **k))(**kw)
    if a.pretrained_hf or a.model_path:                          # architecture from the HF config, weights loaded after sharding
        from neuronx_distributed_b200.models import hf_compat

        mcfg = hf_compat.config_from_hf(a.pretrained_hf or a.model_path, **kw)
    if a.kv_replicator > 1:
        mcfg.kv_size_multiplier = a.kv_replicator
    if a.num_layers > 0:
        mcfg.num_hidden_layers = a.num_layers
    if a.hidden_size > 0:
        mcfg.hidden_size = a.hidden_size
    mcfg.fuse_qkv = bool(a.fuse_qkv)
    mcfg.fp8_training = bool(a.fp8_training)

    def model_fn():
        torch.manual_seed(a.seed)
        if dev.type == "cuda":
            torch.cuda.manual_seed(a.seed)
        return LlamaForCausalLM(mcfg)

    model = nxd.initialize_parallel_model(cfg, model_fn)
    if a.pretrained_hf:
        hf_compat.load_hf_checkpoint(model, a.pretrained_hf)     # every rank keeps its (tp, pp) shard only
    opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=a.lr, betas=(a.beta1, a.beta2),
                                            weight_decay=a.weight_decay)
    sched = linear_warmup_cosine(opt.optimizer if hasattr(opt, "optimizer") else opt, a.warmup_steps, a.max_steps,
                                 min_ratio=(a.min_lr / a.lr) if a.min_lr is not None else 0.1, constant=a.constant_steps)
    dp, dpr = ps.get_data_parallel_size(), ps.get_data_parallel_rank()
    rows = a.batch_size * (a.num_microbatches if pp > 1 else 1)     # a pipeline step consumes all its micro-batches in one call
    if pp > 1:
        a.grad_accum_usteps = 1
    data = (memmap_batches(a.data_path, rows, a.seq_len, dpr, dp, dev) if a.data_path
            else synthetic_batches(mcfg.vocab_size, rows, a.seq_len, a.seed + dpr, dev))
    tb = None
    if a.tb_dir and dist.get_rank() == 0:
        from neuronx_distributed_b200.lightning.logger import NeuronTensorBoardLogger

        tb = NeuronTensorBoardLogger(a.tb_dir, name="pretrain", version="0", log_rank0=True)     # rank 0 holds the averaged loss
    step = 0
    ckpt_dir = a.checkpoint_dir or os.path.join(a.output_dir, "checkpoints")
    if a.loading_step == "latest_if_exists" and a.checkpoint_freq > 0 and nxd.has_checkpoint(ckpt_dir):
        uc = nxd.load_checkpoint(ckpt_dir, tag=None, model=model, optimizer=opt, scheduler=sched)
        step = (uc or {}).get("total_steps", 0)
    os.makedirs(a.output_dir, exist_ok=True)
    metrics = TrainingMetrics(os.path.join(a.output_dir, a.metrics_file))
    metrics.store_parameters(vars(a))
    thr = Throughput(rows, dp, a.grad_accum_usteps, logging_interval=a.logging_interval)
    first_step = step
    tps = []
    while step < a.max_steps and (a.steps_this_run < 0 or step - first_step < a.steps_this_run):
        opt.zero_grad()
        total = 0.0
        for _ in range(a.grad_accum_usteps):
            batch = next(data)
            if a.context_parallel_size > 1:
                from neuronx_distributed_b200.utils.batch_utils import get_batch_on_this_context_parallel_rank

                batch = get_batch_on_this_context_parallel_rank(batch, layout=a.cp_layout)
            loss = model.run_train(**batch)
            total = total + loss.detach() / a.grad_accum_usteps
        opt.step()
        sched.step()
        step += 1
        if step % a.logging_interval == 0:
            if dp > 1:
                dist.all_reduce(total, group=ps.get_data_parallel_group())
                total = total / dp
            tp = thr.get_throughput()
            tps.append(tp)
            if dist.get_rank() == 0:
                gn = float(opt.grad_norm) if opt.grad_norm is not None else float("nan")
                print(f"step {step} loss {float(total):.4f} grad_norm {gn:.3f} lr {sched.get_last_lr()[0]:.2e} "
                      f"throughput {tp:.2f} seq/s ({tp * a.seq_len:.0f} tok/s)", flush=True)
                if tb is not None:
                    tb.log_metrics({"loss": float(total), "grad_norm": gn, "lr": sched.get_last_lr()[0], "throughput_seq_s": tp}, step)
        if a.checkpoint_freq > 0 and step % a.checkpoint_freq == 0:
            nxd.save_checkpoint(ckpt_dir, f"step_{step}", model=model, optimizer=opt, scheduler=sched,
                                user_content={"total_steps": step}, use_xser=bool(a.save_load_xser),
                                num_kept_ckpts=a.num_kept_checkpoint, async_save=bool(a.async_checkpoint_saving),
                                avoid_saving_lower_precision_weights=bool(a.avoid_saving_lower_precision_weights))
    nxd.finalize_checkpoint()
    steady = tps[min(10, len(tps) // 2):] or tps
    metrics.store_metrics({"final_loss": float(total), "average_throughput_seq_s": sum(steady) / max(1, len(steady)),
                           "peak_throughput_seq_s": thr.peak, "steps": step})
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
