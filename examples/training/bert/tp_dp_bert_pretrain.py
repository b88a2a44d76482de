#!/usr/bin/env python
"""BERT-large pre-training (MLM + NSP), TP × DP — counterpart of the reference's
``examples/training/tp_dp_bert_hf_pretrain/tp_dp_bert_large_hf_pretrain_hdf5.py`` with synthetic data.

  torchrun --nproc-per-node 8 examples/training/bert/tp_dp_bert_pretrain.py --model large --tensor_parallel_size 2
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
from neuronx_distributed_b200.models.bert import BertConfig, BertForPreTraining  # noqa: E402
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams  # noqa: E402
from training_utils import Throughput, add_checkpoint_args, init_distributed, maybe_resume, maybe_save  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="tiny", choices=["tiny", "base", "large"])
    p.add_argument("--tensor_parallel_size", type=int, default=1)
    p.add_argument("--batch_size", type=int, default=8)
    p.add_argument("--seq_len", type=int, default=128)
    p.add_argument("--max_steps", type=int, default=10)
    p.add_argument("--mask_prob", type=float, default=0.15)
    p.add_argument("--max_pred_len", type=int, default=0, help="at most this many masked positions per sequence (0 = no limit)")
    p.add_argument("--optimizer", default="AdamW", choices=["AdamW", "LAMB"],
                   help="LAMB is accepted and runs AdamW (layer-wise trust ratios are not implemented)")
    p.add_argument("--lr", type=float, default=1e-4)
    p.add_argument("--dropout", type=float, default=0.0,
                   help="hidden and attention-probability dropout (bert-large-uncased trains with 0.1)")
    add_checkpoint_args(p)
    a = p.parse_args()
    dev = init_distributed()
    cfg = nxd.neuronx_distributed_config(tensor_parallel_size=a.tensor_parallel_size,
                                         optimizer_config={"zero_one_enabled": True, "grad_clipping": True, "max_grad_norm": 1.0})
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    shapes = {"large": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096),
              "base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072),
              "tiny": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=4, intermediate_size=256, vocab_size=1024)}[a.model]
    mcfg = BertConfig(dtype=dtype, device=dev, max_position_embeddings=max(512, a.seq_len), hidden_dropout_prob=a.dropout,
                      attention_probs_dropout_prob=a.dropout, **shapes)

    def model_fn():
        torch.manual_seed(1234)
        return BertForPreTraining(mcfg)

    model = nxd.initialize_parallel_model(cfg, model_fn)
    opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=a.lr, weight_decay=0.01)
    start = maybe_resume(a, nxd, model, opt)
    gen = torch.Generator().manual_seed(17 + ps.get_data_parallel_rank())
    thr = Throughput(a.batch_size, ps.get_data_parallel_size(), 1)
    for step in range(start, a.max_steps):
        if a.steps_this_run >= 0 and step - start >= a.steps_this_run:
            break
        ids = torch.randint(4, mcfg.vocab_size, (a.batch_size, a.seq_len), generator=gen)
        masked = torch.rand(ids.shape, generator=gen) < a.mask_prob
        if a.max_pred_len > 0:                                                       # keep the first max_pred_len masked positions
            masked = masked & (masked.cumsum(-1) <= a.max_pred_len)
        if a.debug and step == start and dist.get_rank() == 0:
            print("batch", tuple(ids.shape), "masked per row", masked.sum(-1).tolist()[:4], flush=True)
        labels = torch.where(masked, ids, torch.full_like(ids, -100))
        ids = torch.where(masked, torch.full_like(ids, 3), ids)                      # [MASK] id 3
        batch = dict(input_ids=ids.to(dev), labels=labels.to(dev), attention_mask=torch.ones_like(ids).to(dev),
                     token_type_ids=torch.zeros_like(ids).to(dev),
                     next_sentence_label=torch.randint(0, 2, (a.batch_size,), generator=gen).to(dev))
        opt.zero_grad()
        loss = model.run_train(**batch)
        opt.step()
        tp = thr.get_throughput()
        if dist.get_rank() == 0:
            print(f"step {step + 1} loss {float(loss):.4f} throughput {tp:.2f} seq/s", flush=True)
        maybe_save(a, nxd, model, opt, step + 1)
    nxd.finalize_checkpoint()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
