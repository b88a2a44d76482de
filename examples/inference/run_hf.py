#!/usr/bin/env python
"""Serve an HF Llama / Mixtral / GPT-NeoX (Pythia) checkpoint and check it against ``transformers`` — counterpart of the reference's
``examples/inference/run_hf.py`` (HF config + weights + tokenizer → TP-sharded model → ``generate``).

  torchrun --nproc-per-node 8 examples/inference/run_hf.py --model_path /models/Llama-2-7b-hf --tp_degree 8 --check_accuracy
  python examples/inference/run_hf.py            # no --model_path: a random tiny HF Llama is created in memory (offline demo)
  python examples/inference/run_hf.py --family gpt_neox     # the same with a tiny random HF GPT-NeoX

Every rank memory-maps the safetensors files and keeps only its shard (``models.hf_compat.load_hf_checkpoint``); the decode
loop is the CUDA-graph captured serving path of ``LlamaForInference`` (``GPTNeoXForInference`` for a ``gpt_neox`` config).  ``--check_accuracy`` also runs the HF model on rank 0
(CPU, fp32) and reports how many greedy tokens agree — the reference runner's ``check_accuracy`` flow."""
import argparse
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "training"))

from neuronx_distributed_b200.models import hf_compat  # noqa: E402
from neuronx_distributed_b200.models.gpt_neox import GPTNeoXConfig  # noqa: E402
from neuronx_distributed_b200.models.gpt_neox_inference import GPTNeoXForInference  # noqa: E402
from neuronx_distributed_b200.models.llama_inference import LlamaForInference  # noqa: E402
from neuronx_distributed_b200.parallel_layers import parallel_state as ps  # noqa: E402
from training_utils import init_distributed  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model_path", default=None, help="HF model directory (config.json + *.safetensors [+ tokenizer])")
    p.add_argument("--tp_degree", type=int, default=None)
    p.add_argument("--family", choices=("llama", "gpt_neox"), default="llama", help="model of the offline demo (no --model_path)")
    p.add_argument("--prompt", action="append", default=None)
    p.add_argument("--max_new_tokens", type=int, default=16)
    p.add_argument("--seq_len", type=int, default=128)
    p.add_argument("--check_accuracy", action="store_true")
    p.add_argument("--do_sample", action="store_true")
    p.add_argument("--top_k", type=int, default=50)
    p.add_argument("--top_p", type=float, default=0.95)
    a = p.parse_args()
    import transformers

    dev = init_distributed()
    ps.initialize_model_parallel(tensor_model_parallel_size=a.tp_degree or dist.get_world_size())
    rank0 = dist.get_rank() == 0
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    tokenizer = hf_model = None
    if a.model_path:
        hf_cfg, state = a.model_path, a.model_path
        if os.path.isfile(os.path.join(a.model_path, "tokenizer_config.json")):
            tokenizer = transformers.AutoTokenizer.from_pretrained(a.model_path, padding_side="right")
    else:
        torch.manual_seed(0)
        if a.family == "gpt_neox":
            hc = transformers.GPTNeoXConfig(vocab_size=512, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                                            num_attention_heads=4, rotary_pct=0.25, hidden_act="gelu_fast",
                                            max_position_embeddings=a.seq_len, attn_implementation="eager")
            hf_model = transformers.GPTNeoXForCausalLM(hc).eval()
        else:
            hc = transformers.LlamaConfig(vocab_size=512, hidden_size=128, intermediate_size=352, num_hidden_layers=2, num_attention_heads=8,
                                          num_key_value_heads=4, max_position_embeddings=a.seq_len, attn_implementation="eager")
            hf_model = transformers.LlamaForCausalLM(hc).eval()
        hf_cfg, state = hc, hf_model.state_dict()
        a.check_accuracy = True
    cfg = hf_compat.config_from_hf(hf_cfg, dtype=dtype, device=dev, max_position_embeddings=a.seq_len)
    prompts = a.prompt or ["I believe the meaning of life is", "The color of the sky is"]
    if tokenizer is not None:
        ids = [tokenizer(t, return_tensors="pt").input_ids[0] for t in prompts]
    else:
        g = torch.Generator().manual_seed(1)
        ids = [torch.randint(3, cfg.vocab_size, (n,), generator=g) for n in (9, 6)][: len(prompts)]
    lm_cls = None
    if hasattr(cfg, "num_local_experts"):                        # Mixtral / DBRX checkpoints: same serving wrapper, MoE decoder
        from neuronx_distributed_b200.models.mixtral import MixtralForCausalLM as lm_cls
    if isinstance(cfg, GPTNeoXConfig):
        model = GPTNeoXForInference(cfg, batch_size=1, max_seq_len=a.seq_len).eval()
    else:
        model = LlamaForInference(cfg, batch_size=1, max_seq_len=a.seq_len, lm_cls=lm_cls).eval()
    res = hf_compat.load_hf_checkpoint(model, state)
    assert not res.missing_keys, res.missing_keys

    from neuronx_distributed_b200.inference.hf_adapter import HuggingFaceGenerationAdapter

    generate = HuggingFaceGenerationAdapter(model, eos_token_id=getattr(tokenizer, "eos_token_id", None), pad_token_id=0).generate
    outs = []
    for seq in ids:                                              # same keyword arguments as transformers' generate()
        full = generate(seq.view(1, -1).to(dev), max_new_tokens=a.max_new_tokens, do_sample=a.do_sample, top_k=a.top_k, top_p=a.top_p)
        outs.append(full[0, seq.numel():].tolist())
    if rank0:
        for i, (seq, gen) in enumerate(zip(ids, outs)):
            text = tokenizer.decode(seq.tolist() + gen, skip_special_tokens=True) if tokenizer is not None else gen
            print(f"Generated {i + 1}: {text}")
    if a.check_accuracy and rank0 and not a.do_sample:
        if hf_model is None:
            hf_model = transformers.AutoModelForCausalLM.from_pretrained(a.model_path, torch_dtype=torch.float32).eval()
        agree = total = 0
        for seq, gen in zip(ids, outs):
            want = hf_model.generate(seq.view(1, -1), max_new_tokens=a.max_new_tokens, do_sample=False, pad_token_id=0)[0, seq.numel():].tolist()
            k = next((j for j, (x, y) in enumerate(zip(gen, want)) if x != y), len(want))
            agree, total = agree + k, total + len(want)
        print(f"accuracy check vs transformers (greedy, matching prefix): {agree}/{total} tokens")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
