"""The token-generation attention kernels on the H100 (sm_90a), slot by slot: ``decode_attention`` (``csrc/decode.cu``
``decode_attn_kernel`` + ``decode_combine_kernel``), flash-decoding's local partial (+ ``decode_combine_partial_kernel``)
and ``speculation_attention`` (``csrc/attention_sm90.cu`` ``spec_attn_kernel``), on the bf16 and the e4m3 cache, at every
head size and GQA group, at real-model shapes and at the split layouts the launchers make rare.  The probes — exact
visibility sums, planted slots and float64 with per-element bounds — and their derivations are in
``test_decode_probes_cpu.py``; the split counts follow the launchers' formulas on this device's SM count."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_decode_probes_cpu import (Case, check_planted, check_random, check_visibility, check_visibility_partial,  # noqa: E402
                                    decode_run, partial_run, spec_run)

pytestmark = pytest.mark.gpu

CACHES = ("bf16", "e4m3")
DIMS = (64, 80, 96, 128)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def counted(_ext, run, per_call=2):
    """``run`` that asserts each call went through the extension's kernels (the attention kernel and a combine)."""
    def wrapped(*a):
        n0 = _ext.launches()
        out = run(*a)
        assert _ext.launches() == n0 + per_call, "fell back to the torch path"
        return out
    return wrapped


# ---- one-token decode -----------------------------------------------------------------------------------------------------
DECODE = [
    # Llama-2-13B at the bench decode shape (40 / 40 heads, 2048-row cache), and its TP = 2 / 4 shards
    Case("llama2-13b-p1024", H=40, Hkv=40, D=128, L=2048, pos=(1024,)),
    Case("llama2-13b-p2047", H=40, Hkv=40, D=128, L=2048, pos=(2047,)),
    Case("llama2-13b-tp2", H=20, Hkv=20, D=128, L=2048, pos=(1500,)),
    Case("llama2-13b-tp4", H=10, Hkv=10, D=128, L=2048, pos=(1024, 2047)),
    # Llama-3-8B / Mistral-7B: 32 / 8 heads; 8192 rows, 32768 rows at the 64-split cap, a 4096 window
    Case("llama3-8b-8k", H=32, Hkv=8, D=128, L=8192, pos=(4999, 8191)),
    Case("llama3-8b-32k", H=32, Hkv=8, D=128, L=32768, pos=(32767,)),
    Case("mistral-7b-32k-sw4096", H=32, Hkv=8, D=128, L=32768, pos=(30000,), window=4096),
    # rolling: 8192 rows, window 4096, positions past L; the ring wraps 95 slots into the range (in the second split)
    Case("mistral-7b-rolling", H=32, Hkv=8, D=128, L=8192, pos=(20384,), window=4096, rolling=True),
    Case("mistral-7b-rolling-b2", H=32, Hkv=8, D=128, L=8192, pos=(4095, 12287), window=4096, rolling=True),
    Case("llama3.2-1b", H=32, Hkv=8, D=64, L=4096, pos=(0, 2047, 4095)),
    Case("phi3-mini", H=32, Hkv=32, D=96, L=4096, pos=(1, 3000)),
    Case("pythia-2.8b", H=32, Hkv=32, D=80, L=2048, pos=(5, 2047)),
    # B·Hkv ≥ 6·SMs: one split per sequence
    Case("single-split", H=32, Hkv=8, D=128, L=512, pos=tuple((37 * i) % 512 for i in range(128))),
    # fewer visible slots than splits; positions 0 and L − 1
    Case("few-visible", H=8, Hkv=2, D=128, L=4096, pos=(0, 1, 7, 4095)),
]
# every head size × GQA group, with and without a window
DECODE += [Case(f"grid-d{D}-g{G}" + ("-sw300" if sw else ""), H=8, Hkv=8 // G, D=D, L=1024, pos=(0, 150, 700, 1023),
                window=sw) for D in DIMS for G in (1, 2, 4, 8) for sw in (0, 300)]
DECODE += [Case(f"grid-rolling-d{D}-g{G}", H=8, Hkv=8 // G, D=D, L=512, pos=(100, 600, 1535), window=300, rolling=True)
           for D in DIMS for G in (1, 8)]
# flash-decoding's local positions: before the shard, inside it and past its end
PARTIAL = [Case(f"local-d{D}-g{G}", H=8, Hkv=8 // G, D=D, L=512, pos=(-40, -1, 0, 63, 511, 512, 700), window=sw)
           for D in DIMS for G in (1, 8) for sw in (0, 100)]


def _id(c):
    return c.name


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", DECODE, ids=_id)
def test_decode_visibility_probe(_ext, case, cache):
    """Probe A through ``decode_attention``'s bf16 output (every band of slots), and through the exact fp32 partial."""
    check_visibility(case, cache, counted(_ext, decode_run(case)), "cuda")
    if not case.rolling:
        check_visibility_partial(case, cache, counted(_ext, partial_run(case)), "cuda")


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", DECODE, ids=_id)
def test_decode_planted_probe(_ext, case, cache):
    check_planted(case, cache, counted(_ext, decode_run(case)), "cuda", sms(), spec=False)


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", DECODE, ids=_id)
def test_decode_random_vs_float64(_ext, case, cache):
    check_random(case, cache, counted(_ext, decode_run(case)), "cuda", sms(), spec=False)


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", PARTIAL, ids=_id)
def test_partial_probes_at_local_positions(_ext, case, cache):
    check_visibility_partial(case, cache, counted(_ext, partial_run(case)), "cuda")
    check_planted(case, cache, counted(_ext, partial_run(case)), "cuda", sms(), spec=False, partial=True)


# ---- verification of W tokens ---------------------------------------------------------------------------------------------
SPEC = [
    Case("llama2-13b-medusa", H=40, Hkv=40, D=128, L=2048, pos=(1024,), W=10, tree="medusa"),
    Case("llama2-13b-tp4-chain5", H=10, Hkv=10, D=128, L=2048, pos=(2043,), W=5),
    Case("llama3-8b-chain5", H=32, Hkv=8, D=128, L=8192, pos=(3000, 8187), W=5),
    Case("llama3-8b-w64", H=32, Hkv=8, D=128, L=8192, pos=(8128,), W=64),                 # W·G = 256: 4 row tiles
    Case("llama3-8b-w63-sw4096", H=32, Hkv=8, D=128, L=32768, pos=(20000,), W=63, window=4096),
    # rolling at window + W − 1 = L, positions past L, W·G > 64
    Case("mistral-7b-rolling-w63", H=32, Hkv=8, D=128, L=4158, pos=(3 * 4158 + 100,), W=63, window=4096, rolling=True),
    Case("mistral-7b-rolling-medusa", H=32, Hkv=8, D=128, L=4105, pos=(5000, 9000), W=10, window=4096, rolling=True,
         tree="medusa"),
    Case("llama3.2-1b-medusa-sw", H=32, Hkv=8, D=64, L=4096, pos=(300, 4086), W=10, window=300, tree="medusa"),
    Case("phi3-random-tree", H=32, Hkv=32, D=96, L=2048, pos=(0, 1500), W=16, tree="random"),
    Case("pythia-chain63", H=32, Hkv=32, D=80, L=2048, pos=(1, 1985), W=63),
    Case("w1", H=32, Hkv=8, D=128, L=2048, pos=(0, 2047), W=1),
    Case("w2-sw", H=32, Hkv=8, D=128, L=2048, pos=(64, 2046), W=2, window=129),
    Case("g8-w64", H=64, Hkv=8, D=128, L=1024, pos=(500,), W=64),                         # W·G = 512: 8 row tiles
    Case("g8-w63-sw-random", H=16, Hkv=2, D=64, L=1024, pos=(700,), W=63, window=200, tree="random"),
]
SPEC += [Case(f"grid-d{D}-g{G}-" + (tree or "chain") + ("-sw200" if sw else ""), H=8, Hkv=8 // G, D=D, L=1024,
              pos=(0, 500, 1019), W=5 if tree is None else (10 if tree == "medusa" else 12), window=sw, tree=tree)
         for D in DIMS for G in (1, 2, 4, 8) for tree, sw in ((None, 0), ("medusa", 200), ("random", 0))]
SPEC += [Case(f"grid-rolling-d{D}-g{G}", H=8, Hkv=8 // G, D=D, L=512, pos=(100, 1400), W=5, window=508, rolling=True)
         for D in DIMS for G in (1, 8)]


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", SPEC, ids=_id)
def test_spec_visibility_probe(_ext, case, cache):
    check_visibility(case, cache, counted(_ext, spec_run(case)), "cuda")


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", SPEC, ids=_id)
def test_spec_planted_probe(_ext, case, cache):
    check_planted(case, cache, counted(_ext, spec_run(case)), "cuda", sms(), spec=True)


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", SPEC, ids=_id)
def test_spec_random_vs_float64(_ext, case, cache):
    check_random(case, cache, counted(_ext, spec_run(case)), "cuda", sms(), spec=True)
