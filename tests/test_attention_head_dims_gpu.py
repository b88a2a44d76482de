"""Flash attention at head_dim 64, 80, 96 and 128, with and without a key-padding mask (H100, sm_90a).

References are computed in float64 from the same bf16 inputs.  Besides the float64 bounds, three properties are checked bit
for bit because the kernels are built to have them:
- zero-padding a head to 128 columns adds exact zeros to every dot product, so a D < 128 run equals the first D columns of
  the padded D = 128 run (every head size uses the same 64-row key tiles and the same per-column accumulation order);
- a key hidden by the mask is treated like a key past S_kv, so right padding equals an unmasked run on the unpadded keys;
- every gradient element is written by one thread (no atomics), so the backward is reproducible.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

DIMS = (64, 80, 96, 128)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _rel(a, b):
    """max |a − b| relative to max |b| (the bound the D = 128 tests use)."""
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _ref64(q, k, v, go, causal, scale, mask=None):
    """float64 (O, LSE, dQ, dK, dV) for bf16 q [B,Sq,H,D], k/v [B,Sk,Hkv,D], go [B,Sq,H,D] and an optional key mask [B,Sk].
    A query row that sees no key gets O = 0, LSE = −inf and zero gradients (the kernels' rule)."""
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    g = H // Hkv
    qd, kd, vd, gd = (t.double() for t in (q, k, v, go))
    kk, vv = kd.repeat_interleave(g, 2), vd.repeat_interleave(g, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qd, kk) * scale
    vis = torch.ones(B, 1, Sq, Sk, dtype=torch.bool, device=q.device)
    if causal:
        vis = vis & torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril()
    if mask is not None:
        vis = vis & mask.bool()[:, None, None, :]
    s = s.masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, -1)                                                   # −inf for empty rows
    p = torch.where(vis, torch.exp(s - lse.unsqueeze(-1).clamp_min(-1e300)), torch.zeros((), dtype=s.dtype, device=s.device))
    o = torch.einsum("bhqk,bkhd->bqhd", p, vv)
    dp = torch.einsum("bqhd,bkhd->bhqk", gd, vv)
    delta = (gd * o).sum(-1).transpose(1, 2).unsqueeze(-1)                         # [B,H,Sq,1]
    ds = p * (dp - delta)
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, qd).view(B, Sk, Hkv, g, D).sum(3) * scale
    dv = torch.einsum("bhqk,bqhd->bkhd", p, gd).view(B, Sk, Hkv, g, D).sum(3)
    return o, lse, dq, dk, dv


def _make(layout, B, Sq, Sk, H, Hkv, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()   # noqa: E731
    if layout == "bshd":
        q, k, v = rn(B, Sq, H, D), rn(B, Sk, Hkv, D), rn(B, Sk, Hkv, D)
    elif layout == "sbhd":
        q, k, v = rn(Sq, B, H, D).transpose(0, 1), rn(Sk, B, Hkv, D).transpose(0, 1), rn(Sk, B, Hkv, D).transpose(0, 1)
    else:                                                                             # slices of a fused QKV projection
        assert Sq == Sk
        f = rn(Sq, B, (H + 2 * Hkv) * D)
        q = f[..., : H * D].view(Sq, B, H, D).transpose(0, 1)
        k = f[..., H * D:(H + Hkv) * D].view(Sq, B, Hkv, D).transpose(0, 1)
        v = f[..., (H + Hkv) * D:].view(Sq, B, Hkv, D).transpose(0, 1)
    return q, k, v, rn(B, Sq, H, D)


def _run(q, k, v, go, causal, scale, mask=None):
    """(O, LSE, dQ, dK, dV) from the extension, through the same calls the autograd front-end makes."""
    from neuronx_distributed_b200.ops import _ext, attention

    e = _ext.ext()
    tv = attention._tma_view
    q, k, v, go = tv(q), tv(k), tv(v), tv(go)
    o, lse = e.flash_attn_fwd(q, k, v, causal, scale, True, mask)
    dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True, None, mask)
    return o, lse, dq, dk, dv


def _check64(got, ref, what):
    o, lse, dq, dk, dv = got
    ro, rl, rdq, rdk, rdv = ref
    assert _rel(o, ro) < 2e-2, what
    fin = torch.isfinite(rl)
    assert torch.equal(torch.isfinite(lse), fin), what
    assert (lse[fin].double() - rl[fin]).abs().max().item() < 2e-2, what
    for name, a, b in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        assert _rel(a, b) < 3e-2, (what, name, _rel(a, b))


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("layout", ["bshd", "sbhd", "fused"])
def test_head_dims_vs_float64(_ext, D, causal, layout):
    """Front-end autograd path and raw extension outputs (O, LSE, dQ, dK, dV) against float64, GQA H=4 / Hkv=2, S=200."""
    from neuronx_distributed_b200.ops import attention

    B, S, H, Hkv = 2, 200, 4, 2
    q, k, v, go = _make(layout, B, S, S, H, Hkv, D, seed=D + 7 * causal)
    scale = 1.0 / math.sqrt(D)
    ref = _ref64(q, k, v, go, causal, scale)
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
    n0 = _ext.launches()
    o = attention.flash_attention(qg, kg, vg, causal=causal)
    o.backward(go)
    assert _ext.launches() >= n0 + 4, "own attention kernels did not run"
    _, lse, *_ = _run(q, k, v, go, causal, scale)
    _check64((o, lse, qg.grad, kg.grad, vg.grad), ref, (D, causal, layout))


@pytest.mark.parametrize("D", DIMS)
def test_head_dims_unequal_lengths_vs_float64(_ext, D):
    """Non-causal S_q = 130, S_kv = 70: ragged query and key tails in the same call."""
    q, k, v, go = _make("bshd", 2, 130, 70, 4, 2, D, seed=3 * D)
    scale = 1.0 / math.sqrt(D)
    n0 = _ext.launches()
    from neuronx_distributed_b200.ops import attention

    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
    attention.flash_attention(qg, kg, vg, causal=False).backward(go)
    assert _ext.launches() > n0
    got = _run(q, k, v, go, False, scale)
    _check64(got, _ref64(q, k, v, go, False, scale), D)
    for a, b in zip((qg.grad, kg.grad, vg.grad), got[2:]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("D", (64, 80, 96))
@pytest.mark.parametrize("causal", [True, False])
def test_zero_padding_to_128_is_bit_identical(_ext, D, causal):
    """D < 128 equals the first D columns of a D = 128 run on zero-padded q, k, v, dO (scale passed explicitly)."""
    q, k, v, go = _make("bshd", 2, 200, 200, 4, 2, D, seed=11 + D)
    pad = lambda t: torch.nn.functional.pad(t, (0, 128 - D))       # noqa: E731
    scale = 1.0 / math.sqrt(D)
    small = _run(q, k, v, go, causal, scale)
    big = _run(pad(q), pad(k), pad(v), pad(go), causal, scale)
    o, lse, dq, dk, dv = small
    po, plse, pdq, pdk, pdv = big
    assert torch.equal(o, po[..., :D]) and torch.equal(lse, plse) and torch.equal(dv, pdv[..., :D])
    assert torch.equal(dq, pdq[..., :D]) and torch.equal(dk, pdk[..., :D])
    for t in (po, pdq, pdk, pdv):
        assert not t[..., D:].any()


@pytest.mark.parametrize("D", DIMS)
def test_right_padding_equals_unpadded_run(_ext, D):
    """Right padding, non-causal: each sequence's masked run equals an unmasked B = 1 run on its first `len` keys."""
    lens = (512, 317, 64, 1)
    B, S, H, Hkv = len(lens), 512, 4, 2
    q, k, v, go = _make("bshd", B, S, S, H, Hkv, D, seed=5 + D)
    mask = torch.arange(S, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    scale = 1.0 / math.sqrt(D)
    o, lse, dq, dk, dv = _run(q, k, v, go, False, scale, mask)
    for b, n in enumerate(lens):
        ro, rlse, rdq, rdk, rdv = _run(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], go[b:b + 1], False, scale)
        assert torch.equal(o[b:b + 1], ro) and torch.equal(lse[b:b + 1], rlse), (D, n)
        assert torch.equal(dq[b:b + 1], rdq), (D, n)
        assert torch.equal(dk[b:b + 1, :n], rdk) and torch.equal(dv[b:b + 1, :n], rdv), (D, n)
        assert not dk[b, n:].any() and not dv[b, n:].any(), (D, n)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["left", "random"])
@pytest.mark.parametrize("causal", [True, False])
def test_mask_vs_float64(_ext, D, kind, causal):
    """Left padding and a random mask, with GQA, against float64; masked keys get dK = dV = 0 exactly, and query rows with
    no visible key (left padding under a causal mask) get O = 0, LSE = −inf, dQ = 0."""
    from neuronx_distributed_b200.ops import attention

    B, S, H, Hkv = 3, 200, 4, 2
    q, k, v, go = _make("bshd", B, S, S, H, Hkv, D, seed=17 + D + causal)
    if kind == "left":
        mask = torch.arange(S, device="cuda")[None, :] >= torch.tensor([0, 37, 150], device="cuda")[:, None]
    else:
        mask = torch.rand(B, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(D)) < 0.7
    scale = 1.0 / math.sqrt(D)
    ref = _ref64(q, k, v, go, causal, scale, mask)
    got = _run(q, k, v, go, causal, scale, mask.to(torch.uint8))
    _check64(got, ref, (D, kind, causal))
    o, lse, dq, dk, dv = got
    hidden = ~mask
    assert not dk[hidden].any() and not dv[hidden].any()
    empty = ~torch.isfinite(ref[1])                                               # [B, H, S]
    assert torch.equal(~torch.isfinite(lse), empty)
    rows = empty.transpose(1, 2)                                                  # [B, S, H]
    assert not o[rows].any() and not dq[rows].any()
    for t in got:
        assert not torch.isnan(t).any()
    # the autograd front-end takes the bool mask and gives the same result
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
    fo = attention.flash_attention(qg, kg, vg, causal=causal, key_padding_mask=mask)
    fo.backward(go)
    assert torch.equal(fo, o) and torch.equal(qg.grad, dq) and torch.equal(kg.grad, dk) and torch.equal(vg.grad, dv)


@pytest.mark.parametrize("D", DIMS)
def test_fully_masked_batch_row(_ext, D):
    """A batch row with every key masked: O = 0, LSE = −inf, dQ = dK = dV = 0, no NaN; the other row is unaffected."""
    B, S, H, Hkv = 2, 130, 4, 2
    q, k, v, go = _make("bshd", B, S, S, H, Hkv, D, seed=23 + D)
    mask = torch.ones(B, S, dtype=torch.bool, device="cuda")
    mask[1] = False
    scale = 1.0 / math.sqrt(D)
    for causal in (False, True):
        o, lse, dq, dk, dv = _run(q, k, v, go, causal, scale, mask)
        for t in (o, lse, dq, dk, dv):
            assert not torch.isnan(t).any()
        assert not o[1].any() and bool((lse[1] == float("-inf")).all()) and not dq[1].any()
        assert not dk[1].any() and not dv[1].any()
        ro, rlse, rdq, rdk, rdv = _run(q[:1], k[:1], v[:1], go[:1], causal, scale)
        assert torch.equal(o[:1], ro) and torch.equal(lse[:1], rlse) and torch.equal(dq[:1], rdq)
        assert torch.equal(dk[:1], rdk) and torch.equal(dv[:1], rdv)


@pytest.mark.parametrize("D", DIMS)
def test_backward_is_bit_reproducible(_ext, D):
    q, k, v, go = _make("sbhd", 2, 333, 333, 8, 2, D, seed=29 + D)
    mask = torch.rand(2, 333, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) < 0.8
    scale = 1.0 / math.sqrt(D)
    for causal, m in ((True, None), (False, mask), (True, mask)):
        a, b = _run(q, k, v, go, causal, scale, m), _run(q, k, v, go, causal, scale, m)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (D, causal, m is not None)


@pytest.mark.parametrize("D", (64, 96))
def test_flash_attention_with_lse_is_differentiable(_ext, D):
    """Ring attention merges blocks through their LSEs: gradients must flow through the LSE output at these head sizes."""
    from neuronx_distributed_b200.ops import attention

    B, S, H = 2, 256, 4
    q, k, v, _ = _make("bshd", B, S, S, H, H, D, seed=31 + D)
    q, k, v = (t.detach().requires_grad_(True) for t in (q, k, v))
    n0 = _ext.launches()
    res = attention.flash_attention_with_lse(q, k, v, False, 1.0 / math.sqrt(D))
    assert res is not None
    o, lse = res
    g = torch.Generator(device="cuda").manual_seed(D)
    w_o = torch.randn(o.shape, device="cuda", generator=g)
    w_l = torch.randn(lse.shape, device="cuda", generator=g)
    ((o.float() * w_o).sum() + (lse * w_l).sum()).backward()
    assert _ext.launches() >= n0 + 4
    qf, kf, vf = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) / math.sqrt(D)
    ro = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), vf)
    rl = torch.logsumexp(s, -1)
    ((ro * w_o.double()).sum() + (rl * w_l.double()).sum()).backward()
    assert _rel(o, ro.detach()) < 2e-2 and (lse.double() - rl.detach()).abs().max().item() < 2e-2
    for a, b in ((q.grad, qf.grad), (k.grad, kf.grad), (v.grad, vf.grad)):
        assert _rel(a, b) < 3e-2


# ---- models on CUDA in bf16: own kernels vs the same seeded model on SDPA (NXD_DISABLE_OWN_ATTENTION=1) -------------------
def _one_rank_model_parallel():
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29544")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    if not ps.model_parallel_is_initialized():
        ps.initialize_model_parallel(1)


def _bert(kw):
    from neuronx_distributed_b200.models import bert

    m = bert.BertModel(bert.BertConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                       num_attention_heads=4, max_position_embeddings=256, hidden_dropout_prob=0.0, **kw))
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, 512, (3, 160), device="cuda", generator=g)
    am = (torch.arange(160, device="cuda")[None, :] < torch.tensor([160, 97, 33], device="cuda")[:, None]).long()
    return m, lambda: m(ids, torch.zeros_like(ids), am)[0]


def _vit(kw):
    from neuronx_distributed_b200.models import vit

    m = vit.ViTForImageClassification(vit.ViTConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                                    num_attention_heads=4, image_size=64, patch_size=8, num_labels=10, **kw))
    px = torch.randn(2, 3, 64, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).bfloat16()
    return m, lambda: m(px)                                                       # 64 patches + CLS: S = 65


def _neox(hidden):
    def make(kw):
        from neuronx_distributed_b200.models import gpt_neox

        m = gpt_neox.GPTNeoXForCausalLM(gpt_neox.GPTNeoXConfig(vocab_size=512, hidden_size=hidden, intermediate_size=4 * hidden,
                                                               num_hidden_layers=2, num_attention_heads=4,
                                                               max_position_embeddings=256, **kw))
        ids = torch.randint(0, 512, (2, 150), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))

        def fwd():
            out = m(ids)
            return out[1] if isinstance(out, tuple) else out
        return m, fwd
    return make


@pytest.mark.parametrize("name,make", [("bert_d64_padded", _bert), ("vit_d64_s65", _vit),
                                       ("neox_d96", _neox(384)), ("neox_d80", _neox(320))])
def test_models_match_sdpa(_ext, monkeypatch, name, make):
    """Loss and every parameter gradient with the own kernels vs the same seeded model with attention on SDPA."""
    _one_rank_model_parallel()
    kw = dict(dtype=torch.bfloat16, device=torch.device("cuda", 0))
    results = []
    for disable in ("0", "1"):
        monkeypatch.setenv("NXD_DISABLE_OWN_ATTENTION", disable)
        torch.manual_seed(0)
        m, fwd = make(kw)
        n0 = _ext.launches()
        out = fwd().float()
        w = torch.randn(out.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        loss = (out * w).sum() / out.numel() ** 0.5
        loss.backward()
        torch.cuda.synchronize()
        launched = _ext.launches() - n0
        results.append((float(loss), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None},
                        launched))
    (l_own, g_own, n_own), (l_ref, g_ref, n_ref) = results
    assert n_own >= n_ref + 2 * 4, "own attention kernels did not run"      # fwd + 3 bwd per layer, 2 layers
    assert abs(l_own - l_ref) <= 2e-2 * max(1.0, abs(l_ref)), (name, l_own, l_ref)
    assert g_own.keys() == g_ref.keys() and g_own
    gmax = max(g.abs().max().item() for g in g_ref.values())
    for n in g_ref:
        if n.endswith("attention.key.bias"):
            # q·(k_j + b) shifts every key score of a query by the same q·b, which softmax ignores: the exact gradient of a
            # key bias is 0 and both runs hold rounding noise only (about 1e-5 here, against a largest gradient of ~0.2)
            assert max(g_own[n].abs().max().item(), g_ref[n].abs().max().item()) < 1e-3 * gmax, (name, n)
            continue
        assert _rel(g_own[n].float(), g_ref[n].double()) < 5e-2, (name, n, _rel(g_own[n].float(), g_ref[n].double()))
