"""``ops.attention.speculation_attention`` off the GPU: its torch path against float64 attention written from the rule.

W new tokens per sequence sit in cache slots p .. p + W − 1 (p = positions[b]); token w sits at sequence position p + d[w]
and has tree-mask row M[w] (a chain: d = arange(W), M lower-triangular).  Token w sees slot c iff
  - c < p and, with a sliding window SW, c > p + d[w] − SW; or
  - c = p + u < p + W with M[w, u] and, with SW, d[u] > d[w] − SW.
"""
import math

import pytest
import torch

from neuronx_distributed_b200.ops import attention

E4M3 = torch.float8_e4m3fn
# the candidate tree of examples/inference/run_llama_medusa.py (10 nodes)
MEDUSA_CHOICES = [[0], [1], [2], [0, 0], [0, 1], [1, 0], [0, 0, 0], [0, 0, 1], [0, 1, 0]]


def medusa_tree(device="cpu"):
    from neuronx_distributed_b200.utils.medusa_utils import generate_medusa_buffers

    buf = generate_medusa_buffers(MEDUSA_CHOICES, device=device, topk=10)
    return buf["medusa_attn_mask"][0, 0].bool(), buf["medusa_position_ids"].long()


def random_tree(W, seed, device="cpu"):
    """A random valid tree of W nodes: node 0 is the root, node i's parent is a random earlier node."""
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(W, W, dtype=torch.bool)
    depth = torch.zeros(W, dtype=torch.long)
    mask[0, 0] = True
    for i in range(1, W):
        par = int(torch.randint(0, i, (1,), generator=g))
        mask[i] = mask[par]
        mask[i, i] = True
        depth[i] = depth[par] + 1
    return mask.to(device), depth.to(device)


def visible(p, w, W, L, mask, depth, sw):
    """Slots token w of a window at p sees, straight from the rule: bool [L]."""
    c = torch.arange(L)
    d = torch.arange(W) if depth is None else depth.cpu()
    m = torch.ones(W, W, dtype=torch.bool).tril() if mask is None else mask.cpu()
    committed = (c < p) & (True if sw is None else c > p + int(d[w]) - sw)
    u = c - p
    ok = (u >= 0) & (u < W)
    uc = u.clamp(0, W - 1)
    win = ok & m[w, uc] & (True if sw is None else d[uc] > int(d[w]) - sw)
    return committed | win


def ref64(q, k, v, pos, mask=None, depth=None, sw=None, scale=None):
    """float64 attention of q [B,W,H,D] over caches [B,L,Hkv,D] (already de-quantised) under the rule; 0 for a token that
    sees nothing."""
    q, k, v = q.double().cpu(), k.double().cpu(), v.double().cpu()
    B, W, H, D = q.shape
    L, Hkv = k.shape[1], k.shape[2]
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    out = torch.zeros(B, W, H, D, dtype=torch.float64)
    for b in range(B):
        for w in range(W):
            idx = visible(int(pos[b]), w, W, L, mask, depth, sw).nonzero()[:, 0]
            if idx.numel() == 0:
                continue
            kk = k[b, idx].repeat_interleave(H // Hkv, 1)                   # [n, H, D]
            vv = v[b, idx].repeat_interleave(H // Hkv, 1)
            s = torch.einsum("hd,nhd->hn", q[b, w], kk) * scale
            out[b, w] = torch.einsum("hn,nhd->hd", s.softmax(-1), vv)
    return out


def rel(a, b):
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def make(B, W, H, Hkv, L, D=16, dtype=torch.float64, seed=0, fp8_scales=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, W, H, D, generator=g).to(dtype)
    k = torch.randn(B, L, Hkv, D, generator=g)
    v = torch.randn(B, L, Hkv, D, generator=g)
    if fp8_scales is None:
        return q, k.to(dtype), v.to(dtype), k.to(dtype), v.to(dtype)
    ks, vs = fp8_scales
    k8, v8 = (k / ks).to(E4M3), (v / vs).to(E4M3)
    return q, k8, v8, (k8.float() * ks).double(), (v8.float() * vs).double()      # the cache's fp32 de-quantisation


TREES = ("chain", "medusa", "random")


def tree_args(kind, W):
    if kind == "chain":
        return None, None
    return medusa_tree() if kind == "medusa" else random_tree(W, 3)


@pytest.mark.parametrize("kind", TREES)
@pytest.mark.parametrize("sw", (None, 4))
@pytest.mark.parametrize("cache", ("float64", "e4m3"))
def test_torch_path_equals_float64_rule(kind, sw, cache):
    """Exact in float64: the torch path applies the rule and nothing else (p = 0, inside and near the end of the cache)."""
    W, H, Hkv, L = 10, 4, 2, 40
    mask, depth = tree_args(kind, W)
    scales = (0.3, 0.7) if cache == "e4m3" else None
    q, kc, vc, kd, vd = make(3, W, H, Hkv, L, fp8_scales=scales)
    pos = torch.tensor([0, 13, L - W])
    kw = {} if scales is None else {"k_scale": scales[0], "v_scale": scales[1]}
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw, **kw)
    assert rel(got, ref64(q, kd, vd, pos, mask, depth, sw)) < 1e-12


@pytest.mark.parametrize("kind", TREES)
@pytest.mark.parametrize("sw", (None, 4))
def test_torch_path_bf16(kind, sw):
    W, H, Hkv, L = 10, 8, 2, 64
    mask, depth = tree_args(kind, W)
    q, kc, vc, kd, vd = make(2, W, H, Hkv, L, dtype=torch.bfloat16, seed=1)
    pos = torch.tensor([0, 30])
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw)
    assert got.dtype == torch.bfloat16
    assert rel(got, ref64(q, kd, vd, pos, mask, depth, sw)) < 2e-2


def test_sliding_window_starts_in_prefix_and_in_window():
    """The SW used above really splits the rows: some windows start in the committed prefix, some inside the new tokens."""
    W, L, sw, p = 10, 40, 4, 13
    for kind in TREES:
        mask, depth = tree_args(kind, W)
        d = torch.arange(W) if depth is None else depth
        starts = [p + int(d[w]) - sw + 1 for w in range(W)]
        assert min(starts) < p and max(starts) >= p, kind


def test_visibility_helper_matches_rule():
    W, L = 10, 40
    pos = torch.tensor([0, 13, 30, 39])
    for kind in TREES:
        mask, depth = tree_args(kind, W)
        for sw in (None, 1, 4, 100):
            got = attention.speculation_visibility(pos, L, W, mask, depth, attention.check_window(sw))
            for b, p in enumerate(pos.tolist()):
                for w in range(W):
                    assert torch.equal(got[b, w], visible(p, w, W, L, mask, depth, sw)), (kind, sw, p, w)


def test_argument_errors():
    q, kc, vc, _, _ = make(1, 4, 4, 2, 16)
    pos = torch.tensor([3])
    mask, depth = random_tree(4, 0)
    with pytest.raises(ValueError, match="go together"):
        attention.speculation_attention(q, kc, vc, pos, tree_mask=mask)
    with pytest.raises(ValueError, match="go together"):
        attention.speculation_attention(q, kc, vc, pos, tree_depth=depth)
    with pytest.raises(ValueError, match=r"\[W, W\]"):
        attention.speculation_attention(q, kc, vc, pos, mask[:3, :3], depth[:3])
    with pytest.raises(ValueError, match=r"\[W, W\]"):
        attention.speculation_attention(q, kc, vc, pos, mask, depth[:3])
    with pytest.raises(ValueError, match="sliding_window"):
        attention.speculation_attention(q, kc, vc, pos, sliding_window=0)
    with pytest.raises(ValueError, match="fp8 caches only"):
        attention.speculation_attention(q, kc, vc, pos, k_scale=0.5)
    with pytest.raises(ValueError, match="same dtype"):
        attention.speculation_attention(q, kc, vc.float(), pos)
    with pytest.raises(ValueError, match="does not match"):
        attention.speculation_attention(q[..., :8], kc, vc, pos)
    with pytest.raises(ValueError, match="expected q"):
        attention.speculation_attention(q[0], kc, vc, pos)
