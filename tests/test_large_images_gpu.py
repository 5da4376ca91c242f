"""Images of more than 1024 pixels: the split KV-cached decode (S > 1024 keys per head), the incremental samplers of
ImageGPT and PixelSNAIL on it, and training parity of all four models at 64x64 (S = 4096).

Above 1024 keys `pg_attn_decode` runs one block per 1024 cache rows and merges their partial (max, sum, output) in
split order.  The kernel tests restate the causal attention in fp32 torch; the model tests use the oracle and the
tolerance of test_parity_gpu.py (1e-2 relative to max(1, max|ref|) on the bf16 path).
"""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

TOL = 1e-2


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def check(name, got, ref, tol=TOL):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    bound = tol * max(1.0, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e}"


# --------------------------------------------------------------------------------------------------
# pg_attn_decode with more than 1024 keys
# --------------------------------------------------------------------------------------------------
def _qkv(N, S, H, dk, dv, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(N * S, H * (2 * dk + dv), generator=g).to(dev()).bfloat16()
    return qkv[:, : H * dk], qkv[:, H * dk: 2 * H * dk], qkv[:, 2 * H * dk:]


def _full_attention(q, k, v, N, S, H, dk, dv, strict):
    """fp32 restatement of the reference's attention core (nn/attention.py:147-160) -> [N, S, H*dv]."""
    qf = q.float().view(N, S, H, dk).transpose(1, 2)
    kf = k.float().view(N, S, H, dk).transpose(1, 2)
    vf = v.float().view(N, S, H, dv).transpose(1, 2)
    mask = torch.tril(torch.ones(S, S, device=q.device), diagonal=-int(strict)).view(1, 1, S, S)
    s = (qf @ kf.transpose(2, 3)) / math.sqrt(dk)
    s = s.masked_fill(mask == 0, float("-inf"))
    p = torch.softmax(s, dim=-1).masked_fill(mask == 0, 0)
    return (p @ vf).transpose(1, 2).reshape(N, S, H * dv)


def _decode_all(L, q, k, v, N, S, H, dk, dv, strict, positions, capacity=None):
    """Appends `positions` one at a time to zeroed caches of `capacity` rows per image -> (outputs [P, N, H*dv],
    k cache, v cache)."""
    cap = capacity or S
    kc = torch.zeros(N * cap, H * dk, device=dev(), dtype=torch.bfloat16)
    vc = torch.zeros(N * cap, H * dv, device=dev(), dtype=torch.bfloat16)
    pos = torch.zeros(1, dtype=torch.int32, device=dev())
    qv, kv_, vv = q.view(N, S, -1), k.view(N, S, -1), v.view(N, S, -1)
    outs = torch.full((len(positions), N, H * dv), float("nan"), device=dev(), dtype=torch.bfloat16)
    for i, p in enumerate(positions):
        pos.fill_(p)
        L.attn_decode(qv[:, p].contiguous(), kv_[:, p].contiguous(), vv[:, p].contiguous(), kc, vc, outs[i], pos, N,
                      cap, H, dk, dv, strict)
    torch.cuda.synchronize()
    return outs, kc, vc


DECODE_CASES = [
    # N, S, H, dk, dv, strict: every value of every axis at least once
    (1, 1025, 1, 64, 64, False),     # one key in the second split
    (3, 1025, 4, 128, 128, True),
    (1, 2048, 4, 64, 128, False),    # two full splits
    (3, 2048, 1, 64, 64, True),
    (1, 3000, 1, 128, 128, True),    # a partial last split
    (3, 3000, 4, 64, 128, False),
    (1, 4096, 4, 64, 64, True),
    (3, 4096, 1, 128, 128, False),
]


@pytest.mark.parametrize("N,S,H,dk,dv,strict", DECODE_CASES)
def test_split_decode_matches_full_attention(L, N, S, H, dk, dv, strict):
    """Appending every position in turn reproduces every row of the full causal attention, on both sides of each
    1024-key split boundary; the caches end up holding exactly k and v; a second run gives the same bits."""
    q, k, v = _qkv(N, S, H, dk, dv, seed=S + dk + dv + H + N)
    ref = _full_attention(q, k, v, N, S, H, dk, dv, strict).transpose(0, 1)   # [S, N, H*dv]
    got, kc, vc = _decode_all(L, q, k, v, N, S, H, dk, dv, strict, range(S))
    err = (got.float() - ref).abs().amax(dim=(1, 2))
    bound = 2e-3 + 2 ** -7 * ref.abs().amax(dim=(1, 2))
    bad = (err > bound) | torch.isnan(got.float()).any(dim=2).any(dim=1)
    assert not bad.any(), f"positions {bad.nonzero().flatten()[:10].tolist()} exceed the bound"
    edges = [p for b in range(1024, S, 1024) for p in (b - 1, b, b + 1) if p < S]
    assert edges and all(not bad[p] for p in edges)
    if strict:
        assert (got[0] == 0).all(), "strict mask: position 0 has no keys and must be exactly zero"
    assert torch.equal(kc, k) and torch.equal(vc, v), "each cache row is written once, with the new key / value"
    again, _, _ = _decode_all(L, q, k, v, N, S, H, dk, dv, strict, range(S))
    assert torch.equal(got, again), "two runs of the split decode differ"


@pytest.mark.parametrize("dk,dv,strict", [(64, 64, False), (128, 128, True), (64, 128, True)])
def test_decode_bits_do_not_depend_on_cache_capacity(L, dk, dv, strict):
    """With pos < 1024 a cache of 4096 rows (four splits, three of them empty, then the merge) gives exactly the bits
    of a cache of 1024 rows (the one-block kernel): empty partials and the merge add exactly nothing."""
    N, H = 3, 2
    q, k, v = _qkv(N, 1024, H, dk, dv, seed=dk + dv)
    positions = list(range(1024))
    small, kc_s, vc_s = _decode_all(L, q, k, v, N, 1024, H, dk, dv, strict, positions)
    large, kc_l, vc_l = _decode_all(L, q, k, v, N, 1024, H, dk, dv, strict, positions, capacity=4096)
    assert torch.equal(small, large), "capacity 4096 and capacity 1024 give different bits"
    assert torch.equal(kc_l.view(N, 4096, -1)[:, :1024], kc_s.view(N, 1024, -1))
    assert torch.equal(vc_l.view(N, 4096, -1)[:, :1024], vc_s.view(N, 1024, -1))
    assert not kc_l.view(N, 4096, -1)[:, 1024:].any() and not vc_l.view(N, 4096, -1)[:, 1024:].any()


# --------------------------------------------------------------------------------------------------
# Incremental samplers at 64x64 and 32x48
# --------------------------------------------------------------------------------------------------
IGPT_64 = dict(in_channels=1, out_channels=1, in_size=64, n_transformer_blocks=2, n_attention_heads=2,
               n_embedding_channels=64)
SNAIL_2 = dict(in_channels=1, out_channels=1, n_channels=64, n_pixel_snail_blocks=2, n_residual_blocks=1,
               attention_key_channels=16, attention_value_channels=32)
SNAIL_1 = dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=1, n_residual_blocks=2,
               attention_key_channels=8, attention_value_channels=32)


def _incremental_states(m):
    return m.__dict__.get("_pixel_states") or {}


def _assert_graphed_incremental(m, shape):
    n, c, h, w = shape
    states = _incremental_states(m)
    assert (n, c, h, w, str(dev())) in states, "sample() did not take the incremental path"
    assert all(st["graph"] for st in states.values()), "per-pixel step was not graph-captured"


@pytest.mark.parametrize("name,cls,cfg,shape", [
    ("image_gpt", "ImageGPT", IGPT_64, (2, 1, 64, 64)),
    ("pixel_snail", "PixelSNAIL", SNAIL_2, (2, 1, 64, 64)),
    ("pixel_snail", "PixelSNAIL", SNAIL_1, (2, 3, 32, 48)),   # not square: S = 1536, row length 48
])
def test_large_image_sampler_logits_match_the_full_forward(name, cls, cfg, shape):
    """Teacher-forced sampling (the protocol of test_incremental_sampler_logits_match_the_full_forward): each pixel's
    logits from the K/V caches, on two calls with the per-pixel step graph-captured, against the oracle in float64 and
    against the full forward.

    Each of the two bf16 paths is held to 1e-2 of the float64 oracle; between themselves they are held to the sum of
    the two bounds.  Their errors are independent and of the same size: with the weights scaled by 1.5, PixelSNAIL
    (SNAIL_2) at 32x32, where the decode does not split, gives incremental and full logits 9.1e-3 apart (of a 1e-2
    bound), and at 64x64 1.01e-2 apart while each stays within 9.4e-3 of the oracle (H100).  The weights here are the
    oracle tests' (initial values plus a 0.02 jitter)."""
    from oracle import reference_path as O

    m, g = _fresh(cls, cfg, seed=7)
    x = torch.bernoulli(torch.full(shape, 0.5), generator=g)
    with torch.no_grad():
        state = {k: v.double() if v.is_floating_point() else v for k, v in m.state_dict().items()}
        exact = O.forward(name, state, x.double(), cfg)
    m = m.to(dev())
    x = x.to(dev())
    with torch.no_grad():
        ref = m(x)
    check("full forward vs oracle", ref, exact)
    n, c, h, w = shape
    for rep in range(2):
        seen = []
        m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), torch.zeros_like(logits))[1]
        out = m.sample(conditioned_on=x)
        assert torch.equal(out, x)
        assert len(seen) == h * w
        got = torch.stack(seen, dim=-1).view(n, c, h, w)
        check(f"incremental logits vs oracle (call {rep})", got, exact)
        check(f"incremental logits vs full forward (call {rep})", got, ref, 2 * TOL)
    _assert_graphed_incremental(m, shape)


@pytest.mark.parametrize("cls,cfg,shape", [
    ("ImageGPT", IGPT_64, (3, 1, 64, 64)),
    ("PixelSNAIL", SNAIL_2, (3, 1, 64, 64)),
])
def test_large_image_sampling_keeps_given_pixels(cls, cfg, shape):
    """64x64 sampling on the KV-cached path: the pixels given in `conditioned_on` come back bit-unchanged and every
    drawn pixel is 0 or 1."""
    from pytorch_generative_b200 import models

    torch.manual_seed(3)
    m = getattr(models, cls)(**cfg).to(dev())
    n, c, h, w = shape
    cond = torch.bernoulli(torch.full(shape, 0.5)).to(dev())
    cond[:, :, h // 2:] = -1
    cond[:, :, h // 2, : w // 3] = 0.0    # given pixels after the first unknown row are kept too
    with torch.no_grad():
        m(cond.clamp(min=0))                # registers the image shape for sample(n_samples=...)
    out = m.sample(conditioned_on=cond)
    given = cond >= 0
    assert torch.equal(out[given], cond[given])
    assert set(out.unique().tolist()) <= {0.0, 1.0}
    _assert_graphed_incremental(m, shape)
    free = m.sample(n_samples=n)
    assert free.shape == shape and set(free.unique().tolist()) <= {0.0, 1.0}


# --------------------------------------------------------------------------------------------------
# Training parity at 64x64
# --------------------------------------------------------------------------------------------------
TRAIN_64 = [
    ("image_gpt", "ImageGPT", IGPT_64),
    ("pixel_cnn", "PixelCNN", dict(in_channels=1, out_channels=1, n_residual=2, residual_channels=32, head_channels=16)),
    ("gated_pixel_cnn", "GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=2, gated_channels=64,
                                              head_channels=32)),
    ("pixel_snail", "PixelSNAIL", SNAIL_2),
]


def _fresh(cls, cfg, seed=0, jitter=0.02):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = getattr(models, cls)(**cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g) * jitter)
    return m, g


@pytest.mark.parametrize("name,cls,cfg", TRAIN_64)
def test_models_match_oracle_at_64x64(name, cls, cfg):
    """Logits, recipe loss and a fixed-cotangent VJP of every parameter at 64x64 (the protocol of
    test_conv_models_match_oracle)."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses

    m, g = _fresh(cls, cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.bernoulli(torch.full((2, 1, 64, 64), 0.5), generator=g)
    pt = O.trainable(state)
    ref_logits = O.forward(name, pt, x, cfg)
    ref_loss = O.recipe_loss(x, ref_logits).detach()
    G = torch.randn(ref_logits.shape, generator=g) / ref_logits[0].numel()
    (ref_logits * G).sum().backward()
    m = m.to(dev())
    xd = x.to(dev())
    logits = m(xd)
    loss = losses.bce_with_logits_sum_mean(logits, xd)
    (logits * G.to(dev())).sum().backward()
    check("logits", logits, ref_logits)
    assert abs(loss.item() - ref_loss.item()) <= TOL * abs(ref_loss.item())
    checked = 0
    for pname, p in m.named_parameters():
        if pt[pname].grad is None:  # parameters the reference's graph never reaches
            continue
        check("d" + pname, p.grad, pt[pname].grad)
        checked += 1
    assert checked > 0


def test_image_gpt_adam_step_matches_oracle_at_64x64():
    """One training step of ImageGPT at 64x64 (loss, gradient norm, fused Adam update) against oracle.TrainState."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses, optim

    lr = 5e-3
    m, g = _fresh("ImageGPT", IGPT_64)
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.bernoulli(torch.full((2, 1, 64, 64), 0.5), generator=g)
    ts = O.TrainState("image_gpt", init, IGPT_64, lr=lr)
    ref_loss, ref_norm = ts.step(x)
    m = m.to(dev()).train()
    opt = optim.FusedAdam(m.parameters(), lr=lr)
    xd = x.to(dev())
    loss = losses.bce_with_logits_sum_mean(m(xd), xd)
    loss.backward()
    norm = opt.clip_and_step(1e50).item()
    assert abs(loss.item() - ref_loss) <= TOL * abs(ref_loss), (loss.item(), ref_loss)
    assert abs(norm - ref_norm) <= 2.5e-2 * abs(ref_norm), (norm, ref_norm)
    num = den = worst = 0.0
    for pname, p in m.named_parameters():
        w, r, w0 = p.detach().float().cpu(), ts.p[pname].detach(), init[pname]
        num += float(((w - w0) - (r - w0)).pow(2).sum())
        den += float((r - w0).pow(2).sum())
        worst = max(worst, float((w - r).abs().max()))
    assert worst <= 2.0 * lr * 1.05, worst     # each of the two updates moves a weight by at most lr
    rel = (num / max(den, 1e-30)) ** 0.5
    assert rel <= 0.15, f"Adam update diverges from the oracle's (relative l2 {rel:.3e})"
