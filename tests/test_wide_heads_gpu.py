"""Attention heads wider than 64 query/key channels: 128-wide q/k head slots of the tensor-core kernels, through the C
ABI, the CausalAttention module, ImageGPT (training, data-parallel buckets, sampling) and PixelSNAIL.

Heads of 65..128 channels run in 128-wide slots (zero padded below 128); the scale stays 1/sqrt(true dk).  Tolerances
are those of test_kernels_gpu.py for the kernels and 1e-2 relative to max(1, max|ref|) for modules and models.
"""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

TOL = 1e-2
GAMMA = 0.999977


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def assert_close(name, got, ref, rtol, atol=0.0):
    ref = ref.float()
    tol = atol + rtol * ref.abs().max().item()
    err = (got.float() - ref).abs().max().item()
    assert err <= tol and not torch.isnan(got.float()).any(), f"{name}: max err {err:.4e} > tol {tol:.3e}"


def check(name, got, ref, tol=TOL):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    bound = tol * max(1.0, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e}"


# --------------------------------------------------------------------------------------------------
# Kernels
# --------------------------------------------------------------------------------------------------
def _attn_inputs(N, S, H, dk, dv, seed=12):
    g = torch.Generator().manual_seed(seed)
    P = N * S
    qkv = torch.randn(P, H * (2 * dk + dv), generator=g).to(dev()).bfloat16()
    q, k, v = qkv[:, : H * dk], qkv[:, H * dk: 2 * H * dk], qkv[:, 2 * H * dk:]
    do = torch.randn(P, H * dv, generator=g).to(dev()).bfloat16()
    return q, k, v, do


def _attn_ref(q, k, v, do, N, S, H, dk, dv, strict):
    """fp32 restatement of the reference's attention core on [P, H*d] pixel-major inputs (with autograd)."""
    qf = q.float().view(N, S, H, dk).transpose(1, 2).requires_grad_(True)
    kf = k.float().view(N, S, H, dk).transpose(1, 2).requires_grad_(True)
    vf = v.float().view(N, S, H, dv).transpose(1, 2).requires_grad_(True)
    mask = torch.tril(torch.ones(S, S, device=q.device), diagonal=-int(strict)).view(1, 1, S, S)
    s = (qf @ kf.transpose(2, 3)) / math.sqrt(dk)
    s = s.masked_fill(mask == 0, float("-inf"))
    p = torch.softmax(s, dim=-1).masked_fill(mask == 0, 0)
    out = (p @ vf).transpose(1, 2).reshape(N * S, H * dv)
    out.backward(do.float())
    g = lambda t, d: t.grad.transpose(1, 2).reshape(N * S, H * d)
    return out.detach(), g(qf, dk), g(kf, dk), g(vf, dv)


def _to_slots(t, H, d, slot):
    P = t.shape[0]
    out = torch.zeros(P, H, slot, device=t.device, dtype=t.dtype)
    out[:, :, :d] = t.reshape(P, H, d)
    return out.reshape(P, H * slot)


def _from_slots(t, H, d, slot):
    return t.reshape(t.shape[0], H, slot)[:, :, :d].reshape(t.shape[0], H * d)


def _run(L, q, k, v, do, N, S, H, dk, ks, vs, strict, impl):
    P = q.shape[0]
    o = torch.full((P, H * vs), float("nan"), device=dev(), dtype=torch.bfloat16)
    lse = torch.empty(N, H, S, device=dev())
    L.causal_attn_fwd(q, k, v, o, lse, N, S, H, ks, vs, strict, impl=impl, dk_true=dk)
    grads = []
    for _ in range(2 if impl == 0 else 1):  # the tensor-core backward twice: it must give the same bits
        dq = torch.full((P, H * ks), float("nan"), device=dev(), dtype=torch.bfloat16)
        dk_ = torch.full((P, H * ks), float("nan"), device=dev(), dtype=torch.bfloat16)
        dv_ = torch.full((P, H * vs), float("nan"), device=dev(), dtype=torch.bfloat16)
        delta = torch.empty(N, H, S, device=dev())
        L.causal_attn_bwd(q, k, v, o, do, lse, delta, None, dq, dk_, dv_, N, S, H, ks, vs, strict, impl=impl, dk_true=dk)
        grads.append((dq, dk_, dv_))
    torch.cuda.synchronize()
    return o, grads


WIDE_CASES = [
    # N, S, H, dk, dv, strict
    (2, 256, 2, 128, 128, False),
    (1, 1024, 4, 128, 128, False),
    (2, 1024, 1, 128, 64, True),
    (3, 100, 2, 96, 96, False),     # partial tile, 96-channel heads padded into 128-wide slots
    (2, 784, 1, 80, 128, True),     # partial last tile, padded q/k slot, strict
    (2, 200, 3, 128, 32, True),     # narrow value heads in 64-wide slots next to 128-wide q/k slots
    (10, 1024, 2, 112, 128, True),  # many work items per (image, head)
]


@pytest.mark.parametrize("case", WIDE_CASES)
def test_wide_head_attention_fwd_bwd(L, case):
    """Tensor-core kernels with 128-wide q/k slots against the fp32 restatement and the SIMT kernels."""
    from pytorch_generative_b200 import ops

    N, S, H, dk, dv, strict = case
    ks, vs = ops.head_slots(dk, dv)
    assert ks == 128
    q, k, v, do = _attn_inputs(N, S, H, dk, dv)
    o_ref, dq_ref, dk_ref, dv_ref = _attn_ref(q, k, v, do, N, S, H, dk, dv, strict)
    o_simt, ((dq_s, dk_s, dv_s),) = _run(L, q, k, v, do, N, S, H, dk, dk, dv, strict, impl=1)
    qs, kslot, vslot, dos = _to_slots(q, H, dk, ks), _to_slots(k, H, dk, ks), _to_slots(v, H, dv, vs), _to_slots(do, H, dv, vs)
    o, grads = _run(L, qs, kslot, vslot, dos, N, S, H, dk, ks, vs, strict, impl=0)
    (dq, dk_, dv_), again = grads
    for ref_name, (o_r, dq_r, dk_r, dv_r) in (("ref", (o_ref, dq_ref, dk_ref, dv_ref)), ("simt", (o_simt, dq_s, dk_s, dv_s))):
        assert_close(f"o vs {ref_name}", _from_slots(o, H, dv, vs), o_r, rtol=2 ** -7, atol=1e-3)
        assert_close(f"dq vs {ref_name}", _from_slots(dq, H, dk, ks), dq_r, rtol=2 ** -6, atol=2e-3)
        assert_close(f"dk vs {ref_name}", _from_slots(dk_, H, dk, ks), dk_r, rtol=2 ** -6, atol=2e-3)
        assert_close(f"dv vs {ref_name}", _from_slots(dv_, H, dv, vs), dv_r, rtol=2 ** -6, atol=2e-3)
    if strict:
        assert (o.view(N, S, -1)[:, 0] == 0).all(), "strict mask: first position must be exactly zero"
    if dk < ks:  # padded q/k columns carry exactly zero gradient
        assert (dq.reshape(-1, H, ks)[:, :, dk:] == 0).all() and (dk_.reshape(-1, H, ks)[:, :, dk:] == 0).all()
    for name, a, b in zip(("dq", "dk", "dv"), (dq, dk_, dv_), again):
        assert torch.equal(a, b), f"{name}: two backward runs differ"


def test_head_slot_limits_are_enforced(L):
    """The tensor-core path takes 64- or 128-wide slots only; the module layer refuses heads wider than 128."""
    from pytorch_generative_b200 import nn as pg_nn

    N, S, H = 1, 64, 1
    q = torch.zeros(N * S, H * 192, device=dev(), dtype=torch.bfloat16)
    v = torch.zeros(N * S, H * 64, device=dev(), dtype=torch.bfloat16)
    o = torch.empty_like(v)
    lse = torch.empty(N, H, S, device=dev())
    with pytest.raises(RuntimeError, match="64 or 128"):
        L.causal_attn_fwd(q, q, v, o, lse, N, S, H, 192, 64, False)
    m = pg_nn.CausalAttention(in_channels=8, n_heads=1, embed_channels=136, out_channels=8).to(dev())
    with pytest.raises(NotImplementedError, match="128"):
        m(torch.zeros(1, 8, 4, 4, device=dev()))


@pytest.mark.parametrize("N,S,H,dk,dv,strict", [(2, 200, 2, 128, 128, False), (3, 64, 1, 128, 64, True)])
def test_wide_head_decode_matches_full_attention(L, N, S, H, dk, dv, strict):
    """pg_attn_decode at dk = 128: appending positions one at a time reproduces the rows of the full attention."""
    q, k, v, do = _attn_inputs(N, S, H, dk, dv, seed=23)
    o_ref, _, _, _ = _attn_ref(q, k, v, do, N, S, H, dk, dv, strict)
    kc = torch.zeros(N * S, H * dk, device=dev(), dtype=torch.bfloat16)
    vc = torch.zeros(N * S, H * dv, device=dev(), dtype=torch.bfloat16)
    pos = torch.zeros(1, dtype=torch.int32, device=dev())
    qv, kv_, vv = q.view(N, S, -1), k.view(N, S, -1), v.view(N, S, -1)
    o = torch.empty(N, H * dv, device=dev(), dtype=torch.bfloat16)
    for p in range(S):
        pos.fill_(p)
        L.attn_decode(qv[:, p].contiguous(), kv_[:, p].contiguous(), vv[:, p].contiguous(), kc, vc, o, pos, N, S, H, dk,
                      dv, strict)
        torch.cuda.synchronize()
        assert_close(f"decode pos {p}", o, o_ref.view(N, S, -1)[:, p], rtol=2 ** -7, atol=2e-3)


# --------------------------------------------------------------------------------------------------
# CausalAttention
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kwargs,shape", [
    (dict(in_channels=32, n_heads=2, embed_channels=256, out_channels=256), (2, 32, 16, 16)),
    (dict(in_channels=16, n_heads=1, embed_channels=128, out_channels=64, mask_center=True, extra_input_channels=3),
     (2, 16, 12, 20)),
])
def test_wide_head_causal_attention_matches_oracle(kwargs, shape):
    from oracle import reference_path as O
    from pytorch_generative_b200 import nn as pg_nn

    torch.manual_seed(4)
    m = pg_nn.CausalAttention(**kwargs)
    g = torch.Generator().manual_seed(5)
    n, _, h, w = shape
    ce = kwargs.get("extra_input_channels", 0)
    x = torch.randn(shape, generator=g)
    extra = torch.randn(n, ce, h, w, generator=g) if ce else None
    dy = torch.randn(n, m._out_channels, h, w, generator=g)
    pt = O.trainable({k: v.detach().clone() for k, v in m.state_dict().items()})
    xr = x.clone().requires_grad_(True)
    er = extra.clone().requires_grad_(True) if ce else None
    yr = O.causal_attention(xr, pt, "", m._n_heads, m._embed_channels, m._out_channels, m._mask_center, er)
    yr.backward(dy)
    m = m.to(dev())
    xd = x.to(dev()).requires_grad_(True)
    ed = extra.to(dev()).requires_grad_(True) if ce else None
    y = m(xd, ed) if ce else m(xd)
    y.backward(dy.to(dev()))
    check("y", y, yr)
    check("dx", xd.grad, xr.grad)
    if ce:
        check("dextra", ed.grad, er.grad)
    for name, p in m.named_parameters():
        check("d" + name, p.grad, pt[name].grad)


# --------------------------------------------------------------------------------------------------
# ImageGPT and PixelSNAIL against the oracle
# --------------------------------------------------------------------------------------------------
IGPT_4x128 = dict(in_channels=3, out_channels=3, in_size=32, n_transformer_blocks=2, n_attention_heads=4,
                  n_embedding_channels=512)
IGPT_2x96 = dict(in_channels=1, out_channels=1, in_size=28, n_transformer_blocks=2, n_attention_heads=2,
                 n_embedding_channels=192)
SNAIL_K128 = dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=2, n_residual_blocks=1,
                  attention_key_channels=128, attention_value_channels=32)


def _synthetic(shape, g):
    if shape[1] == 1:
        return torch.bernoulli(torch.full(shape, 0.5), generator=g)
    return torch.randint(0, 256, shape, generator=g).float() / 255


def _fresh(cls, cfg, seed=0, jitter=0.02):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = getattr(models, cls)(**cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g) * jitter)
    return m, g


@pytest.mark.parametrize("name,cls,cfg,shape", [
    ("image_gpt", "ImageGPT", IGPT_4x128, (2, 3, 32, 32)),
    ("image_gpt", "ImageGPT", IGPT_2x96, (2, 1, 28, 28)),
    ("pixel_snail", "PixelSNAIL", SNAIL_K128, (2, 3, 16, 16)),
])
def test_wide_head_model_matches_oracle(name, cls, cfg, shape):
    """Logits, recipe loss and fixed-cotangent parameter gradients (the protocol of test_image_gpt_matches_oracle)."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses

    m, g = _fresh(cls, cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = _synthetic(shape, g)
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
    for pname, p in m.named_parameters():
        if pt[pname].grad is None:  # parameters the reference's graph never reaches
            continue
        check("d" + pname, p.grad, pt[pname].grad)


def _compare_trajectory(tag, got, ref, model, ref_state, init_state, lr, steps):
    """The budget of test_parity_full_gpu.py's trajectory tests: loss / gradient norm per step, then the updates."""
    for k, ((l, n), (rl, rn)) in enumerate(zip(got, ref)):
        assert abs(l - rl) <= TOL * (1 + k) * abs(rl), (tag, k, l, rl)
        assert abs(n - rn) <= 2.5e-2 * (1 + 1.5 * k) * abs(rn), (tag, k, n, rn)
    num = den = worst = 0.0
    for pname, p in model.named_parameters():
        w, r, w0 = p.detach().float().cpu(), ref_state[pname], init_state[pname]
        num += float(((w - w0) - (r - w0)).pow(2).sum())
        den += float((r - w0).pow(2).sum())
        worst = max(worst, float((w - r).abs().max()))
    assert worst <= 2.0 * steps * lr * 1.05, (tag, worst)
    rel = (num / max(den, 1e-30)) ** 0.5
    assert rel <= 0.15, f"{tag}: parameter updates diverge from the oracle's (relative l2 {rel:.3e})"


@pytest.mark.parametrize("graphed", [False, True])
def test_wide_head_image_gpt_trajectory_matches_oracle(graphed):
    """Three Adam steps of ImageGPT with 4 heads x 128 channels against oracle.TrainState, eager and CUDA-graphed."""
    from oracle import reference_path as O
    from pytorch_generative_b200 import losses, trainstep

    lr, shape = 5e-3, (2, 3, 32, 32)
    m, g = _fresh("ImageGPT", IGPT_4x128)
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    xs = [_synthetic(shape, g) for _ in range(3)]
    ts = O.TrainState("image_gpt", init, IGPT_4x128, lr=lr, lr_gamma=GAMMA)
    ref = [ts.step(x) for x in xs]
    ref_state = {k: v.detach().clone() for k, v in ts.p.items()}
    m = m.to(dev()).train()
    params = list(m.parameters())
    loss_fn = lambda preds, x: losses.bce_with_logits_sum_mean(preds, x)
    if graphed:
        step = trainstep.GraphedTrainStep(m, params, loss_fn, xs[0].to(dev()), lr=lr, lr_gamma=GAMMA)
        step.reset(init)
        got = [step(x.to(dev())) for x in xs]
    else:
        opt = torch.optim.Adam(params, lr=lr)
        sched = torch.optim.lr_scheduler.MultiplicativeLR(opt, lr_lambda=lambda _: GAMMA)
        got = []
        for x in xs:
            xd = x.to(dev())
            opt.zero_grad()
            loss = loss_fn(m(xd), xd)
            loss.backward()
            norm = torch.nn.utils.clip_grad_norm_(params, 1e50)
            opt.step()
            sched.step()
            got.append((loss.item(), norm.item()))
    _compare_trajectory("image_gpt 4x128" + (" graphed" if graphed else ""), got, ref, m, ref_state, init, lr, 3)


def test_wide_head_image_gpt_layout_is_identity_and_uses_the_unscattered_weight_arena():
    """4 heads x 128 channels fill their slots: the packed weights are the one-cast arena, and the block weight
    matrices go to the overlapped data-parallel gradient buckets."""
    from pytorch_generative_b200 import models

    m = models.ImageGPT(**IGPT_4x128).to(dev())
    packed = m._packed_training_weights()
    assert "arena" in packed and all(b["layout"].identity for b in packed["blocks"])
    assert packed["blocks"][0]["layout"].qk_slot == 128
    bucketed = m.bucketed_parameters()
    assert len(bucketed) == 5 * IGPT_4x128["n_transformer_blocks"]
    assert models.ImageGPT(**IGPT_2x96).bucketed_parameters() == []


# --------------------------------------------------------------------------------------------------
# Sampling: the KV-cached per-pixel programs with 128-wide q/k slots
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls,cfg,shape", [
    ("ImageGPT", dict(IGPT_4x128, in_size=16), (2, 3, 16, 16)),
    ("PixelSNAIL", SNAIL_K128, (2, 3, 16, 16)),
])
def test_wide_head_incremental_sampler_matches_the_full_forward(cls, cfg, shape):
    """Teacher-forced sampling (the protocol of test_incremental_sampler_logits_match_the_full_forward): each pixel's
    logits from the K/V caches equal the full forward's, on two calls, with the per-pixel step graph-captured."""
    from pytorch_generative_b200 import models

    torch.manual_seed(7)
    m = getattr(models, cls)(**cfg).to(dev())
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.5)
    x = torch.bernoulli(torch.full(shape, 0.5)).to(dev())
    with torch.no_grad():
        ref = m(x)
    n, c, h, w = shape
    for rep in range(2):
        seen = []
        m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), torch.zeros_like(logits))[1]
        out = m.sample(conditioned_on=x)
        assert torch.equal(out, x)
        got = torch.stack(seen, dim=-1).view(n, c, h, w)
        check(f"incremental logits (call {rep})", got, ref)
    states = getattr(m, "_pixel_states", None)
    assert states and all(st["graph"] for st in states.values()), "per-pixel step was not graph-captured"
