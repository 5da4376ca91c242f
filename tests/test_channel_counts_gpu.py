"""Channel counts that are not multiples of 8 on the CUDA path: GatedActivation at any even width, GatedPixelCNN and
PixelSNAIL at any gated_channels / n_channels (element-by-element gates, zero-padded conv operands) and ImageGPT at any
n_embedding_channels (the padded stream of models.image_gpt.StreamLayout), against the oracle
(oracle/reference_path.py) with the tolerances of test_parity_gpu.py: 1e-3 for fp32-only modules, 1e-2 for the bf16
path, relative to max(1, max|ref|)."""

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL_BF16, TOL_F32 = 1e-2, 1e-3
GAMMA = 0.999977


def dev():
    return torch.device("cuda:0")


def check(name, got, ref, tol):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    bound = tol * max(1.0, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    assert err <= bound and not torch.isnan(got).any(), f"{name}: max err {err:.3e} > {bound:.3e}"


def _recipe_loss(x, logits):
    from pytorch_generative_b200 import losses

    return losses.bce_with_logits_sum_mean(logits, x)


def _image(shape, g):
    return (torch.bernoulli(torch.full(shape, 0.5), generator=g) if shape[1] == 1
            else torch.randint(0, 256, shape, generator=g).float() / 255)


def _perturbed(cls, cfg, seed=0):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = getattr(models, cls)(**cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g) * 0.02)
    return m, g


# --------------------------------------------------------------------------------------------------
# GatedActivation
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["tanh", "identity"])
@pytest.mark.parametrize("half", [1, 3, 12, 100])
def test_gated_activation_matches_oracle(half, act):
    from oracle import reference_path as O
    from pytorch_generative_b200 import nn as pg_nn

    fn = torch.tanh if act == "tanh" else torch.nn.Identity()
    g = torch.Generator().manual_seed(half)
    x = torch.randn(2, 2 * half, 5, 7, generator=g) * 2
    G = torch.randn(2, half, 5, 7, generator=g)
    xr = x.clone().requires_grad_(True)
    ref = O.gated_activation(xr, fn)
    (ref * G).sum().backward()
    xd = x.to(dev()).requires_grad_(True)
    y = pg_nn.GatedActivation(fn)(xd)
    (y * G.to(dev())).sum().backward()
    check(f"gate y C/2={half}", y, ref, TOL_F32)
    check(f"gate dx C/2={half}", xd.grad, xr.grad, TOL_F32)


# --------------------------------------------------------------------------------------------------
# The three models against the oracle: logits, recipe loss, fixed-cotangent VJP of every parameter
# --------------------------------------------------------------------------------------------------
def _gpcnn(c):
    return "gated_pixel_cnn", "GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=2, gated_channels=c,
                                                    head_channels=max(1, c // 2))


def _snail(c, kv):
    return "pixel_snail", "PixelSNAIL", dict(in_channels=1, out_channels=1, n_channels=c, n_pixel_snail_blocks=1,
                                             n_residual_blocks=2, attention_key_channels=kv,
                                             attention_value_channels=kv)


def _igpt(c, heads):
    return "image_gpt", "ImageGPT", dict(in_channels=1, out_channels=1, in_size=32, n_transformer_blocks=2,
                                         n_attention_heads=heads, n_embedding_channels=c)


def _sized(cls, cfg, h):
    """ImageGPT's positional parameter is in_size x in_size, and the oracle adds it whole: images of that size."""
    return dict(cfg, in_size=h) if cls == "ImageGPT" else cfg


# ImageGPT at 15 channels: an odd width, so the MLP's hidden layer (60 channels) is padded too (to 64)
MODELS = {
    "gpcnn1": _gpcnn(1), "gpcnn12": _gpcnn(12), "gpcnn100": _gpcnn(100),
    "snail2": _snail(2, 1), "snail12": _snail(12, 3), "snail100": _snail(100, 20),
    "igpt4": _igpt(4, 2), "igpt12": _igpt(12, 3), "igpt15": _igpt(15, 3), "igpt100": _igpt(100, 4),
}
SHAPES = [(2, 1, 28, 28), (2, 1, 32, 32), (2, 1, 12, 20)]


def _oracle_vjp(name, state, x, cfg, G):
    """Oracle logits, recipe loss and the gradients of <logits, G> for every parameter."""
    from oracle import reference_path as O

    pt = O.trainable(state)
    logits = O.forward(name, pt, x, cfg)
    loss = O.recipe_loss(x, logits).detach()
    (logits * G).sum().backward()
    return logits.detach(), loss, {k: v.grad for k, v in pt.items() if v.requires_grad and v.grad is not None}


def _rel(got, ref):
    return (got.float() - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _image_gpt_budget(state, x, cfg, G, ref_logits, ref_loss, ref_grads):
    """Per-quantity bounds for ImageGPT.  The CUDA path rounds every GEMM operand to bf16: the weight copies and the
    activations they multiply (LayerNorm outputs, q / k / v, the attention output, the MLP hidden layer).  How much such
    rounding moves the result depends on the configuration's conditioning: LayerNorm over a handful of channels
    amplifies it (at 4 channels, rounding only the weights moves the oracle's 32x32 logits by ~2e-2 of max|ref|, at 12
    or more channels by ~3e-3).  So each bound is three times what rounding the GEMM weights alone to bf16 does to the
    oracle (one rounding each for the weights, the activations and the attention probabilities / output), and never
    less than the 1e-2 of the bf16 path."""
    rounded = {k: (v.to(torch.bfloat16).float() if k.endswith("weight") and v.dim() == 4 and not k.startswith("_input")
                   else v) for k, v in state.items()}
    logits_w, loss_w, grads_w = _oracle_vjp("image_gpt", rounded, x, cfg, G)
    budget = {"logits": _rel(logits_w, ref_logits), "loss": abs(loss_w.item() - ref_loss.item()) / abs(ref_loss.item())}
    budget.update({k: _rel(grads_w[k], r) for k, r in ref_grads.items()})
    return {k: max(TOL_BF16, 3 * e) for k, e in budget.items()}


def _record_stream_grads(monkeypatch):
    """Records the gradients ImageGPT's backward hands between its kernels: every LayerNorm backward's incoming
    gradient, residual gradients and outputs, every dgrad GEMM's output, and the stream gradient the input convolution's
    backward reads."""
    from pytorch_generative_b200 import _lib, ops

    seen = []
    ln_bwd, dgrad, conv_bwd = ops.layernorm_bwd, ops.linear_dgrad, _lib.conv_small_bwd

    def layernorm_bwd(dy, x, gamma, mean, rstd, dres0=None, dres1=None, **kw):
        out = ln_bwd(dy, x, gamma, mean, rstd, dres0=dres0, dres1=dres1, **kw)
        seen.extend(("layernorm", t) for t in (dy, dres0, dres1, out[0], out[1]) if t is not None)
        return out

    def linear_dgrad(*args, **kw):
        out = dgrad(*args, **kw)
        seen.extend(("dgrad", t) for t in (out if isinstance(out, tuple) else (out,)) if t is not None)
        return out

    def conv_small_bwd(x, w, dy_pm, *args, **kw):
        seen.append(("input conv", dy_pm))
        return conv_bwd(x, w, dy_pm, *args, **kw)

    monkeypatch.setattr(ops, "layernorm_bwd", layernorm_bwd)
    monkeypatch.setattr(ops, "linear_dgrad", linear_dgrad)
    monkeypatch.setattr(_lib, "conv_small_bwd", conv_small_bwd)
    return seen


def _pads_are_zero(logits, c):
    """ImageGPT's pad columns, exactly zero: every activation the node saves (u holds GELU'(pre), 0.5 in the pad, and
    only ever multiplies a zero gradient) and every gradient recorded by _record_stream_grads.  Stream-wide tensors
    have round_up(c, 8) columns, the MLP's hidden ones round_up(4c, 8); attention-wide gradients have no pad columns."""
    from pytorch_generative_b200.models.image_gpt import stream_layout

    sl = stream_layout(c)
    sv = logits.grad_fn.saved
    for t in (sv["xs_final"], sv["af"]):
        assert t.shape[1] == sl.c_p and not t[:, c:].any()
    for blk in sv["blocks"]:
        for k in ("xs", "a1", "h", "a2"):
            assert blk[k].shape[1] == sl.c_p and not blk[k][:, c:].any(), k
        assert blk["g"].shape[1] == sl.f_p and not blk["g"][:, 4 * c:].any()
    return sl


def _grad_pads_are_zero(seen, sl):
    checked = 0
    for where, t in seen:
        width = {sl.c_p: sl.c, sl.f_p: 4 * sl.c}.get(t.shape[1])
        if width is None:
            continue
        assert not t[:, width:].any(), f"{where}: a gradient of width {t.shape[1]} is nonzero past column {width}"
        checked += 1
    kinds = {w for w, t in seen if t.shape[1] in (sl.c_p, sl.f_p)}
    assert checked and kinds == {"layernorm", "dgrad", "input conv"}, kinds


@pytest.mark.parametrize("shape", SHAPES, ids=["28x28", "32x32", "12x20"])
@pytest.mark.parametrize("key", sorted(MODELS))
def test_models_match_oracle(key, shape, monkeypatch):
    name, cls, cfg = MODELS[key]
    if cls == "ImageGPT" and shape[2] != shape[3]:
        pytest.skip("ImageGPT's positional parameter is square")
    cfg = _sized(cls, cfg, shape[2])
    m, g = _perturbed(cls, cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = _image(shape, g)
    out_shape = (shape[0], cfg["out_channels"], *shape[2:])
    G = torch.randn(out_shape, generator=g) / (cfg["out_channels"] * shape[2] * shape[3])
    ref_logits, ref_loss, ref_grads = _oracle_vjp(name, state, x, cfg, G)
    tol = {}
    if cls == "ImageGPT":
        tol = _image_gpt_budget(state, x, cfg, G, ref_logits, ref_loss, ref_grads)
    padded = cls == "ImageGPT" and cfg["n_embedding_channels"] % 8
    seen = _record_stream_grads(monkeypatch) if padded else None
    m = m.to(dev())
    xd = x.to(dev())
    logits = m(xd)
    loss = _recipe_loss(xd, logits)
    if padded:
        sl = _pads_are_zero(logits, cfg["n_embedding_channels"])
    (logits * G.to(dev())).sum().backward()
    if padded:
        _grad_pads_are_zero(seen, sl)
    report, ok = [], True
    e = _rel(logits.detach().cpu(), ref_logits)
    report.append(f"{'logits':50s} max-rel {e:.3e} bound {tol.get('logits', TOL_BF16):.3e}")
    ok &= e <= tol.get("logits", TOL_BF16) and not torch.isnan(logits).any().item()
    e = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
    report.append(f"{'loss':50s} rel {e:.3e} bound {tol.get('loss', TOL_BF16):.3e}")
    ok &= e <= tol.get("loss", TOL_BF16)
    for pname, p in m.named_parameters():
        if pname not in ref_grads:
            continue
        gq, r = p.grad.detach().float().cpu(), ref_grads[pname]
        assert gq.shape == r.shape, pname
        e = _rel(gq, r)
        report.append(f"{pname:50s} max-rel {e:.3e} bound {tol.get(pname, TOL_BF16):.3e}")
        ok &= e <= tol.get(pname, TOL_BF16)
    print("\n".join(report))
    assert ok, "parity:\n" + "\n".join(report)


# --------------------------------------------------------------------------------------------------
# Standalone NCHW forwards of the blocks (the reference's Module API), at new widths
# --------------------------------------------------------------------------------------------------
def _vjp_check(tag, module, inputs, ref_fn, tol):
    """module(*inputs) against ref_fn(params, *inputs): output and a fixed-cotangent VJP for the inputs and every
    parameter, the cotangent scaled by 1 / (elements per image) as in the model-level VJPs."""
    from oracle import reference_path as O

    state = {k: v.detach().clone() for k, v in module.state_dict().items()}
    pt = O.trainable(state)
    xr = [t.clone().requires_grad_(True) for t in inputs]
    ref = ref_fn(pt, *xr)
    ref = ref if isinstance(ref, tuple) else (ref,)
    g = torch.Generator().manual_seed(3)
    Gs = [torch.randn(r.shape, generator=g) / r[0].numel() for r in ref]
    sum((r * G).sum() for r, G in zip(ref, Gs)).backward()
    module = module.to(dev())
    xd = [t.to(dev()).requires_grad_(True) for t in inputs]
    out = module(*xd)
    out = out if isinstance(out, tuple) else (out,)
    sum((o * G.to(dev())).sum() for o, G in zip(out, Gs)).backward()
    for k, (o, r) in enumerate(zip(out, ref)):
        check(f"{tag} out{k}", o, r, tol)
    for k, (a, b) in enumerate(zip(xd, xr)):
        check(f"{tag} dinput{k}", a.grad, b.grad, tol)
    for pname, p in module.named_parameters():
        if pt[pname].grad is not None:
            check(f"{tag} d{pname}", p.grad, pt[pname].grad, tol)


@pytest.mark.parametrize("c", [1, 3])
def test_standalone_blocks_match_oracle(c):
    from oracle import reference_path as O
    from pytorch_generative_b200.models import gated_pixel_cnn, pixel_snail

    g = torch.Generator().manual_seed(c)
    v, h = torch.randn(2, c, 9, 11, generator=g), torch.randn(2, c, 9, 11, generator=g)
    torch.manual_seed(c)
    layer = gated_pixel_cnn.GatedPixelCNNLayer(c, c, kernel_size=3, mask_center=False)
    _vjp_check(f"GatedPixelCNNLayer({c})", layer, (v, h), lambda p, a, b: O._gated_layer(p, "", a, b, 3, False),
               TOL_BF16)
    rb = pixel_snail.ResidualBlock(c)
    _vjp_check(f"ResidualBlock({c})", rb, (v,), lambda p, a: O._snail_residual(p, "", a), TOL_BF16)

    img = torch.bernoulli(torch.full((2, 1, 9, 11), 0.5), generator=g)
    blk = pixel_snail.PixelSNAILBlock(c, input_img_channels=1, n_residual_blocks=1, attention_key_channels=1,
                                      attention_value_channels=c)

    def block_ref(p, x, im):  # the block of O.pixel_snail_forward, without the stream sum
        res = O._snail_residual(p, "_residual.0.", x)
        attn = O.causal_attention(torch.cat((O.image_positional_encoding(im.shape), res), dim=1), p, "_attention.", 1,
                                  1, c, True, im)
        res = torch.nn.functional.elu(O._conv(torch.nn.functional.elu(res), p, "_residual_out"))
        attn = torch.nn.functional.elu(O._conv(torch.nn.functional.elu(attn), p, "_attention_out"))
        return torch.nn.functional.elu(O._conv(torch.nn.functional.elu(res + attn), p, "_out"))

    _vjp_check(f"PixelSNAILBlock({c})", blk, (v, img), block_ref, TOL_BF16)


# --------------------------------------------------------------------------------------------------
# The reference's own multiple-channel smoke configurations
# --------------------------------------------------------------------------------------------------
SMOKE = {
    "PixelCNN": dict(in_channels=3, out_channels=3, n_residual=1, residual_channels=1, head_channels=1),
    "GatedPixelCNN": dict(in_channels=3, out_channels=3, n_gated=1, gated_channels=1, head_channels=1),
    "PixelSNAIL": dict(in_channels=3, out_channels=3, n_channels=2, n_pixel_snail_blocks=1, n_residual_blocks=1,
                       attention_key_channels=1, attention_value_channels=1),
    "ImageGPT": dict(in_channels=3, out_channels=3, in_size=8, n_transformer_blocks=1, n_attention_heads=2,
                     n_embedding_channels=4),
}


@pytest.mark.parametrize("cls", sorted(SMOKE))
def test_reference_smoke_configurations(cls):
    from pytorch_generative_b200 import models

    torch.manual_seed(0)
    m = getattr(models, cls)(**SMOKE[cls]).to(dev())
    batch = torch.rand(2, 3, 8, 8, device=dev())
    assert torch.isfinite(m(batch)).all()
    s = m.sample(n_samples=2)
    assert s.shape == (2, 3, 8, 8) and set(s.unique().tolist()) <= {0.0, 1.0}
    batch[:, :, 1:, :] = -1
    cs = m.sample(conditioned_on=batch)
    assert torch.equal(cs[:, :, 0, :], batch[:, :, 0, :])
    assert (cs >= 0).all()
    fresh = getattr(models, cls)(**SMOKE[cls]).to(dev())
    fresh.load_state_dict(m.state_dict())
    x = torch.rand(2, 3, 8, 8, device=dev())
    with torch.no_grad():
        assert torch.equal(fresh(x), m(x))
    assert fresh.sample(n_samples=2).shape == (2, 3, 8, 8)


# --------------------------------------------------------------------------------------------------
# Sampling
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c,heads", [(12, 3), (100, 4)])
def test_image_gpt_incremental_logits_match_the_full_forward(c, heads):
    """Teacher-forced KV-cached sampling on the padded stream: each pixel's logits equal the full forward's, over two
    calls (the second replays the captured per-pixel graph)."""
    from pytorch_generative_b200 import models

    torch.manual_seed(7)
    cfg = dict(in_channels=1, out_channels=2, in_size=8, n_transformer_blocks=2, n_attention_heads=heads,
               n_embedding_channels=c)
    m = models.ImageGPT(**cfg).to(dev())
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.5)
    x = torch.bernoulli(torch.full((3, 1, 8, 8), 0.5)).to(dev())
    with torch.no_grad():
        ref = m(x)
    assert m._incremental_ok(x)
    for rep in range(2):
        seen = []
        m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), logits.new_zeros(3, 1))[1]
        assert torch.equal(m.sample(conditioned_on=x), x)
        check(f"incremental logits (call {rep})", torch.stack(seen, dim=-1).view(ref.shape), ref, TOL_BF16)
    assert m._pixel_states and all(st["graph"] for st in m._pixel_states.values())


@pytest.mark.parametrize("key", ["gpcnn12", "snail12", "igpt12"])
def test_sampling_follows_oracle_raster_order(key):
    """Same pre-drawn uniforms in raster order: pixels equal the oracle's sample except, at most, from a knife-edge draw
    (|u - p| within the bf16 tolerance) onwards."""
    from oracle import reference_path as O

    name, cls, cfg = MODELS[key]
    cfg = _sized(cls, cfg, 8)
    m, g = _perturbed(cls, cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    n, shape = 2, (2, 1, 8, 8)
    u = [torch.rand(n, 1, generator=g) for _ in range(64)]  # one draw per image and pixel, in raster order
    ref = O.sample(name, state, cfg, O.uniform_sample_fn(list(u)), n_samples=n, shape=shape[1:])
    m = m.to(dev())
    m._sample_fn = O.uniform_sample_fn(list(u))
    m(torch.zeros(shape, device=dev()))  # registers the image shape like the reference
    got = m.sample(n_samples=n).cpu()
    assert got.shape == ref.shape
    if not torch.equal(got, ref):
        diff = (got != ref).any(dim=1).any(dim=0)
        first = diff.flatten().nonzero()[0].item()
        r, col = divmod(first, shape[3])
        canvas = ref.clone()
        canvas.view(n, 1, -1)[:, :, first:] = -1
        p_ref = torch.sigmoid(O.forward(name, state, canvas, cfg)[:, :, r, col])
        margin = (u[first] - p_ref).abs().min().item()
        assert margin < 2e-2, f"samples diverge at pixel ({r},{col}) without a knife-edge draw (margin {margin:.3e})"


# --------------------------------------------------------------------------------------------------
# Training
# --------------------------------------------------------------------------------------------------
TRAIN = {"gpcnn12": 1e-3, "snail12": 1e-3, "igpt12": 5e-3}


@pytest.mark.parametrize("key", sorted(TRAIN))
def test_fused_adam_trajectory_matches_oracle(key):
    from oracle import reference_path as O
    from pytorch_generative_b200 import optim

    name, cls, cfg = MODELS[key]
    cfg = _sized(cls, cfg, 16)
    lr = TRAIN[key]
    m, g = _perturbed(cls, cfg)
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    xs = [_image((2, 1, 16, 16), g) for _ in range(3)]
    ts = O.TrainState(name, init, cfg, lr=lr, lr_gamma=GAMMA)
    ref = [ts.step(x) for x in xs]
    m = m.to(dev()).train()
    opt = optim.FusedAdam(m.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.MultiplicativeLR(opt, lr_lambda=lambda _: GAMMA)
    for k, x in enumerate(xs):
        xd = x.to(dev())
        opt.zero_grad()
        loss = _recipe_loss(xd, m(xd))
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(list(m.parameters()), 1e50)
        opt.step()
        sched.step()
        rl, rn = ref[k]
        assert abs(loss.item() - rl) <= TOL_BF16 * (1 + k) * abs(rl), (k, loss.item(), rl)
        assert abs(norm.item() - rn) <= 2.5e-2 * (1 + 1.5 * k) * abs(rn), (k, norm.item(), rn)
    worst = max(float((p.detach().cpu() - ts.p[n_].detach()).abs().max()) for n_, p in m.named_parameters())
    assert worst <= 2.0 * 3 * lr * 1.05


def _step(m, x):
    m.zero_grad(set_to_none=True)
    logits = m(x)
    loss = _recipe_loss(x, logits)
    loss.backward()
    out = dict(logits=logits.detach(), loss=loss.detach())
    out.update({n: p.grad.detach().clone() for n, p in m.named_parameters()})
    return out


def test_image_gpt_recompute_and_graphed_steps_are_bit_identical(monkeypatch):
    """At 12 channels: a forced-recompute step and a GraphedTrainStep step give the logits, loss and parameter
    gradients of the eager keep-everything step, bit for bit."""
    from pytorch_generative_b200 import losses, models, trainstep
    from pytorch_generative_b200.models import image_gpt

    cfg = _sized("ImageGPT", MODELS["igpt12"][2], 16)
    torch.manual_seed(0)
    m = models.ImageGPT(**cfg).to(dev()).train()
    x = torch.bernoulli(torch.full((2, 1, 16, 16), 0.5)).to(dev())
    monkeypatch.setattr(image_gpt, "recompute_activations", lambda mem, available: False)
    stored = _step(m, x)
    monkeypatch.setattr(image_gpt, "recompute_activations", lambda mem, available: True)
    recomputed = _step(m, x)
    for k in stored:
        assert torch.equal(stored[k], recomputed[k]), f"recompute: {k}"

    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    monkeypatch.setattr(image_gpt, "recompute_activations", lambda mem, available: False)
    params = list(m.parameters())
    step = trainstep.GraphedTrainStep(m, params, lambda preds, xx: losses.bce_with_logits_sum_mean(preds, xx), x,
                                      lr=1e-3, lr_gamma=GAMMA)
    step.reset(init)
    step(x)
    assert torch.equal(step.static_preds, stored["logits"])
    assert torch.equal(step.static_loss, stored["loss"])
    for n, p in m.named_parameters():  # the replay leaves its gradients in .grad (the Adam step does not clear them)
        assert torch.equal(p.grad, stored[n]), f"graphed: {n}"
