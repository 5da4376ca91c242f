"""The categorical likelihood on an H100: pg_categorical_xent_fwd_bwd against float64 with per-element bounds, the four
image models at out_channels = 256 C (loss and every parameter gradient), a FusedAdam trajectory, a graphed step bit for
bit, pg_categorical_sample against the float64 inverse CDF and in a chi-square test, sample() of every model, and the
8-bit ImageGPT recipe."""

import copy
import json
import math

import pytest
import torch
import torch.nn.functional as F

import _categorical_reference as R

pytestmark = pytest.mark.gpu

F64 = torch.float64
THREADS = 256  # threads per block of the loss kernel: its per-image sums have ceil(C H W / 256) block partials


def dev():
    return torch.device("cuda:0")


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), err[bad].max().item(), (err / bound)[bad].max().item())
    return (err / bound).max().item()


def _grid(k, K):
    """k / (K - 1) rounded once to fp32 (the quotient in float64 is rounded to fp32 without a double-rounding error:
    53 >= 2 * 24 + 2).  torch's CUDA division by a scalar multiplies by its reciprocal, which can be 1 ulp away."""
    return (k.double() / (K - 1)).float()


def _grid_input(N, C, H, W, K, g):
    return _grid(torch.randint(0, K, (N, C, H, W), generator=g), K).to(dev())


def _run_kernel(logits, x):
    """(nll, image_nll, dlogits) of one launch with grad_scale 1 / N."""
    from pytorch_generative_b200 import _lib as L

    N = x.shape[0]
    nll = torch.empty(x.shape, device=dev())
    image_nll = torch.zeros(N, device=dev())
    dlogits = torch.empty_like(logits)
    L.categorical_xent(logits, x, 1.0 / N, nll=nll, image_nll=image_nll, dlogits=dlogits)
    return nll, image_nll, dlogits


def _check_kernel(logits, x):
    N, C = x.shape[:2]
    nll, image_nll, dlogits = _run_kernel(logits, x)
    worst = _within(nll, R.nll(logits, x), R.nll_bound(logits, x), "nll")
    blocks = -(-x[0].numel() // THREADS)
    ref_sums = R.nll(logits, x).reshape(N, -1).sum(dim=1)
    worst = max(worst, _within(image_nll, ref_sums, R.image_sum_bound(logits, x, blocks), "per-image sums"))
    worst = max(worst, _within(dlogits, R.dlogits(logits, x, 1.0 / N), R.dlogits_bound(logits, x, 1.0 / N), "dlogits"))
    return worst, (nll, image_nll, dlogits)


SIDES = [(1, 1), (7, 13), (28, 28), (32, 32)]
CASES = [(K, C, h, w) for K in (2, 17, 256, 1000) for C in (1, 3) for h, w in SIDES]


@pytest.mark.parametrize("K,C,H,W", CASES)
def test_loss_kernel_against_float64(K, C, H, W):
    """Random logits (scale 3) over every K, C and side, the batch cycling through 1, 5 and 64: the NLL, the per-image
    sums and every dlogits element within their float64 bounds."""
    i = CASES.index((K, C, H, W))
    N = (1, 5, 64)[i % 3]
    g = torch.Generator().manual_seed(100 + i)
    logits = (torch.randn(N, K * C, H, W, generator=g) * 3).to(dev())
    x = _grid_input(N, C, H, W, K, g)
    worst, _ = _check_kernel(logits, x)
    print(f"K {K} C {C} {H}x{W} N {N}: worst error / bound {worst:.3f}")


def test_loss_kernel_at_the_c5_shape():
    """[64, 768, 32, 32], the shape the 8-bit recipe trains at."""
    g = torch.Generator().manual_seed(7)
    logits = (torch.randn(64, 768, 32, 32, generator=g) * 2).to(dev())
    x = _grid_input(64, 3, 32, 32, 256, g)
    worst, _ = _check_kernel(logits, x)
    print(f"C5 shape: worst error / bound {worst:.3f}")


@pytest.mark.parametrize("K", [2, 256, 1000])
@pytest.mark.parametrize("kind", ["equal", "peaked", "huge", "ends"])
def test_loss_kernel_hard_logits(K, kind):
    """Equal logits, one logit raised by 80 (at the target for half the pixels), logits of +-1e4, and inputs at (and
    beyond) the ends of [0, 1]: within the bounds, and two runs give the same bits."""
    N, C, H, W = 5, 3, 7, 13
    g = torch.Generator().manual_seed(K + len(kind))
    x = _grid_input(N, C, H, W, K, g)
    if kind == "equal":
        logits = torch.full((N, K * C, H, W), 5.0, device=dev())
    elif kind == "peaked":
        logits = torch.randn(N, K, C, H, W, generator=g)
        t = R.target(x, K).cpu()
        other = torch.randint(0, K, t.shape, generator=g)
        peak = torch.where(torch.rand(t.shape, generator=g) < 0.5, t, other)
        logits.scatter_add_(1, peak.unsqueeze(1), torch.full((N, 1, C, H, W), 80.0))
        logits = logits.reshape(N, K * C, H, W).to(dev())
    elif kind == "huge":
        logits = (torch.randint(0, 2, (N, K * C, H, W), generator=g).float() * 2e4 - 1e4).to(dev())
    else:
        logits = torch.randn(N, K * C, H, W, generator=g).to(dev())
        ends = torch.tensor([0.0, 1.0, -0.25, 1.25, -0.0])
        x = ends[torch.randint(0, 5, (N, C, H, W), generator=g)].to(dev())
        assert set(R.target(x, K).unique().tolist()) == {0, K - 1}
    worst, first = _check_kernel(logits, x)
    second = _run_kernel(logits, x)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    if kind == "equal":
        assert _within(first[0], torch.full(x.shape, math.log(K), dtype=F64, device=dev()),
                       R.nll_bound(logits, x), "log K")
    print(f"{kind} K {K}: worst error / bound {worst:.3f}")


def test_loss_kernel_refuses_bad_shapes():
    from pytorch_generative_b200 import _lib as L

    x = torch.zeros(2, 3, 4, 4, device=dev())
    with pytest.raises(RuntimeError):  # K = 1
        L.categorical_xent(torch.zeros(2, 3, 4, 4, device=dev()), x, image_nll=torch.zeros(2, device=dev()))


# --------------------------------------------------------------------------------------------------
# the four models
# --------------------------------------------------------------------------------------------------
def _model_cfg(cls, C):
    out = 256 * C
    return {
        "PixelCNN": dict(in_channels=C, out_channels=out, n_residual=1, residual_channels=16, head_channels=32),
        "GatedPixelCNN": dict(in_channels=C, out_channels=out, n_gated=2, gated_channels=16, head_channels=32),
        "PixelSNAIL": dict(in_channels=C, out_channels=out, n_channels=16, n_pixel_snail_blocks=1, n_residual_blocks=1,
                           attention_key_channels=4, attention_value_channels=8),
        "ImageGPT": dict(in_channels=C, out_channels=out, in_size=8, n_transformer_blocks=1, n_attention_heads=2,
                         n_embedding_channels=32),
    }[cls]


MODELS = ["PixelCNN", "GatedPixelCNN", "PixelSNAIL", "ImageGPT"]
GRAD_TOL = 1e-2  # each gradient tensor within 1e-2 of its own largest entry (test_vae_gpu.py's per-tensor scale)


def _model(cls, C, seed=0, sample_fn=None):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    return getattr(models, cls)(**_model_cfg(cls, C), sample_fn=sample_fn).to(dev())


def _loss_bound(logits, x):
    N = x.shape[0]
    blocks = -(-x[0].numel() // THREADS)
    ref = R.loss(logits, x)[0].item()
    return R.image_sum_bound(logits, x, blocks).mean().item() + 4 * N * R.U * ref


def _grads(loss_or_logits, params, **kw):
    """{name: gradient} (zeros for a parameter the output does not reach)."""
    gs = torch.autograd.grad(loss_or_logits, list(params.values()), allow_unused=True, **kw)
    return {k: torch.zeros_like(p) if gr is None else gr for (k, p), gr in zip(params.items(), gs)}


def _grads_close(got, ref, what):
    ratios = []
    for k, r in ref.items():
        gk, r = got[k].double(), r.double()
        ratios.append(((gk - r).abs().max().item() / max(r.abs().max().item(), 1e-30), k))
    ratios.sort(reverse=True)
    assert ratios[0][0] <= GRAD_TOL, (what, ratios[:5])
    return ratios


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("cls", MODELS)
def test_models_loss_and_gradients(cls, C):
    """categorical_nll on each model's logits equals F.cross_entropy in float64 within the kernel bound, and every
    parameter gradient equals the one the same backward gives for the float64 dlogits."""
    from pytorch_generative_b200 import losses

    m = _model(cls, C).train()
    g = torch.Generator().manual_seed(3)
    N, H, W = 3, 8, 8
    x = _grid_input(N, C, H, W, 256, g)
    logits = m(x)
    assert logits.shape == (N, 256 * C, H, W)
    out = losses.categorical_nll(x, None, logits)
    lg = logits.detach()
    ce = F.cross_entropy(lg.double().reshape(N, 256, C, H, W), losses.categorical_target(x, 256), reduction="sum") / N
    assert abs(out["loss"].item() - ce.item()) <= _loss_bound(lg, x), (out["loss"].item(), ce.item())
    assert abs(out["bits_per_dim"].item() - out["loss"].item() / (C * H * W * math.log(2))) <= 1e-6 * out["loss"].item()
    params = dict(m.named_parameters())
    got = _grads(out["loss"], params)
    again = m(x)  # a second forward for the second backward: ImageGPT's fused stack frees its activations in backward
    assert torch.equal(again, logits)
    ref = _grads(again, params, grad_outputs=R.dlogits(lg, x, 1.0 / N).float())
    ratios = _grads_close(got, ref, cls)
    print(cls, C, "worst gradient errors over own scale:", ratios[:3])


def test_fused_adam_trajectory():
    """Three FusedAdam steps of ImageGPT (C = 3) on one batch: at every step the loss is the float64 cross-entropy of
    that step's logits within the kernel bound, every gradient is the float64 dlogits' within GRAD_TOL, no weight moves
    by more than the learning rate, and the loss falls."""
    from pytorch_generative_b200 import losses, optim

    m = _model("ImageGPT", 3, seed=4).train()
    lr = 1e-3
    opt = optim.FusedAdam(m.parameters(), lr=lr)
    x = _grid_input(4, 3, 8, 8, 256, torch.Generator().manual_seed(5))
    params = dict(m.named_parameters())
    seen = []
    for step in range(3):
        opt.zero_grad()
        first = m(x)
        ref = _grads(first, params, grad_outputs=R.dlogits(first.detach(), x, 1.0 / 4).float())
        logits = m(x)
        assert torch.equal(logits, first)
        out = losses.categorical_nll(x, None, logits)
        lg = logits.detach()
        assert abs(out["loss"].item() - R.loss(lg, x)[0].item()) <= _loss_bound(lg, x), step
        out["loss"].backward()
        _grads_close({k: torch.zeros_like(p) if p.grad is None else p.grad for k, p in params.items()}, ref,
                     f"step {step}")
        before = {k: p.detach().clone() for k, p in params.items()}
        opt.clip_and_step(1e50)
        moved = max((p.detach() - before[k]).abs().max().item() for k, p in params.items())
        assert 0 < moved <= lr * 1.01, (step, moved)
        seen.append(out["loss"].item())
    assert seen[2] < seen[0], seen


def test_graphed_step_is_bit_identical_to_eager():
    """A GraphedTrainStep replay with categorical_nll gives the eager step's logits, loss and gradients bit for bit."""
    from pytorch_generative_b200 import losses, trainstep

    m = _model("ImageGPT", 3, seed=6).train()
    x = _grid_input(2, 3, 8, 8, 256, torch.Generator().manual_seed(7))
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.zero_grad(set_to_none=True)
    logits = m(x)
    loss = losses.categorical_nll(x, None, logits)["loss"]
    loss.backward()
    stored = dict(logits=logits.detach().clone(), loss=loss.detach().clone())
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters()}
    del logits, loss  # nothing may keep the eager forward's autograd node (and its activations) alive into the capture
    step = trainstep.GraphedTrainStep(m, list(m.parameters()), lambda p, xx: losses.categorical_nll(xx, None, p)["loss"],
                                      x, lr=1e-3, lr_gamma=1.0)
    step.reset(init)
    step(x)
    assert torch.equal(step.static_preds, stored["logits"])
    assert torch.equal(step.static_loss, stored["loss"])
    for n, p in m.named_parameters():
        assert torch.equal(p.grad, grads[n]), n


# --------------------------------------------------------------------------------------------------
# sampling
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 17, 256, 1000])
@pytest.mark.parametrize("C", [1, 3])
def test_sampler_is_the_inverse_cdf(K, C):
    """Under recorded uniforms each draw is the float64 inverse CDF wherever u is not within the fp32 bound of a CDF
    boundary; every output is k / (K - 1) in fp32; a padded row pitch gives the same draws."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(K * 7 + C)
    n = 4096
    logits = (torch.randn(n, K * C, generator=g) * 2).to(dev())
    u = torch.rand(n, C, generator=g).to(dev())
    out = torch.empty(n, C, device=dev())
    L.categorical_sample(logits, u, out)
    k = torch.round(out.double() * (K - 1)).long()
    assert torch.equal(out.cpu(), _grid(k.cpu(), K)), "off the k / (K - 1) grid"
    ref = R.inverse_cdf(logits, u)
    clear = ~R.near_boundary(logits, u)
    assert clear.float().mean().item() > 0.5
    assert torch.equal(k[clear], ref[clear]), int((k[clear] != ref[clear]).sum())
    assert ((k - ref).abs() <= 1).all()
    wide = torch.zeros(n, K * C + 5, device=dev())
    wide[:, : K * C] = logits
    again = torch.empty_like(out)
    L.categorical_sample(wide[:, : K * C], u, again)
    assert torch.equal(again, out)


@pytest.mark.parametrize("K,C", [(17, 3), (256, 1)])
def test_sampler_chi_square(K, C):
    """2e5 seeded draws of categorical_sample_fn from one row of logits against its softmax probabilities (bins with
    fewer than 5 expected draws merged), per channel."""
    from scipy import stats

    from pytorch_generative_b200 import models

    g = torch.Generator().manual_seed(K + C)
    row = torch.randn(1, K * C, generator=g) * 1.5
    n = 200_000
    torch.manual_seed(11)
    out = models.categorical_sample_fn(K)(row.to(dev()).repeat(n, 1))
    k = torch.round(out.double() * (K - 1)).long().cpu()
    p = R.probabilities(row, C)[0]
    for c in range(C):
        counts = torch.bincount(k[:, c], minlength=K).double()
        expected = p[:, c] * n
        order = torch.argsort(expected)
        obs, exp, acc_o, acc_e = [], [], 0.0, 0.0
        for i in order.tolist():
            acc_o += counts[i].item()
            acc_e += expected[i].item()
            if acc_e >= 5:
                obs.append(acc_o)
                exp.append(acc_e)
                acc_o = acc_e = 0.0
        obs[-1] += acc_o
        exp[-1] += acc_e
        chi2 = sum((o - e) ** 2 / e for o, e in zip(obs, exp))
        pval = stats.chi2.sf(chi2, len(obs) - 1)
        assert pval > 1e-4, (c, chi2, len(obs), pval)


class _Recording:
    """categorical_sample_fn that keeps every logits batch it is handed."""

    def __init__(self):
        from pytorch_generative_b200 import models

        self.fn, self.seen = models.categorical_sample_fn(256), []

    def __call__(self, logits):
        self.seen.append(logits.detach().clone())
        return self.fn(logits)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("cls", MODELS)
def test_model_sample(cls, C):
    """sample() with categorical_sample_fn: teacher-forced (every pixel given) it returns the input and hands each pixel's
    768- (or 256-) way logits, equal to the full forward's; with the top rows given it keeps them and draws the rest on
    the k / 255 grid; n_samples draws land on the grid too."""
    rec = _Recording()
    m = _model(cls, C, seed=8, sample_fn=rec).eval()
    n, H, W = 2, 8, 8
    x = _grid_input(n, C, H, W, 256, torch.Generator().manual_seed(9))
    with torch.no_grad():
        ref = m(x)
    assert torch.equal(m.sample(conditioned_on=x), x)
    got = torch.stack(rec.seen, dim=-1).view(ref.shape)
    err = (got - ref).abs().max().item()
    assert err <= 1e-2 * max(1.0, ref.abs().max().item()), err
    cond = x.clone()
    cond[:, :, 3:] = -1
    out = m.sample(conditioned_on=cond)
    assert torch.equal(out[:, :, :3], x[:, :, :3])
    for s in (out, m.sample(n_samples=2)):
        assert s.shape == (n, C, H, W)
        s = s.cpu()
        assert torch.equal(s, _grid(torch.round(s.double() * 255).long(), 256)) and (s >= 0).all() and (s <= 1).all()
    copy.deepcopy(m)


def test_recipe_trains_one_epoch(tmp_path):
    """reproduce_image_gpt_8bit on two batches of random 8-bit images: one epoch, a checkpoint, and loss and bits/dim in
    metrics.jsonl."""
    from pytorch_generative_b200 import recipes

    g = torch.Generator().manual_seed(12)
    loader = [(torch.randint(0, 256, (4, 3, 32, 32), generator=g).float().div(255).to(dev()), None) for _ in range(2)]
    trainer = recipes.reproduce_image_gpt_8bit(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    assert trainer.model._sample_fn.n_classes == 256
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["model"]["_out.weight"].shape[0] == 768
    rows = [json.loads(line) for line in open(tmp_path / "metrics.jsonl")]
    tags = {r["tag"] for r in rows}
    assert {"metrics/loss", "metrics/bits_per_dim"} <= tags
    bpd = [r["train"] for r in rows if r["tag"] == "metrics/bits_per_dim" and "train" in r]
    loss = [r["train"] for r in rows if r["tag"] == "metrics/loss" and "train" in r]
    assert len(bpd) == 2 and all(math.isfinite(v) and v > 0 for v in bpd)
    for lv, bv in zip(loss, bpd):
        assert abs(bv - lv / (3 * 32 * 32 * math.log(2))) <= 1e-5 * bv
