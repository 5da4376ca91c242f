"""The discretised logistic mixture likelihood on an H100: pg_logistic_mixture_fwd_bwd against float64 with per-element
bounds (and bug models the bounds must see), the four image models at out_channels = M G (loss and every parameter
gradient), a FusedAdam trajectory, a graphed step bit for bit, pg_logistic_mixture_sample against the float64 inverse
map and in chi-square tests, sample() of every model, and the 8-bit PixelSNAIL recipe."""

import copy
import json
import math

import pytest
import torch

import _logistic_mixture_reference as R

pytestmark = pytest.mark.gpu

F64 = torch.float64
THREADS = 128  # threads per block of the loss kernel: its per-image sums have ceil(H W / 128) block partials


def dev():
    return torch.device("cuda:0")


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), err[bad].max().item(), (err / bound)[bad].max().item())
    return (err / bound).max().item()


def _grid(k, K):
    """k / (K - 1) rounded once to fp32 (see test_categorical_gpu.py)."""
    return (k.double() / (K - 1)).float()


def _grid_input(N, C, H, W, K, g):
    return _grid(torch.randint(0, K, (N, C, H, W), generator=g), K).to(dev())


def _preds(M, C, N, H, W, g, coupling=1.0):
    """Random parameters: logits ~ N(0, 1), means ~ N(0, 0.25), log-scales in [-5, 0], coefficients ~ coupling N(0, 1)."""
    T = C * (C - 1) // 2
    pi = torch.randn(N, M, H, W, generator=g)
    mu = torch.randn(N, M * C, H, W, generator=g) * 0.5
    ls = torch.rand(N, M * C, H, W, generator=g) * 5 - 5
    r = torch.randn(N, M * T, H, W, generator=g) * coupling
    return torch.cat([pi, mu, ls, r], dim=1)


def _run_kernel(preds, x, M, K):
    """(nll, image_nll, dpreds) of one launch with grad_scale 1 / N."""
    from pytorch_generative_b200 import _lib as L

    N = x.shape[0]
    nll = torch.empty(N, *x.shape[2:], device=dev())
    image_nll = torch.zeros(N, device=dev())
    dp = torch.empty_like(preds)
    L.logistic_mixture_nll_kernel(preds, x, M, K, 1.0 / N, nll=nll, image_nll=image_nll, dpreds=dp)
    return nll, image_nll, dp


def _check_kernel(preds, x, M, K):
    N = x.shape[0]
    nll, image_nll, dp = _run_kernel(preds, x, M, K)
    ref = R.nll(preds, x, K)
    worst = _within(nll, ref, R.nll_bound(preds, x, K), "nll")
    blocks = -(-x[0, 0].numel() // THREADS)
    worst = max(worst, _within(image_nll, ref.reshape(N, -1).sum(dim=1), R.image_sum_bound(preds, x, K, blocks),
                               "per-image sums"))
    worst = max(worst, _within(dp, R.dpreds(preds, x, K, 1.0 / N), R.dpreds_bound(preds, x, K, 1.0 / N), "dpreds"))
    return worst, (nll, image_nll, dp)


SIDES = [(1, 1), (7, 13), (28, 28), (32, 32)]
CASES = [(M, C, K, h, w) for M in (1, 5, 10) for C in (1, 3) for K in (2, 256) for h, w in SIDES]


@pytest.mark.parametrize("M,C,K,H,W", CASES)
def test_loss_kernel_against_float64(M, C, K, H, W):
    """Random parameters over every M, C, K and side, the batch cycling through 1, 5 and 64: the NLL, the per-image
    sums and every dpreds element within their float64 bounds."""
    i = CASES.index((M, C, K, H, W))
    N = (1, 5, 64)[i % 3]
    g = torch.Generator().manual_seed(200 + i)
    preds = _preds(M, C, N, H, W, g).to(dev())
    x = _grid_input(N, C, H, W, K, g)
    worst, _ = _check_kernel(preds, x, M, K)
    print(f"M {M} C {C} K {K} {H}x{W} N {N}: worst error / bound {worst:.3f}")


def _hard(kind, M, C, K, N, H, W, g):
    preds = _preds(M, C, N, H, W, g)
    x = _grid_input(N, C, H, W, K, g)
    ls = slice(M + M * C, M + 2 * M * C)
    if kind == "peaked":  # one component ahead by 80 nats
        preds[:, 0] += 80.0
    elif kind == "clamp":  # raw log-scales at, just above and just below -7
        at = torch.tensor([-7.0, math.nextafter(-7.0, 0.0), math.nextafter(-7.0, -8.0), -7.5, -6.5])
        preds[:, ls] = at[torch.randint(0, 5, preds[:, ls].shape, generator=g)]
    elif kind == "wide":  # log-scales of +10: a bin carries a tiny share of the mass
        preds[:, ls] = 10.0
    elif kind == "saturated":  # coefficients at +-20
        preds[:, M + 2 * M * C:] = torch.randint(0, 2, preds[:, M + 2 * M * C:].shape, generator=g).float() * 40 - 20
    elif kind == "ends":  # inputs at and beyond the ends of [0, 1]
        ends = torch.tensor([0.0, 1.0, -0.25, 1.25, -0.0])
        x = ends[torch.randint(0, 5, (N, C, H, W), generator=g)].to(dev())
    return preds.to(dev()), x


@pytest.mark.parametrize("K", [2, 256])
@pytest.mark.parametrize("kind", ["peaked", "clamp", "wide", "saturated", "ends"])
def test_loss_kernel_hard_cases(kind, K):
    """Hard parameters within the bounds, and two runs give the same bits."""
    M, C, N, H, W = 5, 3, 5, 7, 13
    preds, x = _hard(kind, M, C, K, N, H, W, torch.Generator().manual_seed(K + len(kind)))
    worst, first = _check_kernel(preds, x, M, K)
    second = _run_kernel(preds, x, M, K)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    print(f"{kind} K {K}: worst error / bound {worst:.3f}")


def test_bounds_see_bug_models():
    """Each bug model misses the bound around the kernel's output by a wide factor, where the kernel itself is within
    it: half-width 1 / K, no clamp of the log-scale, coupling to the wrong channel, the edge bins swapped, and
    1 - tanh^2 in fp32 instead of sech^2."""
    M, C, K, N, H, W = 5, 3, 256, 4, 16, 16
    g = torch.Generator().manual_seed(31)
    preds = _preds(M, C, N, H, W, g, coupling=1.0)
    ls = preds[:, M + M * C:M + 2 * M * C]
    ls[:, :, :4] = -9.0  # below the clamp
    preds[:, M + 2 * M * C:, 4:8] = 20.0  # saturated coefficients
    preds = preds.to(dev())
    x = _grid_input(N, C, H, W, K, g)
    x[:, :, 8:12] = 0.0
    x[:, :, 12:] = 1.0
    worst, (nll, _, dp) = _check_kernel(preds, x, M, K)
    bound = R.nll_bound(preds, x, K)
    for bug in R.BUGS:
        miss = ((R.nll(preds, x, K, bug) - nll.double()).abs() / bound).max().item()
        print(f"{bug}: misses the NLL bound by {miss:.3g}")
        assert miss > 100, (bug, miss)
    dbound = R.dpreds_bound(preds, x, K, 1.0 / N)
    miss = ((R.dpreds(preds, x, K, 1.0 / N, bug="one_minus_tanh2") - dp.double()).abs() / dbound).max().item()
    print(f"one_minus_tanh2: misses the dpreds bound by {miss:.3g}; the kernel's worst error / bound {worst:.3f}")
    assert miss > 100, miss


def test_loss_kernel_refuses_bad_shapes():
    from pytorch_generative_b200 import _lib as L

    x = torch.zeros(2, 3, 4, 4, device=dev())
    with pytest.raises(RuntimeError):  # K = 1
        L.logistic_mixture_nll_kernel(torch.zeros(2, 10, 4, 4, device=dev()), x, 1, 1,
                                      image_nll=torch.zeros(2, device=dev()))


# --------------------------------------------------------------------------------------------------
# the four models
# --------------------------------------------------------------------------------------------------
M_MODELS = 5


def _model_cfg(cls, C):
    out = M_MODELS * R.groups(C)
    return {
        "PixelCNN": dict(in_channels=C, out_channels=out, n_residual=1, residual_channels=16, head_channels=32),
        "GatedPixelCNN": dict(in_channels=C, out_channels=out, n_gated=2, gated_channels=16, head_channels=32),
        "PixelSNAIL": dict(in_channels=C, out_channels=out, n_channels=16, n_pixel_snail_blocks=1, n_residual_blocks=1,
                           attention_key_channels=4, attention_value_channels=8),
        "ImageGPT": dict(in_channels=C, out_channels=out, in_size=8, n_transformer_blocks=1, n_attention_heads=2,
                         n_embedding_channels=32),
    }[cls]


MODELS = ["PixelCNN", "GatedPixelCNN", "PixelSNAIL", "ImageGPT"]
GRAD_TOL = 1e-2  # each gradient tensor within 1e-2 of its own largest entry (test_categorical_gpu.py's per-tensor scale)


def _model(cls, C, seed=0, sample_fn=None):
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    return getattr(models, cls)(**_model_cfg(cls, C), sample_fn=sample_fn).to(dev())


def _loss_bound(preds, x, K):
    N = x.shape[0]
    blocks = -(-x[0, 0].numel() // THREADS)
    ref = R.loss(preds, x, K)[0].item()
    return R.image_sum_bound(preds, x, K, blocks).mean().item() + 4 * N * R.U * abs(ref)


def _grads(loss_or_preds, params, **kw):
    gs = torch.autograd.grad(loss_or_preds, list(params.values()), allow_unused=True, **kw)
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
    """logistic_mixture_nll on each model's output equals the float64 restatement within the kernel bound, and every
    parameter gradient equals the one the same backward gives for the float64 dpreds."""
    from pytorch_generative_b200 import losses

    m = _model(cls, C).train()
    g = torch.Generator().manual_seed(3)
    N, H, W = 3, 8, 8
    x = _grid_input(N, C, H, W, 256, g)
    preds = m(x)
    assert preds.shape == (N, M_MODELS * R.groups(C), H, W)
    out = losses.logistic_mixture_nll(x, None, preds)
    pd = preds.detach()
    ref = R.loss(pd, x, 256)[0].item()
    assert abs(out["loss"].item() - ref) <= _loss_bound(pd, x, 256), (out["loss"].item(), ref)
    assert abs(out["bits_per_dim"].item() - out["loss"].item() / (C * H * W * math.log(2))) <= 1e-6 * out["loss"].item()
    params = dict(m.named_parameters())
    got = _grads(out["loss"], params)
    again = m(x)  # a second forward for the second backward: ImageGPT's fused stack frees its activations in backward
    assert torch.equal(again, preds)
    want = _grads(again, params, grad_outputs=R.dpreds(pd, x, 256, 1.0 / N).float())
    ratios = _grads_close(got, want, cls)
    print(cls, C, "worst gradient errors over own scale:", ratios[:3])


def _adam_step_bound(lr, t, b1=0.9, b2=0.999):
    """Largest |update| of Adam's t-th step (t >= 1, eps ignored): Cauchy-Schwarz on the bias-corrected moment sums
    gives lr (1 - b1) / (1 - b1^t) sqrt(sum_{k<t} (b1^2 / b2)^k) sqrt((1 - b2^t) / (1 - b2)); lr at t = 1."""
    s = sum((b1 * b1 / b2) ** k for k in range(t))
    return lr * (1 - b1) / (1 - b1 ** t) * math.sqrt(s) * math.sqrt((1 - b2 ** t) / (1 - b2))


def test_fused_adam_trajectory():
    """Five FusedAdam steps of PixelSNAIL (C = 3) on one batch: at every step the loss is the float64 restatement's
    within the kernel bound, every gradient is the float64 dpreds' within GRAD_TOL, no weight moves by more than Adam's
    largest step, and the loss falls."""
    from pytorch_generative_b200 import losses, optim

    m = _model("PixelSNAIL", 3, seed=4).train()
    lr = 1e-3
    opt = optim.FusedAdam(m.parameters(), lr=lr)
    x = _grid_input(4, 3, 8, 8, 256, torch.Generator().manual_seed(5))
    params = dict(m.named_parameters())
    seen = []
    for step in range(5):
        opt.zero_grad()
        first = m(x)
        ref = _grads(first, params, grad_outputs=R.dpreds(first.detach(), x, 256, 1.0 / 4).float())
        preds = m(x)
        assert torch.equal(preds, first)
        out = losses.logistic_mixture_nll(x, None, preds)
        pd = preds.detach()
        assert abs(out["loss"].item() - R.loss(pd, x, 256)[0].item()) <= _loss_bound(pd, x, 256), step
        out["loss"].backward()
        _grads_close({k: torch.zeros_like(p) if p.grad is None else p.grad for k, p in params.items()}, ref,
                     f"step {step}")
        before = {k: p.detach().clone() for k, p in params.items()}
        opt.clip_and_step(1e50)
        moved = max((p.detach() - before[k]).abs().max().item() for k, p in params.items())
        assert 0 < moved <= _adam_step_bound(lr, step + 1) * 1.01, (step, moved)
        seen.append(out["loss"].item())
    assert seen[-1] < seen[0], seen


def test_graphed_step_is_bit_identical_to_eager():
    """A GraphedTrainStep replay with logistic_mixture_nll gives the eager step's output, loss and gradients bit for
    bit."""
    from pytorch_generative_b200 import losses, trainstep

    m = _model("ImageGPT", 3, seed=6).train()
    x = _grid_input(2, 3, 8, 8, 256, torch.Generator().manual_seed(7))
    init = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m.zero_grad(set_to_none=True)
    preds = m(x)
    loss = losses.logistic_mixture_nll(x, None, preds)["loss"]
    loss.backward()
    stored = dict(preds=preds.detach().clone(), loss=loss.detach().clone())
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters()}
    del preds, loss
    step = trainstep.GraphedTrainStep(m, list(m.parameters()),
                                      lambda p, xx: losses.logistic_mixture_nll(xx, None, p)["loss"], x, lr=1e-3,
                                      lr_gamma=1.0)
    step.reset(init)
    step(x)
    assert torch.equal(step.static_preds, stored["preds"])
    assert torch.equal(step.static_loss, stored["loss"])
    for n, p in m.named_parameters():
        assert torch.equal(p.grad, grads[n]), n


# --------------------------------------------------------------------------------------------------
# sampling
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,C,K", [(1, 1, 256), (10, 1, 2), (10, 3, 256), (5, 3, 5), (3, 2, 17)])
def test_sampler_is_the_inverse_map(M, C, K):
    """Under recorded uniforms (including u = 0 and u = 1 - 2^-24) each draw equals the float64 inverse map wherever it
    is not within the fp32 bound of a bin edge or a component boundary; every output is k / (K - 1) in fp32; a padded
    row pitch gives the same draws."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(M * 100 + C * 10 + K)
    n = 8192
    preds = _preds(M, C, n, 1, 1, g, coupling=1.5)[:, :, 0, 0].contiguous().to(dev())
    u = torch.rand(n, 1 + C, generator=g)
    u[:64] = 0.0
    u[64:128] = 1.0 - 2.0 ** -24
    u[128:192, 1:] = 0.0
    u[192:256, 1:] = 1.0 - 2.0 ** -24
    u = u.to(dev())
    out = torch.empty(n, C, device=dev())
    L.logistic_mixture_sample(preds, u, out, M, K)
    k = torch.round(out.double() * (K - 1)).long().cpu()
    assert torch.equal(out.cpu(), _grid(k, K)), "off the k / (K - 1) grid"
    ref, near = R.inverse_map(preds.cpu(), u.cpu(), K)
    clear = ~near
    assert clear.float().mean().item() > 0.9
    assert torch.equal(k[clear], ref[clear]), int((k[clear] != ref[clear]).any(dim=1).sum())
    assert (k[128:192] == 0).all()  # u = 0: v = -inf, bin 0 in every channel
    wide = torch.zeros(n, preds.shape[1] + 7, device=dev())
    wide[:, : preds.shape[1]] = preds
    again = torch.empty_like(out)
    L.logistic_mixture_sample(wide[:, : preds.shape[1]], u, again, M, K)
    assert torch.equal(again, out)


def _chi_square(counts, expected):
    """(chi2, degrees of freedom) with cells of fewer than 5 expected draws merged in ascending order of expectation."""
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
    return sum((o - e) ** 2 / e for o, e in zip(obs, exp)), len(obs) - 1


@pytest.mark.parametrize("M,C,K", [(10, 1, 256), (4, 3, 5)])
def test_sampler_chi_square(M, C, K):
    """2e5 seeded draws of logistic_mixture_sample_fn from one pixel against the float64 joint bin probabilities: per
    bin at C = 1, per joint cell at C = 3 and K = 5 with coupling."""
    from scipy import stats

    from pytorch_generative_b200 import models

    g = torch.Generator().manual_seed(M + C + K)
    row = _preds(M, C, 1, 1, 1, g, coupling=1.5)[0, :, 0, 0]
    if K == 5:  # scales comparable to the bins, so every cell is drawn
        row[M + M * C:M + 2 * M * C] = torch.rand(M * C, generator=g) - 1.5
    n = 200_000
    torch.manual_seed(11)
    out = models.logistic_mixture_sample_fn(M, K)(row.to(dev()).repeat(n, 1))
    k = torch.round(out.double() * (K - 1)).long().cpu()
    cell = torch.zeros(n, dtype=torch.long)
    for c in range(C):
        cell = cell * K + k[:, c]
    counts = torch.bincount(cell, minlength=K ** C).double()
    p = R.joint_probabilities(row, C, K).reshape(-1)
    chi2, dof = _chi_square(counts, p * n)
    pval = stats.chi2.sf(chi2, dof)
    print(f"M {M} C {C} K {K}: chi2 {chi2:.1f} on {dof} dof, p {pval:.3g}")
    assert pval > 1e-4, (chi2, dof, pval)


class _Recording:
    """logistic_mixture_sample_fn that keeps every parameter batch it is handed."""

    def __init__(self):
        from pytorch_generative_b200 import models

        self.fn, self.seen = models.logistic_mixture_sample_fn(M_MODELS, 256), []

    def __call__(self, logits):
        self.seen.append(logits.detach().clone())
        return self.fn(logits)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("cls", MODELS)
def test_model_sample(cls, C):
    """sample() with logistic_mixture_sample_fn: teacher-forced (every pixel given) it returns the input and hands each
    pixel's M G parameters, equal to the full forward's; with the top rows given it keeps them and draws the rest on
    the k / 255 grid; n_samples draws land on the grid too; the model deep-copies after sampling."""
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
    twin = copy.deepcopy(m)
    assert twin._sample_fn.fn.n_mixtures == M_MODELS


def test_recipe_trains_one_epoch(tmp_path):
    """reproduce_pixel_snail_8bit on two batches of random 8-bit images: one epoch, a checkpoint whose last output layer
    has 100 channels, and loss and bits/dim in metrics.jsonl consistent with each other."""
    from pytorch_generative_b200 import recipes

    g = torch.Generator().manual_seed(12)
    loader = [(torch.randint(0, 256, (4, 3, 32, 32), generator=g).float().div(255).to(dev()), None) for _ in range(2)]
    trainer = recipes.reproduce_pixel_snail_8bit(n_epochs=1, log_dir=str(tmp_path), debug_loader=loader)
    assert trainer.model._sample_fn.n_mixtures == 10
    ckpt = torch.load(tmp_path / "trainer_state_1.ckpt", weights_only=False)
    assert ckpt["model"]["_output.1.weight"].shape[0] == 100
    rows = [json.loads(line) for line in open(tmp_path / "metrics.jsonl")]
    tags = {r["tag"] for r in rows}
    assert {"metrics/loss", "metrics/bits_per_dim"} <= tags
    bpd = [r["train"] for r in rows if r["tag"] == "metrics/bits_per_dim" and "train" in r]
    loss = [r["train"] for r in rows if r["tag"] == "metrics/loss" and "train" in r]
    assert len(bpd) == 2 and all(math.isfinite(v) and v > 0 for v in bpd)
    for lv, bv in zip(loss, bpd):
        assert abs(bv - lv / (3 * 32 * 32 * math.log(2))) <= 1e-5 * bv
