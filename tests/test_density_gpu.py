"""Mixture models and KDE on the H100: the kernels of csrc/pg_density.cu against float64 with per-element bounds, Parzen
counts equal to the CPU reference's, the reference's outputs (tests/golden/density.pt) and its two known-answer tests,
memory at a size the reference cannot run, determinism and launch counts, sampling, and training (FusedAdam against
torch.optim.Adam on the restatement, the graphed step against the eager one)."""

import copy
import math
import os

import pytest
import torch

import _density_reference as R
from _checks import check, check_equal

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "density.pt")
EPS = 2.0 ** -24
F64, F32 = torch.float64, torch.float32
GAUSS, BERN = 0, 1


def dev():
    return torch.device("cuda:0")


def gamma(k):
    return k * EPS / (1 - k * EPS)


@pytest.fixture(scope="module")
def fixture():
    return torch.load(GOLD, weights_only=False)


def _clustered(n, m, d, seed, spread=1.0):
    """Training points around a few far-apart centres and queries near some of them, so that each query's density is
    dominated by training rows that sit in different codebook splits (a merge without the exp(m_s - max) rescale
    fails)."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn((4, d), generator=g) * 3
    t = centres[torch.randint(0, 4, (m,), generator=g)] + torch.randn((m, d), generator=g) * spread
    x = centres[torch.randint(0, 4, (n,), generator=g)] + torch.randn((n, d), generator=g) * spread
    return x.to(dev()), t.to(dev())


# --------------------------------------------------------------------------------------------------
# Gaussian KDE
# --------------------------------------------------------------------------------------------------
def _gauss_ref(x, t, h):
    """float64 log p, lse, w = exp(s - lse), |s| via matrix products (the expanded form is exact enough in float64)."""
    x64, t64 = x.to(F64), t.to(F64)
    M, D = t.shape
    sq = ((x64 * x64).sum(1)[:, None] + (t64 * t64).sum(1)[None, :] - 2 * x64 @ t64.T).clamp(min=0)
    s = -0.5 * sq / h ** 2
    lse = torch.logsumexp(s, 1)
    w = torch.exp(s - lse[:, None])
    return lse, s, w


GAUSS_CASES = [(1, 1, 1, 1.0), (5, 63, 2, 0.5), (300, 65, 37, 2.0), (0, 100, 2, 1.0), (5, 60000, 784, 1.5),
               (300, 100, 3072, 4.0), (4096, 65, 784, 1.5), (1, 60000, 37, 0.3), (300, 60000, 2, 0.05)]


@pytest.mark.parametrize("N, M, D, h", GAUSS_CASES)
def test_gauss_forward_and_backward_against_float64(N, M, D, h):
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.models import kde

    x, t = _clustered(N, M, D, seed=N + M + D)
    Z = kde.gaussian_log_normaliser(M, D, h)
    out = torch.full((N,), float("nan"), dtype=F32, device=dev())
    lse = torch.full((N,), float("nan"), dtype=F32, device=dev())
    L.kde_gauss_fwd(x, t, h, Z, out, lse)
    if N == 0:
        return
    lse_ref, s, w = _gauss_ref(x, t, h)
    Z64 = 0.5 * D * math.log(2 * math.pi) + D * math.log(h) + math.log(M)
    # each pair value carries gamma(D + 5) |s| (D fmaf, the scale's two roundings); the logsumexp adds the relative error
    # of its sum of exps (the per-thread chains, the butterfly and the split merge: at most M / 16 + 40 roundings, two
    # per exp) and the roundings of max + log(l) and of - Z
    lse_bound = (w * s.abs()).sum(1) * gamma(D + 5) + gamma(2 * (M // 16) + 80) + gamma(2) * lse_ref.abs()
    check("lse", lse, lse_ref, lse_bound)
    check("log p", out, lse_ref - Z64, lse_bound + gamma(2) * (lse_ref - Z64).abs() + abs(Z - Z64) + gamma(1) * abs(Z64))
    # backward: dx = -(g / h^2) sum_m w (x - t)
    g = torch.randn(N, generator=torch.Generator().manual_seed(7)).to(dev())
    dx = torch.zeros_like(x)
    L.kde_gauss_bwd(x, t, h, lse, g, dx)
    x64, t64, g64 = x.to(F64), t.to(F64), g.to(F64)
    c = -g64 / h ** 2
    dx_ref = c[:, None] * (x64 * w.sum(1, keepdim=True) - w @ t64)
    # |x - t| <= |x| + |t|; per weight the relative error of s - lse and of exp, then the chain of the sum over m and
    # the split partials
    mag = x64.abs() * w.sum(1, keepdim=True) + w @ t64.abs()
    mag_rel = (w * (s.abs() * gamma(D + 5))) @ t64.abs() + x64.abs() * (w * s.abs() * gamma(D + 5)).sum(1, keepdim=True)
    bound = c.abs()[:, None] * (mag_rel + mag * (lse_bound[:, None].to(F64) + gamma(M + 16)))
    check("dx", dx, dx_ref, bound)


def test_gauss_split_merge_needs_the_rescale():
    """Peaked distances over many splits: the per-split maxima differ by hundreds, so l_s summed without exp(m_s - max)
    would be off by orders of magnitude; the merged result holds the bound."""
    from pytorch_generative_b200 import _lib as L
    from pytorch_generative_b200.models import kde

    x, t = _clustered(7, 60000, 16, seed=3, spread=0.3)
    h = 0.2
    out = torch.empty(7, dtype=F32, device=dev())
    L.kde_gauss_fwd(x, t, h, kde.gaussian_log_normaliser(60000, 16, h), out)
    lse_ref, s, w = _gauss_ref(x, t, h)
    assert ((s.amax(1) - s.amin(1)) > 100).all()
    Z64 = 0.5 * 16 * math.log(2 * math.pi) + 16 * math.log(h) + math.log(60000)
    bound = (w * s.abs()).sum(1) * gamma(21) + gamma(2 * 3750 + 80) + gamma(4) * lse_ref.abs() + 1e-5
    check("peaked log p", out, lse_ref - Z64, bound)


# --------------------------------------------------------------------------------------------------
# Parzen window
# --------------------------------------------------------------------------------------------------
def _cpu_counts(x, t, h, strict=False):
    x, t = x.cpu(), t.cpu()
    return torch.cat([R.parzen_inside(x[i:i + 16], t, h, strict).sum(1) for i in range(0, x.shape[0], 16)]).int()


def _check_log_density(name, got, ref):
    """-inf exactly where the reference has it; elsewhere within two fp32 roundings (the fp64 logs are formed in a
    different order before they are rounded)."""
    assert torch.equal(torch.isinf(got), torch.isinf(ref)), name
    fin = ~torch.isinf(ref)
    check(name, got[fin], ref[fin].to(F64), gamma(2) * ref[fin].to(F64).abs())


PARZEN_CASES = [(1, 1, 1), (5, 63, 2), (300, 65, 37), (5, 100, 784), (300, 60000, 2), (64, 60000, 37), (5, 65, 3072)]


@pytest.mark.parametrize("N, M, D", PARZEN_CASES)
def test_parzen_counts_equal_the_cpu_reference(N, M, D):
    """Grid data: every difference is a multiple of 1/8, so many |x - t| / h are exactly 0.5 at h = 0.25; a second run at
    h = 0.1 (not a power of two) has quotients that round to 0.5 from either side."""
    from pytorch_generative_b200 import _lib as L

    g = torch.Generator().manual_seed(N * 7 + M + D)
    t = torch.randint(0, 3, (M, D), generator=g).float() / 8
    x = torch.randint(0, 3, (N, D), generator=g).float() / 8
    for h, xs in ((0.25, x), (0.1, x * 0.4)):
        ts = t if h == 0.25 else t * 0.4
        count = torch.empty(N, dtype=torch.int32, device=dev())
        out = torch.empty(N, dtype=F32, device=dev())
        L.kde_parzen_count(xs.to(dev()), ts.to(dev()), h, count=count, out=out)
        ref = _cpu_counts(xs, ts, h)
        check_equal("count", count.cpu(), ref)
        _check_log_density("log p", out.cpu(), R.parzen_log_density(ref, M, D, h))
        if h == 0.25 and D <= 2:
            assert ref.sum() > 0


def test_parzen_boundary_set_and_the_strict_bug_model(fixture):
    from pytorch_generative_b200 import models

    fx = fixture["kde"]["parzen_boundary"]
    kde = models.KernelDensityEstimator(fx["train"].to(dev()), models.ParzenWindowKernel(fx["bandwidth"]))
    got = kde(fx["x"].to(dev()))
    _check_log_density("boundary", got.cpu(), fx["out"])  # D = 2, h = 0.1: the reference's coef is finite
    strict = _cpu_counts(fx["x"], fx["train"], fx["bandwidth"], strict=True)
    assert not torch.equal(strict > 0, ~torch.isinf(got.cpu()))


# --------------------------------------------------------------------------------------------------
# mixture models
# --------------------------------------------------------------------------------------------------
def _mixture_params(kind, K, D, seed):
    g = torch.Generator().manual_seed(seed)
    p = {"mixture_logits": torch.randn(K, generator=g)}
    if kind == GAUSS:
        p.update(mean=torch.randn((K, D), generator=g) * 0.5, log_std=torch.randn((K, D), generator=g) * 0.3)
    else:
        p.update(logits=torch.randn((K, D), generator=g) * 2)
    return {k: v.to(dev()) for k, v in p.items()}


def _mixture_x(kind, N, D, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, D), generator=g) if kind == GAUSS else (torch.rand((N, D), generator=g) < 0.3).float()
    return x.to(dev())


def _mixture_magnitudes(kind, p, x):
    """float64 (a [N, K], sum over d of the magnitudes of the rounded quantities of each term [N, K], the per-element
    derivative factors by parameter [N, K, D] and for x)."""
    p64 = {k: v.to(F64) for k, v in p.items()}
    x64 = x.to(F64)[:, None, :]
    lsm = torch.log_softmax(p64["mixture_logits"], -1)
    if kind == GAUSS:
        sd = p64["log_std"].exp()
        q = (x64 - p64["mean"]) / sd
        terms = (-p64["log_std"] - 0.5 * math.log(2 * math.pi)) - 0.5 * q * q
        mag = (p64["log_std"].abs() + 1 + 0.5 * q * q).sum(-1)
        facs = {"mean": q / sd, "log_std": q * q - 1}
        fac_mag = {"mean": (q / sd).abs(), "log_std": q * q + 1}
        fx = -q / sd
    else:
        lg = p64["logits"]
        terms = lg * x64 - (lg.clamp(min=0) + torch.log1p(torch.exp(-lg.abs())))
        mag = ((lg * x64).abs() + lg.clamp(min=0) + torch.log1p(torch.exp(-lg.abs()))).sum(-1)
        facs = {"logits": x64 - torch.sigmoid(lg)}
        fac_mag = {"logits": x64.abs() + torch.sigmoid(lg)}  # the operands of x - sigmoid(l): sigmoid carries the error
        fx = lg.expand_as(terms)
    return lsm + terms.sum(-1), mag, facs, fac_mag, fx


MIX_CASES = [(kind, N, K, D) for kind in (GAUSS, BERN)
             for (N, K, D) in ((0, 3, 2), (1, 1, 1), (5, 3, 37), (300, 13, 784), (4096, 3, 2), (300, 256, 37),
                               (5, 13, 3072), (1024, 64, 784))]


@pytest.mark.parametrize("kind, N, K, D", MIX_CASES)
def test_mixture_forward_and_backward_against_float64(kind, N, K, D):
    from pytorch_generative_b200 import _lib as L

    p = _mixture_params(kind, K, D, seed=K * 3 + D)
    x = _mixture_x(kind, N, D, seed=N + 1)
    p0, p1 = (p["mean"], p["log_std"]) if kind == GAUSS else (p["logits"], None)
    a = torch.full((N, K), float("nan"), dtype=F32, device=dev())
    out = torch.full((N,), float("nan"), dtype=F32, device=dev())
    L.mixture_fwd(kind, x, p["mixture_logits"], p0, p1, a, out)
    if N == 0:
        return
    a_ref, mag, facs, fac_mag, fx = _mixture_magnitudes(kind, p, x)
    lsm_mag = p["mixture_logits"].to(F64).abs() + p["mixture_logits"].to(F64).abs().max() + math.log(K) + 1
    a_bound = gamma(D + 10) * mag + gamma(K + 8) * lsm_mag
    check("a", a, a_ref, a_bound)
    out_ref = torch.logsumexp(a_ref, 1)
    r = torch.exp(a_ref - out_ref[:, None])
    out_bound = (r * a_bound).sum(1) + gamma(2 * K + 8) * (1 + out_ref.abs())
    check("out", out, out_ref, out_bound)
    # backward
    g = torch.randn(N, generator=torch.Generator().manual_seed(11)).to(dev())
    g64 = g.to(F64)
    names = list(facs)
    flat = torch.zeros(len(names) * K * D + K, dtype=F32, device=dev())
    dx = torch.full((N, D), float("nan"), dtype=F32, device=dev())
    L.mixture_bwd(kind, x, p["mixture_logits"], p0, p1, a, out, g, flat, dx)
    r_rel = a_bound + out_bound[:, None] + gamma(8)  # relative error of each responsibility
    gr = g64[:, None] * r
    for i, name in enumerate(names):
        ref = torch.einsum("nk,nkd->kd", gr, facs[name])
        bound = torch.einsum("nk,nkd->kd", gr.abs() * r_rel, fac_mag[name]) * (1 + gamma(8)) + \
            gamma(N + 40) * torch.einsum("nk,nkd->kd", gr.abs(), fac_mag[name] + gamma(8))
        check(f"d{name}", flat[i * K * D:(i + 1) * K * D].view(K, D), ref, bound)
    sm = torch.softmax(p["mixture_logits"].to(F64), 0)
    dml_ref = gr.sum(0) - sm * g64.sum()
    dml_bound = (gr.abs() * r_rel).sum(0) + gamma(N + 40) * (gr.abs().sum(0) + sm * g64.abs().sum()) + \
        gamma(K + 8) * sm * g64.abs().sum()
    check("dmixture_logits", flat[len(names) * K * D:], dml_ref, dml_bound)
    dx_ref = torch.einsum("nk,nkd->nd", gr, fx)
    dx_bound = torch.einsum("nk,nkd->nd", gr.abs() * (r_rel + gamma(K + 8)), fx.abs() * (1 + gamma(6)))
    check("dx", dx, dx_ref, dx_bound)


# --------------------------------------------------------------------------------------------------
# models against the reference's outputs
# --------------------------------------------------------------------------------------------------
def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def test_mixture_models_match_the_fixture(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture["mixture"].items():
        m = getattr(models, fx["cls"])(**fx["kwargs"])
        m.load_state_dict(fx["state"])
        m = m.to(dev())
        x = fx["x"].to(dev()).requires_grad_(True)
        out = m(x)
        assert out.shape == fx["out"].shape and out.dtype == F32, name
        assert _rel(out, fx["out"]) <= 1e-5, name
        (out * fx["cot"].to(dev())).sum().backward()
        # each gradient against its own scale; float64 restatement gives the scale of the fp32 reference's own error
        _, g64, xg64 = R.mixture_loss_and_grads(fx["cls"], fx["state"], fx["x"], fx["cot"], F64)
        for k, prm in m.named_parameters():
            assert _rel(prm.grad, g64[k]) <= 1e-4, (name, k, _rel(prm.grad, g64[k]))
        assert x.grad.shape == fx["x"].shape and _rel(x.grad, xg64) <= 1e-4, name


def test_kde_matches_the_fixture(fixture):
    from pytorch_generative_b200 import models

    for name, fx in fixture["kde"].items():
        kde = models.KernelDensityEstimator(fx["train"].to(dev()), getattr(models, fx["kernel"])(fx["bandwidth"]))
        x = fx["x"].to(dev()).requires_grad_(fx["kernel"] == "GaussianKernel")
        out = kde(x)
        if fx["kernel"] == "GaussianKernel":
            assert _rel(out, fx["out"]) <= 1e-5, name
            (out * fx["cot"].to(dev())).sum().backward()
            assert _rel(x.grad, fx["x_grad"]) <= 1e-4, name
        else:
            assert out.grad_fn is None
            assert torch.equal(torch.isinf(out.cpu()), torch.isinf(fx["out"])), name
            fin = ~torch.isinf(fx["out"])
            assert _rel(out.cpu()[fin], fx["out"][fin]) <= 1e-6, name


@pytest.mark.parametrize("kernel", ["GaussianKernel", "ParzenWindowKernel"])
def test_reference_known_answer_integral_is_one(kernel):
    """The reference's tests.py:201-233 with the data on CUDA: the density over a 0.1-spaced mesh integrates to 1."""
    from pytorch_generative_b200 import models

    torch.manual_seed(0)
    train_Xs = torch.normal(torch.zeros((100, 2)), torch.ones((100, 2))).to(dev())
    model = models.KernelDensityEstimator(train_Xs, getattr(models, kernel)(bandwidth=1.0))
    dx = 0.1
    X = torch.arange(-8, 8, dx)
    xx, yy = torch.meshgrid(X, X, indexing="ij")
    meshgrid = torch.stack((xx, yy), axis=2).view(-1, 2).to(dev())
    log_probs = model(meshgrid)
    integral = torch.sum(torch.exp(log_probs) * dx * dx)
    torch.testing.assert_close(integral.cpu(), torch.tensor(1.0))


def test_other_dtypes_and_requires_grad_training_data_raise():
    from pytorch_generative_b200 import _lib as L, models

    before = L.launch_count()
    with pytest.raises(RuntimeError, match="fp32"):
        models.GaussianMixtureModel(3, 4).to(dev())(torch.zeros(2, 4, dtype=F64, device=dev()))
    with pytest.raises(RuntimeError, match="fp32"):
        models.GaussianMixtureModel(3, 4).to(dev()).double()(torch.zeros(2, 4, device=dev()))
    with pytest.raises(RuntimeError, match="fp32"):
        models.KernelDensityEstimator(torch.rand(5, 3, device=dev()))(torch.rand(2, 3, dtype=F64, device=dev()))
    with pytest.raises(NotImplementedError):
        models.KernelDensityEstimator(torch.rand(5, 3, device=dev(), requires_grad=True))(torch.rand(2, 3, device=dev()))
    assert L.launch_count() == before


# --------------------------------------------------------------------------------------------------
# memory, determinism, launch counts
# --------------------------------------------------------------------------------------------------
def test_gaussian_kde_at_a_size_the_reference_cannot_hold():
    """N = 4096 queries against M = 65536 training points of D = 784: the reference's [N, M, D] intermediate would be
    842 GB.  Above the inputs the forward allocates O(N) through torch (out, lse; the split partials, 32 N floats, live
    in the library scratch): the budget asserted is (N + M) D floats, one more copy of the inputs."""
    from pytorch_generative_b200 import models

    N, M, D = 4096, 65536, 784
    g = torch.Generator(device=dev()).manual_seed(5)
    t = torch.rand((M, D), device=dev(), generator=g)
    x = t[:N] + 0.01 * torch.randn((N, D), device=dev(), generator=g)
    kde = models.KernelDensityEstimator(t, models.GaussianKernel(bandwidth=0.5))
    kde(x[:64])  # grows the scratch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = kde(x)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= (N + M) * D * 4
    assert torch.isfinite(out).all()
    # each query lies near its own training point, so log p is dominated by exp(-0.5 |x - t|^2 / h^2) / M
    sq = ((x - t[:N]) ** 2).sum(1).double()
    nearest = -0.5 * sq / 0.25 - (0.5 * D * math.log(2 * math.pi) + D * math.log(0.5) + math.log(M))
    assert (out.double() >= nearest - 1e-3 * nearest.abs()).all()


def test_repeat_runs_and_sub_batches_are_bit_identical():
    from pytorch_generative_b200 import models

    x, t = _clustered(300, 5000, 37, seed=9)
    for kernel in (models.GaussianKernel(0.8), models.ParzenWindowKernel(6.0)):
        kde = models.KernelDensityEstimator(t, kernel)
        xs = x.clone().requires_grad_(isinstance(kernel, models.GaussianKernel))
        a, b = kde(xs), kde(xs)
        check_equal("repeat", a, b)
        check_equal("sub-batch", kde(x[17:40]), a[17:40].detach())
        if xs.requires_grad:
            g1 = torch.autograd.grad(a.sum(), xs)[0]
            g2 = torch.autograd.grad(b.sum(), xs)[0]
            check_equal("dx repeat", g1, g2)
            xsub = x[17:40].clone().requires_grad_(True)
            check_equal("dx sub-batch", torch.autograd.grad(kde(xsub).sum(), xsub)[0], g1[17:40])
    for cls in (models.GaussianMixtureModel, models.BernoulliMixtureModel):
        torch.manual_seed(1)
        m = cls(64, 784).to(dev())
        xb = _mixture_x(GAUSS if cls is models.GaussianMixtureModel else BERN, 300, 784, seed=2)
        runs = []
        for _ in range(2):
            m.zero_grad()
            out = m(xb)
            out.sum().backward()
            runs.append((out.detach(), [p.grad.clone() for p in m.parameters()]))
        check_equal("mixture repeat", runs[0][0], runs[1][0])
        for u, v in zip(runs[0][1], runs[1][1]):
            check_equal("mixture grad repeat", u, v)
        with torch.no_grad():
            check_equal("mixture sub-batch", m(xb[17:40]), runs[0][0][17:40])


def test_launch_counts_match_the_header():
    """Gaussian forward 2, its backward 2; Parzen 2; mixture forward 2, backward 2 and 3 with an input gradient, at
    every size."""
    from pytorch_generative_b200 import _lib as L, models

    def launches(fn):
        torch.cuda.synchronize()
        before = L.launch_count()
        fn()
        torch.cuda.synchronize()
        return L.launch_count() - before

    for N, M, D in ((1, 1, 1), (300, 60000, 37), (4096, 65, 784)):
        x, t = _clustered(N, M, D, seed=1)
        g = models.KernelDensityEstimator(t, models.GaussianKernel(1.0))
        p = models.KernelDensityEstimator(t, models.ParzenWindowKernel(1.0))
        xg = x.clone().requires_grad_(True)
        with torch.no_grad():
            assert launches(lambda: g(x)) == 2
        assert launches(lambda: p(x)) == 2
        assert launches(lambda: g(xg).sum().backward()) == 4
    for cls in (models.GaussianMixtureModel, models.BernoulliMixtureModel):
        for N, K, D in ((1, 1, 1), (300, 13, 784), (4096, 256, 37)):
            m = cls(K, D).to(dev())
            x = torch.rand((N, D), device=dev())
            with torch.no_grad():
                assert launches(lambda: m(x)) == 2
            assert launches(lambda: m(x).sum().backward()) == 4
            xg = x.clone().requires_grad_(True)
            assert launches(lambda: m(xg).sum().backward()) == 5


# --------------------------------------------------------------------------------------------------
# sampling and training
# --------------------------------------------------------------------------------------------------
def test_seeded_samples_equal_the_restatement_on_the_device(fixture):
    import numpy as np

    from pytorch_generative_b200 import models

    for name, fx in fixture["mixture"].items():
        m = getattr(models, fx["cls"])(**fx["kwargs"])
        m.load_state_dict(fx["state"])
        m = m.to(dev())
        m(fx["x"].to(dev()))
        torch.manual_seed(fx["sample_seed"])
        got = m.sample(5)
        torch.manual_seed(fx["sample_seed"])
        ref = R.mixture_sample(fx["cls"], {k: v.to(dev()) for k, v in fx["state"].items()}, 5, fx["x"].shape)
        assert got.device.type == "cuda"
        check_equal(name, got, ref)
    t = torch.rand(50, 3, device=dev())
    kde = models.KernelDensityEstimator(t, models.GaussianKernel(0.3))
    np.random.seed(1)
    torch.manual_seed(2)
    got = kde.sample(7)
    np.random.seed(1)
    torch.manual_seed(2)
    idxs = np.random.choice(range(50), size=7)
    check_equal("kde sample", got, t[idxs] + torch.randn(t[idxs].shape, device=dev()) * 0.3)


@pytest.mark.parametrize("cls", ["GaussianMixtureModel", "BernoulliMixtureModel"])
def test_fused_adam_trajectory_matches_the_restatement(cls):
    from pytorch_generative_b200 import models, optim

    torch.manual_seed(4)
    m = getattr(models, cls)(16, 3 * 8 * 8).to(dev())
    params = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters()}
    ref_opt = torch.optim.Adam(list(params.values()), lr=1e-2)
    opt = optim.FusedAdam(m.parameters(), lr=1e-2)
    kind = GAUSS if cls == "GaussianMixtureModel" else BERN
    for s in range(3):
        x = _mixture_x(kind, 64, 192, seed=30 + s).view(64, 3, 8, 8)
        ref_opt.zero_grad()
        ref_loss = -R.mixture_forward(cls, params, x).mean()
        ref_loss.backward()
        ref_norm = torch.nn.utils.clip_grad_norm_(list(params.values()), 1e50).item()
        ref_opt.step()
        opt.zero_grad()
        loss = -m(x).mean()
        loss.backward()
        norm = opt.clip_and_step(1e50).item()
        assert abs(loss.item() - ref_loss.item()) <= 1e-4 * max(1.0, abs(ref_loss.item())), s
        assert abs(norm - ref_norm) <= 1e-4 * ref_norm, (s, norm, ref_norm)
    for k, prm in m.named_parameters():
        assert _rel(prm, params[k]) <= 1e-3, k


def _nll(preds, x):
    return -preds.mean()


@pytest.mark.parametrize("cls", ["GaussianMixtureModel", "BernoulliMixtureModel"])
def test_graphed_train_step_equals_the_eager_step(cls):
    """Forward and backward never synchronise with the host: the step captures as a CUDA graph, and two replays equal
    two eager steps bit for bit."""
    from pytorch_generative_b200 import models, trainstep

    torch.manual_seed(5)
    init = getattr(models, cls)(64, 784).to(dev())
    state = {k: v.clone() for k, v in init.state_dict().items()}
    kind = GAUSS if cls == "GaussianMixtureModel" else BERN
    xs = [_mixture_x(kind, 1024, 784, seed=40 + s).view(1024, 1, 28, 28) for s in range(2)]
    graphed = copy.deepcopy(init)
    step = trainstep.GraphedTrainStep(graphed, graphed.parameters(), _nll, xs[0], lr=1e-3, lr_gamma=1.0)
    step.reset(state, lr=1e-3)
    eager = copy.deepcopy(init)
    eager.load_state_dict(state)
    params = list(eager.parameters())
    opt = torch.optim.Adam(params, lr=torch.tensor(1e-3, device=dev()), capturable=True)
    for x in xs:
        loss_g, norm_g = step(x)
        opt.zero_grad(set_to_none=True)
        loss = _nll(eager(x), x)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 1e50, foreach=True)
        opt.step()
        assert loss_g == loss.item() and norm_g == norm.item()
    for (k, a), b in zip(graphed.named_parameters(), params):
        check_equal(k, a.detach(), b.detach())
