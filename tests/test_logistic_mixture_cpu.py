"""CPU checks of the discretised logistic mixture likelihood: the float64 restatement (bin masses that sum to 1, bin
masses against scipy's logistic CDF, closed-form gradients against autograd, the target rule, the channel layout),
the argument checks of losses.logistic_mixture_nll, the sample function's channel inference and pickling, the 8-bit
PixelSNAIL recipe's signature and the library's new symbols."""

import copy
import inspect
import math
import pickle

import pytest
import torch

import _logistic_mixture_reference as R

F64 = torch.float64


def _preds(M, C, N, P, g, scale=1.0, coupling=1.0):
    """Random parameters [N, M * G, P, 1]: logits and means ~ scale N(0, 1), log-scales in [-4, -1], coefficients ~
    coupling N(0, 1)."""
    T = C * (C - 1) // 2
    pi = torch.randn(N, M, P, generator=g) * scale
    mu = torch.randn(N, M * C, P, generator=g) * 0.5 * scale
    ls = torch.rand(N, M * C, P, generator=g) * 3 - 4
    r = torch.randn(N, M * T, P, generator=g) * coupling
    return torch.cat([pi, mu, ls, r], dim=1).unsqueeze(-1).float()


def _every_cell(C, K):
    cells = torch.cartesian_prod(*[torch.arange(K)] * C).reshape(-1, C) if C > 1 else torch.arange(K).reshape(-1, 1)
    return cells, (cells.double() / (K - 1)).float().reshape(-1, C, 1, 1)


@pytest.mark.parametrize("M,C,K", [(1, 1, 256), (4, 1, 256), (3, 1, 2), (3, 3, 5), (2, 3, 2), (2, 2, 7)])
def test_bin_masses_sum_to_one(M, C, K):
    """Over all K^C cells of one pixel (all 256 bins at C = 1; all 125 at C = 3, K = 5, with coupling), the masses
    sum to 1 within 1e-12."""
    g = torch.Generator().manual_seed(M * 100 + C * 10 + K)
    for _ in range(3):
        row = _preds(M, C, 1, 1, g, coupling=1.5)[0, :, 0, 0]
        p = R.joint_probabilities(row, C, K)
        assert p.shape == (K,) * C and (p > 0).all()
        assert abs(p.sum().item() - 1.0) <= 1e-12, p.sum().item()


@pytest.mark.parametrize("K", [2, 5, 256])
def test_bin_masses_equal_logistic_cdf_differences(K):
    """One component, one channel: the mass of every bin is the difference of scipy's logistic CDF at its edges, the end
    bins taking the tails, in float64."""
    from scipy import stats

    for mu, ls in [(0.1, -3.0), (-0.8, -5.5), (0.3, 0.5), (0.0, -9.0)]:
        row = torch.tensor([0.0, mu, ls], dtype=torch.float32)
        p = R.joint_probabilities(row, 1, K)
        s = math.exp(max(float(row[2]), -7.0))
        m = float(row[1])
        edges = [(2 * k / (K - 1) - 1) for k in range(K)]
        h = 1.0 / (K - 1)
        for k in range(K):
            hi = 1.0 if k == K - 1 else stats.logistic.cdf(edges[k] + h, loc=m, scale=s)
            lo = 0.0 if k == 0 else stats.logistic.cdf(edges[k] - h, loc=m, scale=s)
            want = hi - lo
            assert abs(p[k].item() - want) <= 1e-12 * max(1.0, 1 / max(want, 1e-300)) * want + 1e-15, (k, p[k], want)


@pytest.mark.parametrize("M,C,K", [(1, 1, 256), (3, 1, 2), (5, 3, 256), (2, 3, 2), (2, 2, 9)])
def test_closed_form_gradients_equal_autograd(M, C, K):
    """The gradient formulas of the convention equal float64 autograd of the restatement (log-scales on both sides of
    -7, including exactly -7, every bin kind and saturated coefficients)."""
    g = torch.Generator().manual_seed(M + C + K)
    N, P = 3, 40
    preds = _preds(M, C, N, P, g, coupling=2.0)
    G = R.groups(C)
    ls_rows = slice(M + M * C, M + 2 * M * C)
    preds[:, ls_rows, :8] = -7.0
    preds[:, ls_rows, 8:12] = -8.5
    if C > 1:
        preds[:, M + 2 * M * C:, 12:16] = 20.0
    x = torch.randint(0, K, (N, C, P, 1), generator=g).double().div(K - 1).float()
    x[:, :, 20:24] = 0.0
    x[:, :, 24:28] = 1.0
    assert preds.shape[1] == M * G
    leaf = preds.double().requires_grad_(True)
    (R.nll(leaf, x, K).sum() * 0.25).backward()
    got = R.dpreds(preds, x, K, 0.25)
    err = (got - leaf.grad).abs().max().item()
    assert err <= 1e-12 * max(1.0, leaf.grad.abs().max().item()), err


@pytest.mark.parametrize("K", [2, 17, 256])
def test_target_rule_is_the_categorical_rule(K):
    from pytorch_generative_b200 import losses

    k = torch.arange(K)
    x = (k.double() / (K - 1)).float()
    assert torch.equal(R.target(x, K), losses.categorical_target(x, K))
    assert torch.equal(R.target(x, K), k)
    ends = torch.tensor([-0.5, -0.0, 1.0, 1.5])
    assert torch.equal(R.target(ends, K), losses.categorical_target(ends, K))


def test_layout_moves_exactly_the_named_parameter():
    """A preds tensor of zeros with one nonzero parameter changes exactly the component, channel and coefficient the
    layout table names: the mixture logit of m, the mean / log-scale of (m, c), the coupling of (m, c, j)."""
    M, C, K = 3, 3, 256
    G, T = R.groups(C), C * (C - 1) // 2
    base = torch.zeros(1, M * G, 1, 1)
    for m in range(M):
        p = base.clone()
        p[0, m] = 1.5
        pi, mu, ls, r = R.split(p, C)
        assert pi[0, m, 0] == 1.5 and pi.abs().sum() == 1.5 and mu.abs().sum() == 0 and ls.abs().sum() == 0
        for c in range(C):
            p = base.clone()
            p[0, M + m * C + c] = 0.25
            pi, mu, ls, r = R.split(p, C)
            assert mu[0, m, c, 0] == 0.25 and mu.abs().sum() == 0.25 and pi.abs().sum() == 0 and r.abs().sum() == 0
            p = base.clone()
            p[0, M + M * C + m * C + c] = -2.0
            pi, mu, ls, r = R.split(p, C)
            assert ls[0, m, c, 0] == -2.0 and ls.abs().sum() == 2.0 and mu.abs().sum() == 0
            for j in range(c):
                t = c * (c - 1) // 2 + j
                p = base.clone()
                p[0, M + 2 * M * C + m * T + t] = 3.0
                pi, mu, ls, r = R.split(p, C)
                assert r[0, m, t, 0] == 3.0 and r.abs().sum() == 3.0
                # the coefficient moves the mean of (m, c) by tanh(3) x'_j and no other
                x = torch.tensor([0.2, 0.9, 0.5]).reshape(1, C, 1, 1)
                t0, t1 = R._terms(base, x, K), R._terms(p, x, K)
                moved = (t1["mup"] - t0["mup"]).abs() > 0
                assert moved.sum() == 1 and moved[0, m, c, 0]
                want = math.tanh(3.0) * R.centre(R.target(x[0, j], K), K).item()
                assert abs((t1["mup"] - t0["mup"])[0, m, c, 0].item() - want) <= 1e-15


@pytest.mark.parametrize("preds_shape,x_shape", [
    ((2, 9, 4, 4), (2, 3, 4, 4)),      # 9 channels are not a multiple of G = 10
    ((2, 0, 4, 4), (2, 3, 4, 4)),      # M = 0
    ((2, 4, 4, 4), (2, 1, 4, 4)),      # 4 channels are not a multiple of G = 3
    ((2, 100, 4, 4), (2, 3, 4, 5)),    # spatial shapes differ
    ((3, 100, 4, 4), (2, 3, 4, 4)),    # batch sizes differ
    ((2, 100, 16), (2, 3, 4, 4)),      # ranks differ
])
def test_argument_checks(preds_shape, x_shape):
    from pytorch_generative_b200 import losses

    with pytest.raises(ValueError):
        losses.logistic_mixture_nll(torch.zeros(x_shape), None, torch.zeros(preds_shape))


def test_bad_bin_count_and_cpu_tensors():
    from pytorch_generative_b200 import losses, models

    with pytest.raises(ValueError):
        losses.logistic_mixture_nll(torch.zeros(1, 3, 2, 2), None, torch.zeros(1, 100, 2, 2), n_bins=1)
    with pytest.raises(RuntimeError):
        losses.logistic_mixture_nll(torch.zeros(1, 3, 2, 2), None, torch.zeros(1, 100, 2, 2))
    with pytest.raises(RuntimeError):
        models.logistic_mixture_sample_fn()(torch.zeros(2, 100))


def test_bits_per_dim_arithmetic(monkeypatch):
    """logistic_mixture_nll divides its loss by C H W ln 2 (the autograd Function is replaced by the restatement so
    the arithmetic runs on the CPU)."""
    from pytorch_generative_b200 import losses

    monkeypatch.setattr(losses._LogisticMixtureNLL, "apply", lambda p, x, m, k: R.loss(p, x, k)[0])
    g = torch.Generator().manual_seed(3)
    preds = _preds(10, 3, 2, 24, g).reshape(2, 100, 4, 6)
    x = torch.randint(0, 256, (2, 3, 4, 6), generator=g).float() / 255
    out = losses.logistic_mixture_nll(x, None, preds)
    assert set(out) == {"loss", "bits_per_dim"}
    ref, ref_bpd = R.loss(preds, x, 256)
    assert out["loss"].item() == ref.item()
    assert abs(out["bits_per_dim"].item() - ref.item() / (3 * 4 * 6 * math.log(2))) <= 1e-12 * ref_bpd.item()


def test_sample_fn_channels_repr_and_pickling():
    from pytorch_generative_b200 import models

    sig = inspect.signature(models.logistic_mixture_sample_fn)
    assert list(sig.parameters) == ["n_mixtures", "n_bins"]
    assert sig.parameters["n_mixtures"].default == 10 and sig.parameters["n_bins"].default == 256
    fn = models.logistic_mixture_sample_fn()
    assert isinstance(fn, models.LogisticMixtureSampleFn)
    assert fn.channels(100) == 3 and fn.channels(30) == 1 and fn.channels(60) == 2 and fn.channels(150) == 4
    for bad in (99, 40, 10, 0):
        with pytest.raises(ValueError):
            fn.channels(bad)
    with pytest.raises(ValueError):
        fn(torch.zeros(2, 99))
    assert models.logistic_mixture_sample_fn(5).channels(15) == 1
    assert repr(models.logistic_mixture_sample_fn(5, 17)) == "logistic_mixture_sample_fn(n_mixtures=5, n_bins=17)"
    for bad in ((0, 256), (10, 1)):
        with pytest.raises(ValueError):
            models.logistic_mixture_sample_fn(*bad)
    fn = models.logistic_mixture_sample_fn(5, 17)
    for twin in (pickle.loads(pickle.dumps(fn)), copy.deepcopy(fn)):
        assert type(twin) is models.LogisticMixtureSampleFn and (twin.n_mixtures, twin.n_bins) == (5, 17)
    m = models.PixelCNN(in_channels=3, out_channels=100, n_residual=1, residual_channels=8, head_channels=8,
                        sample_fn=models.logistic_mixture_sample_fn())
    for twin in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert twin._sample_fn.n_mixtures == 10


def test_recipe_signature():
    from pytorch_generative_b200 import recipes

    sig = inspect.signature(recipes.reproduce_pixel_snail_8bit)
    ref = inspect.signature(recipes.reproduce_pixel_snail)
    assert list(sig.parameters) == list(ref.parameters)
    assert {k: p.default for k, p in sig.parameters.items()} == {k: p.default for k, p in ref.parameters.items()}
    assert "not validated" in recipes.reproduce_pixel_snail_8bit.__doc__


def test_new_symbols_are_exported():
    from pytorch_generative_b200 import _build, _lib, losses, models

    assert callable(losses.logistic_mixture_nll)
    for name in ("LogisticMixtureSampleFn", "logistic_mixture_sample_fn"):
        assert name in models.__all__ and hasattr(models, name)
    _build.build(verbose=False)
    lib = _lib.load()
    for sym in ("pg_logistic_mixture_fwd_bwd", "pg_logistic_mixture_sample"):
        assert sym in _lib.EXPORTED_SYMBOLS
        getattr(lib, sym)
    assert callable(_lib.logistic_mixture_nll_kernel) and callable(_lib.logistic_mixture_sample)
