"""Restatement of the reference mixture models (models/mixture_models.py) and kernel density estimators (models/kde.py)
in plain torch, on any device and in any dtype; not a test module.  In fp32 on the CPU it performs the reference's
operations in the reference's order, so it equals tests/golden/density.pt bit for bit; in float64 it is the reference
the kernels are held to.  It broadcasts [N, M, D] as the reference does, so it only runs at test sizes."""

import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import distributions

F64 = torch.float64


def mixture_names(cls):
    return ["mixture_logits", "mean", "log_std"] if cls == "GaussianMixtureModel" else ["mixture_logits", "logits"]


def gmm_component_log_prob(mean, log_std, x):
    """[N, 1, K] of x [N, 1, F] (the reference's broadcast, mixture_models.py:74-79)."""
    z = -log_std - 0.5 * torch.log(torch.tensor(2 * np.pi, dtype=mean.dtype))
    log_prob = z - 0.5 * ((x.unsqueeze(dim=1) - mean) / log_std.exp()) ** 2
    return log_prob.sum(-1)


def bmm_component_log_prob(logits, x):
    """[N, K] of x [N, 1, F]."""
    logits, x = torch.broadcast_tensors(logits, x)
    return -F.binary_cross_entropy_with_logits(logits, x, reduction="none").sum(-1)


def mixture_forward(cls, params, x):
    """The reference's forward of x in any shape [N, ...] (viewed as [N, 1, F]); params by name."""
    x = x.reshape(x.shape[0], 1, -1)
    mixture_log_prob = torch.log_softmax(params["mixture_logits"], dim=-1)
    if cls == "GaussianMixtureModel":
        comp = gmm_component_log_prob(params["mean"], params["log_std"], x)
    else:
        comp = bmm_component_log_prob(params["logits"], x)
    return torch.logsumexp(mixture_log_prob + comp, dim=-1)


def mixture_terms(cls, params, x):
    """float64 a [N, K] (the per-component log-likelihoods with the mixture weights) and the sum over the features of
    |term| [N, K], the scale of a's rounding error."""
    p = {k: v.to(F64) for k, v in params.items()}
    x = x.to(F64).reshape(x.shape[0], 1, -1)
    lsm = torch.log_softmax(p["mixture_logits"], -1)
    if cls == "GaussianMixtureModel":
        terms = (-p["log_std"] - 0.5 * math.log(2 * math.pi)) - 0.5 * ((x - p["mean"]) / p["log_std"].exp()) ** 2
    else:
        lg = p["logits"]
        terms = -(lg.clamp(min=0) - lg * x + torch.log1p(torch.exp(-lg.abs())))
    return lsm + terms.sum(-1), terms.abs().sum(-1)


def mixture_loss_and_grads(cls, params, x, cot, dtype=torch.float32):
    """(out, parameter gradients by name, x's gradient) of sum(forward(x) * cot)."""
    p = {k: v.to(dtype).clone().requires_grad_(True) for k, v in params.items()}
    x = x.to(dtype).clone().requires_grad_(True)
    out = mixture_forward(cls, p, x)
    (out * cot.to(dtype).reshape(out.shape)).sum().backward()
    return out.detach(), {k: v.grad for k, v in p.items()}, x.grad


def mixture_sample(cls, params, n, original_shape):
    """The reference's sample(n): Categorical over the mixture logits, then the component draw."""
    idxs = distributions.Categorical(logits=params["mixture_logits"]).sample((n,))
    if cls == "GaussianMixtureModel":
        s = distributions.Normal(params["mean"][idxs], params["log_std"][idxs].exp()).sample()
    else:
        s = distributions.Bernoulli(logits=params["logits"][idxs]).sample()
    return s.view(n, *original_shape[1:])


def gaussian_kde(test_Xs, train_Xs, bandwidth):
    """The reference's GaussianKernel.forward (kde.py:70-79) in the inputs' dtype."""
    dtype = test_Xs.dtype
    n, d = train_Xs.shape
    n, h = torch.tensor(n, dtype=dtype), torch.tensor(bandwidth, dtype=dtype)
    pi = torch.tensor(np.pi, dtype=dtype)
    Z = 0.5 * d * torch.log(2 * pi) + d * torch.log(h) + torch.log(n)
    diffs = (test_Xs.view(test_Xs.shape[0], 1, -1) - train_Xs.view(1, *train_Xs.shape)) / h.to(test_Xs.device)
    log_exp = -0.5 * torch.norm(diffs, p=2, dim=-1) ** 2
    return torch.logsumexp(log_exp - Z.to(test_Xs.device), dim=-1)


def parzen_inside(test_Xs, train_Xs, bandwidth, strict=False):
    """[N, M] bool: every |x_d - t_d| / h <= 0.5 (`<` when strict, a bug model), divided as the inputs' dtype divides."""
    abs_diffs = torch.abs(test_Xs.view(test_Xs.shape[0], 1, -1) - train_Xs.view(1, *train_Xs.shape))
    q = abs_diffs / bandwidth
    return ((q < 0.5) if strict else (q <= 0.5)).all(-1)


def parzen_kde(test_Xs, train_Xs, bandwidth):
    """The reference's ParzenWindowKernel.forward (kde.py:52-58), including its Python-float coefficient."""
    abs_diffs = torch.abs(test_Xs.view(test_Xs.shape[0], 1, -1) - train_Xs.view(1, *train_Xs.shape))
    dims = tuple(range(len(abs_diffs.shape))[2:])
    dim = np.prod(abs_diffs.shape[2:])
    inside = torch.sum(abs_diffs / bandwidth <= 0.5, dim=dims) == dim
    coef = 1 / bandwidth**dim
    return torch.log((coef * inside).mean(dim=1))


def parzen_log_density(count, M, D, bandwidth):
    """log(count) - log(M) - D log(h) in float64 (the product's formula, which does not overflow)."""
    c = count.to(F64)
    return torch.log(c) - math.log(M) - D * math.log(bandwidth)


def gaussian_kde_f64(test_Xs, train_Xs, bandwidth):
    """float64 (log p [N], the pair values s [N, M] = -0.5 |x_n - t_m|^2 / h^2)."""
    x, t = test_Xs.to(F64), train_Xs.to(F64)
    M, D = t.shape
    sq = ((x[:, None, :] - t[None, :, :]) ** 2).sum(-1)
    s = -0.5 * sq / bandwidth**2
    Z = 0.5 * D * math.log(2 * math.pi) + D * math.log(bandwidth) + math.log(M)
    return torch.logsumexp(s, -1) - Z, s
