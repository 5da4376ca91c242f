"""Float64 restatement of the categorical likelihood (losses.categorical_nll, models.categorical_sample_fn) and the
per-element bounds its fp32 kernels are held to.

Layout: logits [N, K * C, *spatial], class k of channel c at logit channel k * C + c, i.e. viewed as [N, K, C, *spatial];
target class of x: rint(clamp(x, 0, 1) * (K - 1)) in fp32.  U = 2^-24, the unit roundoff of fp32."""

import math

import torch

F64 = torch.float64
U = 2.0 ** -24


def target(x, K):
    """Class index of each input value, computed in fp32 as the kernel does."""
    return torch.round(x.float().clamp(0, 1) * float(K - 1)).long()


def classes_view(logits, C):
    """[N, K * C, *spatial] -> [N, K, C, *spatial]."""
    return logits.reshape(logits.shape[0], logits.shape[1] // C, C, *logits.shape[2:])


def parts(logits, x):
    """(m, log s, l_target, t) in float64: the max over k, log of sum exp(l - m), the target logit and the target, each
    [N, C, *spatial]."""
    C = x.shape[1]
    lv = classes_view(logits.to(F64), C)
    t = target(x, lv.shape[1]).to(lv.device)
    m = lv.max(dim=1).values
    log_s = torch.log(torch.exp(lv - m.unsqueeze(1)).sum(dim=1))
    lt = lv.gather(1, t.unsqueeze(1)).squeeze(1)
    return m, log_s, lt, t


def nll(logits, x):
    """Per (image, channel, pixel) negative log-likelihood in nats, float64: logsumexp - logit[target]."""
    m, log_s, lt, _ = parts(logits, x)
    return log_s + (m - lt)


def loss(logits, x):
    """(mean over images of the summed NLL, bits/dim) in float64."""
    per_image = nll(logits, x).reshape(x.shape[0], -1).sum(dim=1)
    value = per_image.mean()
    return value, value / (x[0].numel() * math.log(2.0))


def dlogits(logits, x, grad_scale):
    """(softmax - onehot) * grad_scale in float64, in the logits' layout."""
    C = x.shape[1]
    lv = classes_view(logits.to(F64), C)
    t = target(x, lv.shape[1]).to(lv.device)
    p = torch.softmax(lv, dim=1)
    onehot = torch.zeros_like(p).scatter_(1, t.unsqueeze(1), 1.0)
    return ((p - onehot) * grad_scale).reshape(logits.shape)


def sum_relative_bound(K):
    """Relative error bound of the kernel's fp32 sum s = sum exp(l - m) over k (s >= 1): each expf within 2 ulp plus
    the rounding of its argument (u |l - m| relative, and |l - m| e^(l - m) <= 1/e), one rounding per addition and per
    rescale of the running sum."""
    return (3 * K + 16) * U


def nll_bound(logits, x):
    """Per-element bound of the kernel's NLL: the sum's relative error carried through the log, the log's own 1 ulp, and
    the roundings of m - l_target and of the final addition; doubled for slack."""
    m, log_s, lt, _ = parts(logits, x)
    K = logits.shape[1] // x.shape[1]
    return 2 * (1.01 * sum_relative_bound(K) + 3 * U * log_s.abs() + 2 * U * (m - lt).abs())


def dlogits_bound(logits, x, grad_scale):
    """Per-element bound of the kernel's dlogits: p = expf(l - m) (2 ulp + argument rounding) times 1 / s (the sum's
    relative error + 1 rounding), one rounding each for the product, the onehot subtraction and the scale; doubled."""
    C = x.shape[1]
    lv = classes_view(logits.to(F64), C)
    K = lv.shape[1]
    t = target(x, K).to(lv.device)
    m = lv.max(dim=1, keepdim=True).values
    p = torch.softmax(lv, dim=1)
    onehot = torch.zeros_like(p).scatter_(1, t.unsqueeze(1), 1.0)
    rel = sum_relative_bound(K) + 8 * U + U * (lv - m).abs()
    b = 2 * abs(grad_scale) * (p * rel + 2 * U * (p - onehot).abs()) + 1e-43
    return b.reshape(logits.shape)


def image_sum_bound(logits, x, n_blocks):
    """Bound of the per-image sums: every element's bound plus the fp32 additions of the reduction (a 5-level warp
    butterfly, a 5-level block butterfly, then at most n_blocks sequential additions of the block partials)."""
    b = nll_bound(logits, x).reshape(x.shape[0], -1).sum(dim=1)
    v = nll(logits, x).abs().reshape(x.shape[0], -1).sum(dim=1)
    return b + 1.1 * (12 + n_blocks) * U * v


def cdf(logits, C):
    """[n, K, C] float64 cumulative probabilities over k ascending of logits [n, K * C]."""
    lv = logits.to(F64).reshape(logits.shape[0], -1, C)
    return torch.softmax(lv, dim=1).cumsum(dim=1)


def inverse_cdf(logits, u):
    """First class k with cdf(k) >= u, per (row, channel): logits [n, K * C], u [n, C] -> [n, C] int64."""
    F = cdf(logits, u.shape[1])
    K = F.shape[1]
    return (F < u.to(F64).unsqueeze(1)).sum(dim=1).clamp(max=K - 1)


def near_boundary(logits, u):
    """True where u is within the fp32 bound of a CDF boundary: there the kernel's cumulative sum, its total and the
    product u * s can fall on either side, and its draw may be the neighbouring class."""
    F = cdf(logits, u.shape[1])
    K = F.shape[1]
    eps = 4 * sum_relative_bound(K)
    return ((F - u.to(F64).unsqueeze(1)).abs() <= eps).any(dim=1)


def probabilities(logits, C):
    """[n, K, C] float64 softmax probabilities of logits [n, K * C]."""
    return torch.softmax(logits.to(F64).reshape(logits.shape[0], -1, C), dim=1)
