"""Mixture models on the CUDA path — API of reference models/mixture_models.py (`MixtureModel`, `GaussianMixtureModel`,
`BernoulliMixtureModel`).

Same constructors, parameters (`mixture_logits`, then `mean` / `log_std` or `logits`, created in the reference's order so
that seeded inits are bit-equal), state-dict keys and output shapes.  `__call__` records `_original_shape` and views x as
[N, 1, n_features] as the reference does, so the input is 3-D and no `_c/_h/_w` buffers are registered.

`forward` is one autograd Function over `pg_mixture_fwd` / `pg_mixture_bwd` (csrc/pg_density.cu): the per-(row,
component) log-likelihoods a [N, K] are reduced over the features in fp32 tiles and never broadcast to [N, K, D]; the
backward recomputes the responsibilities exp(a - out) from the saved a and out and sums every parameter gradient in a
fixed order.  Neither direction synchronises with the host, so a training step captures as a CUDA graph.

`sample(n)` makes the reference's own torch calls on the parameters' device (`Categorical`, then `Normal` / `Bernoulli`):
sampling is not a hot path, and seeded samples equal the reference's.
"""

import torch
from torch import distributions, nn

from .. import _lib as L
from . import base
from .nice import _require

F32 = torch.float32


class _Mixture(torch.autograd.Function):
    """log p(x) [N] of x [N, D] under the mixture; p1 is None for the Bernoulli kind."""

    @staticmethod
    def forward(ctx, x, kind, mixture_logits, p0, p1):
        N, D = x.shape
        K = mixture_logits.numel()
        a = torch.empty((N, K), dtype=F32, device=x.device)
        out = torch.empty(N, dtype=F32, device=x.device)
        L.mixture_fwd(kind, x, mixture_logits, p0, p1, a, out)
        ctx.save_for_backward(x, mixture_logits, p0, p1, a, out)
        ctx.kind = kind
        return out

    @staticmethod
    def backward(ctx, g):
        x, mixture_logits, p0, p1, a, out = ctx.saved_tensors
        N, D = x.shape
        K = mixture_logits.numel()
        n_tensors = 1 if p1 is None else 2
        flat = torch.zeros(n_tensors * K * D + K, dtype=F32, device=x.device)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        L.mixture_bwd(ctx.kind, x, mixture_logits, p0, p1, a, out, g.contiguous(), flat, dx)
        dp0 = flat[: K * D].view(K, D)
        dp1 = None if p1 is None else flat[K * D: 2 * K * D].view(K, D)
        return dx, None, flat[n_tensors * K * D:], dp0, dp1


class MixtureModel(base.GenerativeModel):
    """Base of the mixture models (reference mixture_models.py:13-62): log-likelihoods from `forward`, samples from
    `sample`; the component distribution is the subclass's."""

    _KIND = None

    def __init__(self, n_components, n_features):
        super().__init__()
        self.n_components = n_components
        self.n_features = n_features
        self.mixture_logits = nn.Parameter(torch.ones((n_components,)))

    def __call__(self, *args, **kwargs):
        x = args[0]
        self._original_shape = x.shape
        x = x.view(self._original_shape[0], 1, self.n_features)
        return super().__call__(x, *args[1:], **kwargs)

    def _component_params(self):
        raise NotImplementedError

    def forward(self, x):
        """log p(x) of x [N, 1, n_features] (the view `__call__` makes)."""
        p0, p1 = self._component_params()
        params = [self.mixture_logits, p0] + ([] if p1 is None else [p1])
        _require(x, params, type(self).__name__)
        x = x.reshape(x.shape[0], self.n_features).contiguous()
        return _Mixture.apply(x, self._KIND, self.mixture_logits, p0, p1)

    def _component_sample(self, idxs):
        raise NotImplementedError

    @torch.no_grad()
    def sample(self, n_samples):
        shape = (n_samples,)
        idxs = distributions.Categorical(logits=self.mixture_logits).sample(shape)
        sample = self._component_sample(idxs)
        return sample.view(n_samples, *self._original_shape[1:])


class GaussianMixtureModel(MixtureModel):
    """A categorical mixture of Gaussians with diagonal covariance (reference mixture_models.py:65-83).  Its forward
    returns [N, 1], as the reference's broadcast does."""

    _KIND = L.MIXTURE_GAUSSIAN

    def __init__(self, n_components, n_features):
        super().__init__(n_components, n_features)
        self.mean = nn.Parameter(torch.randn(n_components, n_features) * 0.01)
        # std = exp(log_std) = 1 at init
        self.log_std = nn.Parameter(torch.zeros(n_components, n_features))

    def _component_params(self):
        return self.mean, self.log_std

    def forward(self, x):
        return super().forward(x).unsqueeze(1)

    def _component_sample(self, idxs):
        mean, std = self.mean[idxs], self.log_std[idxs].exp()
        return distributions.Normal(mean, std).sample()


class BernoulliMixtureModel(MixtureModel):
    """A categorical mixture of Bernoulli distributions (reference mixture_models.py:86-100); its forward returns [N]."""

    _KIND = L.MIXTURE_BERNOULLI

    def __init__(self, n_components, n_features):
        super().__init__(n_components, n_features)
        self.logits = nn.Parameter(torch.rand(n_components, n_features))

    def _component_params(self):
        return self.logits, None

    def _component_sample(self, idxs):
        return distributions.Bernoulli(logits=self.logits[idxs]).sample()
