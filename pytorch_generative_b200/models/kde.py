"""Kernel density estimation on the CUDA path — API of reference models/kde.py (`Kernel`, `ParzenWindowKernel`,
`GaussianKernel`, `KernelDensityEstimator`).

Same constructors and attributes (`bandwidth`, `kernel`, and `train_Xs` as a plain attribute, not a buffer), the same
results and the same sampling calls.  The reference broadcasts every query against every training point, an
[N, M, D] tensor (188 GB for 1000 MNIST test images against the 60000 training images); here the kernels of
csrc/pg_density.cu stream 64 x 64 tiles of pairs through shared memory and keep only [N]-sized state:
  * GaussianKernel: `pg_kde_gauss_fwd` gives logsumexp_m(-0.5 |x - t_m|^2 / h^2) from direct differences, minus the
    normaliser Z = 0.5 d log(2 pi) + d log h + log n, computed on the host with the reference's fp32 scalar ops.  The
    output has a gradient with respect to the queries (`pg_kde_gauss_bwd`); a training set that requires grad is refused.
  * ParzenWindowKernel: `pg_kde_parzen_count` counts, per query, the training points whose every |x_d - t_d| / h <= 0.5 in
    IEEE fp32 division, and returns log(count) - log(M) - D log(h) computed in fp64.  The reference forms
    coef = 1 / h**D as a Python float, which is 0, inf or a ZeroDivisionError at MNIST's D for common bandwidths; the log
    of the same density does not overflow (DESIGN.md §2).  As in the reference, the output has no grad_fn.
"""

import abc

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from . import base

F32 = torch.float32


def _operands(test_Xs, train_Xs, who):
    """Contiguous fp32 [N, D] queries and [M, D] training points on one CUDA device; no CPU fallback."""
    for t in (test_Xs, train_Xs):
        if not t.is_cuda:
            raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {t.device}")
        if t.dtype != F32:
            raise RuntimeError(f"{who}: the CUDA path takes fp32 inputs; got {t.dtype}")
    if train_Xs.dim() != 2:
        raise ValueError(f"{who}: the training data must be [M, D]; got {tuple(train_Xs.shape)}")
    if test_Xs.dim() != 2 or test_Xs.shape[1] != train_Xs.shape[1]:
        raise ValueError(f"{who}: queries must be [N, {train_Xs.shape[1]}]; got {tuple(test_Xs.shape)}")
    return test_Xs.contiguous(), train_Xs.contiguous()


def gaussian_log_normaliser(n, d, bandwidth):
    """Z = 0.5 d log(2 pi) + d log(h) + log(n) with the reference's fp32 tensor ops (kde.py:71-75), as a float."""
    n, h = torch.tensor(n, dtype=torch.float32), torch.tensor(bandwidth)
    pi = torch.tensor(np.pi)
    return float(0.5 * d * torch.log(2 * pi) + d * torch.log(h) + torch.log(n))


class _GaussianKDE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, t, bandwidth):
        N, D = x.shape
        M = t.shape[0]
        out = torch.empty(N, dtype=F32, device=x.device)
        lse = torch.empty(N, dtype=F32, device=x.device)
        L.kde_gauss_fwd(x, t, bandwidth, gaussian_log_normaliser(M, D, bandwidth), out, lse)
        ctx.save_for_backward(x, t, lse)
        ctx.bandwidth = bandwidth
        return out

    @staticmethod
    def backward(ctx, g):
        x, t, lse = ctx.saved_tensors
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.zeros_like(x)
            L.kde_gauss_bwd(x, t, ctx.bandwidth, lse, g.contiguous(), dx)
        return dx, None, None


class Kernel(abc.ABC, nn.Module):
    """Base class of the kernels (reference kde.py:22-46)."""

    def __init__(self, bandwidth=1.0):
        super().__init__()
        self.bandwidth = bandwidth

    @abc.abstractmethod
    def forward(self, test_Xs, train_Xs):
        """log p(x) [N] of each query given the training points."""

    @abc.abstractmethod
    def sample(self, train_Xs):
        """One draw from the kernel placed on each row of train_Xs."""


class ParzenWindowKernel(Kernel):
    """The Parzen window (box) kernel of width h (reference kde.py:49-64)."""

    def forward(self, test_Xs, train_Xs):
        x, t = _operands(test_Xs, train_Xs, "ParzenWindowKernel")
        out = torch.empty(x.shape[0], dtype=F32, device=x.device)
        L.kde_parzen_count(x, t, self.bandwidth, out=out)
        return out

    @torch.no_grad()
    def sample(self, train_Xs):
        noise = (torch.rand(train_Xs.shape, device=train_Xs.device) - 0.5) * self.bandwidth
        return train_Xs + noise


class GaussianKernel(Kernel):
    """The Gaussian kernel of standard deviation h (reference kde.py:67-85)."""

    def forward(self, test_Xs, train_Xs):
        if torch.is_grad_enabled() and train_Xs.requires_grad:
            raise NotImplementedError("GaussianKernel: the CUDA path has no gradient with respect to the training data "
                                      "(only the queries'); detach train_Xs")
        x, t = _operands(test_Xs, train_Xs, "GaussianKernel")
        return _GaussianKDE.apply(x, t, self.bandwidth)

    @torch.no_grad()
    def sample(self, train_Xs):
        noise = torch.randn(train_Xs.shape, device=train_Xs.device) * self.bandwidth
        return train_Xs + noise


class KernelDensityEstimator(base.GenerativeModel):
    """p(x) = 1 / |D| sum over the training points of K(x, x_i) (reference kde.py:88-115)."""

    def __init__(self, train_Xs, kernel=None):
        super().__init__()
        self.kernel = kernel or GaussianKernel()
        self.train_Xs = train_Xs
        assert len(self.train_Xs.shape) == 2, "Input cannot have more than two axes."

    @property
    def device(self):
        return self.train_Xs.device

    def forward(self, x):
        return self.kernel(x, self.train_Xs)

    @torch.no_grad()
    def sample(self, n_samples):
        idxs = np.random.choice(range(len(self.train_Xs)), size=n_samples)
        return self.kernel.sample(self.train_Xs[idxs])
