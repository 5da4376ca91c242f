"""Gaussian process on the CUDA path — API of reference models/gaussian_process.py (`GaussianProcess`).

Same constructor, attributes (`mean` and `kernel` as submodules when they are modules, the `noise_var` buffer, plain
`train_x` / `train_y` attributes) and results.  The mean and kernel functions run in torch; the posterior's dense
linear algebra runs in fp64 on csrc/pg_gp.cu:
  * `predict` after `fit` factors A = kernel(train_x, train_x) + noise_var I with `pg_gp_potrf` (blocked Cholesky,
    semi-definite pivot rule), solves [V | beta] = L^-1 [kernel(train_x, x) | train_y - mean(train_x)] with one
    `pg_gp_trsm`, and forms [Q | P] = V^T [V | beta] with one `pg_gemm_f64`: mu = mean(x) + P, sig = kernel(x, x) - Q.
    That is 5 ceil(M / 64) - 1 launches for M training points.  The reference solves with LU instead; both give
    A^-1 for a positive-definite A.  Where the training covariance is numerically singular (a repeated point, no
    noise), a dropped pivot conditions that point out: the result is the posterior given the points kept (DESIGN.md §2).
  * The backward recomputes [W | alpha] = L^-T [V | beta] (one more `pg_gp_trsm`) and forms the gradients of the
    reference's expression with `pg_gemm_f64`: dr = W G_P, Z = W G_Q^T + alpha G_P^T, dKts = W G_Q + Z,
    dKtt = -Z W^T (the full-matrix gradient `torch.linalg.solve` gives a symmetric A).
  * `sample` factors sig with `pg_gp_potrf` (no noise, same pivot rule) and returns mu^T + z L^T through
    `pg_gemm_f64`, z = torch.randn(n_samples, N) in fp64 on the device, so `torch.manual_seed` controls it.  A prior that
    is numerically rank-deficient (the reference's TODO) samples without error.
No kernel synchronises with the host: `predict`, its backward and `sample` can be captured in a CUDA graph once the
noise value has been read (the first call).
"""

import torch

from .. import _lib as L
from . import base

F64 = torch.float64


def _device_operands(who, *tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {t.device}")
        if not t.is_floating_point():
            raise RuntimeError(f"{who}: the CUDA path takes floating-point operands; got {t.dtype}")


def _f64(t):
    """A contiguous fp64 copy of t that the kernels may overwrite."""
    return t.detach().to(dtype=F64, memory_format=torch.contiguous_format, copy=True)


class _Posterior(torch.autograd.Function):
    """(P, Q) = (V^T beta, V^T V) with V = L^-1 Kts, beta = L^-1 r, L L^T = Ktt + noise I."""

    @staticmethod
    def forward(ctx, Ktt, Kts, r, noise, dropped):
        out_dtype = torch.promote_types(torch.promote_types(Ktt.dtype, Kts.dtype), r.dtype)
        M, N = Kts.shape
        r2 = r.reshape(M, -1)
        k = r2.shape[1]
        Lf = _f64(Ktt)
        L.gp_potrf(Lf, noise, dropped)
        VB = torch.empty(M, N + k, dtype=F64, device=Kts.device)
        VB[:, :N].copy_(Kts)
        VB[:, N:].copy_(r2)
        L.gp_trsm(Lf, VB)
        QP = torch.empty(N, N + k, dtype=F64, device=Kts.device)
        L.gemm_f64(VB[:, :N], VB, QP, trans_a=True)
        ctx.save_for_backward(Lf, VB)
        ctx.shapes = (M, N, k, r.shape)
        ctx.dtypes = (Ktt.dtype, Kts.dtype, r.dtype)
        P = QP[:, N:].to(out_dtype)
        Q = QP[:, :N].to(out_dtype)
        return (P if r.dim() == 2 else P.reshape(N)), Q

    @staticmethod
    def backward(ctx, gP, gQ):
        Lf, VB = ctx.saved_tensors
        M, N, k, r_shape = ctx.shapes
        dev = VB.device
        WA = VB.clone()
        L.gp_trsm(Lf, WA, transpose=True)
        W, alpha = WA[:, :N], WA[:, N:]
        gP = None if gP is None else _f64(gP.reshape(N, k))
        gQ = None if gQ is None else _f64(gQ)
        dr = torch.zeros(M, k, dtype=F64, device=dev)
        Z = torch.zeros(M, N, dtype=F64, device=dev)
        if gP is not None:
            L.gemm_f64(W, gP, dr)
            L.gemm_f64(alpha, gP, Z, trans_b=True)
        if gQ is not None:
            L.gemm_f64(W, gQ, Z, trans_b=True, beta=0.0 if gP is None else 1.0)
        dKts = Z.clone()
        if gQ is not None:
            L.gemm_f64(W, gQ, dKts, beta=1.0)
        dKtt = None
        if ctx.needs_input_grad[0]:
            dKtt = torch.empty(M, M, dtype=F64, device=dev)
            L.gemm_f64(Z, W, dKtt, trans_b=True, alpha=-1.0)
            dKtt = dKtt.to(ctx.dtypes[0])
        return dKtt, dKts.to(ctx.dtypes[1]), dr.reshape(r_shape).to(ctx.dtypes[2]), None, None


class GaussianProcess(base.GenerativeModel):
    """The Gaussian process model (reference gaussian_process.py:17-91)."""

    def __init__(self, mean, kernel, noise_var=None):
        """mean: prior mean function mu(x); kernel: prior covariance function K(x, x'); noise_var: the variance of the
        observation noise (None: noiseless observations)."""
        super().__init__()
        self.mean = mean
        self.kernel = kernel
        self.register_buffer("noise_var", torch.tensor(noise_var or 0.0))
        self.train_x = None
        self.train_y = None
        self.dropped = None  # device int32 [1]: the pivots dropped by the latest factorisation
        self._noise_seen = None

    def fit(self, x, y):
        """Fits the Gaussian process on the given training data."""
        if self.train_x is None:
            self.train_x, self.train_y = x, y
        else:
            self.train_x = torch.cat([self.train_x, x])
            self.train_y = torch.cat([self.train_y, y])

    def _noise(self):
        """noise_var's stored value as a Python float (exact: fp32 widens to fp64).  Read once per buffer version, so a
        CUDA-graph capture after the first call does not synchronise."""
        key = (self.noise_var.data_ptr(), self.noise_var._version, self.noise_var.dtype)
        if self._noise_seen is None or self._noise_seen[0] != key:
            self._noise_seen = (key, float(self.noise_var))
        return self._noise_seen[1]

    def _counter(self, device):
        if self.dropped is None or self.dropped.device != device:
            self.dropped = torch.zeros(1, dtype=torch.int32, device=device)
        return self.dropped

    @torch.no_grad()
    def sample(self, x, n_samples):
        """n_samples draws [n_samples, N] (fp64) from the posterior at x if `fit()` has been called, else the prior."""
        mu, sig = self.predict(x)
        if mu.dim() == 2 and mu.shape[1] != 1:
            raise ValueError(f"GaussianProcess.sample: needs one output per location; got mu of shape {tuple(mu.shape)}")
        _device_operands("GaussianProcess.sample", mu, sig)
        N = sig.shape[0]
        Ls = _f64(sig)
        L.gp_potrf(Ls, 0.0, self._counter(sig.device))
        z = torch.randn(n_samples, N, dtype=F64, device=sig.device)
        out = mu.detach().reshape(1, N).to(F64).expand(n_samples, N).contiguous()
        return L.gemm_f64(z, Ls, out, trans_b=True, beta=1.0)

    def predict(self, x):
        """(mu, sig): the posterior means and covariances at x if `fit()` has been called, else the prior's."""
        if self.train_x is None:
            return self.mean(x), self.kernel(x, x)
        train_mu, x_mu = self.mean(self.train_x), self.mean(x)
        r = self.train_y - train_mu
        Ktt = self.kernel(self.train_x, self.train_x)
        x_sig, cross_sig = self.kernel(x, x), self.kernel(self.train_x, x)
        _device_operands("GaussianProcess.predict", Ktt, cross_sig, r, x_sig, x_mu)
        if r.dim() not in (1, 2) or r.shape[0] != Ktt.shape[0]:
            raise ValueError(f"GaussianProcess.predict: train_y - mean(train_x) must be [M] or [M, k]; got "
                             f"{tuple(r.shape)} for M = {Ktt.shape[0]}")
        P, Q = _Posterior.apply(Ktt, cross_sig, r, self._noise(), self._counter(Ktt.device))
        return x_mu + P, x_sig - Q
