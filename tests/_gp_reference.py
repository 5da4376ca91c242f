"""Float restatements for GaussianProcess (reference models/gaussian_process.py), CPU only.

  * `ConstMean` / `SqExp`: the mean and kernel the tests and tests/golden/make_gp_golden.py use (a constant mean with one
    Parameter; s^2 exp(-0.5 |a - b|^2 / l^2) from direct differences, Parameters s and l).
  * `reference_predict`: the reference's posterior, op for op (noise_var * eye, torch.linalg.solve, the transposed
    solve times the residual); reproduces tests/golden/gp.pt bit for bit on the CPU.
  * `psd_cholesky`: an unblocked float64 Cholesky with the kernels' semi-definite rule (a finite pivot d <= tau,
    tau = n 2^-52 max_i A_ii after the noise, is dropped: its column of L is 0), and `cholesky_predict`, the posterior
    through it, which conditions dropped points out.
"""

import torch
from torch import nn


class ConstMean(nn.Module):
    def __init__(self, c=0.0):
        super().__init__()
        self.c = nn.Parameter(torch.tensor(float(c)))

    def forward(self, x):
        return torch.ones(x.shape[0], 1, dtype=x.dtype, device=x.device) * self.c


class SqExp(nn.Module):
    def __init__(self, s=1.0, ell=1.0):
        super().__init__()
        self.s = nn.Parameter(torch.tensor(float(s)))
        self.ell = nn.Parameter(torch.tensor(float(ell)))

    def forward(self, a, b):
        d = a[:, None, :] - b[None, :, :]
        return self.s ** 2 * torch.exp(-0.5 * (d * d).sum(-1) / self.ell ** 2)


def cotangents(seed, mu, sig):
    """The fixture's cotangents c1, c2 (tests/golden/make_gp_golden.py)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(mu.shape, generator=g, dtype=mu.dtype), torch.randn(sig.shape, generator=g, dtype=sig.dtype))


def reference_predict(mean, kernel, noise_var, train_x, train_y, x):
    """The reference's predict after fit (gaussian_process.py:79-91)."""
    train_mu, x_mu = mean(train_x), mean(x)
    train_sig = kernel(train_x, train_x) + noise_var * torch.eye(train_x.shape[0])
    x_sig, cross_sig = kernel(x, x), kernel(train_x, x)
    solved = torch.linalg.solve(train_sig, cross_sig).T
    mu = x_mu + solved @ (train_y - train_mu)
    sig = x_sig - (solved @ cross_sig)
    return mu, sig


def psd_cholesky(A, noise=0.0):
    """(L, dropped) of A + noise I in float64 with the semi-definite pivot rule."""
    A = A.detach().to(torch.float64).clone()
    n = A.shape[0]
    A.diagonal().add_(noise)
    tau = n * 2.0 ** -52 * float(A.diagonal().max()) if n else 0.0
    L = torch.zeros_like(A)
    dropped = 0
    for k in range(n):
        d = float(A[k, k])
        if torch.isfinite(torch.tensor(d)) and d <= tau:
            dropped += 1
            continue
        piv = d ** 0.5 if d >= 0 else float("nan")
        L[k, k] = piv
        L[k + 1:, k] = A[k + 1:, k] / piv
        A[k + 1:, k + 1:] -= torch.outer(L[k + 1:, k], L[k + 1:, k])
    return L, dropped


def tri_solve(L, B, transpose=False):
    """L X = B or L^T X = B in float64 by substitution; a zero diagonal entry gives a zero row."""
    L, X = L.to(torch.float64), B.to(torch.float64).clone()
    n = L.shape[0]
    order = range(n - 1, -1, -1) if transpose else range(n)
    for r in order:
        d = L[r, r]
        X[r] = 0.0 if d == 0 else X[r] / d
        if transpose:
            X[:r] -= torch.outer(L[r, :r], X[r])
        else:
            X[r + 1:] -= torch.outer(L[r + 1:, r], X[r])
    return X


def cholesky_predict(Ktt, Kts, Kss, r, x_mu, noise):
    """(mu, sig) in float64 through psd_cholesky: the posterior given the points whose pivots were kept."""
    L, _ = psd_cholesky(Ktt, noise)
    V = tri_solve(L, Kts.to(torch.float64))
    beta = tri_solve(L, r.to(torch.float64).reshape(Ktt.shape[0], -1))
    P = V.T @ beta
    return x_mu.to(torch.float64) + (P if r.dim() == 2 else P.reshape(-1)), Kss.to(torch.float64) - V.T @ V


def replay(case, predict, device="cpu", dtype=None):
    """Runs a fixture case through predict(mean, kernel, noise_var, train_x, train_y, x) -> (mu, sig): the prediction
    after each fit, then the gradients of sum(mu c1) + sum(sig c2).  Returns (steps, mu, sig, grads) with the
    leaves named as in the fixture."""
    p = case["params"]
    mean, kernel = ConstMean(p["c"]).to(device), SqExp(p["s"], p["ell"]).to(device)
    noise_var = torch.tensor(case["noise"] or 0.0)
    cast = lambda t: t.to(device=device, dtype=dtype or t.dtype)
    steps, tx, ty = [], [], []
    x = cast(case["x"])
    for fx, fy in case["fits"]:
        tx.append(cast(fx))
        ty.append(cast(fy))
        with torch.no_grad():
            steps.append(predict(mean, kernel, noise_var, torch.cat(tx), torch.cat(ty), x))
    train_x = torch.cat(tx).requires_grad_(True)
    train_y = torch.cat(ty).requires_grad_(True)
    xs = x.clone().requires_grad_(True)
    mu, sig = predict(mean, kernel, noise_var, train_x, train_y, xs)
    c1, c2 = cotangents(case["seed"], mu.detach().cpu(), sig.detach().cpu())
    ((mu * c1.to(mu.device)).sum() + (sig * c2.to(sig.device)).sum()).backward()
    grads = dict(x=xs.grad, train_x=train_x.grad, train_y=train_y.grad, c=mean.c.grad, s=kernel.s.grad,
                 ell=kernel.ell.grad)
    return steps, mu.detach(), sig.detach(), grads


def model_predict(mean, kernel, noise_var, train_x, train_y, x):
    """The same prediction through pytorch_generative_b200's GaussianProcess."""
    from pytorch_generative_b200.models import GaussianProcess

    gp = GaussianProcess(mean, kernel, float(noise_var) or None)
    gp.fit(train_x, train_y)
    return gp.predict(x)
