"""Generates tests/golden/gp.pt by running the UNMODIFIED reference GaussianProcess (models/gaussian_process.py) on the
CPU.

    python tests/golden/make_gp_golden.py <path to the reference checkout>

The mean and kernel are defined here: a constant mean with one Parameter `c`, and s^2 exp(-0.5 |a - b|^2 / l^2) from
direct differences with Parameters `s` and `ell`.  Cases:
  * `notebook`: D = 1, fp64, five noisy observations of a smooth function fitted one at a time, noise_var 0.01 (the
    fp32 buffer), predictions on 100 points of [0, 6] after each fit;
  * `d3`: D = 3, M = 200, N = 150, fp64, noise_var 1e-3;
  * `fp32`: D = 2, M = 64, N = 48, fp32 operands, noise_var 1e-2;
  * `multi`: D = 2, M = 40, N = 30, fp64, y of shape [40, 3], noise_var 1e-2.
Each case records (mu, sig) and the gradients of sum(mu c1) + sum(sig c2), fixed cotangents c1, c2, with respect to x,
train_x, train_y and the parameters c, s, ell.
"""

import os
import sys

import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))


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
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(mu.shape, generator=g, dtype=mu.dtype), torch.randn(sig.shape, generator=g, dtype=sig.dtype))


def run(GP, params, noise, fits, x, seed):
    mean, kernel = ConstMean(params["c"]), SqExp(params["s"], params["ell"])
    gp = GP(mean, kernel, noise)
    xs = x.clone().requires_grad_(True)
    steps = []
    for tx, ty in fits:
        gp.fit(tx.clone().requires_grad_(True), ty.clone().requires_grad_(True))
        with torch.no_grad():
            mu, sig = gp.predict(x)
        steps.append((mu.clone(), sig.clone()))
    # one leaf for all training points, so the gradients land on [M, D] / [M, k] tensors
    train_x = torch.cat([f[0] for f in fits]).clone().requires_grad_(True)
    train_y = torch.cat([f[1] for f in fits]).clone().requires_grad_(True)
    gp.train_x, gp.train_y = train_x, train_y
    mu, sig = gp.predict(xs)
    c1, c2 = cotangents(seed, mu, sig)
    assert torch.equal(mu.detach(), steps[-1][0]) and torch.equal(sig.detach(), steps[-1][1])
    ((mu * c1).sum() + (sig * c2).sum()).backward()
    # c1, c2 are not stored: cotangents(seed, mu, sig) rebuilds them; the last step is the final (mu, sig)
    return dict(params=params, noise=noise, fits=fits, x=x, seed=seed, steps=steps, grads=dict(x=xs.grad, train_x=train_x.grad, train_y=train_y.grad, c=mean.c.grad, s=kernel.s.grad,
                           ell=kernel.ell.grad))


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.gaussian_process import GaussianProcess as GP

    g = torch.Generator().manual_seed(0)
    f64 = torch.float64
    fn = lambda t: torch.sin(2 * t) + 0.3 * t
    grid = torch.linspace(0, 6, 100, dtype=f64)[:, None]
    nb_x = torch.rand(5, 1, 1, generator=g, dtype=f64) * 6
    fits = [(t, fn(t) + 0.1 * torch.randn(t.shape, generator=g, dtype=f64)) for t in nb_x]
    cases = dict(notebook=run(GP, dict(c=0.2, s=1.3, ell=0.7), 0.1 ** 2, fits, grid, 1))
    tx = torch.rand(200, 3, generator=g, dtype=f64) * 3
    ty = fn(tx).sum(1, keepdim=True) + 0.03 * torch.randn(200, 1, generator=g, dtype=f64)
    cases["d3"] = run(GP, dict(c=-0.1, s=1.1, ell=0.9), 1e-3, [(tx, ty)], torch.rand(150, 3, generator=g, dtype=f64) * 3,
                      2)
    tx = torch.rand(64, 2, generator=g) * 2
    ty = fn(tx).sum(1, keepdim=True) + 0.1 * torch.randn(64, 1, generator=g)
    cases["fp32"] = run(GP, dict(c=0.3, s=0.8, ell=0.6), 1e-2, [(tx, ty)], torch.rand(48, 2, generator=g) * 2, 3)
    tx = torch.rand(40, 2, generator=g, dtype=f64) * 2
    ty = torch.cat([fn(tx).sum(1, keepdim=True), torch.cos(tx[:, :1]), tx[:, 1:] ** 2], 1)
    cases["multi"] = run(GP, dict(c=0.0, s=1.0, ell=0.5), 1e-2, [(tx, ty)], torch.rand(30, 2, generator=g, dtype=f64) * 2,
                         4)
    torch.save(cases, os.path.join(HERE, "gp.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
