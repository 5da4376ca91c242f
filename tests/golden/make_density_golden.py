"""Generates tests/golden/density.pt by running the UNMODIFIED reference mixture models (models/mixture_models.py) and
kernel density estimators (models/kde.py) on the CPU.

    python tests/golden/make_density_golden.py <path to the reference checkout>

Mixture models (`mixture`): GaussianMixtureModel and BernoulliMixtureModel at the reference test's K = 3 on 3x8x8 images
and at K = 13 on 3x5x7 images (105 features, odd).  Per case: the constructor arguments, the state dict right after
`torch.manual_seed(seed)` and the constructor (the init check), a state with noise added to every parameter, and under
it the input batch x (4-D), the forward, every parameter gradient and x's gradient of sum(out * cot) with a fixed
cotangent `cot`, and `sample(n)` right after `torch.manual_seed(sample_seed)`.

Kernel density estimators (`kde`), each with the queries' gradient under a fixed cotangent for the Gaussian kernel:
  * `gauss_2d` / `parzen_2d`: [100, 2] standard-normal training data, queries on a 0.5-spaced mesh over [-8, 8)^2;
  * `gauss_37` / `parzen_37`: [64, 37] training data, 40 queries: perturbed training points and fresh draws;
  * `parzen_boundary`: h = 0.1, queries whose first feature lies at |x - t| / h == 0.5 in fp32 (and the neighbours one
    ulp either side), on training points with varied offsets.
"""

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

MIXTURES = {
    "gmm_3": dict(cls="GaussianMixtureModel", kwargs=dict(n_components=3, n_features=3 * 8 * 8), shape=(6, 3, 8, 8)),
    "bmm_3": dict(cls="BernoulliMixtureModel", kwargs=dict(n_components=3, n_features=3 * 8 * 8), shape=(6, 3, 8, 8)),
    "gmm_13": dict(cls="GaussianMixtureModel", kwargs=dict(n_components=13, n_features=105), shape=(9, 3, 5, 7)),
    "bmm_13": dict(cls="BernoulliMixtureModel", kwargs=dict(n_components=13, n_features=105), shape=(9, 3, 5, 7)),
}


def run_mixture(models, cfg, seed):
    torch.manual_seed(seed)
    model = getattr(models, cfg["cls"])(**cfg["kwargs"])
    out = dict(cls=cfg["cls"], kwargs=cfg["kwargs"], seed=seed,
               state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.5)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    if cfg["cls"] == "GaussianMixtureModel":
        x = torch.randn(cfg["shape"], generator=g)
    else:
        x = (torch.rand(cfg["shape"], generator=g) < 0.4).float()
    out["x"] = x.clone()
    x = x.clone().requires_grad_(True)
    y = model(x)
    cot = torch.randn(y.shape, generator=g)
    (y * cot).sum().backward()
    out.update(out=y.detach().clone(), cot=cot, x_grad=x.grad.clone(),
               grads={k: p.grad.clone() for k, p in model.named_parameters()})
    out["sample_seed"] = seed + 2
    torch.manual_seed(seed + 2)
    out["sample"] = model.sample(5).clone()
    return out


def run_kde(models, train, queries, kernel, bandwidth, seed):
    model = models.KernelDensityEstimator(train, getattr(models, kernel)(bandwidth=bandwidth))
    x = queries.clone().requires_grad_(kernel == "GaussianKernel")
    y = model(x)
    out = dict(kernel=kernel, bandwidth=bandwidth, train=train.clone(), x=queries.clone(), out=y.detach().clone())
    if kernel == "GaussianKernel":
        cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed))
        (y * cot).sum().backward()
        out.update(cot=cot, x_grad=x.grad.clone())
    return out


def boundary_case():
    """Queries at |x - t| / h == 0.5 in fp32 and one ulp either side, h = 0.1, D = 2."""
    h = 0.1
    hf = np.float32(h)
    train = np.array([[0.0, 0.0], [1.0, -0.5], [-3.25, 2.0], [0.3, 0.7]], dtype=np.float32)
    rows = []
    for t in train:
        # the fp32 values a with fl(a / h) == 0.5, and the neighbours of the extreme ones
        a = np.float32(0.05)
        while np.float32(np.float32(a) / hf) >= np.float32(0.5):
            a = np.nextafter(a, np.float32(0), dtype=np.float32)
        a = np.nextafter(a, np.float32(1), dtype=np.float32)  # the smallest a with quotient >= 0.5
        cands = [np.nextafter(a, np.float32(0), dtype=np.float32)]
        while np.float32(a / hf) == np.float32(0.5):
            cands.append(a)
            a = np.nextafter(a, np.float32(1), dtype=np.float32)
        cands.append(a)
        for c in cands:
            for sign in (1, -1):
                x0 = np.float32(t[0] + np.float32(sign) * c)
                rows.append([x0, t[1]])
    return torch.tensor(train), torch.tensor(np.array(rows, dtype=np.float32)), h


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative import models

    mixture = {name: run_mixture(models, cfg, 10 * i) for i, (name, cfg) in enumerate(MIXTURES.items())}
    g = torch.Generator().manual_seed(100)
    train_2d = torch.normal(torch.zeros((100, 2)), torch.ones((100, 2)), generator=g)
    axis = torch.arange(-8, 8, 0.5)
    xx, yy = torch.meshgrid(axis, axis, indexing="ij")
    mesh = torch.stack((xx, yy), axis=2).view(-1, 2)
    train_37 = torch.rand((64, 37), generator=g)
    queries_37 = torch.cat([train_37[:30] + (torch.rand((30, 37), generator=g) - 0.5) * 0.45,
                            torch.rand((10, 37), generator=g)])
    b_train, b_x, b_h = boundary_case()
    kde = {
        "gauss_2d": run_kde(models, train_2d, mesh, "GaussianKernel", 1.0, 201),
        "parzen_2d": run_kde(models, train_2d, mesh, "ParzenWindowKernel", 1.0, 202),
        "gauss_37": run_kde(models, train_37, queries_37, "GaussianKernel", 0.3, 203),
        "parzen_37": run_kde(models, train_37, queries_37, "ParzenWindowKernel", 0.5, 204),
        "parzen_boundary": run_kde(models, b_train, b_x, "ParzenWindowKernel", b_h, 205),
    }
    torch.save(dict(mixture=mixture, kde=kde), os.path.join(HERE, "density.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
