"""Generates tests/golden/fvbn.pt by running the UNMODIFIED reference FullyVisibleBeliefNetwork
(models/autoregressive/fvbn.py) on the CPU.

    python tests/golden/make_fvbn_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments, the state dict after `torch.manual_seed(seed)` and the
constructor (no noise, for the init check), a state with N(0, 0.05) noise added, and under that state:
  * `binary` / `negative`: an input (0/1, or 0/1 with about 30% of the entries -1), the logits, the recipe loss, every
    parameter gradient and the input gradient (through the model, the target held fixed; None at n_dims 1, where the
    input feeds no row);
  * `unconditional` / `conditional`: a sample drawn through a `sample_fn` that compares recorded uniforms with
    sigmoid(logits), one [n, c] tensor per pixel in raster order (a conditional canvas keeps about half its entries).
The configurations are 1x8x8 (n_dims 64), 3x4x4 (n_dims 48: a pixel's later channels enter the forward as -1 while it
is drawn) and 1x1x1 (n_dims 1: row 0 alone).
"""

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "image_1x8x8": dict(kwargs=dict(n_dims=64), shape=(4, 1, 8, 8)),
    "image_3x4x4": dict(kwargs=dict(n_dims=48), shape=(4, 3, 4, 4)),
    "image_1x1x1": dict(kwargs=dict(n_dims=1), shape=(5, 1, 1, 1)),
}


def loss_fn(x, preds):
    b = x.shape[0]
    loss = torch.nn.functional.binary_cross_entropy_with_logits(preds.view(b, -1), x.view(b, -1), reduction="none")
    return loss.sum(dim=1).mean()


def uniform_sample_fn(uniforms):
    it = iter(uniforms)
    return lambda logits: (next(it) < torch.sigmoid(logits)).float()


def run(fvbn_mod, cfg, seed):
    torch.manual_seed(seed)
    model = fvbn_mod.FullyVisibleBeliefNetwork(**cfg["kwargs"])
    out = dict(kwargs=cfg["kwargs"], state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    n, c, h, w = cfg["shape"]
    binary = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g)
    negative = torch.where(torch.rand(cfg["shape"], generator=g) < 0.3, -torch.ones(cfg["shape"]), binary)
    for kind, x in (("binary", binary), ("negative", negative)):
        x = x.clone().requires_grad_(True)
        model.zero_grad()
        logits = model(x)
        loss = loss_fn(x.detach(), logits)
        loss.backward()
        out[kind] = dict(x=x.detach().clone(), logits=logits.detach().clone(), loss=loss.detach().clone(),
                         x_grad=None if x.grad is None else x.grad.clone(),
                         grads={k: prm.grad.clone() for k, prm in model.named_parameters()})
    for kind in ("unconditional", "conditional"):
        uniforms = torch.rand(h * w, n, c, generator=g)
        model._sample_fn = uniform_sample_fn(uniforms)
        cond = None
        if kind == "conditional":
            given = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g)
            keep = torch.rand(cfg["shape"], generator=g) < 0.5
            cond = torch.where(keep, given, torch.full_like(given, -1.0))
        sample = model.sample(None if cond is not None else n, cond)
        out[kind] = dict(uniforms=uniforms, conditioned_on=cond, sample=sample.clone())
    out["state_after"] = {k: v.clone() for k, v in model.state_dict().items()}  # with the _c/_h/_w of an image forward
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.autoregressive import fvbn as fvbn_mod

    fixture = {name: run(fvbn_mod, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    torch.save(fixture, os.path.join(HERE, "fvbn.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
