"""Generates tests/golden/nice.pt by running the UNMODIFIED reference NICE (models/flow/nice.py) on the CPU.

    python tests/golden/make_nice_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments, the state dict after `torch.manual_seed(seed)` and the
constructor (for the init check), a state with N(0, 0.05) noise added to every parameter (so the scaling is not the
identity), and under that state:
  * `x`: a dequantised image batch, (255 u + U[0, 1)) / 256 with u an 8-bit image scaled to [0, 1];
  * `z`, `log_det_J` of the forward, the recipe loss dict (the reference's `loss_fn`, nice.py:205-213), every parameter
    gradient of the loss and the input gradient;
  * `inverse`: `_inverse(z)`;
  * `sample`: `sample(n, temp=0.7)` right after `torch.manual_seed(sample_seed)`.
The configurations are NICE(64, 4 blocks, 2 hidden layers, 32 units) on 1x8x8 images and NICE(30, 3, 1, 20) on 3x2x5
images, whose halves (15) and hidden layers (20) are not multiples of 8.
"""

import os
import sys

import torch
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "nice_64": dict(kwargs=dict(n_features=64, n_coupling_blocks=4, n_hidden_layers=2, n_hidden_features=32),
                    shape=(4, 1, 8, 8)),
    "nice_30": dict(kwargs=dict(n_features=30, n_coupling_blocks=3, n_hidden_layers=1, n_hidden_features=20),
                    shape=(4, 3, 2, 5)),
}


def loss_fn(preds):
    preds, log_det_J = preds
    log_prob = -(F.softplus(preds) + F.softplus(-preds)).sum(dim=(1, 2, 3))
    loss = log_prob + log_det_J
    return {"loss": -loss.mean(), "prior_log_likelihood": log_prob.mean(), "log_det_J": log_det_J.mean()}


def run(nice_mod, cfg, seed):
    torch.manual_seed(seed)
    model = nice_mod.NICE(**cfg["kwargs"])
    out = dict(kwargs=cfg["kwargs"], seed=seed, state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    images = torch.randint(0, 256, cfg["shape"], generator=g).float() / 255
    x = (images * 255 + torch.rand(cfg["shape"], generator=g)) / 256
    out["x"] = x.clone()
    x = x.clone().requires_grad_(True)
    z, log_det_J = model(x)
    losses = loss_fn((z, log_det_J))
    losses["loss"].backward()
    out.update(z=z.detach().clone(), log_det_J=log_det_J.detach().clone(),
               losses={k: v.detach().clone() for k, v in losses.items()}, x_grad=x.grad.clone(),
               grads={k: prm.grad.clone() for k, prm in model.named_parameters()})
    with torch.no_grad():
        out["inverse"] = model._inverse(z.detach()).clone()
    out["sample_seed"] = seed + 2
    torch.manual_seed(seed + 2)
    out["sample"] = model.sample(cfg["shape"][0], temp=0.7).detach().clone()
    out["state_after"] = {k: v.clone() for k, v in model.state_dict().items()}  # with the _c/_h/_w of an image forward
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.flow import nice as nice_mod

    fixture = {name: run(nice_mod, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    torch.save(fixture, os.path.join(HERE, "nice.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
