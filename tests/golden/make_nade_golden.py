"""Generates tests/golden/nade.pt by running the UNMODIFIED reference NADE (models/autoregressive/nade.py) on the CPU.

    python tests/golden/make_nade_golden.py <path to the reference checkout>

`distributions.Bernoulli` in the reference module is replaced by a class that draws `u < probs` from pre-generated
uniforms, one [n, 1] column per call, so every draw is recorded as a uniform [n, D] per call of the model.  Per
configuration the fixture holds the constructor arguments, the state dict after `torch.manual_seed(seed)` and the
constructor (no noise, for the init check), a state with N(0, 0.05) noise added, and under that state:
  * `binary`: a 0/1 input, p, the recipe loss, every parameter gradient and the input gradient (through the model, the
    target held fixed);
  * `negative`: the same for an input with negative entries (drawn under the recorded uniforms), with x~;
  * `unconditional` / `conditional`: a sample under recorded uniforms (a conditional canvas keeps about half its
    entries).
"""

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "image_192_10": dict(kwargs=dict(input_dim=192, hidden_dim=10), shape=(4, 3, 8, 8)),
    "image_64_32": dict(kwargs=dict(input_dim=64, hidden_dim=32), shape=(4, 1, 8, 8)),
    "vector_37_1": dict(kwargs=dict(input_dim=37, hidden_dim=1), shape=(5, 37)),
}


class _UniformBernoulli:
    """Stand-in for torch.distributions.Bernoulli(probs=p).sample(): u < p with u the next [n, 1] column of `columns`."""

    columns = None

    def __init__(self, probs=None, logits=None):
        self.probs = probs

    def sample(self):
        return (next(_UniformBernoulli.columns) < self.probs).to(self.probs.dtype)


def _draw_with(uniforms):
    _UniformBernoulli.columns = iter(uniforms.t().unsqueeze(-1))  # [D, n, 1]: one column per dimension


def loss_fn(x, preds):
    b = x.shape[0]
    loss = torch.nn.functional.binary_cross_entropy_with_logits(preds.view(b, -1), x.view(b, -1), reduction="none")
    return loss.sum(dim=1).mean()


def run(nade_mod, cfg, seed):
    torch.manual_seed(seed)
    model = nade_mod.NADE(**cfg["kwargs"])
    out = dict(kwargs=cfg["kwargs"], state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    n, D = cfg["shape"][0], cfg["kwargs"]["input_dim"]
    binary = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g)
    negative = torch.where(torch.rand(cfg["shape"], generator=g) < 0.3, -torch.ones(cfg["shape"]), binary)
    for kind, x in (("binary", binary), ("negative", negative)):
        uniforms = torch.rand(n, D, generator=g)
        _draw_with(uniforms)
        x = x.clone().requires_grad_(True)
        model.zero_grad()
        p = model(x)
        loss = loss_fn(x.detach(), p)
        loss.backward()
        _draw_with(uniforms)
        with torch.no_grad():
            xt = model._forward(x.detach().view(n, -1))[1]
        out[kind] = dict(x=x.detach().clone(), uniforms=uniforms, p=p.detach().clone(), loss=loss.detach().clone(),
                         x_grad=x.grad.clone(), xt=xt.clone(),
                         grads={k: prm.grad.clone() for k, prm in model.named_parameters()})
    for kind in ("unconditional", "conditional"):
        uniforms = torch.rand(n, D, generator=g)
        cond = None
        if kind == "conditional" or len(cfg["shape"]) != 4:  # a vector model has no image shape to sample from
            given = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g)
            keep = torch.rand(cfg["shape"], generator=g) < (0.5 if kind == "conditional" else 0.0)
            cond = torch.where(keep, given, torch.full_like(given, -1.0))
        _draw_with(uniforms)
        sample = model.sample(None if cond is not None else n, cond)
        out[kind] = dict(uniforms=uniforms, conditioned_on=cond, sample=sample.clone())
    out["state_after"] = {k: v.clone() for k, v in model.state_dict().items()}  # with the _c/_h/_w of an image forward
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.autoregressive import nade as nade_mod

    nade_mod.distributions.Bernoulli = _UniformBernoulli
    fixture = {name: run(nade_mod, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    torch.save(fixture, os.path.join(HERE, "nade.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
