"""Generates tests/golden/made.pt by running the UNMODIFIED reference MADE (models/autoregressive/made.py).

    python tests/golden/make_made_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments, the initial state dict (default init under manual_seed
plus N(0, 0.05) noise), the connectivity vectors of every mask set the run uses (recorded from the reference's own
RandomState calls), and for each forward in sequence: the input, the `mask` buffers after it, the logits, the recipe
loss, every parameter gradient and the input gradient (through the model, the target held fixed).  Then the state after
those forwards (masked weights) and an unconditional and a conditional sample drawn with pre-generated uniforms, one [n]
tensor per dimension in sampling order.
"""

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "one_hidden": dict(kwargs=dict(input_dim=192, hidden_dims=[10]), shape=(4, 3, 8, 8), n_forwards=1),
    "two_hidden_three_masks": dict(kwargs=dict(input_dim=64, hidden_dims=[32, 48], n_masks=3), shape=(4, 1, 8, 8),
                                   n_forwards=4),
    "no_hidden": dict(kwargs=dict(input_dim=64), shape=(4, 1, 8, 8), n_forwards=1),
}


class _RecordingRandomState(np.random.RandomState):
    """RandomState that records what `permutation` and `randint` return, keyed by its seed."""

    log = {}

    def __init__(self, seed=None):
        super().__init__(seed)
        self._vectors = _RecordingRandomState.log.setdefault(int(seed), [])
        self._vectors.clear()

    def permutation(self, *a, **k):
        out = super().permutation(*a, **k)
        self._vectors.append(out.copy())
        return out

    def randint(self, *a, **k):
        out = super().randint(*a, **k)
        self._vectors.append(out.copy())
        return out


def loss_fn(x, preds):
    b = x.shape[0]
    loss = torch.nn.functional.binary_cross_entropy_with_logits(preds.view(b, -1), x.view(b, -1), reduction="none")
    return loss.sum(dim=1).mean()


def uniform_sample_fn(uniforms):
    it = iter(uniforms)
    return lambda logits: (next(it) < torch.sigmoid(logits)).float()


def run(made_mod, cfg, seed):
    torch.manual_seed(seed)
    model = made_mod.MADE(**cfg["kwargs"])
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out = dict(kwargs=cfg["kwargs"], state_before={k: v.clone() for k, v in model.state_dict().items()}, forwards=[])
    _RecordingRandomState.log.clear()
    for f in range(cfg["n_forwards"]):
        x = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g).requires_grad_(True)
        model.zero_grad()
        logits = model(x)
        loss = loss_fn(x.detach(), logits)  # x_grad: the gradient through the model's input, not through the target
        loss.backward()
        out["forwards"].append(dict(
            x=x.detach().clone(), logits=logits.detach().clone(), loss=loss.detach().clone(), x_grad=x.grad.clone(),
            grads={k: p.grad.clone() for k, p in model.named_parameters()},
            masks={k: v.clone() for k, v in model.state_dict().items() if k.endswith("mask")}))
    out["state_after"] = {k: v.clone() for k, v in model.state_dict().items()}
    n, D = cfg["shape"][0], cfg["kwargs"]["input_dim"]
    for kind in ("unconditional", "conditional"):
        uniforms = torch.rand(D, n, generator=g)
        model._sample_fn = uniform_sample_fn(uniforms)
        cond = None
        if kind == "conditional":
            given = torch.bernoulli(torch.full(cfg["shape"], 0.5), generator=g)
            keep = torch.rand(cfg["shape"], generator=g) < 0.5
            cond = torch.where(keep, given, torch.full_like(given, -1.0))
        seed_before = model._mask_seed
        sample = model.sample(None if cond is not None else n, cond)
        out[kind] = dict(uniforms=uniforms, conditioned_on=cond, sample=sample.clone(), mask_seed_before=seed_before,
                         masks={k: v.clone() for k, v in model.state_dict().items() if k.endswith("mask")})
    out["mask_seed_after"] = model._mask_seed
    out["connectivity"] = {s: [torch.from_numpy(v.astype(np.int64)) for v in vecs]
                           for s, vecs in _RecordingRandomState.log.items()}
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.autoregressive import made as made_mod

    made_mod.np.random.RandomState = _RecordingRandomState
    fixture = {name: run(made_mod, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    torch.save(fixture, os.path.join(HERE, "made.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
