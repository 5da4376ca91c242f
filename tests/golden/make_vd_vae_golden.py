"""Generates tests/golden/vd_vae.pt by running the UNMODIFIED reference VeryDeepVAE (models/vae/vd_vae.py) on the CPU.

    python tests/golden/make_vd_vae_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments (stack configs as (encoder, decoder) pairs), the state
dict after `torch.manual_seed(seed)` and the constructor (for the init check), and the outputs of a state with
N(0, 0.05) noise added to every parameter:
  * `x`: a binary image batch;
  * `logits`, `kl` of the forward, the recipe loss dict (the reference's `loss_fn` in vd_vae.py `reproduce`) and every
    parameter gradient of its `loss`;
  * `sample_logits`: the output of `_sample(n)` right after `torch.manual_seed(sample_seed)`.
To keep the file small, the state dict and the gradients are stored as one flat tensor each (`keys`, `shapes`), x as
uint8, and what follows from seeds is not stored: the perturbed state (the parameters in order plus 0.05 randn from a
generator seeded with seed + 1) and each TopDownBlock's noise in decoder order (randn of `noise_shapes` after
`manual_seed(fwd_seed)` or `manual_seed(sample_seed)`).  `tests/_vd_vae_reference.load_fixture` rebuilds them; this
script checks that it does so exactly.
The configurations are (a) `VeryDeepVAE()` on 1x32x32 images (six stacks down to 1x1: every decoder `_out` block has
1x1 middle convolutions) and (b) three stacks on 3x16x16 images with 3x3 decoder `_out` blocks, unequal encoder and
decoder counts and widths that are not multiples of 8 (2L + C = 18, p_h at column 6).
"""

import os
import sys

import torch
from torch.nn import functional as F


HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "default_32": dict(kwargs=dict(), stacks=None, shape=(3, 1, 32, 32)),
    "rgb_16": dict(kwargs=dict(in_channels=3, out_channels=3, input_resolution=16, latent_channels=3,
                               hidden_channels=12, bottleneck_channels=6),
                   stacks=[(2, 3), (1, 2), (1, 1)], shape=(2, 3, 16, 16)),
}


def loss_fn(x, _, preds):
    preds, kl_div = preds
    recon_loss = F.binary_cross_entropy_with_logits(preds, x, reduction="none")
    recon_loss = recon_loss.sum(dim=(1, 2, 3))
    elbo = recon_loss + kl_div
    return {"recon_loss": recon_loss.mean(), "kl_div": kl_div.mean(), "loss": elbo.mean()}


def noise_shapes(model, n):
    """(n, L, side, side) of each TopDownBlock in decoder order."""
    shapes = []
    side = None
    for stack, bias in zip(model._decoder, reversed(model._biases)):
        side = bias.shape[-1] * (2 if stack._unpool is not None else 1)
        for block in stack._topdowns:
            shapes.append((n, block._latent_channels, side, side))
    return shapes


def run(vd_vae, cfg, seed):
    kwargs = dict(cfg["kwargs"])
    if cfg["stacks"] is not None:
        kwargs["stack_configs"] = [vd_vae.StackConfig(e, d) for e, d in cfg["stacks"]]
    torch.manual_seed(seed)
    model = vd_vae.VeryDeepVAE(**kwargs)
    out = dict(kwargs=cfg["kwargs"], stacks=cfg["stacks"], seed=seed,
               state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    x = torch.randint(0, 2, cfg["shape"], generator=g).float()
    out["x"] = x.clone()
    out["fwd_seed"] = seed + 2
    torch.manual_seed(seed + 2)
    logits, kl = model(x)
    losses = loss_fn(x, None, (logits, kl))
    losses["loss"].backward()
    out.update(logits=logits.detach().clone(), kl=kl.detach().clone(),
               losses={k: v.detach().clone() for k, v in losses.items()},
               grads={k: prm.grad.clone() for k, prm in model.named_parameters()})
    n = x.shape[0]
    torch.manual_seed(seed + 2)
    out["eps"] = [torch.randn(s) for s in noise_shapes(model, n)]
    out["sample_seed"] = seed + 3
    torch.manual_seed(seed + 3)
    with torch.no_grad():
        out["sample_logits"] = model._sample(n).clone()
    torch.manual_seed(seed + 3)
    out["sample_eps"] = [torch.randn(s) for s in noise_shapes(model, n)]
    out["noise_shapes"] = noise_shapes(model, n)
    return out


def pack(case):
    """The stored form of a case: flat state and gradients, no seeded tensors."""
    keys = list(case["state_init"])
    packed = {k: v for k, v in case.items() if k not in ("state_init", "state", "grads", "eps", "sample_eps")}
    packed.update(keys=keys, shapes=[tuple(case["state_init"][k].shape) for k in keys],
                  state_init=torch.cat([case["state_init"][k].reshape(-1) for k in keys]),
                  grads=torch.cat([case["grads"][k].reshape(-1) for k in keys]), x=case["x"].to(torch.uint8))
    return packed


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.vae import vd_vae

    sys.path.insert(0, os.path.dirname(HERE))
    import _vd_vae_reference as R

    full = {name: run(vd_vae, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    path = os.path.join(HERE, "vd_vae.pt")
    torch.save({name: pack(case) for name, case in full.items()}, path)
    for name, case in R.load_fixture(path).items():
        for key in ("state_init", "state", "grads"):
            assert all(torch.equal(case[key][k], v) for k, v in full[name][key].items()), (name, key)
        assert torch.equal(case["x"], full[name]["x"]), name
        for key in ("eps", "sample_eps"):
            assert all(torch.equal(a, b) for a, b in zip(case[key], full[name][key], strict=True)), (name, key)


if __name__ == "__main__":
    main(sys.argv[1])
