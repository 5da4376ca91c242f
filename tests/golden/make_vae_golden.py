"""Generates tests/golden/vae.pt by running the UNMODIFIED reference VAE / BetaVAE (models/vae/{vae,beta_vae}.py) on the
CPU.

    python tests/golden/make_vae_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments, the state dict after `torch.manual_seed(seed)` and the
constructor (for the init check), a state with N(0, 0.05) noise added to every parameter, and under that state:
  * `x`: a binary image batch;
  * `eps`: the forward's reparameterisation noise, re-drawn under the seed the forward ran under (`fwd_seed`);
  * `logits`, `kl` of the forward, the recipe loss dict (the reference's `loss_fn` in vae.py `reproduce`) and every
    parameter gradient of its `loss`;
  * `sample_latents` and `sample_logits`: the latent batch `_sample(n)` draws right after
    `torch.manual_seed(sample_seed)` and the decoder's output for it;
  * `shape_buffers`: the `_c`, `_h`, `_w` buffers the image forward registered.
The configurations are VAE(1, 1, 4, [2, 2], 16, 8) on 1x16x16 images, BetaVAE(1, 1, 4.0, 4, [4], 12, 8) on 1x12x12
images (hidden // 2 = 6 and 12 channels, neither a multiple of 8, and a 3x3 latent) and the reference's multi-channel
smoke configuration VAE(3, 3, 1, [2, 2], 1, 1) on 3x8x8 images.
"""

import os
import sys

import torch
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = {
    "vae_16": dict(cls="VAE", kwargs=dict(in_channels=1, out_channels=1, latent_channels=4, strides=[2, 2],
                                          hidden_channels=16, residual_channels=8), shape=(4, 1, 16, 16)),
    "beta_vae_12": dict(cls="BetaVAE", kwargs=dict(in_channels=1, out_channels=1, beta=4.0, latent_channels=4,
                                                   strides=[4], hidden_channels=12, residual_channels=8),
                        shape=(3, 1, 12, 12)),
    "vae_rgb_8": dict(cls="VAE", kwargs=dict(in_channels=3, out_channels=3, latent_channels=1, strides=[2, 2],
                                             hidden_channels=1, residual_channels=1), shape=(2, 3, 8, 8)),
}


def loss_fn(x, _, preds):
    preds, kl_div = preds
    recon_loss = F.binary_cross_entropy_with_logits(preds, x, reduction="none")
    recon_loss = recon_loss.sum(dim=(1, 2, 3))
    elbo = recon_loss + kl_div
    return {"recon_loss": recon_loss.mean(), "kl_div": kl_div.mean(), "loss": elbo.mean()}


def run(modules, cfg, seed):
    torch.manual_seed(seed)
    model = getattr(modules[cfg["cls"]], cfg["cls"])(**cfg["kwargs"])
    out = dict(cls=cfg["cls"], kwargs=cfg["kwargs"], seed=seed,
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
    n, L = x.shape[0], cfg["kwargs"]["latent_channels"]
    side = x.shape[2] // 2 ** (sum(cfg["kwargs"]["strides"]) // 2)  # the latent's side (square images)
    torch.manual_seed(seed + 2)
    out["eps"] = torch.randn(n, L, side, side)
    out["sample_seed"] = seed + 3
    torch.manual_seed(seed + 3)
    with torch.no_grad():
        out["sample_logits"] = model._sample(n).clone()
    torch.manual_seed(seed + 3)
    out["sample_latents"] = torch.randn(n, L, side, side)
    out["shape_buffers"] = {k: model.state_dict()[k].clone() for k in ("_c", "_h", "_w")}  # of the image forward
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative.models.vae import beta_vae, vae

    modules = {"VAE": vae, "BetaVAE": beta_vae}
    fixture = {name: run(modules, cfg, 10 * i) for i, (name, cfg) in enumerate(CONFIGS.items())}
    torch.save(fixture, os.path.join(HERE, "vae.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
