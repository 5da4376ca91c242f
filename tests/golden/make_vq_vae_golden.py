"""Generates tests/golden/vq_vae.pt by running the UNMODIFIED reference VQ-VAE / VQ-VAE-2 (models/vae/vq_vae.py,
vq_vae_2.py) and VectorQuantizer (nn/utils.py) on the CPU.

    python tests/golden/make_vq_vae_golden.py <path to the reference checkout>

Per configuration the fixture holds the constructor arguments, the state dict after `torch.manual_seed(seed)` and the
constructor (for the init check), a state with N(0, 0.05) noise added to every parameter (the EMA buffers are kept),
and under that state:
  * `x`: an input batch (N(0, 1), like normalised CIFAR-10 images);
  * `vq_inputs`: per quantizer (by module name), the input it received, the codebook it used and the indices it chose;
  * the outputs, the recipe's loss dict (the reference's `loss_fn` in vq_vae.py / vq_vae_2.py `reproduce`), every
    parameter gradient of its `loss` and the buffers after the forward.
For every row of every quantizer the generator asserts that the relative margin (second - best) / best between the two
smallest distances (float64) is at least MARGIN: far more than the CUDA path's bf16 operands move a distance, so the
device must choose the same indices.  A configuration whose seed fails that is retried with the next seed, and the
seed used is recorded.  Configurations: VQ-VAE(3, 3, 12, 2, 8, 10, 6) on 3x16x16 (widths that are not multiples of 8),
the same model in eval(), VQ-VAE-2(3, 3, 16, 1, 8, 12, 5) on 3x8x8, and a standalone VectorQuantizer(10, 6,
use_ema=False) whose loss adds the sum of its output times fixed cotangents.
"""

import os
import sys

import torch
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
MARGIN = 0.05

CONFIGS = {
    "vq_vae": dict(cls="VectorQuantizedVAE", kwargs=dict(in_channels=3, out_channels=3, hidden_channels=12,
                                                         n_residual_blocks=2, residual_channels=8, n_embeddings=10,
                                                         embedding_dim=6), shape=(2, 3, 16, 16), train=True, seed=0),
    "vq_vae_eval": dict(cls="VectorQuantizedVAE", kwargs=dict(in_channels=3, out_channels=3, hidden_channels=12,
                                                              n_residual_blocks=2, residual_channels=8,
                                                              n_embeddings=10, embedding_dim=6),
                        shape=(2, 3, 16, 16), train=False, seed=100),
    "vq_vae_2": dict(cls="VectorQuantizedVAE2", kwargs=dict(in_channels=3, out_channels=3, hidden_channels=16,
                                                            n_residual_blocks=1, residual_channels=8, n_embeddings=12,
                                                            embedding_dim=5), shape=(1, 3, 8, 8), train=True,
                     seed=200),
    "vq_no_ema": dict(cls="VectorQuantizer", kwargs=dict(n_embeddings=10, embedding_dim=6, use_ema=False),
                      shape=(1, 6, 3, 4), train=True, seed=300),
}


def loss_fn(weight):
    def fn(x, _, preds):
        preds, vq_loss = preds
        recon_loss = F.mse_loss(preds, x)
        return {"vq_loss": vq_loss, "reconstruction_loss": recon_loss, "loss": recon_loss + weight * vq_loss}
    return fn


def margins(x, emb):
    """(second - best) / best of every row's two smallest float64 distances."""
    flat = x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).double()
    d = torch.cdist(flat, emb.double()) ** 2
    two = d.topk(2, dim=1, largest=False).values
    return (two[:, 1] - two[:, 0]) / two[:, 0]


def run(ref_nn, models, cfg, seed):
    torch.manual_seed(seed)
    if cfg["cls"] == "VectorQuantizer":
        model = ref_nn.VectorQuantizer(**cfg["kwargs"])
    else:
        model = getattr(models, cfg["cls"])(**cfg["kwargs"])
    out = dict(cls=cfg["cls"], kwargs=cfg["kwargs"], seed=seed, train=cfg["train"],
               state_init={k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in model.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.05)
    out["state"] = {k: v.clone() for k, v in model.state_dict().items()}
    x = torch.randn(cfg["shape"], generator=g)
    out["x"] = x.clone()
    model.train(cfg["train"])
    seen = {}

    def hook(name):
        def pre(module, args):
            seen[name] = dict(input=args[0].detach().clone(), embedding=module._embedding.detach().clone())
        return pre
    for name, m in model.named_modules():
        if isinstance(m, ref_nn.VectorQuantizer):
            m.register_forward_pre_hook(hook(name))
    if cfg["cls"] == "VectorQuantizer":
        xg = x.clone().requires_grad_(True)
        q, vq_loss = model(xg)
        cot = torch.randn(q.shape, generator=g)
        total = (q * cot).sum() + vq_loss
        total.backward()
        out.update(cot=cot, outputs=q.detach().clone(), vq_loss=vq_loss.detach().clone(), x_grad=xg.grad.clone())
    else:
        x_hat, vq_loss = model(x)
        losses = loss_fn(1.0 if cfg["cls"] == "VectorQuantizedVAE" else 0.25)(x, None, (x_hat, vq_loss))
        losses["loss"].backward()
        out.update(outputs=x_hat.detach().clone(), vq_loss=vq_loss.detach().clone(),
                   losses={k: v.detach().clone() for k, v in losses.items()})
    out["grads"] = {k: prm.grad.clone() for k, prm in model.named_parameters()}
    out["buffers"] = {k: v.clone() for k, v in model.state_dict().items() if k not in dict(model.named_parameters())}
    for name, s in seen.items():
        flat = s["input"].permute(0, 2, 3, 1).contiguous().view(-1, s["input"].shape[1])
        dist = torch.sum(flat ** 2, dim=1, keepdim=True) + torch.sum(s["embedding"] ** 2, dim=1) - 2 * flat @ s["embedding"].t()
        s["idx"] = torch.argmin(dist, dim=1)
        s["margin"] = margins(s["input"], s["embedding"])
    out["vq_inputs"] = seen
    return out


def main(reference):
    sys.path.insert(0, os.path.abspath(reference))
    from pytorch_generative import models
    from pytorch_generative import nn as ref_nn

    fixture = {}
    for name, cfg in CONFIGS.items():
        seed = cfg["seed"]
        for _ in range(5000):
            fx = run(ref_nn, models, cfg, seed)
            worst = min(s["margin"].min().item() for s in fx["vq_inputs"].values())
            if worst >= MARGIN:
                break
            seed += 1
        else:
            raise RuntimeError(f"{name}: no seed from {cfg['seed']} gives every row a margin of {MARGIN}")
        print(name, "seed", seed, "smallest margin", worst)
        fixture[name] = fx
    torch.save(fixture, os.path.join(HERE, "vq_vae.pt"))


if __name__ == "__main__":
    main(sys.argv[1])
