"""A plain-torch restatement of reference models/vae/{vae,beta_vae,vaes}.py on a state dict: the reference's operations
in the reference's order, so in fp32 on the CPU it reproduces the reference's outputs bit for bit
(tests/golden/vae.pt).  `eps` is the reparameterisation noise the forward's `randn_like` draws.

`q`, when given, rounds a tensor where the CUDA path keeps it in bf16: every convolution weight and operand (the image,
the ReLU outputs the strided convolutions and the residual blocks' 3x3 convolutions emit, the activated stream a
convolution reads, a non-last encoder's or decoder's output) and the latent z.  With `device_rounding` in float64 the
forward then takes the CUDA path's ReLU decisions (its fp32 sums differ from float64 by far less than bf16 rounds),
so gradients can be compared element by element without a ReLU flipping between the two."""

import torch
from torch.nn import functional as F


def _same(t):
    return t


def device_rounding(t):
    """bf16 rounding in the forward, the identity in the backward (the CUDA path's gradient of a bf16 operand is the
    gradient of the value it stands for)."""
    return t + (t.to(torch.bfloat16).to(t.dtype) - t).detach()


def _conv(state, key, x, q=_same, **kw):
    return F.conv2d(x, q(state[key + ".weight"]), state[key + ".bias"], **kw)


def _res_stack(state, key, x, q=_same, n_blocks=2):
    for b in range(n_blocks):
        k = f"{key}._net.{b}._net"
        h = _conv(state, f"{k}.1", q(F.relu(x)), q, padding=1)
        x = x + _conv(state, f"{k}.3", q(F.relu(h)), q)
    return F.relu(x)


def _n_strided(state, prefix):
    """Strided (de)convolutions of one Encoder / Decoder: stride // 2."""
    return sum(1 for k in state if k.startswith(prefix) and k.endswith(".weight") and state[k].shape[-1] == 4)


def encoder(state, i, x, q=_same):
    key = f"_encoder.{i}._net"
    k = _n_strided(state, key + ".")
    for j in range(k):
        x = q(F.relu(_conv(state, f"{key}.{2 * j}", q(x), q, stride=2, padding=1)))
    x = _res_stack(state, f"{key}.{2 * k}", x, q)
    return _conv(state, f"{key}.{2 * k + 1}", q(x), q, padding=1)


def decoder(state, i, x, q=_same):
    key = f"_decoder.{i}._net"
    x = _conv(state, f"{key}.0", q(x), q, padding=1)
    x = _res_stack(state, f"{key}.1", x, q)
    k = _n_strided(state, key + ".")
    j = 2
    for t in range(k):
        x = F.conv_transpose2d(q(x), q(state[f"{key}.{j}.weight"]), state[f"{key}.{j}.bias"], stride=2, padding=1)
        j += 1
        if t < k - 1:
            x = F.relu(x)
            j += 1
    return x


def _count(state, prefix):
    return len({k.split(".")[1] for k in state if k.startswith(prefix)})


def decode(state, z, q=_same):
    for i in range(_count(state, "_decoder.")):
        z = decoder(state, i, z, q)
    return z


@torch.jit.script
def _unit_gaussian_kl_div(mean, log_std):
    """vaes.py unit_gaussian_kl_div, scripted like the reference's (TorchScript's autodiff rounds its backward
    differently from eager autograd)."""
    return -0.5 * (1 + 2 * log_std - log_std.exp().pow(2) - mean**2)


@torch.jit.script
def _reparameterise(mu, log_sig, eps):
    """vaes.py sample_from_gaussian with its randn_like drawn beforehand (eps)."""
    return mu + log_sig.exp() * eps


def forward(state, x, eps, latent_channels, beta=None, q=_same):
    """(logits, kl) of VAE.forward (BetaVAE.forward when beta is given) with the noise eps."""
    h = x
    for i in range(_count(state, "_encoder.")):
        h = encoder(state, i, h, q)
    mean, log_std = torch.split(h, latent_channels, dim=1)
    kl = _unit_gaussian_kl_div(mean, log_std).sum(dim=(1, 2, 3))
    z = _reparameterise(mean, log_std, eps)
    out = decode(state, z, q)
    return (out, kl) if beta is None else (out, beta * kl)


def loss_fn(x, logits, kl):
    """The recipe's loss dict (reference vae.py `reproduce`)."""
    recon_loss = F.binary_cross_entropy_with_logits(logits, x, reduction="none").sum(dim=(1, 2, 3))
    elbo = recon_loss + kl
    return {"recon_loss": recon_loss.mean(), "kl_div": kl.mean(), "loss": elbo.mean()}


def params_of(state, dtype=torch.float32):
    """The parameters of a state dict (shape buffers left out), as leaf tensors that require grad."""
    return {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in state.items() if k not in ("_c", "_h", "_w")}


def loss_and_grads(state, x, eps, latent_channels, beta=None, dtype=torch.float32, q=_same):
    """(logits, kl, loss dict, {name: gradient of loss}) in `dtype`, on the device of x."""
    params = {k: v.to(x.device) for k, v in params_of(state, dtype).items()}
    logits, kl = forward(params, x.to(dtype), eps.to(x.device, dtype), latent_channels, beta, q)
    losses = loss_fn(x.to(dtype), logits, kl)
    grads = torch.autograd.grad(losses["loss"], list(params.values()))
    return logits.detach(), kl.detach(), {k: v.detach() for k, v in losses.items()}, dict(zip(params, grads))
