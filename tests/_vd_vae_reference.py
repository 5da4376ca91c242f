"""Functional torch restatement of reference models/vae/vd_vae.py VeryDeepVAE, in any dtype, with the noise given.

`forward(state, x, cfg, eps)` -> (logits, kl) and `sample(state, cfg, n, eps)` -> logits take the state dict of a
VeryDeepVAE (keys `_input.*`, `_encoder.{i}._residuals.{j}._net.{k}.*`, `_biases.{i}`, `_decoder.{i}._topdowns.{j}.*`,
`_output.*`) and `cfg` = (input_resolution, stacks [(n_enc, n_dec), ...], latent_channels).  eps: one tensor per
TopDownBlock in decoder order.  Kernel sizes follow the state's weight shapes, so the reference's decoder kernel size
(DESIGN §2) needs no restating; the padding is (k - 1) / 2, as the reference's 1 for k = 3 and 0 for k = 1."""

import torch
from torch.nn import functional as F


def _conv(state, x, key):
    w = state[key + ".weight"]
    return F.conv2d(x, w.to(x.dtype), state[key + ".bias"].to(x.dtype), padding=(w.shape[-1] - 1) // 2)


def bottleneck(state, x, key, residual):
    h = x
    for k in (1, 3, 5, 7):
        h = _conv(state, F.gelu(h), f"{key}._net.{k}")
    return x + h if residual else h


def gaussian_kl_div(q_mean, q_log_std, p_mean, p_log_std):
    """KL(q || p) in the reference's order of operations (vaes.py gaussian_kl_div)."""
    mean_delta, log_std_delta = (q_mean - p_mean) ** 2, p_log_std - q_log_std
    q_var, p_var = q_log_std.exp().pow(2), 2 * p_log_std.exp().pow(2)
    return -0.5 + log_std_delta + (q_var + mean_delta) / p_var


def topdown(state, x, mixin, key, L, eps):
    C = x.shape[1]
    p_mean, p_log_std, p_h = torch.split(bottleneck(state, x, key + "._prior", False), [L, L, C], dim=1)
    if mixin is None:
        z, kl = p_mean + p_log_std.exp() * eps, None
    else:
        q_mean, q_log_std = torch.split(bottleneck(state, torch.cat((x, mixin), dim=1), key + "._posterior", False), L,
                                        dim=1)
        z = q_mean + q_log_std.exp() * eps
        kl = gaussian_kl_div(q_mean, q_log_std, p_mean, p_log_std)
    return bottleneck(state, x + p_h + _conv(state, z, key + "._latents"), key + "._out", True), kl


def _decode(state, cfg, n, mixins, eps, dtype):
    _, stacks, L = cfg
    n_biases = len(stacks)
    x = torch.zeros_like(state[f"_biases.{n_biases - 1}"].to(dtype)).repeat(n, 1, 1, 1)
    kls, e = [], 0
    for i, (_, n_dec) in enumerate(reversed(stacks)):
        x = x + state[f"_biases.{n_biases - 1 - i}"].to(dtype).repeat(n, 1, 1, 1)
        if i > 0:
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        mixin = None if mixins is None else mixins[len(mixins) - 1 - i]
        for j in range(n_dec):
            x, kl = topdown(state, x, mixin, f"_decoder.{i}._topdowns.{j}", L, eps[e].to(dtype))
            e += 1
            kls.append(kl)
    return _conv(state, x, "_output"), kls


def forward(state, x, cfg, eps):
    _, stacks, _ = cfg
    dtype = x.dtype
    x = _conv(state, x, "_input")
    mixins = []
    for i, (n_enc, _) in enumerate(stacks):
        for j in range(n_enc):
            x = bottleneck(state, x, f"_encoder.{i}._residuals.{j}", True)
        mixins.append(x)
        if i < len(stacks) - 1:
            x = F.avg_pool2d(x, 2, 2)
    logits, kls = _decode(state, cfg, x.shape[0], mixins, eps, dtype)
    kl = torch.zeros(x.shape[0], dtype=dtype)
    for div in kls:
        kl = kl + div.sum(dim=(1, 2, 3))
    return logits, kl


def sample(state, cfg, n, eps, dtype=torch.float32):
    logits, _ = _decode(state, cfg, n, None, eps, dtype)
    return logits


def elbo_loss(logits, kl, x):
    recon = F.binary_cross_entropy_with_logits(logits, x, reduction="none").sum(dim=(1, 2, 3))
    return (recon + kl).mean()


def cfg_of(model):
    """(input_resolution, stacks, latent_channels) of a VeryDeepVAE (this package's or the reference's)."""
    stacks = [(len(e._residuals), len(d._topdowns)) for e, d in zip(model._encoder, reversed(model._decoder))]
    L = model._decoder[0]._topdowns[0]._latent_channels if len(model._decoder[0]._topdowns) else None
    if L is None:
        L = next(b._latent_channels for d in model._decoder for b in d._topdowns)
    return model._biases[-1].shape[-1] * 2 ** (len(stacks) - 1), stacks, L


def grads(state, x, cfg, eps, dtype=torch.float64):
    """Every parameter's gradient of the recipe's ELBO in `dtype`."""
    st = {k: v.detach().to(dtype).requires_grad_(v.is_floating_point()) for k, v in state.items()}
    logits, kl = forward(st, x.to(dtype), cfg, eps)
    loss = elbo_loss(logits, kl, x.to(dtype))
    loss.backward()
    return {k: v.grad for k, v in st.items() if v.grad is not None}, logits.detach(), kl.detach(), loss.detach()


def load_fixture(path):
    """tests/golden/vd_vae.pt with what its generator leaves to seeds rebuilt (see make_vd_vae_golden.py): per case
    `state_init`, `state` and `grads` as dicts, and the recorded noise `eps` / `sample_eps` as lists in decoder order."""
    fixture = torch.load(path, weights_only=False)
    for case in fixture.values():
        keys, shapes = case.pop("keys"), case.pop("shapes")

        def unflat(flat):
            out, i = {}, 0
            for k, shape in zip(keys, shapes):
                n = int(torch.Size(shape).numel())
                out[k] = flat[i:i + n].reshape(shape).clone()
                i += n
            return out
        case["state_init"], case["grads"] = unflat(case["state_init"]), unflat(case["grads"])
        case["x"] = case["x"].float()
        g = torch.Generator().manual_seed(case["seed"] + 1)
        case["state"] = {k: v + torch.randn(v.shape, generator=g) * 0.05 for k, v in case["state_init"].items()}
        for key, seed in (("eps", case["fwd_seed"]), ("sample_eps", case["sample_seed"])):
            g = torch.Generator().manual_seed(seed)
            case[key] = [torch.randn(s, generator=g) for s in case["noise_shapes"]]
    return fixture
