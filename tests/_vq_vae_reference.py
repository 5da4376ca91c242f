"""A plain-torch restatement of reference nn/utils.py `VectorQuantizer` and models/vae/{vq_vae,vq_vae_2}.py on a state
dict: the reference's operations in the reference's order, so in fp32 on the CPU it reproduces the reference's outputs,
gradients and buffers bit for bit (tests/golden/vq_vae.pt).  The convolution stages are those of tests/_vae_reference.py.

`q`, when given, rounds a tensor where the CUDA path keeps it in bf16 (see tests/_vae_reference.py), here also the
encoder output the quantizer's 1x1 convolution reads, the quantized operand of a decoder and VQ-VAE-2's `_conv` output.
`idx`, when given, fixes each quantizer's choice (by module name), so a float64 restatement takes the device's indices.
"""

import torch
from torch.nn import functional as F

import _vae_reference as V

device_rounding = V.device_rounding


def _same(t):
    return t


def encoder(state, key, x, q=_same):
    k = V._n_strided(state, key + ".")
    for j in range(k):
        x = q(F.relu(V._conv(state, f"{key}.{2 * j}", q(x), q, stride=2, padding=1)))
    x = V._res_stack(state, f"{key}.{2 * k}", x, q, _n_blocks(state, f"{key}.{2 * k}"))
    return V._conv(state, f"{key}.{2 * k + 1}", q(x), q, padding=1)


def _n_blocks(state, key):
    return len({k[len(key) + 6:].split(".")[0] for k in state if k.startswith(key + "._net.")})


def decoder(state, key, x, q=_same):
    x = V._conv(state, f"{key}.0", q(x), q, padding=1)
    x = V._res_stack(state, f"{key}.1", x, q, _n_blocks(state, f"{key}.1"))
    k = V._n_strided(state, key + ".")
    j = 2
    for t in range(k):
        x = F.conv_transpose2d(q(x), q(state[f"{key}.{j}.weight"]), state[f"{key}.{j}.bias"], stride=2, padding=1)
        j += 1
        if t < k - 1:
            x = F.relu(x)
            j += 1
    return x


def quantize(x, embedding, cluster_size=None, embedding_avg=None, use_ema=True, decay=0.99, training=True, idx=None):
    """(x + (q - x).detach(), loss, idx, new buffers or None) of VectorQuantizer.forward; the buffers are not modified."""
    n, c, h, w = x.shape
    flat_x = x.permute(0, 2, 3, 1).contiguous().view(-1, c)
    if idx is None:
        distances = torch.sum(flat_x**2, dim=1, keepdim=True) + torch.sum(embedding**2, dim=1) - 2 * flat_x @ embedding.t()
        idx = torch.argmin(distances, dim=1)
    one_hot = torch.zeros(idx.shape[0], embedding.shape[0], dtype=x.dtype, device=x.device)
    one_hot.scatter_(1, idx.view(-1, 1).to(x.device), 1)
    quantized = one_hot @ embedding
    quantized = quantized.view(n, h, w, c).permute(0, 3, 1, 2).contiguous()
    loss = F.mse_loss(x, quantized.detach())
    buffers = None
    if use_ema and training:
        with torch.no_grad():
            batch_cluster_size = one_hot.sum(axis=0)
            batch_embedding_avg = (flat_x.t() @ one_hot).t()
            cs = cluster_size.clone().mul_(decay).add_(batch_cluster_size, alpha=1 - decay)
            avg = embedding_avg.clone().mul_(decay).add_(batch_embedding_avg, alpha=1 - decay)
            buffers = (cs, avg, avg / (cs + 1e-5).unsqueeze(1))
    elif not use_ema:
        loss += F.mse_loss(quantized, x.detach())
    return x + (quantized - x).detach(), loss, idx, buffers


def _quantizer(state, key, x, q, training, idx, found, use_ema=True):
    """A vaes.Quantizer: the 1x1 convolution of q(x), then the quantizer.  Records (input, idx, buffers) in `found`."""
    z = V._conv(state, f"{key}._net.0", q(x), q)
    p = f"{key}._net.1."
    out, loss, i, bufs = quantize(z, state[p + "_embedding"], state.get(p + "_cluster_size"),
                                  state.get(p + "_embedding_avg"), use_ema, training=training,
                                  idx=None if idx is None else idx[f"{key}._net.1"])
    found[f"{key}._net.1"] = dict(input=z, idx=i, buffers=bufs)
    return q(out), loss


def vq_vae(state, x, q=_same, training=True, idx=None):
    """(x_hat, vq_loss, {quantizer name: (input, idx, new buffers)}) of VectorQuantizedVAE.forward."""
    found = {}
    h = encoder(state, "_encoder._net", x, q)
    quantized, vq_loss = _quantizer(state, "_quantizer", h, q, training, idx, found)
    return decoder(state, "_decoder._net", quantized, q), vq_loss, found


def vq_vae_2(state, x, q=_same, training=True, idx=None):
    """(x_hat, loss, found) of VectorQuantizedVAE2.forward."""
    found = {}
    encoded_b = encoder(state, "_encoder_b._net", x, q)
    encoded_t = encoder(state, "_encoder_t._net", encoded_b, q)
    quantized_t, vq_loss_t = _quantizer(state, "_quantizer_t", encoded_t, q, training, idx, found)
    quantized_b, vq_loss_b = _quantizer(state, "_quantizer_b", encoded_b, q, training, idx, found)
    decoded_t = decoder(state, "_decoder_t._net", quantized_t, q)
    left = q(V._conv(state, "_conv", q(decoded_t), q))
    xhat = decoder(state, "_decoder_b._net", torch.cat((left, quantized_b), dim=1), q)
    return xhat, 0.5 * (vq_loss_b + vq_loss_t) + F.mse_loss(decoded_t, encoded_b), found


def loss_fn(x, x_hat, vq_loss, weight):
    recon_loss = F.mse_loss(x_hat, x)
    return {"vq_loss": vq_loss, "reconstruction_loss": recon_loss, "loss": recon_loss + weight * vq_loss}


MODELS = {"VectorQuantizedVAE": (vq_vae, 1.0), "VectorQuantizedVAE2": (vq_vae_2, 0.25)}


def is_param(k):
    return not k.endswith(("_cluster_size", "_embedding_avg")) and not (k.endswith("_embedding") and
                                                                          "._net.1." in k)


def run(fx, dtype=torch.float32, device="cpu", q=_same, idx=None, state=None):
    """(outputs, loss dict or vq_loss, {name: gradient}, found) of a fixture configuration in `dtype` on `device`."""
    state = {k: v.to(device, dtype) for k, v in (state or fx["state"]).items()}
    params = {k: v.clone().requires_grad_(True) for k, v in state.items() if is_param(k) or fx["cls"] == "VectorQuantizer"
              and k == "_embedding" and not fx["kwargs"].get("use_ema", True)}
    state.update(params)
    x = fx["x"].to(device, dtype)
    if fx["cls"] == "VectorQuantizer":
        xg = x.clone().requires_grad_(True)
        out, loss, i, _ = quantize(xg, state["_embedding"], use_ema=False, idx=None if idx is None else idx[""])
        total = (out * fx["cot"].to(device, dtype)).sum() + loss
        grads = torch.autograd.grad(total, [xg] + list(params.values()))
        return out.detach(), loss.detach(), dict(zip(["x"] + list(params), grads)), {"": dict(input=x, idx=i, buffers=None)}
    fn, weight = MODELS[fx["cls"]]
    x_hat, vq_loss, found = fn(state, x, q, fx["train"], idx)
    losses = loss_fn(x, x_hat, vq_loss, weight)
    grads = torch.autograd.grad(losses["loss"], list(params.values()))
    return x_hat.detach(), {k: v.detach() for k, v in losses.items()}, dict(zip(params, grads)), found
