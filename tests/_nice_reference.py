"""A CPU restatement of the reference NICE (models/flow/nice.py) and its recipe loss, in any float dtype, from a state
dict; pinned to the reference's own outputs by tests/test_nice_cpu.py (tests/golden/nice.pt).  Not a test module.

Block b couples with `reverse = b % 2 == 1`: the MLP net.{b}.net (Linear / ReLU, no ReLU after the last Linear) reads
the first half x[:, :D/2] and is added to the second (reverse: reads the second, added to the first); then
z = y * exp(scaling.log_scale) and log_det_J = sum(log_scale)."""

import torch
from torch.nn import functional as F


def n_blocks(state):
    return len({k.split(".")[1] for k in state if k.startswith("net.")})


def layers(state, b):
    """[(weight, bias)] of block b's MLP in order."""
    idx = sorted({int(k.split(".")[3]) for k in state if k.startswith(f"net.{b}.net.")})
    return [(state[f"net.{b}.net.{i}.weight"], state[f"net.{b}.net.{i}.bias"]) for i in idx]


def names(state):
    """parameters() order of the reference: every block's Linear weights and biases, then scaling.log_scale."""
    return [f"net.{b}.net.{i}.{w}" for b in range(n_blocks(state))
            for i in sorted({int(k.split(".")[3]) for k in state if k.startswith(f"net.{b}.net.")})
            for w in ("weight", "bias")] + ["scaling.log_scale"]


def mlp(params, b, h):
    ls = layers(params, b)
    for i, (w, bias) in enumerate(ls):
        h = F.linear(h, w, bias)
        if i + 1 < len(ls):
            h = torch.relu(h)
    return h


def couple(params, b, x, sign):
    D = x.shape[1]
    h1, h2 = x[:, : D // 2], x[:, D // 2:]
    if b % 2 == 1:
        h1 = h1 + sign * mlp(params, b, h2)
    else:
        h2 = h2 + sign * mlp(params, b, h1)
    return torch.cat((h1, h2), dim=1)


def forward(params, x):
    """(z in x's shape, log_det_J) in the dtype of `params`."""
    shape = x.shape
    y = x.reshape(shape[0], -1)
    for b in range(n_blocks(params)):
        y = couple(params, b, y, 1)
    log_scale = params["scaling.log_scale"]
    return (y * torch.exp(log_scale)).view(shape), torch.sum(log_scale)


def inverse(params, z):
    shape = z.shape
    y = z.reshape(shape[0], -1) * torch.exp(-params["scaling.log_scale"])
    for b in reversed(range(n_blocks(params))):
        y = couple(params, b, y, -1)
    return y.view(shape)


def loss(z, log_det_J):
    """The recipe's loss dict (reference nice.py:205-213), z of any shape [n, ...]."""
    log_prob = -(F.softplus(z) + F.softplus(-z)).reshape(z.shape[0], -1).sum(dim=1)
    total = log_prob + log_det_J
    return {"loss": -total.mean(), "prior_log_likelihood": log_prob.mean(), "log_det_J": log_det_J.mean()}


def params_of(state, dtype=torch.float32, device="cpu"):
    return {k: v.to(device, dtype) for k, v in state.items() if k.startswith(("net.", "scaling."))}


def loss_and_grads(state, x, dtype=torch.float32, device="cpu"):
    """(z, log_det_J, loss dict, {name: grad}, x_grad) of the recipe loss, in `dtype` on `device`."""
    params = {k: v.clone().requires_grad_(True) for k, v in params_of(state, dtype, device).items()}
    xx = x.to(device, dtype).clone().requires_grad_(True)
    z, log_det_J = forward(params, xx)
    losses = loss(z, log_det_J)
    losses["loss"].backward()
    return (z.detach(), log_det_J.detach(), {k: v.detach() for k, v in losses.items()},
            {k: params[k].grad for k in names(state)}, xx.grad)
