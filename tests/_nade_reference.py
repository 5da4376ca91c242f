"""Restatement of the reference NADE (models/autoregressive/nade.py) in torch: the per-dimension loop of `_forward` with
draws from given uniforms, the recipe loss, gradients, sampling and the recipe's training step.  Any dtype and device
(float32 on the CPU is pinned to the reference's own outputs in tests/golden/nade.pt; float64 on the GPU is the
kernels' yardstick; float32 on the GPU is the comparison arm of tools/bench_nade.py).  Tests and tools only.  State
dicts use the reference's keys (`_in_W`, `_in_b`, `_h_W`, `_h_b`)."""

import torch
import torch.nn.functional as F

PARAMS = ("_in_W", "_in_b", "_h_W", "_h_b")


def forward(p, x, u):
    """(probabilities, x~) of a flat batch x [n, D]: a_0 = _in_b; per dimension i, p_i = sigmoid(relu(a) . _h_W[i] +
    _h_b[i]), x~_i = (u[:, i] < p_i) where x_i < 0 (else x_i), a += x~_i _in_W[:, i] (one product, then the add)."""
    n, D = x.shape
    a = p["_in_b"].expand(n, -1)
    probs, xt = [], []
    for i in range(D):
        p_i = torch.sigmoid(torch.relu(a) @ p["_h_W"][i : i + 1, :].t() + p["_h_b"][i : i + 1])
        probs.append(p_i)
        x_i = x[:, i : i + 1]
        x_i = torch.where(x_i < 0, (u[:, i : i + 1] < p_i).to(x.dtype), x_i)
        xt.append(x_i)
        a = a + x_i @ p["_in_W"][:, i : i + 1].t()
    return torch.cat(probs, dim=1), torch.cat(xt, dim=1)


def hidden_preactivations(p, xt):
    """a_d for every d, [n, D, H], with the reference's arithmetic (exactly what the kernels compute in float32)."""
    n, D = xt.shape
    a = p["_in_b"].expand(n, -1)
    out = []
    for i in range(D):
        out.append(a)
        a = a + xt[:, i : i + 1] * p["_in_W"][:, i].unsqueeze(0)
    return torch.stack(out, dim=1)


def recipe_loss(x, preds):
    b = x.shape[0]
    return F.binary_cross_entropy_with_logits(preds.reshape(b, -1), x.reshape(b, -1), reduction="none").sum(1).mean()


def trainable(state, dtype=torch.float32, device="cpu"):
    return {k: state[k].detach().to(device=device, dtype=dtype).clone().requires_grad_(True) for k in PARAMS}


def loss_and_grads(state, x, u, dtype=torch.float32, device="cpu"):
    """One forward of x (any shape with n rows) under uniforms u [n, D], the recipe loss on the probabilities and the
    backward.  Returns (p in x's shape, x~, loss, {param: grad}, x grad)."""
    pt = trainable(state, dtype, device)
    xg = x.detach().to(device=device, dtype=dtype).clone().requires_grad_(True)
    probs, xt = forward(pt, xg.view(x.shape[0], -1), u.to(device=device, dtype=dtype))
    probs = probs.view(x.shape)
    loss = recipe_loss(xg.detach(), probs)  # the input gradient goes through the model only
    loss.backward()
    return probs.detach(), xt.detach(), loss.detach(), {k: pt[k].grad for k in PARAMS}, xg.grad


@torch.no_grad()
def sample(state, conditioned_on, u):
    """NADE.sample: x~ of one forward over the canvas; entries >= 0 kept."""
    pt = {k: state[k] for k in PARAMS}
    n = conditioned_on.shape[0]
    return forward(pt, conditioned_on.reshape(n, -1), u)[1].view(conditioned_on.shape)


class TrainState:
    """The NADE recipe's training step: zero_grad, forward, loss, backward, clip_grad_norm_(1e50), Adam at its default
    learning rate, no scheduler (reference nade.py:127-146, trainer.py:173-193)."""

    def __init__(self, state, lr=1e-3, dtype=torch.float32, device="cpu"):
        self.p = trainable(state, dtype, device)
        self.params = [self.p[k] for k in PARAMS]
        self.opt = torch.optim.Adam(self.params, lr=lr)

    def step(self, x, u):
        self.opt.zero_grad()
        probs = forward(self.p, x.reshape(x.shape[0], -1), u)[0]
        loss = recipe_loss(x, probs)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(self.params, 1e50)
        self.opt.step()
        return loss.item(), norm.item()
