"""Restatement of the reference FullyVisibleBeliefNetwork (models/autoregressive/fvbn.py) in torch: the D row weights
packed into one triangle and the forward as one `tril(W, -1)` contraction, plus row 0's constant input, the recipe loss,
gradients, raster-order sampling and the recipe's training step.  Any dtype and device (float32 on the CPU is pinned to
the reference's own outputs in tests/golden/fvbn.pt; float64 on the GPU is the kernels' yardstick; the comparison arm of
tools/bench_fvbn.py is its own module).  Tests and tools only.  State dicts use the reference's keys (`_net.{i}.weight`
[1, max(1, i)], `_net.{i}.bias` [1])."""

import torch
import torch.nn.functional as F


def names(D):
    """Parameter names in the reference's `parameters()` order."""
    return [f"_net.{i}.{kind}" for i in range(D) for kind in ("weight", "bias")]


def n_dims(state):
    return sum(1 for k in state if k.endswith(".bias"))


def offsets(D):
    """Start of row i in the packed triangle: 0 for i = 0, 1 + i (i - 1) / 2 otherwise; T = 1 + D (D - 1) / 2."""
    return [0 if i == 0 else 1 + i * (i - 1) // 2 for i in range(D)], 1 + D * (D - 1) // 2


def dense(p, D):
    """(tril(W, -1) [D, D] with W[i, :i] = the weight of row i >= 1, w0 [1] = row 0's weight, b [D])."""
    rows = [torch.zeros(1, D, dtype=p["_net.0.weight"].dtype, device=p["_net.0.weight"].device)]
    rows += [F.pad(p[f"_net.{i}.weight"], (0, D - i)) for i in range(1, D)]
    W = torch.cat(rows, dim=0)
    b = torch.cat([p[f"_net.{i}.bias"] for i in range(D)])
    return W, p["_net.0.weight"].reshape(1), b


def forward(p, x):
    """Logits of a flat batch x [n, D]: x @ tril(W, -1)^T + b, and row 0's b_0 + w_0 * 0."""
    n, D = x.shape
    W, w0, b = dense(p, D)
    out = x @ W.t() + b
    row0 = b[0] + w0 * torch.zeros(n, 1, dtype=x.dtype, device=x.device)
    return torch.cat([row0, out[:, 1:]], dim=1)


def recipe_loss(x, preds):
    b = x.shape[0]
    return F.binary_cross_entropy_with_logits(preds.reshape(b, -1), x.reshape(b, -1), reduction="none").sum(1).mean()


def trainable(state, dtype=torch.float32, device="cpu"):
    D = n_dims(state)
    return {k: state[k].detach().to(device=device, dtype=dtype).clone().requires_grad_(True) for k in names(D)}


def loss_and_grads(state, x, dtype=torch.float32, device="cpu"):
    """One forward of x (any shape with n rows), the recipe loss and the backward.  Returns (logits in x's shape, loss,
    {param: grad}, x grad)."""
    pt = trainable(state, dtype, device)
    xg = x.detach().to(device=device, dtype=dtype).clone().requires_grad_(True)
    logits = forward(pt, xg.view(x.shape[0], -1)).view(x.shape)
    loss = recipe_loss(xg.detach(), logits)  # the input gradient goes through the model only
    loss.backward()
    return logits.detach(), loss.detach(), {k: t.grad for k, t in pt.items()}, xg.grad


def uniform_sample_fn(uniforms):
    """sample_fn drawing u < sigmoid(logits) from recorded uniforms [h * w, n, c], one [n, c] tensor per call."""
    it = iter(uniforms)
    return lambda logits: (next(it).to(logits.device) < torch.sigmoid(logits)).float()


@torch.no_grad()
def sample(state, canvas, sample_fn):
    """base.AutoregressiveModel.sample: raster order, every channel of a pixel from the full forward of the canvas as it
    stands, entries >= 0 kept."""
    canvas = canvas.clone()
    n, c, h, w = canvas.shape
    p = {k: state[k].to(canvas.dtype) for k in names(c * h * w)}
    for row in range(h):
        for col in range(w):
            logits = forward(p, canvas.view(n, -1)).view(n, c, h, w)[:, :, row, col]
            drawn = sample_fn(logits).view(n, c)
            canvas[:, :, row, col] = torch.where(canvas[:, :, row, col] < 0, drawn, canvas[:, :, row, col])
    return canvas


class TrainState:
    """The FVBN recipe's training step: zero_grad, forward, loss, backward, clip_grad_norm_(1e50), Adam at lr 1e-3, no
    scheduler (reference fvbn.py:80-97, trainer.py:173-193)."""

    def __init__(self, state, lr=1e-3, dtype=torch.float32, device="cpu"):
        self.p = trainable(state, dtype, device)
        self.params = list(self.p.values())
        self.opt = torch.optim.Adam(self.params, lr=lr)

    def step(self, x):
        self.opt.zero_grad()
        logits = forward(self.p, x.reshape(x.shape[0], -1))
        loss = recipe_loss(x, logits)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(self.params, 1e50)
        self.opt.step()
        return loss.item(), norm.item()
