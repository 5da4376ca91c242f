"""CPU restatement of the reference MADE (models/autoregressive/made.py) in float32 torch: connectivity vectors, masks,
forward, recipe loss, a training step and the per-dimension sampler.  Tests only; tests/golden/made.pt (written by the
reference itself) pins it.  State dicts use the reference's keys (`_net.{2l}.weight / bias / mask`)."""

import numpy as np
import torch
import torch.nn.functional as F


def connectivity(input_dim, hidden_dims, mask_set):
    """RandomState(mask_set): permutation of the inputs; per hidden layer l, randint(low_l, input_dim - 1) with low_0 = 0
    and low_l = min of the vector of layer l - 2 (the inputs for l = 1); the outputs repeat the input permutation."""
    rng = np.random.RandomState(seed=mask_set)
    vecs = [rng.permutation(input_dim)]
    for layer, width in enumerate(hidden_dims):
        low = 0 if layer == 0 else int(vecs[layer - 1].min())
        vecs.append(rng.randint(low, input_dim - 1, size=width))
    return vecs + [vecs[0].copy()]


def masks(vecs):
    """0/1 float masks [out, in] per layer: in <= out between hidden layers, in < out into the outputs."""
    out = []
    for layer in range(1, len(vecs)):
        c_in, c_out = torch.from_numpy(vecs[layer - 1]), torch.from_numpy(vecs[layer])
        rel = c_in[None, :] < c_out[:, None] if layer == len(vecs) - 1 else c_in[None, :] <= c_out[:, None]
        out.append(rel.float())
    return out


def n_layers(p):
    return len([k for k in p if k.endswith(".weight")])


def forward(p, x, layer_masks):
    """Sets every `mask`, zeroes the masked weights in place (outside autograd), then Linear/ReLU/.../Linear on
    x.view(n, -1); returns logits of x's shape."""
    h = x.reshape(x.shape[0], -1)
    count = n_layers(p)
    for layer in range(count):
        pre = f"_net.{2 * layer}."
        with torch.no_grad():
            p[pre + "mask"].copy_(layer_masks[layer])
            p[pre + "weight"].mul_(p[pre + "mask"])
        h = F.linear(h, p[pre + "weight"], p[pre + "bias"])
        if layer + 1 < count:
            h = F.relu(h)
    return h.view(x.shape)


def recipe_loss(x, preds):
    b = x.shape[0]
    return F.binary_cross_entropy_with_logits(preds.reshape(b, -1), x.reshape(b, -1), reduction="none").sum(1).mean()


def trainable(p):
    out = {}
    for k, v in p.items():
        t = v.detach().clone().float()
        if not k.endswith("mask") and k not in ("_c", "_h", "_w"):
            t.requires_grad_(True)
        out[k] = t
    return out


def hidden_dims(p):
    count = n_layers(p)
    return [p[f"_net.{2 * layer}.weight"].shape[0] for layer in range(count - 1)]


def loss_and_grads(p, x, mask_set, n_masks=1):
    """One forward with mask set `mask_set % n_masks`, the recipe loss and backward.  Returns (logits, loss,
    {param: grad}, x grad, state after)."""
    pt = trainable(p)
    D = pt["_net.0.weight"].shape[1]
    xg = x.detach().clone().float().requires_grad_(True)
    logits = forward(pt, xg, masks(connectivity(D, hidden_dims(pt), mask_set % n_masks)))
    loss = recipe_loss(xg.detach(), logits)  # the input gradient goes through the model only
    loss.backward()
    grads = {k: v.grad for k, v in pt.items() if v.requires_grad}
    return logits.detach(), loss.detach(), grads, xg.grad, {k: v.detach() for k, v in pt.items()}


class TrainState:
    """The MADE recipe's training step: zero_grad, forward, loss, backward, clip_grad_norm_(1e50), Adam at its default
    learning rate, no scheduler (reference made.py:170-189, trainer.py:173-193)."""

    def __init__(self, p, n_masks=1, lr=1e-3):
        self.p, self.n_masks, self.seed = trainable(p), n_masks, 0
        self.params = [v for v in self.p.values() if v.requires_grad]
        self.opt = torch.optim.Adam(self.params, lr=lr)

    def step(self, x):
        self.opt.zero_grad()
        D = self.p["_net.0.weight"].shape[1]
        vecs = connectivity(D, hidden_dims(self.p), self.seed % self.n_masks)
        self.seed += 1
        loss = recipe_loss(x, forward(self.p, x, masks(vecs)))
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(self.params, 1e50)
        self.opt.step()
        return loss.item(), norm.item()


@torch.no_grad()
def sample(p, mask_set, sample_fn, conditioned_on, n_masks=1):
    """MADE.sample: the dimensions in argsort(ordering), one full forward per dimension, `sample_fn` on the [n] logits
    of that dimension, only entries < 0 overwritten."""
    p = {k: v.clone() for k, v in p.items()}
    D = p["_net.0.weight"].shape[1]
    vecs = connectivity(D, hidden_dims(p), mask_set % n_masks)
    layer_masks = masks(vecs)
    x = conditioned_on.clone()
    flat = x.view(x.shape[0], -1)
    for d in np.argsort(vecs[-1]):
        logits = forward(p, flat, layer_masks)[:, d]
        drawn = sample_fn(logits)
        flat[:, d] = torch.where(flat[:, d] < 0, drawn, flat[:, d])
    return x


def uniform_sample_fn(uniforms):
    """Bernoulli draws from pre-drawn uniforms, one [n] tensor per call."""
    it = iter(uniforms)
    return lambda logits: (next(it).to(logits.device) < torch.sigmoid(logits)).float()
