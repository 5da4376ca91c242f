"""NADE on the CUDA path — API of reference models/autoregressive/nade.py (`NADE`, `reproduce`).

Same constructor, parameters (`_in_W [H, D]`, `_in_b [H]`, `_h_W [D, H]`, `_h_b [D]`, in that order, the weights
`kaiming_normal_` in that order, the biases zero), `auto_reshape` behaviour and results:

  * `forward` returns the probabilities p (not logits), viewed to the input's shape;
  * entries < 0 are drawn, in `forward` too: x~_d = Bernoulli(p_d) where x_d < 0, and x~ feeds the hidden layer.  No
    gradient flows through a drawn entry (dx is 0 there) and the `_in_W` gradient uses x~;
  * `sample` returns x~ with every entry >= 0 of `conditioned_on` kept bit for bit.  `sample_fn` is stored and never
    called: the draws are Bernoulli(probs=p), as in the reference.

The scan over the D dimensions is one launch of `pg_nade_fwd` (after a transpose of `_in_W`): one image per warp at
H <= 512, the hidden pre-activation `a` in registers, accumulated with the reference's separately rounded multiply and
add, and each probability complete before `a` takes the next input.  So the training forward, a forward with entries
to draw and `sample()` are the same kernel, and the forward never asks the host whether an entry is negative.  The
uniforms come from `torch.rand(n, D)` on the model's device (the global CUDA generator) on every call.  With gradients
the forward also keeps `a` every `_lib.NADE_CHUNK` dimensions; `pg_nade_bwd` recomputes each chunk from them and walks
it backwards.
"""

import torch
from torch import nn

from .. import _lib as L
from . import base


def _require_cuda(x, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")


class _NadeScan(torch.autograd.Function):
    """p = NADE(x) for x [n, D] under uniforms u [n, D]; returns (p, x~), x~ without gradient.  `grads`: whether a
    backward can follow (the checkpoints are kept only then)."""

    @staticmethod
    def forward(ctx, grads, x, u, in_w, in_b, h_w, h_b):
        n, D = x.shape
        H = in_b.numel()
        p = torch.empty(n, D, dtype=torch.float32, device=x.device)
        xt = torch.empty_like(p)
        ckpt = torch.empty(n, -(-D // L.NADE_CHUNK), H, dtype=torch.float32, device=x.device) if grads else None
        L.nade_fwd(x, u, in_w, in_b, h_w, h_b, p, xt, ckpt)
        ctx.mark_non_differentiable(xt)
        if grads:
            ctx.save_for_backward(x, xt, p, ckpt, in_w, h_w)
        return p, xt

    @staticmethod
    def backward(ctx, g, _):
        x, xt, p, ckpt, in_w, h_w = ctx.saved_tensors
        zeros = lambda t: torch.zeros_like(t, dtype=torch.float32)
        d_in_w, d_in_b, d_h_w, d_h_b = zeros(in_w), torch.zeros(in_w.shape[0], device=x.device), zeros(h_w), \
            torch.zeros(h_w.shape[0], device=x.device)
        dx = zeros(x) if ctx.needs_input_grad[1] else None
        L.nade_bwd(x, xt, p, g.contiguous().float(), ckpt, in_w, h_w, d_in_w, d_in_b, d_h_w, d_h_b, dx)
        return None, dx, None, d_in_w, d_in_b, d_h_w, d_h_b


class NADE(base.AutoregressiveModel):
    """The Neural Autoregressive Distribution Estimator (reference nade.py:18-90)."""

    def __init__(self, input_dim, hidden_dim, sample_fn=None):
        super().__init__(sample_fn)
        self._input_dim = input_dim
        self._in_W = nn.Parameter(torch.zeros(hidden_dim, self._input_dim))
        self._in_b = nn.Parameter(torch.zeros(hidden_dim,))
        self._h_W = nn.Parameter(torch.zeros(self._input_dim, hidden_dim))
        self._h_b = nn.Parameter(torch.zeros(self._input_dim,))
        nn.init.kaiming_normal_(self._in_W)
        nn.init.kaiming_normal_(self._h_W)

    def _uniforms(self, n, device):
        """The uniforms of one call's draws, [n, input_dim] (tests replace this to supply their own)."""
        return torch.rand(n, self._input_dim, device=device)

    def _forward(self, x):
        """(p, x~) of a flat batch x [n, input_dim]."""
        _require_cuda(x, "NADE")
        x = x.contiguous().float()
        u = self._uniforms(x.shape[0], x.device)
        params = (self._in_W, self._in_b, self._h_W, self._h_b)
        # Function.forward sees needs_input_grad from requires_grad alone, whatever the grad mode
        grads = torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in params))
        return _NadeScan.apply(grads, x, u, *params)

    def forward(self, x):
        """Probabilities of every dimension; x is (n, input_dim) or an image batch (n, c, h, w) with c*h*w = input_dim."""
        return self._forward(x.view(x.shape[0], -1))[0].view(x.shape)

    @torch.no_grad()
    def sample(self, n_samples=None, conditioned_on=None):
        """Draws the entries < 0 of `conditioned_on` (or of a fresh canvas of n_samples images) in one scan."""
        canvas = self._start_canvas(n_samples, conditioned_on)
        return self._forward(canvas.view(canvas.shape[0], -1))[1].view(canvas.shape)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference nade.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_nade(*args, **kwargs)
