"""`ReZeroWrapper`: the reference's nn/utils.py ReZeroWrapper (ReZero, Bachlechner et al. 2020, arXiv:2003.04887) on
the library's kernels: y = x + alpha * module(x) with a trainable [1] fp32 scalar alpha initialised to 0."""

import torch
from torch import nn

from .. import _lib as L


class _ReZero(torch.autograd.Function):
    """y = x + alpha f (pg_rezero_fwd, one launch); backward dx = dy, df = alpha dy and dalpha = sum(dy f) in a fixed
    order (pg_rezero_bwd: two launches, one when alpha needs no gradient).  x and f are contiguous fp32 CUDA tensors of
    one shape."""

    @staticmethod
    def forward(ctx, x, f, alpha):
        y = torch.empty_like(x)
        L.rezero_fwd(x, f, alpha, y)
        ctx.save_for_backward(f if ctx.needs_input_grad[2] else None, alpha)
        return y

    @staticmethod
    def backward(ctx, dy):
        f, alpha = ctx.saved_tensors
        dy = dy.contiguous()
        need_x, need_f, need_alpha = ctx.needs_input_grad
        df = torch.empty_like(dy) if need_f else None
        dalpha = torch.empty_like(alpha) if need_alpha else None
        if need_f or need_alpha:
            L.rezero_bwd(dy, f, alpha, df, dalpha)
        return dy if need_x else None, df, dalpha


class ReZeroWrapper(nn.Module):
    """Wraps a given module into a ReZero function: `x + alpha * module(x)` for an input `x`, with `alpha` a trainable
    scalar initialised to 0.  `module(x)` must have `x`'s shape; a different shape raises ValueError (the reference
    would broadcast).

    CUDA fp32 only, with no fallback.  Both operands are made contiguous before the kernels run (a no-op when they
    already are; a copy when the module returns a strided view, as NCHWLayerNorm does), and the output is a contiguous
    tensor.  The forward is fp32 `x + alpha * f` rounded after each operation, bit-identical to torch's; the gradient
    of alpha is summed in a fixed order, so every run gives the same bits."""

    def __init__(self, module):
        """Initializes a new ReZeroWrapper.

        Args:
            module: The module to wrap.
        """
        super().__init__()
        self._module = module
        self._alpha = nn.Parameter(torch.tensor([0.0]))

    def forward(self, x):
        f = self._module(x)
        if f.shape != x.shape:
            raise ValueError(f"ReZeroWrapper: the module's output has shape {tuple(f.shape)}, its input {tuple(x.shape)}; "
                             "ReZero needs them equal")
        if not all(t.is_cuda and t.dtype == torch.float32 for t in (x, f)):
            raise RuntimeError("ReZeroWrapper: x and the module's output must be fp32 CUDA tensors (the CUDA path has no "
                               "CPU fallback)")
        return _ReZero.apply(x.contiguous(), f.contiguous(), self._alpha)
