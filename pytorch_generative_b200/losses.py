"""The recipes' loss on the CUDA path: `BCEWithLogits(preds, x, reduction="none").sum(dim=1).mean()`
(reference models/autoregressive/image_gpt.py:158-162, identical in pixel_cnn.py:159-163, gated_pixel_cnn.py:234-238,
pixel_snail.py:237-241).  One fused kernel (`pg_bce_logits_fwd_bwd`) computes the summed loss and, in the same pass,
d loss / d logits, so backward is a scale of a saved tensor."""

import torch

from . import _lib as L


class _BCESumMean(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target):
        if not logits.is_cuda:
            raise RuntimeError("bce_with_logits_sum_mean: CUDA tensors only (no CPU fallback)")
        n = logits.shape[0]
        lg = logits.contiguous().float()
        tg = target.contiguous().float()
        loss_sum = torch.zeros(1, dtype=torch.float32, device=lg.device)
        dlogits = torch.empty_like(lg) if ctx.needs_input_grad[0] else None
        L.bce_logits(lg.view(-1), tg.view(-1), 1.0 / n, loss_sum, None if dlogits is None else dlogits.view(-1))
        ctx.save_for_backward(dlogits)
        return (loss_sum / n).reshape(())

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None


def bce_with_logits_sum_mean(preds, x):
    """loss_fn(x, _, preds) of the reference recipes; works on any memory layout (elementwise + full reduction)."""
    assert preds.shape == x.shape or preds.numel() == x.numel()
    return _BCESumMean.apply(preds.reshape(x.shape), x)
