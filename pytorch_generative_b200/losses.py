"""The recipes' losses on the CUDA path.

* `bce_with_logits_sum_mean`: `BCEWithLogits(preds, x, reduction="none").sum(dim=1).mean()` (reference
  models/autoregressive/image_gpt.py:158-162, identical in pixel_cnn.py:159-163, gated_pixel_cnn.py:234-238,
  pixel_snail.py:237-241).  One fused kernel (`pg_bce_logits_fwd_bwd`) computes the summed loss and, in the same pass,
  d loss / d logits, so backward is a scale of a saved tensor.
* `logistic_prior_nll`: NICE's negative log-likelihood under a logistic prior (reference models/flow/nice.py:205-213).
  `pg_logistic_prior_fwd_bwd` gives each image's prior log-likelihood and, in the same pass, its gradient, so backward
  is again a scale of a saved tensor.
* `vae_elbo`: the VAE recipes' negative ELBO dict (reference models/vae/vae.py `loss_fn` in `reproduce`); the
  reconstruction term is `pg_bce_logits_fwd_bwd` again."""

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


class _LogisticPrior(torch.autograd.Function):
    """log_prob[b] = -sum over the image of softplus(z) + softplus(-z), the logistic prior's log-density."""

    @staticmethod
    def forward(ctx, z):
        if not z.is_cuda:
            raise RuntimeError("logistic_prior_nll: CUDA tensors only (no CPU fallback)")
        n = z.shape[0]
        zf = z.reshape(n, -1).contiguous().float()
        log_prob = torch.empty(n, dtype=torch.float32, device=zf.device)
        dz = torch.empty_like(zf) if ctx.needs_input_grad[0] else None
        L.logistic_prior_fwd_bwd(zf, log_prob, dz, grad_scale=-1.0)  # dz = d log_prob[b] / dz = -tanh(z / 2)
        ctx.save_for_backward(dz)
        ctx.shape = z.shape
        return log_prob

    @staticmethod
    def backward(ctx, g):
        (dz,) = ctx.saved_tensors
        return (dz * g.view(-1, 1)).view(ctx.shape)


def logistic_prior_nll(x, _, preds):
    """loss_fn(x, _, preds) of the NICE recipe: preds = (z, log_det_J); returns the reference's dict
    {loss: -mean(log_prob + log_det_J), prior_log_likelihood: mean(log_prob), log_det_J: mean(log_det_J)}."""
    z, log_det_J = preds
    log_prob = _LogisticPrior.apply(z)
    loss = log_prob + log_det_J
    return {"loss": -loss.mean(), "prior_log_likelihood": log_prob.mean(), "log_det_J": log_det_J.mean()}


def vae_elbo(x, _, preds):
    """loss_fn(x, _, preds) of the VAE / BetaVAE recipes: preds = (logits, kl); returns the reference's dict
    {recon_loss: mean over images of the summed BCE, kl_div: mean(kl), loss: their sum, the mean negative ELBO}."""
    logits, kl_div = preds
    recon_loss = bce_with_logits_sum_mean(logits, x)
    kl_div = kl_div.mean()
    return {"recon_loss": recon_loss, "kl_div": kl_div, "loss": recon_loss + kl_div}
