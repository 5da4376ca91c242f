"""The recipes' losses on the CUDA path.

* `bce_with_logits_sum_mean`: `BCEWithLogits(preds, x, reduction="none").sum(dim=1).mean()` (reference
  models/autoregressive/image_gpt.py:158-162, identical in pixel_cnn.py:159-163, gated_pixel_cnn.py:234-238,
  pixel_snail.py:237-241).  One fused kernel (`pg_bce_logits_fwd_bwd`) computes the summed loss and, in the same pass,
  d loss / d logits, so backward is a scale of a saved tensor.
* `categorical_nll`: a 256-way (K-way) categorical likelihood of 8-bit images, with its bits/dim.  Convention, owned
  here: an image of C channels is modelled with `out_channels = K * C` logits per pixel, and class k of channel c is
  logit channel `k * C + c` -- the NCHW logits viewed as `[N, K, C, H, W]`, the input `F.cross_entropy` takes with
  targets `[N, C, H, W]`.  K is `preds.shape[1] // x.shape[1]` (256 for 8-bit data); the target class of an input value
  x is `categorical_target(x, K)` = `rint(clamp(x, 0, 1) * (K - 1))`, exactly k for the loaders' `k / 255`.
  `pg_categorical_xent_fwd_bwd` computes each image's summed NLL and, in the same launch, d loss / d logits.
* `logistic_mixture_nll`: the discretised mixture of logistics (DMOL) of PixelCNN++, with its bits/dim.  Convention,
  owned here: an image of C channels, values in [0, 1], is modelled with M logistic components per pixel and K bins per
  channel (K = 256 for 8-bit data) by `out_channels = M * G` channels, `G = (C + 1)(C + 2) / 2` (10 for RGB, 3 for one
  channel); M is `preds.shape[1] // G`.  With `T = C (C - 1) / 2`, the NCHW channel of each parameter is: mixture logit
  `pi_m` at `m`; mean `mu_{m,c}` at `M + m*C + c`; raw log-scale `ls_{m,c}` at `M + M*C + m*C + c`; raw coupling
  coefficient `r_{m,t}` at `M + 2*M*C + m*T + t`, `t = c(c-1)/2 + j` for `j < c` -- grouped by kind, not PixelCNN++'s
  per-channel interleaving, which does not extend past C = 3.  The bin of x is `categorical_target(x, K)`, its centre
  `x'_k = 2k/(K-1) - 1` and half-width `h = 1/(K-1)`.  Per component and channel: `log_s = max(ls, -7)`;
  `mu' = mu + sum_{j<c} tanh(r_{m,t(c,j)}) x'_{k_j}` (coupled to the bin centres of the pixel's earlier channels);
  `a = (x' - mu' + h) e^-log_s`, `b = (x' - mu' - h) e^-log_s`; the bin's log-mass `lp` is `-softplus(-a)` for bin 0,
  `-softplus(b)` for bin K - 1 and `-softplus(-a) - softplus(b) + log(-expm1(-(a - b)))` otherwise: the exact
  `log(sigmoid(a) - sigmoid(b))`, without PixelCNN++'s `cdf_delta > 1e-5` switch to `log_pdf_mid - log(127.5)`, so
  the loss is the exact discrete NLL and its bits/dim compares directly with the papers'.  Per-pixel NLL:
  `-logsumexp_m(log_softmax(pi)_m + sum_c lp_{m,c})`.  `pg_logistic_mixture_fwd_bwd` computes each image's summed NLL
  and, in the same launch, d loss / d preds.
* `logistic_prior_nll`: NICE's negative log-likelihood under a logistic prior (reference models/flow/nice.py:205-213).
  `pg_logistic_prior_fwd_bwd` gives each image's prior log-likelihood and, in the same pass, its gradient, so backward
  is again a scale of a saved tensor.
* `vae_elbo`: the VAE recipes' negative ELBO dict (reference models/vae/vae.py `loss_fn` in `reproduce`); the
  reconstruction term is `pg_bce_logits_fwd_bwd` again.
* `mse_loss` / `mse_loss_pm`: F.mse_loss (the mean over every element) on `pg_mse_mean`, with a fixed-order sum and a
  gradient for both operands; `vq_vae_loss` / `vq_vae_2_loss` are the VQ-VAE recipes' loss dicts (reference
  models/vae/{vq_vae,vq_vae_2}.py `loss_fn` in `reproduce`)."""

import math

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


def categorical_target(x, n_classes):
    """The class index of each input value under `categorical_nll`: rint(clamp(x, 0, 1) * (n_classes - 1)) in fp32 (the
    rule the loss kernel applies; for x = k / (n_classes - 1) in fp32 it is k)."""
    return torch.round(x.float().clamp(0, 1) * float(n_classes - 1)).long()


def _categorical_classes(preds, x):
    """K of `preds` [N, K * C, ...] against `x` [N, C, ...]; raises ValueError on shapes the convention does not fit."""
    if preds.dim() < 2 or x.dim() != preds.dim() or preds.shape[0] != x.shape[0] or preds.shape[2:] != x.shape[2:]:
        raise ValueError(f"categorical_nll: preds {tuple(preds.shape)} is not [N, K * C, ...] for x {tuple(x.shape)}")
    c = x.shape[1]
    if c < 1 or preds.shape[1] % c != 0 or preds.shape[1] // c < 2:
        raise ValueError(f"categorical_nll: {preds.shape[1]} logit channels are not K * C with K >= 2 for C = {c}")
    return preds.shape[1] // c


class _CategoricalNLL(torch.autograd.Function):
    """Mean over images of the summed categorical NLL (nats); backward scales the saved d loss / d logits."""

    @staticmethod
    def forward(ctx, logits, x):
        if not logits.is_cuda or not x.is_cuda:
            raise RuntimeError("categorical_nll: CUDA tensors only (no CPU fallback)")
        n = x.shape[0]
        lg = logits.contiguous().float()
        image_nll = torch.zeros(n, dtype=torch.float32, device=lg.device)
        dlogits = torch.empty_like(lg) if ctx.needs_input_grad[0] else None
        L.categorical_xent(lg, x.contiguous().float(), 1.0 / n, image_nll=image_nll, dlogits=dlogits)
        ctx.save_for_backward(dlogits)
        return image_nll.mean()

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None


def categorical_nll(x, _, preds):
    """loss_fn(x, _, preds) of the 8-bit recipes: preds [N, K * C, H, W] logits, x [N, C, H, W] in [0, 1] (see the
    convention above).  Returns {"loss": mean over images of the summed NLL in nats,
    "bits_per_dim": loss / (C H W ln 2)}."""
    _categorical_classes(preds, x)
    loss = _CategoricalNLL.apply(preds, x)
    dims = x[0].numel()
    return {"loss": loss, "bits_per_dim": loss / (dims * math.log(2.0))}


def _logistic_mixture_shape(preds, x):
    """(M, C) of `preds` [N, M * G, ...] against `x` [N, C, ...]; raises ValueError on shapes the convention does not
    fit."""
    if preds.dim() < 2 or x.dim() != preds.dim() or preds.shape[0] != x.shape[0] or preds.shape[2:] != x.shape[2:]:
        raise ValueError(f"logistic_mixture_nll: preds {tuple(preds.shape)} is not [N, M * G, ...] for x "
                         f"{tuple(x.shape)}")
    c = x.shape[1]
    g = (c + 1) * (c + 2) // 2
    if c < 1 or preds.shape[1] < g or preds.shape[1] % g != 0:
        raise ValueError(f"logistic_mixture_nll: {preds.shape[1]} channels are not a positive multiple of "
                         f"G = (C + 1)(C + 2) / 2 = {g} for C = {c}")
    return preds.shape[1] // g, c


class _LogisticMixtureNLL(torch.autograd.Function):
    """Mean over images of the summed discretised logistic mixture NLL (nats); backward scales the saved
    d loss / d preds."""

    @staticmethod
    def forward(ctx, preds, x, n_mixtures, n_bins):
        if not preds.is_cuda or not x.is_cuda:
            raise RuntimeError("logistic_mixture_nll: CUDA tensors only (no CPU fallback)")
        n = x.shape[0]
        p = preds.contiguous().float()
        image_nll = torch.zeros(n, dtype=torch.float32, device=p.device)
        dpreds = torch.empty_like(p) if ctx.needs_input_grad[0] else None
        L.logistic_mixture_nll_kernel(p, x.contiguous().float(), n_mixtures, n_bins, 1.0 / n, image_nll=image_nll,
                                      dpreds=dpreds)
        ctx.save_for_backward(dpreds)
        return image_nll.mean()

    @staticmethod
    def backward(ctx, g):
        (dpreds,) = ctx.saved_tensors
        return dpreds * g, None, None, None


def logistic_mixture_nll(x, _, preds, n_bins=256):
    """loss_fn(x, _, preds) for a discretised logistic mixture head: preds [N, M * G, H, W], x [N, C, H, W] in [0, 1],
    `n_bins` bins per channel (see the convention above).  Returns {"loss": mean over images of the summed NLL in nats,
    "bits_per_dim": loss / (C H W ln 2)}.  The bin's mass is the exact difference of the logistic CDF at its edges (the
    edge bins take the tails), with no PixelCNN++ `cdf_delta > 1e-5` threshold, so bits/dim is the exact discrete NLL."""
    if int(n_bins) < 2:
        raise ValueError(f"logistic_mixture_nll: n_bins {n_bins} < 2")
    m, _c = _logistic_mixture_shape(preds, x)
    loss = _LogisticMixtureNLL.apply(preds, x, m, int(n_bins))
    dims = x[0].numel()
    return {"loss": loss, "bits_per_dim": loss / (dims * math.log(2.0))}


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


class _MSEMean(torch.autograd.Function):
    """mean((a - b)^2) over the first `cols` columns of two fp32 [rows, pitch] matrices; both get a gradient."""

    @staticmethod
    def forward(ctx, a, b, cols, numel):
        loss_sum = torch.zeros(1, dtype=torch.float32, device=a.device)
        L.mse_mean(a, b, cols, loss_sum=loss_sum)
        ctx.save_for_backward(a, b)
        ctx.cols, ctx.numel = cols, numel
        return (loss_sum / numel).reshape(())

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        da = torch.empty(a.shape, dtype=torch.float32, device=a.device) if ctx.needs_input_grad[0] else None
        db = torch.empty(b.shape, dtype=torch.float32, device=b.device) if ctx.needs_input_grad[1] else None
        L.mse_mean(a, b, ctx.cols, g=g.reshape(1).float().contiguous(), scale=2.0 / ctx.numel, da=da, db=db)
        return da, db, None, None


def _mse_operand(t, who):
    if not t.is_cuda:
        raise RuntimeError(f"{who}: CUDA tensors only (no CPU fallback)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{who}: fp32 tensors only; got {t.dtype}")
    return t.contiguous()


def mse_loss(preds, x):
    """F.mse_loss(preds, x): the mean of (preds - x)^2 over every element of two tensors of one shape."""
    if preds.shape != x.shape:
        raise ValueError(f"mse_loss: shapes {tuple(preds.shape)} and {tuple(x.shape)} differ")
    a, b = _mse_operand(preds, "mse_loss"), _mse_operand(x, "mse_loss")
    w = a.shape[-1] if a.dim() else 1
    return _MSEMean.apply(a.view(-1, w), b.view(-1, w), w, a.numel())


def mse_loss_pm(a, b, cols):
    """F.mse_loss of two pixel-major activations: the first `cols` columns of fp32 [P, >=cols] matrices, each a whole
    matrix (their pad columns, if any, get a zero gradient)."""
    a, b = _mse_operand(a, "mse_loss_pm"), _mse_operand(b, "mse_loss_pm")
    assert a.shape[0] == b.shape[0] and min(a.shape[1], b.shape[1]) >= cols
    return _MSEMean.apply(a, b, cols, a.shape[0] * cols)


def vq_vae_loss(x, _, preds):
    """loss_fn(x, _, preds) of the VQ-VAE recipe: preds = (x_hat, vq_loss); returns the reference's dict
    {vq_loss, reconstruction_loss: mse(x_hat, x), loss: reconstruction_loss + vq_loss}."""
    preds, vq_loss = preds
    recon_loss = mse_loss(preds, x)
    return {"vq_loss": vq_loss, "reconstruction_loss": recon_loss, "loss": recon_loss + vq_loss}


def vq_vae_2_loss(x, _, preds):
    """loss_fn(x, _, preds) of the VQ-VAE-2 recipe: as `vq_vae_loss` with loss = reconstruction_loss + 0.25 vq_loss."""
    preds, vq_loss = preds
    recon_loss = mse_loss(preds, x)
    return {"vq_loss": vq_loss, "reconstruction_loss": recon_loss, "loss": recon_loss + 0.25 * vq_loss}
