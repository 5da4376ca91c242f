"""Base classes of the drop-in models (API of reference pytorch_generative/models/base.py:28-120).

Behavioural contract kept from the reference (SURVEY.md §8a row 11):
  * `__call__` records the image shape of the first 4-D input in buffers `_c, _h, _w` (int64 scalars that are
    part of the state dict) — base.py:41-46, 55-61;
  * `load_state_dict` registers those buffers first when the checkpoint has them — base.py:48-53;
  * `sample(n_samples=None, conditioned_on=None)` walks the image in raster order, draws all channels of one
    pixel from `sample_fn(logits[:, :, r, c])` and only overwrites entries < 0 — base.py:97-120;
  * `device` property — base.py:63-65.
"""

import abc

import torch
from torch import nn

from .. import _lib as L


def _bernoulli_from_logits(logits):
    """Default `sample_fn` (reference base.py:9-10): one Bernoulli draw per logit."""
    return torch.bernoulli(torch.sigmoid(logits))


class CategoricalSampleFn:
    """`sample_fn` of models trained with `losses.categorical_nll`: for one pixel's logits [n, n_classes * C] (class k of
    channel c at k * C + c), draws each channel's class k with `pg_categorical_sample` from uniforms of `torch.rand` on
    the logits' device and returns [n, C] fp32 values k / (n_classes - 1), the grid the 8-bit loaders produce."""

    def __init__(self, n_classes=256):
        if int(n_classes) < 2:
            raise ValueError(f"categorical_sample_fn: n_classes {n_classes} < 2")
        self.n_classes = int(n_classes)

    def __call__(self, logits):
        n = logits.shape[0]
        logits = logits.reshape(n, -1)
        if logits.shape[1] % self.n_classes:
            raise ValueError(f"categorical_sample_fn: {logits.shape[1]} logits per pixel are not a multiple of "
                             f"{self.n_classes} classes")
        logits = logits.float()
        if logits.stride(1) != 1:
            logits = logits.contiguous()
        c = logits.shape[1] // self.n_classes
        u = torch.rand(n, c, device=logits.device)
        out = torch.empty(n, c, dtype=torch.float32, device=logits.device)
        L.categorical_sample(logits, u, out)
        return out

    def __repr__(self):
        return f"categorical_sample_fn(n_classes={self.n_classes})"


def categorical_sample_fn(n_classes=256):
    """The `sample_fn` for `n_classes`-way categorical logits (see `CategoricalSampleFn`); picklable and deep-copyable."""
    return CategoricalSampleFn(n_classes)


class LogisticMixtureSampleFn:
    """`sample_fn` of models trained with `losses.logistic_mixture_nll`: for one pixel's parameters [n, n_mixtures * G]
    (the layout `losses` states), draws a component and then each channel's bin in ascending channel order with
    `pg_logistic_mixture_sample`, from uniforms of `torch.rand` on the logits' device, and returns [n, C] fp32 values
    k / (n_bins - 1), the grid the 8-bit loaders produce.  C is the channel count whose G = (C + 1)(C + 2) / 2 is the
    number of parameters per component.

    Limitation: the channels of one pixel are drawn together, each coupled to the bins drawn for the earlier ones.
    When `sample()` is conditioned on some channels of a pixel but not others, the drawn channels are coupled to the
    drawn values, not the given ones (which `sample()` then keeps in place of the draws)."""

    def __init__(self, n_mixtures=10, n_bins=256):
        if int(n_mixtures) < 1:
            raise ValueError(f"logistic_mixture_sample_fn: n_mixtures {n_mixtures} < 1")
        if int(n_bins) < 2:
            raise ValueError(f"logistic_mixture_sample_fn: n_bins {n_bins} < 2")
        self.n_mixtures, self.n_bins = int(n_mixtures), int(n_bins)

    def channels(self, n_params):
        """C of a pixel with `n_params` parameters: n_params = n_mixtures * (C + 1)(C + 2) / 2, else ValueError."""
        if n_params % self.n_mixtures == 0:
            g = n_params // self.n_mixtures
            c = 1
            while (c + 1) * (c + 2) // 2 < g:
                c += 1
            if (c + 1) * (c + 2) // 2 == g:
                return c
        raise ValueError(f"logistic_mixture_sample_fn: {n_params} parameters per pixel are not "
                         f"{self.n_mixtures} x (C + 1)(C + 2) / 2 for any C >= 1")

    def __call__(self, logits):
        n = logits.shape[0]
        logits = logits.reshape(n, -1)
        c = self.channels(logits.shape[1])
        logits = logits.float()
        if logits.stride(1) != 1:
            logits = logits.contiguous()
        u = torch.rand(n, 1 + c, device=logits.device)
        out = torch.empty(n, c, dtype=torch.float32, device=logits.device)
        L.logistic_mixture_sample(logits, u, out, self.n_mixtures, self.n_bins)
        return out

    def __repr__(self):
        return f"logistic_mixture_sample_fn(n_mixtures={self.n_mixtures}, n_bins={self.n_bins})"


def logistic_mixture_sample_fn(n_mixtures=10, n_bins=256):
    """The `sample_fn` for a discretised logistic mixture head of `n_mixtures` components (see
    `LogisticMixtureSampleFn`); picklable and deep-copyable."""
    return LogisticMixtureSampleFn(n_mixtures, n_bins)


class GenerativeModel(abc.ABC, nn.Module):
    """Shape-tracking nn.Module base."""

    def __call__(self, x, *args, **kwargs):
        if getattr(self, "_c", None) is None and x.dim() == 4:
            self._register_shape(*x.shape[1:])
        return super().__call__(x, *args, **kwargs)

    def load_state_dict(self, state_dict, strict=True):
        if "_c" in state_dict and not getattr(self, "_c", None):
            self._register_shape(state_dict["_c"], state_dict["_h"], state_dict["_w"])
        return super().load_state_dict(state_dict, strict)

    def _register_shape(self, c, h, w):
        as_t = lambda v: v if torch.is_tensor(v) else torch.tensor(v)
        self.register_buffer("_c", as_t(c))
        self.register_buffer("_h", as_t(h))
        self.register_buffer("_w", as_t(w))

    @property
    def device(self):
        return next(self.parameters()).device

    # Runtime caches (sampler graphs and buffers, ImageGPT's cast plan, the bucket hook) stay out of pickles and deep
    # copies: they are rebuilt on demand, a CUDA graph cannot be copied, and a copy must not use the original's buffers.
    _RUNTIME_CACHES = ("_pixel_states", "_cast_plan", "_grad_bucket_hook")

    def __getstate__(self):
        state = self.__dict__.copy()
        for key in self._RUNTIME_CACHES:
            state.pop(key, None)
        return state

    @abc.abstractmethod
    def sample(self, n_samples):
        ...


class AutoregressiveModel(GenerativeModel):
    """Adds raster-scan ancestral sampling on top of `forward`."""

    def __init__(self, sample_fn=None):
        super().__init__()
        self._sample_fn = sample_fn or _bernoulli_from_logits

    def _start_canvas(self, n_samples, conditioned_on):
        assert (
            n_samples is not None or conditioned_on is not None
        ), 'Must provided one, and only one, of "n_samples" or "conditioned_on"'
        if conditioned_on is not None:
            return conditioned_on.clone()
        shape = (n_samples, int(self._c), int(self._h), int(self._w))
        return torch.full(shape, -1.0, device=self.device)

    # Models whose forward is exactly row-causal (the logits of image row r depend on rows <= r only, and every
    # kernel computes an output row from the same operands in the same order whatever the image height) can evaluate
    # a pixel on the top (r + 1) rows of the canvas: bit-identical logits for roughly half the work on average.
    _row_truncated_sampling = True

    @torch.no_grad()
    def sample(self, n_samples=None, conditioned_on=None):
        """Generates samples pixel by pixel; entries of `conditioned_on` that are >= 0 are kept."""
        canvas = self._start_canvas(n_samples, conditioned_on)
        n, c, h, w = canvas.shape
        for row in range(h):
            rows = row + 1 if self._row_truncated_sampling else h
            for col in range(w):
                logits = self.forward(canvas[:, :, :rows])[:, :, row, col]
                drawn = self._sample_fn(logits).view(n, c)
                current = canvas[:, :, row, col]
                canvas[:, :, row, col] = torch.where(current < 0, drawn, current)
        return canvas


class VariationalAutoEncoder(GenerativeModel):
    """Base of the VAEs (reference base.py:123-134): `sample(n)` is `sample_fn(_sample(n))` without autograd."""

    def __init__(self, sample_fn=None):
        super().__init__()
        self._sample_fn = sample_fn or _bernoulli_from_logits

    @abc.abstractmethod
    def _sample(self, n_samples):
        ...

    @torch.no_grad()
    def sample(self, n_samples):
        return self._sample_fn(self._sample(n_samples))
