"""MADE on the CUDA path — API of reference models/autoregressive/made.py (`MaskedLinear`, `MADE`, `reproduce`).

Same constructor, module tree and state-dict keys (`_net.{0,2,...}.weight / bias / mask`, plus `_c/_h/_w` after an
image forward), the same `auto_reshape` behaviour and the same mask bookkeeping:

  * mask set `s` is drawn from `np.random.RandomState(s)` with the reference's call sequence (`permutation` of the
    inputs, then one `randint` per hidden layer), and `forward` and `sample` each take the next set of the rotation
    `_mask_seed % n_masks` and advance `_mask_seed` by one;
  * every layer's `mask` buffer holds the last set used, and masked weights are zeroed in place (and stay zero: once
    `n_masks > 1` sets have been applied, a weight carries the product of their masks, as the reference's in-place
    multiply leaves it).

The masks themselves are never built on the host: the connectivity vectors (D + sum(hidden_dims) ints per set) are
cached per set on the device, and `pg_made_mask_cast` derives mask[o, i] = conn_in[i] <= conn_out[o] (`<` on the output
layer) while it zeroes the fp32 weight and writes the bf16 GEMM operand.  Each layer then runs on the tensor-core GEMM:
`ops.linear_fwd` with the ReLU in its epilogue, `ops.linear_dgrad` with ReLU' from the layer's output, `ops.linear_wgrad`
with the fused bias gradient.  As in the reference the mask is outside autograd, so weight gradients are dense.  The
inputs become a bf16 operand, which is exact for the 0/1 images of the recipe.

`sample` visits the dimensions in `argsort(ordering)` and calls `sample_fn` once per dimension with the [n] logits of
that dimension.  With hidden layers it is incremental: the first layer's pre-activation h1 = W1 x + b1 is kept in fp32
for the current canvas and updated by one column of W1 per drawn dimension (`pg_made_sample_step`), and only row d of
the output layer is evaluated, so a step costs O(hidden) per image instead of a full forward.  Deeper stacks recompute
their middle layers per step on the GEMM.  The step is captured once in a CUDA graph and replayed D times.  A MADE
without hidden layers samples with one full forward per dimension.
"""

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .. import ops
from . import base

BF16, F32 = torch.bfloat16, torch.float32


def _pitch(d):
    """Columns of a GEMM operand holding `d` features: the 16-byte operand pitch, zero in the pad."""
    return ops.round_up(d, 8)


def _require_cuda(x, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")


def _operand(x):
    """bf16 [n, pitch(d)] copy of an fp32 [n, d] matrix, zero in the pad columns."""
    n, d = x.shape
    out = (torch.empty if _pitch(d) == d else torch.zeros)((n, _pitch(d)), dtype=BF16, device=x.device)
    L.act_cast(x.contiguous().float(), L.ACT_NONE, out[:, :d])
    return out


def _padded_bias(bias):
    if bias is None:
        return None
    bias = bias.detach()
    if _pitch(bias.numel()) == bias.numel():
        return bias
    return torch.nn.functional.pad(bias, (0, _pitch(bias.numel()) - bias.numel()))


def connectivity(input_dim, hidden_dims, mask_set):
    """The connectivity vectors [inputs, hidden layer 1, ..., outputs] of one mask set, drawn from
    `RandomState(mask_set)` in the reference's order: a permutation of the inputs, then per hidden layer integers in
    [low, input_dim - 1) where `low` is 0 for the first hidden layer and, for layer l > 1, the minimum of the vector two
    below it.  The outputs reuse the input permutation."""
    rng = np.random.RandomState(seed=mask_set)
    vectors = [rng.permutation(input_dim)]
    for layer, width in enumerate(hidden_dims):
        low = np.min(vectors[layer - 1]) if layer > 0 else 0
        vectors.append(rng.randint(low, input_dim - 1, size=width))
    vectors.append(vectors[0].copy())
    return vectors


class _MaskedStack(torch.autograd.Function):
    """x -> relu(W_0 x + b_0) -> ... -> W_L h + b_L over bf16 operands [pitch(out), pitch(in)] whose masks are already
    applied.  `layers`: [(w_bf16, padded bias or None, out_features)]; `params`: each layer's weight, then its bias if
    it has one (the gradients flow to those)."""

    @staticmethod
    def forward(ctx, x, layers, *params):
        acts = [_operand(x)]
        for i, (wq, bias, _) in enumerate(layers):
            if i + 1 < len(layers):
                acts.append(ops.linear_fwd(acts[-1], wq, bias, act=L.ACT_RELU)[0])
            else:
                y = ops.linear_fwd(acts[-1], wq, bias, want_bf16=False, want_f32=True)[2]
        ctx.save_for_backward(*acts)
        ctx.layers, ctx.in_features = layers, x.shape[1]
        out = layers[-1][2]
        return y if y.shape[1] == out else y[:, :out].contiguous()

    @staticmethod
    def backward(ctx, g):
        acts = ctx.saved_tensors
        dy = _operand(g)
        grads = []
        for i in reversed(range(len(ctx.layers))):
            wq, bias, out = ctx.layers[i]
            a = acts[i]
            dw = torch.zeros(wq.shape, dtype=F32, device=g.device)
            db = None if bias is None else torch.zeros(wq.shape[0], dtype=F32, device=g.device)
            ops.linear_wgrad(dy, a, dw, db)
            cin = ctx.layers[i - 1][2] if i > 0 else ctx.in_features
            dw = dw if dw.shape == (out, cin) else dw[:out, :cin].contiguous()
            grads = [dw] + ([] if db is None else [db[:out]]) + grads
            if i > 0:
                dy = ops.linear_dgrad(dy, wq, aux=a, dact=L.ACT_RELU_OUT)   # ReLU' from the layer's input activation
            elif ctx.needs_input_grad[0]:
                dx = ops.linear_dgrad(dy, wq, want_f32=True)[1]
                dx_in = dx if dx.shape[1] == cin else dx[:, :cin].contiguous()
        return (dx_in if ctx.needs_input_grad[0] else None, None, *grads)


def _stack(x, layers, modules):
    params = [t for m in modules for t in (m.weight, m.bias) if t is not None]
    return _MaskedStack.apply(x, layers, *params)


class MaskedLinear(nn.Linear):
    """A Linear layer whose weights are multiplied by a 0/1 `mask` buffer (reference made.py:22-34).  `forward` zeroes
    the masked weights in place, as the reference does, and contracts on the bf16 tensor-core GEMM."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__(in_features, out_features, bias)
        self.register_buffer("mask", torch.ones((out_features, in_features)))

    def set_mask(self, mask):
        self.mask.data.copy_(mask)

    def forward(self, x):
        _require_cuda(x, "MaskedLinear")
        self.weight.data *= self.mask
        wq = _operand(self.weight.detach())
        if wq.shape[0] != _pitch(self.out_features):
            rows = torch.zeros(_pitch(self.out_features), wq.shape[1], dtype=BF16, device=wq.device)
            rows[: self.out_features] = wq
            wq = rows
        lead = x.shape[:-1]
        y = _stack(x.reshape(-1, self.in_features), [(wq, _padded_bias(self.bias), self.out_features)], [self])
        return y.view(*lead, self.out_features)


class MADE(base.AutoregressiveModel):
    """The Masked Autoencoder Distribution Estimator (reference made.py:37-133)."""

    _RUNTIME_CACHES = base.GenerativeModel._RUNTIME_CACHES + ("_made_conn", "_made_sampler")
    _incremental_sampling = True  # False: one full forward per dimension, as the reference samples (for comparisons)

    def __init__(self, input_dim, hidden_dims=None, n_masks=1, sample_fn=None):
        super().__init__(sample_fn)
        self._input_dim = input_dim
        self._dims = [self._input_dim] + (hidden_dims or []) + [self._input_dim]
        self._n_masks = n_masks
        self._mask_seed = 0
        self._applied_mask = None  # the mask set the weights and `mask` buffers were last given

        layers = []
        for i in range(len(self._dims) - 1):
            layers.append(MaskedLinear(self._dims[i], self._dims[i + 1]))
            layers.append(nn.ReLU())
        self._net = nn.Sequential(*layers[:-1])

    def load_state_dict(self, state_dict, strict=True):
        self._applied_mask = None  # the loaded `mask` buffers may hold any set
        return super().load_state_dict(state_dict, strict)

    def _masked_layers(self):
        return [m for m in self._net if isinstance(m, MaskedLinear)]

    def _next_mask_set(self):
        """The mask set of the next forward / sample call; advances `_mask_seed` (reference made.py:76-77)."""
        mask_set = self._mask_seed % self._n_masks
        self._mask_seed += 1
        return mask_set

    def _connectivity(self, mask_set, device=None):
        """The connectivity vectors of a mask set: host numpy arrays, or int32 tensors on `device`; cached."""
        cache = self.__dict__.setdefault("_made_conn", {})
        if mask_set not in cache:
            cache[mask_set] = connectivity(self._input_dim, self._dims[1:-1], mask_set)
        if device is None:
            return cache[mask_set]
        key = (mask_set, str(device))
        if key not in cache:
            cache[key] = [torch.from_numpy(v.astype(np.int32)).to(device) for v in cache[mask_set]]
        return cache[key]

    def _apply_masks(self, mask_set, device):
        """Zeroes every layer's masked weights for `mask_set` and returns the layers' bf16 operands for _MaskedStack.
        While the mask set stays the one last applied (always, with n_masks = 1) the operands are cached until an
        optimizer step; a new set rewrites the `mask` buffers and builds fresh operands, because zeroing under it changes
        weights whose cached operands were built under another set."""
        conn = self._connectivity(mask_set, device)
        changed = self._applied_mask != mask_set
        packed = []
        modules = self._masked_layers()
        for i, m in enumerate(modules):
            strict = i == len(modules) - 1

            def build(m=m, i=i, strict=strict):
                wq = torch.empty(_pitch(m.out_features), _pitch(m.in_features), dtype=BF16, device=device)
                L.made_mask_cast(m.weight.detach(), conn[i], conn[i + 1], strict, wq, m.mask if changed else None)
                return wq

            wq = build() if changed else ops.cached_copy((m.weight,), ("made", mask_set), build)
            packed.append((wq, _padded_bias(m.bias), m.out_features))
        self._applied_mask = mask_set
        return packed

    def forward(self, x):
        """Logits of every dimension; x is (n, input_dim) or an image batch (n, c, h, w) with c*h*w = input_dim."""
        _require_cuda(x, "MADE")
        shape = x.shape
        packed = self._apply_masks(self._next_mask_set(), x.device)
        return _stack(x.reshape(shape[0], -1), packed, self._masked_layers()).view(shape)

    @torch.no_grad()
    def sample(self, n_samples=None, conditioned_on=None):
        """Draws the entries < 0 of `conditioned_on` (or of a fresh canvas of n_samples images), one dimension at a time
        in the order of the mask set this call uses (reference made.py:119-133)."""
        canvas = self._start_canvas(n_samples, conditioned_on)
        _require_cuda(canvas, "MADE.sample")
        shape = canvas.shape
        x = canvas.reshape(shape[0], -1)
        mask_set = self._next_mask_set()
        packed = self._apply_masks(mask_set, x.device)
        order = np.argsort(self._connectivity(mask_set)[-1])
        if len(self._dims) > 2 and self._incremental_sampling:
            self._sample_incremental(x, packed, order)
        else:
            for d in order:
                logits = _stack(x, packed, self._masked_layers())[:, d]
                drawn = self._sample_fn(logits)
                x[:, d] = torch.where(x[:, d] < 0, drawn, x[:, d])
        return x.view(shape)

    # ---- incremental sampler ----
    def _sampler_state(self, n, device):
        cache = self.__dict__.setdefault("_made_sampler", {})
        key = (n, str(device))
        if key not in cache:
            D, hidden = self._input_dim, self._dims[1:-1]
            f32 = dict(dtype=F32, device=device)
            st = dict(pos=torch.zeros(1, dtype=torch.int64, device=device),
                      order=torch.zeros(D, dtype=torch.int32, device=device),
                      canvas=torch.zeros(n, D, **f32), x_in=torch.zeros(n, D, **f32), h1=torch.zeros(n, hidden[0], **f32),
                      w1t=torch.zeros(D, hidden[0], **f32), w_out=torch.zeros(D, hidden[-1], **f32),
                      b_out=torch.zeros(D, **f32), logits=torch.zeros(n, **f32), a1=None, mids=[], graph=None)
            if len(hidden) > 1:
                st["a1"] = torch.zeros(n, _pitch(hidden[0]), dtype=BF16, device=device)
                for h_in, h_out in zip(hidden[:-1], hidden[1:]):
                    st["mids"].append((torch.zeros(_pitch(h_out), _pitch(h_in), dtype=BF16, device=device),
                                       torch.zeros(_pitch(h_out), **f32)))
            cache[key] = st
        return cache[key]

    def _sample_step(self, st):
        """The per-dimension program: the rank-1 update of h1, then the logit of dimension order[pos]."""
        n = st["canvas"].shape[0]
        common = (st["pos"], st["order"], n)
        if st["a1"] is None:
            L.made_sample_step(*common, st["canvas"], st["x_in"], st["w1t"], st["h1"], 1, st["w_out"], st["b_out"],
                               st["logits"])
            return
        L.made_sample_step(*common, st["canvas"], st["x_in"], st["w1t"], st["h1"], 1, None, None, None, a1=st["a1"])
        a = st["a1"]
        for wq, bias in st["mids"]:
            a = ops.linear_fwd(a, wq, bias, act=L.ACT_RELU, skinny=True)[0]
        L.made_sample_step(*common, None, None, None, None, 0, st["w_out"], st["b_out"], st["logits"], hl=a)

    def _sample_incremental(self, x, packed, order):
        n, D = x.shape
        modules = self._masked_layers()
        st = self._sampler_state(n, x.device)
        # the sampler's own buffers, refreshed in place (a captured graph keeps reading them): weights may have been
        # trained and the mask set may differ since the last call
        st["order"].copy_(torch.from_numpy(order.astype(np.int32)))
        st["w1t"].copy_(modules[0].weight.detach().t())
        st["w_out"].copy_(modules[-1].weight.detach())
        st["b_out"].copy_(modules[-1].bias.detach())
        for (wq, bias), (src_w, src_b, _) in zip(st["mids"], packed[1:-1]):
            wq.copy_(src_w)
            bias[: src_b.numel()].copy_(src_b)
        st["canvas"].copy_(x)
        st["x_in"].zero_()
        st["h1"].copy_(modules[0].bias.detach().expand_as(st["h1"]))
        st["pos"].zero_()
        L.made_sample_step(st["pos"], st["order"], n, st["canvas"], st["x_in"], st["w1t"], st["h1"], 2, None, None, None)
        if st["graph"] is None:
            self._sample_step(st)  # warm-up outside capture (at position 0 the step leaves h1 alone)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._sample_step(st)
            st["graph"] = graph
        canvas, logits = st["canvas"], st["logits"]
        for t, d in enumerate(order):
            st["pos"].fill_(t)
            st["graph"].replay()
            drawn = self._sample_fn(logits.clone())  # the graph overwrites `logits` at the next step
            current = canvas[:, d]
            canvas[:, d] = torch.where(current < 0, drawn, current)
        x.copy_(canvas)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference made.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_made(*args, **kwargs)
