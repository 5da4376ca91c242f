"""FVBN on the CUDA path — API of reference models/autoregressive/fvbn.py (`FullyVisibleBeliefNetwork`, `reproduce`).

Same constructor, module tree and state-dict keys: `_net` is an nn.ModuleList of nn.Linear(max(1, i), 1), built in the
reference's order, so `_net.{i}.weight` [1, max(1, i)], `_net.{i}.bias` [1], the `parameters()` order and the init bits
under a seed match, and trainer and optimizer checkpoints interchange with the reference's.  `forward` returns logits in
the input's shape; the input is (n, n_dims) or an image batch with c*h*w = n_dims, flattened with `view`.  Row 0 takes
the constant input 0 (its logit is b_0 + w_0 * 0, computed, so a non-finite w_0 propagates) and row i >= 1 takes
x[:, :i].

The rows stay separate parameters.  `ParamTable` owns their layout: a device table of the 2 * n_dims parameter addresses
that the kernels read them through (no copies, no rebinding of `.data`), and the packed triangular layout of the weight
gradient.  `pg_fvbn_fwd` is the whole forward in one launch, `pg_fvbn_bwd` the whole backward in two; the autograd
Function returns each weight gradient as a [1, len] view of one packed gradient buffer and each bias gradient as a view
of one [n_dims] buffer, so AccumulateGrad adopts them without a copy.

`sample` keeps the reference's semantics (base `AutoregressiveModel.sample`): pixels in raster order, `sample_fn` called
once per pixel with the [n, c] logits computed from the canvas as it stands at that step (for c > 1 the entries of later
channels not drawn yet enter as -1, as in the reference), only entries < 0 overwritten.  The logit step
(`pg_fvbn_sample_step`, in the forward's summation order) is captured once per (n, shape) in a CUDA graph and replayed
h*w times.  The forward is not defined on a truncated image, so `_row_truncated_sampling` does not apply.
"""

import torch
from torch import nn

from .. import _lib as L
from . import base


def _require_cuda(x, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")


def packed_offsets(n_dims):
    """(offsets, lengths, T) of the packed weight gradient: row i starts at 0 for i = 0 and 1 + i (i - 1) / 2 otherwise
    and has max(1, i) entries; T = 1 + n_dims (n_dims - 1) / 2 in all."""
    lengths = [max(1, i) for i in range(n_dims)]
    offsets = [0 if i == 0 else 1 + i * (i - 1) // 2 for i in range(n_dims)]
    return offsets, lengths, 1 + n_dims * (n_dims - 1) // 2


class ParamTable:
    """The one owner of the parameter layout: per device, the int64 table (W_0, ..., W_{D-1}, b_0, ..., b_{D-1}) of
    parameter addresses the kernels read, and the packed layout of the weight gradient.  The table is rebuilt (in place,
    so captured graphs keep reading it) only when a parameter's storage changed, e.g. after `.to()`; like FusedAdam's
    plan it is keyed by the parameters' data pointers, and it is never rebuilt during graph capture.

    The kernels read every row as len(i) contiguous fp32 values, so a rebuild first checks that each parameter is one:
    a CUDA fp32 contiguous tensor of max(1, i) (weight) or 1 (bias) elements on the table's device.  Any change of
    dtype, device or shape gives a parameter new storage, hence a new key and this check before the kernels see it."""

    def __init__(self, n_dims):
        self.n_dims = n_dims
        _, self.lengths, self.total = packed_offsets(n_dims)
        self._tables = {}  # device -> (key, int64 [2 * D] table)

    def _check(self, weights, biases, device):
        expected = [(w, "weight", n) for w, n in zip(weights, self.lengths)] + [(b, "bias", 1) for b in biases]
        for i, (t, kind, numel) in enumerate(expected):
            if not (device.type == "cuda" and t.device == device and t.dtype == torch.float32 and t.is_contiguous()
                    and t.numel() == numel):
                raise RuntimeError(
                    f"FullyVisibleBeliefNetwork: the CUDA path needs every row's parameters as contiguous fp32 tensors on "
                    f"one CUDA device; _net.{i % self.n_dims}.{kind} is {t.dtype} on {t.device} with {t.numel()} "
                    f"elements (expected {numel}{'' if t.is_contiguous() else ', contiguous'}; no CPU or other-dtype "
                    f"fallback)")

    def table(self, weights, biases):
        params = weights + biases
        key = tuple(p.data_ptr() for p in params)
        device = params[0].device
        entry = self._tables.get(device)
        if entry is None or entry[0] != key:
            self._check(weights, biases, device)
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FullyVisibleBeliefNetwork: the parameters moved during CUDA graph capture")
            host = torch.tensor(key, dtype=torch.int64)
            dev = entry[1] if entry is not None else torch.empty(len(key), dtype=torch.int64, device=device)
            dev.copy_(host)
            entry = self._tables[device] = (key, dev)
        return entry[1]

    def grads(self, buf):
        """The gradients of one backward from its buffer [T + D] (packed weight gradient, then the biases): a [1, len(i)]
        view per weight and a [1] view per bias, in `parameters()` order."""
        ws = buf[: self.total].view(1, self.total).split(self.lengths, dim=1)
        bs = buf[self.total:].split(1)
        return [t for pair in zip(ws, bs) for t in pair]


class _FvbnLogits(torch.autograd.Function):
    """logits = FVBN(x) for x [n, D]; `params` are the D weights and D biases interleaved (`parameters()` order), read by
    the kernels through `table`."""

    @staticmethod
    def forward(ctx, layout, table, x, *params):
        n, D = x.shape
        logits = torch.empty(n, D, dtype=torch.float32, device=x.device)
        L.fvbn_fwd(table, x, logits)
        ctx.layout, ctx.table = layout, table
        ctx.save_for_backward(x)
        return logits

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        n, D = x.shape
        layout = ctx.layout
        buf = torch.zeros(layout.total + D, dtype=torch.float32, device=x.device)
        # at D = 1 the input feeds no row (row 0 takes the constant 0): no input gradient, as in the reference
        dx = torch.empty(n, D, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[2] and D > 1 else None
        L.fvbn_bwd(ctx.table, x, g.contiguous().float(), buf[: layout.total], buf[layout.total:], dx)
        return (None, None, dx, *layout.grads(buf))


class FullyVisibleBeliefNetwork(base.AutoregressiveModel):
    """The Fully Visible Belief Network (reference fvbn.py:19-45)."""

    _RUNTIME_CACHES = base.GenerativeModel._RUNTIME_CACHES + ("_fvbn_table", "_fvbn_sampler")
    _row_truncated_sampling = False  # the forward needs every dimension of the image

    def __init__(self, n_dims, sample_fn=None):
        super().__init__(sample_fn)
        self.n_dims = n_dims
        # As in the reference: row 0 has one weight and always takes the input 0 (PyTorch has no zero-width Linear).
        self._net = nn.ModuleList(nn.Linear(in_features=max(1, i), out_features=1) for i in range(self.n_dims))

    def _params(self):
        """Every row's weight and bias, interleaved (`parameters()` order)."""
        return [t for m in self._net for t in (m.weight, m.bias)]

    def _table(self, params):
        layout = self.__dict__.get("_fvbn_table")
        if layout is None:
            layout = self.__dict__["_fvbn_table"] = ParamTable(self.n_dims)
        return layout, layout.table(params[0::2], params[1::2])

    def forward(self, x):
        """Logits of every dimension; x is (n, n_dims) or an image batch (n, c, h, w) with c*h*w = n_dims."""
        _require_cuda(x, "FullyVisibleBeliefNetwork")
        original_shape = x.shape
        flat = x.view(original_shape[0], -1)
        if flat.shape[1] != self.n_dims:
            raise ValueError(f"FullyVisibleBeliefNetwork({self.n_dims}): an input of {flat.shape[1]} dimensions per "
                             f"example ({tuple(original_shape)})")
        params = self._params()
        layout, table = self._table(params)
        logits = _FvbnLogits.apply(layout, table, flat.contiguous().float(), *params)
        return logits.view(original_shape)

    # ---- sampling ----
    def _sampler_state(self, shape, device):
        cache = self.__dict__.setdefault("_fvbn_sampler", {})
        key = (tuple(shape), str(device))
        if key not in cache:
            n, c = shape[0], shape[1]
            cache[key] = dict(pos=torch.zeros((), dtype=torch.int64, device=device),
                              canvas=torch.zeros(shape, dtype=torch.float32, device=device),
                              logits=torch.zeros(n, c, dtype=torch.float32, device=device), graph=None)
        return cache[key]

    @torch.no_grad()
    def sample(self, n_samples=None, conditioned_on=None):
        """Draws the entries < 0 of `conditioned_on` (or of a fresh canvas of n_samples images) pixel by pixel in raster
        order, calling `sample_fn` once per pixel with that pixel's [n, c] logits (reference base.py:97-120)."""
        canvas = self._start_canvas(n_samples, conditioned_on)
        _require_cuda(canvas, "FullyVisibleBeliefNetwork.sample")
        n, c, h, w = canvas.shape
        if c * h * w != self.n_dims:
            raise ValueError(f"FullyVisibleBeliefNetwork({self.n_dims}): a canvas of shape {tuple(canvas.shape)}")
        _, table = self._table(self._params())  # refreshed outside capture; the graph reads the table in place
        st = self._sampler_state(canvas.shape, canvas.device)
        live, pos, logits = st["canvas"], st["pos"], st["logits"]
        live.copy_(canvas)
        if st["graph"] is None:
            pos.zero_()
            L.fvbn_sample_step(table, pos, live, logits)  # warm-up outside capture
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                L.fvbn_sample_step(table, pos, live, logits)
            st["graph"] = graph
        for p in range(h * w):
            row, col = divmod(p, w)
            pos.fill_(p)
            st["graph"].replay()
            drawn = self._sample_fn(logits.clone()).view(n, c)  # the graph overwrites `logits` at the next step
            current = live[:, :, row, col]
            live[:, :, row, col] = torch.where(current < 0, drawn, current)
        canvas.copy_(live)
        return canvas


def reproduce(*args, **kwargs):
    """The recipe of this model (reference fvbn.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_fvbn(*args, **kwargs)
