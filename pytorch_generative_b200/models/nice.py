"""NICE on the CUDA path — API of reference models/flow/nice.py (`AdditiveCouplingBlock`, `ScalingLayer`, `NICE`,
`reproduce`).

Same constructors, module tree and state-dict keys (`net.{b}.net.{0,2,...}.weight / bias`, `scaling.log_scale` [1, D]),
the same init bits under a seed and the same results: `NICE.forward(x)` returns `(z, log_det_J)` with `z` in x's shape
(2-D or an image batch, as under the reference's `auto_reshape`) and `log_det_J = sum(log_scale)`, a 0-d tensor;
`_forward` / `_inverse` keep the reference's meaning; `sample(n, temp)` draws its latents with `torch.randn` on the CPU
default generator exactly as the reference does and runs the inverse on the device.

The flow's stream is two fp32 half buffers, lo = x[:, :D/2] and hi = x[:, D/2:], each of pitch round_up(D/2, 8) with
zero pad columns (the GEMM operand pitch).  A coupling block reads one half as a bf16 operand and writes a NEW buffer for
the other, so nothing aliases and nothing is copied:
  * hidden layers: `ops.linear_fwd` with the ReLU in the epilogue, bf16 outputs;
  * the last layer: one GEMM whose epilogue adds the bias, adds the transformed half as `res0` into a fresh fp32 half,
    and writes bf16 of that half, the next block's operand (`reverse` alternates, so the half a block writes is the half
    the next one conditions on);
  * the inverse runs the same GEMMs with alpha = -1 and a negated bias copy: negation is exact, so the last layer gives
    y - fl(acc + b), the forward's m subtracted with the forward's rounding.
`pg_nice_split` / `pg_nice_join` are the two ends (with the diagonal scaling and the sum of the log-scales at the join),
`pg_nice_scale_bwd` starts the backward.  The backward walks the blocks in reverse: the transformed half's gradient
passes through and its bf16 copy is `dm`; dgrad uses ReLU' from the saved outputs, the wgrads the fused bias gradient,
and the first layer's dgrad adds the conditioning half's gradient as `res0` into a new fp32 half while it writes the
bf16 copy that the previous block needs as its `dm`.  Only the bf16 operands (each block's conditioning operand and its
hidden activations) and z are saved for the backward.  The inverse is inference-only.
"""

import torch
from torch import nn

from .. import _lib as L
from .. import ops
from . import base

BF16, F32 = torch.bfloat16, torch.float32


def _pitch(d):
    """Columns of a GEMM operand holding `d` features: the 16-byte operand pitch, zero in the pad."""
    return ops.round_up(d, 8)


def _half_pitch(D):
    """Pitch of the two half buffers of a D-feature stream (the wider half is hi = x[:, D/2:])."""
    return _pitch(D - D // 2)


def _weight(lin):
    """bf16 [pitch(out), pitch(in)] operand of an nn.Linear, zero in the pads; cached until the weight changes."""
    def build():
        w = lin.weight.detach()
        out_f, in_f = w.shape
        shape = (_pitch(out_f), _pitch(in_f))
        out = (torch.empty if shape == (out_f, in_f) else torch.zeros)(shape, dtype=BF16, device=w.device)
        L.act_cast(w, L.ACT_NONE, out[:out_f, :in_f])
        return out
    return ops.cached_copy((lin.weight,), ("nice",), build)


def _bias(lin, negate=False):
    """fp32 bias padded with zeros to pitch(out) (negated for the inverse's last layer); cached like the weights."""
    b = lin.bias.detach()
    if not negate and _pitch(b.numel()) == b.numel():
        return b

    def build():
        out = torch.zeros(_pitch(b.numel()), dtype=F32, device=b.device)
        out[: b.numel()].copy_(b)
        return out.neg_() if negate else out
    return ops.cached_copy((lin.bias,), ("nice", negate), build)


def _require(x, params, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")
    for p in params:
        if p.dtype != F32 or not p.is_cuda or not p.is_contiguous():
            raise RuntimeError(f"{who}: the CUDA path needs contiguous fp32 CUDA parameters; got {p.dtype} on {p.device}")
    if x.dtype != F32:
        raise RuntimeError(f"{who}: the CUDA path takes fp32 inputs; got {x.dtype}")


def _check_features(D, blocks, scaling, who):
    if blocks and D % 2:
        raise ValueError(f"{who}: the coupling blocks split the features into two halves of D/2, so D must be even; "
                         f"got D = {D}")
    for b in blocks:
        if b.half_features != D // 2:
            raise ValueError(f"{who}: a coupling block of {2 * b.half_features} features got inputs of {D} features")
    if scaling is not None and scaling.log_scale.numel() != D:
        raise ValueError(f"{who}: a scaling layer of {scaling.log_scale.numel()} features got inputs of {D} features")


class _Flow(torch.autograd.Function):
    """x [n, D] -> coupling blocks -> scaling -> z [n, D] (and log_det = sum(log_scale) when there is a scaling layer).
    `blocks`: [(reverse, [(w_bf16, padded bias, out_features, in_features) per layer])], alternating `reverse`;
    `log_scale`: [1, D] or None; `params`: every block's weights and biases in parameters() order."""

    @staticmethod
    def forward(ctx, x, blocks, log_scale, *params):
        n, D = x.shape
        ld = _half_pitch(D)
        halves = [torch.empty((n, ld), dtype=F32, device=x.device) for _ in range(2)]
        a = torch.empty((n, ld), dtype=BF16, device=x.device) if blocks else None
        L.nice_split(x.contiguous(), halves[0], halves[1], out_bf16=a, bf16_half=int(blocks[0][0]) if blocks else 0)
        saved = []
        for k, (reverse, layers) in enumerate(blocks):
            t = 0 if reverse else 1  # the transformed half
            acts = [a]
            for wq, bias, _, _ in layers[:-1]:
                acts.append(ops.linear_fwd(acts[-1], wq, bias, act=L.ACT_RELU)[0])
            wq, bias, _, _ = layers[-1]
            _, a, halves[t] = ops.linear_fwd(acts[-1], wq, bias, res0=halves[t], want_bf16=False,
                                             want_pre=k + 1 < len(blocks), want_f32=True)
            saved += acts
        z = torch.empty((n, D), dtype=F32, device=x.device)
        log_det = None if log_scale is None else torch.empty((), dtype=F32, device=x.device)
        L.nice_join(halves[0], halves[1], z, log_scale, log_det=log_det)
        ctx.save_for_backward(z, log_scale, *saved)
        ctx.blocks = blocks
        return z if log_det is None else (z, log_det)

    @staticmethod
    def backward(ctx, gz, g_log_det=None):
        z, log_scale, *acts = ctx.saved_tensors
        blocks = ctx.blocks
        n, D = z.shape
        ld = _half_pitch(D)
        d = [torch.empty((n, ld), dtype=F32, device=z.device) for _ in range(2)]
        last_t = (0 if blocks[-1][0] else 1) if blocks else 0
        dm = torch.empty((n, ld), dtype=BF16, device=z.device) if blocks else None
        d_log_scale = None
        if log_scale is not None:
            d_log_scale = torch.empty_like(log_scale)
            L.nice_scale_bwd(gz.contiguous(), z, log_scale, g_log_det.contiguous(), d[0], d[1], d_log_scale,
                             dm_bf16=dm, bf16_half=last_t)
        else:
            L.nice_split(gz.contiguous(), d[0], d[1], out_bf16=dm, bf16_half=last_t)
        grads, end = [], len(acts)
        for k in reversed(range(len(blocks))):
            reverse, layers = blocks[k]
            c = 1 if reverse else 0  # the conditioning half
            block_acts = acts[end - len(layers): end]
            end -= len(layers)
            dy, block_grads = dm, []
            for i in reversed(range(len(layers))):
                wq, bias, out_f, in_f = layers[i]
                dw = torch.zeros(wq.shape, dtype=F32, device=z.device)
                db = torch.zeros(wq.shape[0], dtype=F32, device=z.device)
                ops.linear_wgrad(dy, block_acts[i], dw, db)
                dw = dw if dw.shape == (out_f, in_f) else dw[:out_f, :in_f].contiguous()
                block_grads = [dw, db[:out_f]] + block_grads
                if i > 0:
                    dy = ops.linear_dgrad(dy, wq, aux=block_acts[i], dact=L.ACT_RELU_OUT)  # ReLU' from the layer's input
                elif k > 0 or ctx.needs_input_grad[0]:
                    # the conditioning half's gradient: dy W + the gradient that passed through it, and (for the previous
                    # block, which transformed this half) its bf16 copy
                    dm = torch.empty((n, ld), dtype=BF16, device=z.device) if k > 0 else None
                    new = torch.empty((n, ld), dtype=F32, device=z.device)
                    L.gemm(dy, wq, n, ld, dy.shape[1], b_mn=True, res0=d[c], out_bf16=dm, out_f32=new,
                           impl=ops.GEMM_IMPL)
                    d[c] = new
            grads = block_grads + grads
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((n, D), dtype=F32, device=z.device)
            L.nice_join(d[0], d[1], dx)
        return (dx, None, d_log_scale, *grads)


def _flow(x, blocks, scaling, who):
    """(z, log_det) of x [n, D] through `blocks` and `scaling` (either may be absent; log_det only with a scaling layer)."""
    params = [p for b in blocks for p in b._params()]
    log_scale = None if scaling is None else scaling.log_scale
    _check_features(x.shape[1], blocks, scaling, who)
    _require(x, params + ([] if log_scale is None else [log_scale]), who)
    specs = [b._spec() for b in blocks]
    for prev, cur in zip(specs, specs[1:]):
        assert prev[0] != cur[0], "the flow's coupling blocks alternate `reverse`"
    out = _Flow.apply(x, specs, log_scale, *params)
    return (out, None) if log_scale is None else out


def _inverse(y, blocks, scaling, who):
    """x of y [n, D] under the inverse of `blocks` then `scaling`: the scaling's inverse, then the blocks in reverse.
    Inference only: under autograd recording it raises rather than return a tensor without a gradient."""
    params = [p for b in blocks for p in b._params()]
    log_scale = None if scaling is None else scaling.log_scale
    _check_features(y.shape[1], blocks, scaling, who)
    _require(y, params + ([] if log_scale is None else [log_scale]), who)
    if torch.is_grad_enabled() and (y.requires_grad or any(p.requires_grad for p in params) or
                                    (log_scale is not None and log_scale.requires_grad)):
        raise RuntimeError(f"{who}: the inverse is inference-only on the CUDA path (it has no backward); call it under "
                           "torch.no_grad()")
    n, D = y.shape
    ld = _half_pitch(D)
    halves = [torch.empty((n, ld), dtype=F32, device=y.device) for _ in range(2)]
    specs = [b._spec(negate_last=True) for b in blocks]
    a = torch.empty((n, ld), dtype=BF16, device=y.device) if blocks else None
    L.nice_split(y.contiguous(), halves[0], halves[1], log_scale, sign=-1.0, out_bf16=a,
                 bf16_half=int(specs[-1][0]) if blocks else 0)
    for k in reversed(range(len(specs))):
        reverse, layers = specs[k]
        t = 0 if reverse else 1
        for wq, bias, _, _ in layers[:-1]:
            a = ops.linear_fwd(a, wq, bias, act=L.ACT_RELU)[0]
        wq, neg_bias, _, _ = layers[-1]
        nxt = torch.empty((n, ld), dtype=BF16, device=y.device) if k > 0 else None
        new = torch.empty((n, ld), dtype=F32, device=y.device)
        L.gemm(a, wq, n, ld, a.shape[1], bias=neg_bias, res0=halves[t], out_pre=nxt, out_f32=new, alpha=-1.0,
               impl=ops.GEMM_IMPL)
        halves[t], a = new, nxt
    x = torch.empty((n, D), dtype=F32, device=y.device)
    L.nice_join(halves[0], halves[1], x)
    return x


class AdditiveCouplingBlock(nn.Module):
    """Additive coupling (reference nice.py:15-63): with x1, x2 the halves of x and m the coupling MLP, `forward` gives
    (x1, x2 + m(x1)) and `inverse` (y1, y2 - m(y1)); `reverse` swaps the roles of the halves."""

    def __init__(self, n_features, n_hidden_layers, n_hidden_features, reverse):
        super().__init__()
        self.reverse = reverse
        half_features = n_features // 2
        net = [nn.Linear(in_features=half_features, out_features=n_hidden_features), nn.ReLU()]
        for _ in range(n_hidden_layers - 1):
            net.append(nn.Linear(in_features=n_hidden_features, out_features=n_hidden_features))
            net.append(nn.ReLU())
        net.append(nn.Linear(in_features=n_hidden_features, out_features=half_features))
        self.net = nn.Sequential(*net)

    @property
    def half_features(self):
        return self.net[0].in_features

    def _linears(self):
        return [m for m in self.net if isinstance(m, nn.Linear)]

    def _params(self):
        return [t for m in self._linears() for t in (m.weight, m.bias)]

    def _spec(self, negate_last=False):
        lins = self._linears()
        return (bool(self.reverse), [(_weight(m), _bias(m, negate_last and i == len(lins) - 1), m.out_features,
                                      m.in_features) for i, m in enumerate(lins)])

    def forward(self, x):
        """Inverse mapping from the inputs to the prior (X -> Z); x is [n, D]."""
        return _flow(x, [self], None, "AdditiveCouplingBlock")[0]

    def inverse(self, y):
        """Forward mapping from the prior to the inputs (Z -> X); inference only."""
        return _inverse(y, [self], None, "AdditiveCouplingBlock.inverse")


class ScalingLayer(nn.Module):
    """Diagonal scaling by exp(log_scale) (reference nice.py:66-97)."""

    def __init__(self, n_features):
        super().__init__()
        self.log_scale = nn.Parameter(torch.zeros((1, n_features)))

    def log_det_J(self):
        """log det S = sum(log_scale), summed in ascending order on the device (the value NICE.forward returns)."""
        x = torch.empty((0, self.log_scale.numel()), dtype=F32, device=self.log_scale.device)
        return _flow(x, [], self, "ScalingLayer")[1]

    def forward(self, x):
        """Inverse mapping from the inputs to the prior (X -> Z): x * exp(log_scale) over the flattened features."""
        return _flow(x.reshape(x.shape[0], -1), [], self, "ScalingLayer")[0].view(x.shape)

    def inverse(self, y):
        """Forward mapping from the prior to the inputs (Z -> X): y * exp(-log_scale); inference only."""
        return _inverse(y.reshape(y.shape[0], -1), [], self, "ScalingLayer.inverse").view(y.shape)


class NICE(base.GenerativeModel):
    """Non-linear Independent Components Estimation (reference nice.py:100-161)."""

    def __init__(self, n_features, n_coupling_blocks=4, n_hidden_layers=5, n_hidden_features=1000):
        super().__init__()
        net = []
        reverse = False
        for _ in range(n_coupling_blocks):
            net.append(AdditiveCouplingBlock(n_features=n_features, n_hidden_layers=n_hidden_layers,
                                             n_hidden_features=n_hidden_features, reverse=reverse))
            reverse = not reverse
        self.net = nn.Sequential(*net)
        self.scaling = ScalingLayer(n_features)

    def forward(self, x):
        """Inverse mapping from the inputs to the prior (X -> Z): (z, log_det_J), z in x's shape."""
        z, log_det = _flow(x.reshape(x.shape[0], -1), list(self.net), self.scaling, "NICE")
        return z.view(x.shape), log_det

    def _forward(self, x):
        return self.forward(x)[0]

    @torch.no_grad()
    def sample(self, n_samples, temp=1.0):
        """Latents from the standard normal times `temp`, drawn on the CPU default generator as the reference draws them,
        mapped to the inputs by the inverse."""
        x = torch.randn((n_samples, self._c, self._h, self._w)) * temp
        x = x.to(self.device)
        return self._inverse(x)

    def _inverse(self, x):
        return _inverse(x.reshape(x.shape[0], -1), list(self.net), self.scaling, "NICE._inverse").view(x.shape)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference nice.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_nice(*args, **kwargs)
