"""Drives the pixel-major stacks of VAE, VQ-VAE and VQ-VAE-2 for the stage-replay tests: builds a model with parameters
away from their initial values, records every call of the stacks' autograd Functions (nn/pm.py, nn/vq.py, the VAE
latent and the MSE), holds each record to its stage of tests/_conv_stack_reference.py and keeps the bug models the
replay must reject.  Shared by tests/test_conv_stack_bounds_cpu.py and tests/test_conv_stack_stages_gpu.py; not a test
module."""

import types

import torch

import _block_replay as BR
import _conv_stack_reference as R

BF16 = torch.bfloat16


def build(cls, kwargs, shape, seed=0, device="cpu"):
    """(model, x, cotangents): a `cls(**kwargs)` from models whose biases are N(0, 0.5^2) (the weights keep their
    initialisation), an image batch of `shape` in [0, 1) and unit-scale cotangents of every model output (the logits or
    x_hat, and kl or vq_loss)."""
    from pytorch_generative_b200 import models

    torch.manual_seed(seed)
    m = getattr(models, cls)(**kwargs)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.5 * torch.randn(p.shape, generator=g))
    x = torch.rand(shape, generator=g)
    n, _, h, w = shape
    cout = kwargs.get("out_channels", 1)
    G = torch.randn(n, cout, h, w, generator=g)
    G2 = torch.randn(n, generator=g) if cls in ("VAE", "BetaVAE") else torch.ones(())
    return m.to(device), x.to(device), (G.to(device), G2.to(device))


def step(m, x, G):
    """One training-mode forward and backward with the cotangents G; returns the outputs."""
    for p in m.parameters():
        p.grad = None
    out = m(x)
    (out[0] * G[0]).sum().add((out[1] * G[1]).sum()).backward()
    return out


class Recorder:
    """Wraps the forward and backward of pm._Conv, pm._StridedConv, pm._TransposedConv, vq._Quantize, vae._Latent and
    losses._MSEMean, and _lib.vq_assign.  A record is labelled by the identity of its weight (a convolution) or of its
    quantizer module, never by call order.  Install it after the stand-ins and the bug model under test."""

    def __init__(self, monkeypatch):
        from pytorch_generative_b200 import _lib, losses
        from pytorch_generative_b200.models import vae
        from pytorch_generative_b200.nn import pm, vq

        self.records = []
        self._idx = []
        assign = _lib.vq_assign

        def vq_assign(x, emb, idx, *a, **kw):
            assign(x, emb, idx, *a, **kw)
            self._idx.append(idx)
        monkeypatch.setattr(_lib, "vq_assign", vq_assign)
        for cls, kind in ((pm._Conv, "conv"), (pm._StridedConv, "strided"), (pm._TransposedConv, "transposed"),
                          (vq._Quantize, "quantizer"), (vae._Latent, "latent"), (losses._MSEMean, "mse")):
            self._wrap(monkeypatch, cls, kind)

    def _wrap(self, monkeypatch, cls, kind):
        fwd, bwd = cls.forward, cls.backward

        def forward(ctx, *args):
            r = types.SimpleNamespace(kind=kind, args=args, grads=None, res=None)
            if kind == "quantizer":
                r.emb = args[2].detach().clone()  # the codebook the loss uses, before the EMA update
            r.out = fwd(ctx, *args)
            if kind == "conv":
                r.mode = ctx.meta[2]  # the path the product took: POINTWISE, TAP_LOOP or GATHER
            if kind == "quantizer":
                r.idx = self._idx[-1]
            ctx._stage_record = len(self.records)  # an index: the record holds the outputs, whose node holds ctx
            self.records.append(r)
            return r.out

        def backward(ctx, *grads):
            r = self.records[ctx._stage_record]
            r.grads = grads
            r.res = bwd(ctx, *grads)
            return r.res

        monkeypatch.setattr(cls, "forward", staticmethod(forward))
        monkeypatch.setattr(cls, "backward", staticmethod(backward))


def _conv_view(r):
    """The record of a convolution in the reference's terms (input, operand, geometries, outputs, gradients)."""
    from pytorch_generative_b200.nn import pm

    a = r.args
    v = types.SimpleNamespace(x=a[0], xa=a[1], weight=a[2], bias=a[3])
    res = r.res or (None,) * 5
    v.dx, v.dw, v.db = res[0], res[2], res[3]
    if r.kind == "conv":
        _, _, _, _, resid, geom, taps, _, emit, _, out_f32, _ = a
        v.in_geom = v.out_geom = tuple(geom)
        v.y, v.ya = r.out
        v.grads = r.grads
        v.has_res, v.res_dtype, v.dres = resid is not None, None if resid is None else resid.dtype, res[4]
        v.mode = r.mode
        v.bf16_partials = v.mode == pm.GATHER
    else:
        rows, spatial, emit = a[4], a[5], a[9]
        v.in_geom, v.out_geom = (spatial, rows) if r.kind == "strided" else (rows, spatial)
        v.y, v.ya = (None, r.out) if emit is not None else (r.out, None)
        g = None if r.grads is None else r.grads[0]
        v.grads = None if r.grads is None else ((None, g) if emit is not None else (g, None))
        v.has_res, v.mode, v.dres = False, None, None
        v.bf16_partials = r.kind == "strided"
    return v


def replay(m, rec):
    """Every recorded stage against the stage table of m's state dict: (Checks, {stage kind: count}, conv modes)."""
    state = m.state_dict()
    T = R.table(state)
    params = dict(m.named_parameters())
    by_weight = {id(p): k[: -len(".weight")] for k, p in params.items() if k.endswith(".weight")}
    names = {id(mod): k for k, mod in m.named_modules()}
    C = R.Checks()
    views, counts, modes = {}, {}, set()
    for r in rec.records:
        counts[r.kind] = counts.get(r.kind, 0) + 1
        if r.kind in ("conv", "strided", "transposed"):
            name = by_weight[id(r.args[2])]
            assert name not in views, f"{name} recorded twice"
            views[name] = _conv_view(r)
    assert set(views) == set(T), (sorted(set(views) ^ set(T)))
    for name, layer in T.items():
        v = views[name]
        modes.add(v.mode)
        res_in = views[layer.res].x if layer.res else None
        R.conv_stage(C, name, layer, v, res_in, params[name + ".weight"], params[name + ".bias"])
    for r in rec.records:
        if r.kind == "quantizer":
            R.quantizer_stage(C, names[id(r.args[4])], r)
        elif r.kind == "latent":
            R.latent_stage(C, r)
        elif r.kind == "mse":
            R.mse_stage(C, r)
    return C, counts, modes


# ----------------------------------------------------------------------------------------------------------------------
# bug models: each changes only which valid tensor or argument the product passes
# ----------------------------------------------------------------------------------------------------------------------
def bug_fp32_dres_from_bf16_operand(monkeypatch):
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._Conv, "backward",
               "dres = dy if dy.dtype == res_dtype else", "dres = dyb if dy.dtype == res_dtype else")


def bug_transposed_bias_grad_before_emit(monkeypatch):
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._TransposedConv, "backward", "db = ops.bias_grad(dyb[:, :cout])",
               "db = ops.bias_grad(dy.contiguous()[:, :cout])")


def bug_pack_taps_t_kh_kw_swapped(monkeypatch):
    from pytorch_generative_b200 import ops

    pack = ops.pack_taps_t
    monkeypatch.setattr(ops, "pack_taps_t", lambda w, cin_p, cout_p: pack(w.transpose(2, 3).contiguous(), cin_p, cout_p))


def bug_commitment_scale_per_row(monkeypatch):
    from pytorch_generative_b200.nn import vq

    BR._mutate(monkeypatch, vq._Quantize, "backward", "L.vq_bwd(z, emb, idx, dq, c0, g, 2.0 / numel, dx)",
               "L.vq_bwd(z, emb, idx, dq, c0, g, 2.0 / z.shape[0], dx)")


def bug_transposed_dx_without_in_act(monkeypatch):
    """The first transposed convolution's input gradient leaves without the decoder stack's trailing ReLU'."""
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._TransposedConv, "backward", "dact = L.DACT_FROM_OUT.get(in_act, L.ACT_NONE)",
               "dact = L.ACT_NONE")


def bug_gather_dx_without_in_act(monkeypatch):
    """On the tap-gather path, `_Conv`'s input gradient is folded back without the input activation's derivative."""
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._Conv, "backward", "cin_p, taps, dact, aux,", "cin_p, taps, L.ACT_NONE, None,")


# name -> (apply(monkeypatch), the stage kind (R.kind_of) that must fail, the geometries that run the code it changes)
BUGS = {
    "fp32_dres_from_bf16_operand": (bug_fp32_dres_from_bf16_operand, "conv.dres", None),
    "transposed_bias_grad_before_emit": (bug_transposed_bias_grad_before_emit, "transposed.db", "stride4"),
    "pack_taps_t_kh_kw_swapped": (bug_pack_taps_t_kh_kw_swapped, "transposed.y", None),
    "commitment_scale_per_row": (bug_commitment_scale_per_row, "quantizer.dx", "vq"),
    "transposed_dx_without_in_act": (bug_transposed_dx_without_in_act, "transposed.dx", None),
    "gather_dx_without_in_act": (bug_gather_dx_without_in_act, "conv.dx", None),
}
