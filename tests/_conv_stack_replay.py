"""Drives the pixel-major stacks of GatedPixelCNN, PixelSNAIL, VAE, VQ-VAE and VQ-VAE-2 for the stage-replay tests:
builds a model with parameters away from their initial values, records every call of the stacks' autograd Functions
(nn/pm.py, the pixel-major attention of nn/modules.py, nn/vq.py, the VAE latent and the MSE), holds each record to its
stage of tests/_conv_stack_reference.py, each hand-off between GatedPixelCNN's and PixelSNAIL's stages to the stage
graph, and keeps the bug models the replay must reject.  Shared by tests/test_conv_stack_bounds_cpu.py and
tests/test_conv_stack_stages_gpu.py; not a test module."""

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
    """One training-mode forward and backward with the cotangents G (of as many outputs as the model returns); returns
    the outputs."""
    for p in m.parameters():
        p.grad = None
    out = m(x)
    out = out if isinstance(out, tuple) else (out,)  # GatedPixelCNN: the logits alone
    sum((o * g).sum() for o, g in zip(out, G)).backward()
    return out


class Recorder:
    """Wraps the forward and backward of pm._Conv, pm._StridedConv, pm._TransposedConv, pm._SmallConv, pm._Gated,
    pm._GatedRes, pm._ActCast, modules._AttentionPMFn, vq._Quantize, vae._Latent and losses._MSEMean, and
    _lib.vq_assign.  A record is labelled by the identity of its weight (a convolution, the attention by its `_q`), of
    its quantizer module, or of the GatedPixelCNN layer, PixelSNAIL ResidualBlock or PixelSNAILBlock whose forward_pm
    made it (`owner`; a gate by its order within the layer, v then h), never by its place in the whole step.  It also
    keeps what PixelSNAIL hands between kernels inside one stage: the operand _lib.dact_from_out forms for an activated
    output (by that output), the attention's saved tensors, its bf16 output gradient and the do, dq, dk and dv of
    ops.attn_bwd; and, per PixelSNAILBlock call, the stream it read and the gradient that stream received (`blocks`),
    and the model input (`image`).  Install it after the stand-ins and the bug model under test."""

    def __init__(self, monkeypatch):
        from pytorch_generative_b200 import _lib, losses, ops
        from pytorch_generative_b200.models import gated_pixel_cnn, pixel_snail, vae
        from pytorch_generative_b200.nn import modules, pm, vq

        self.records, self.blocks, self.dact, self.image = [], [], {}, None
        self._idx = []
        self._owner = None
        self._attn = None
        assign, dact_from_out = _lib.vq_assign, _lib.dact_from_out
        attention_bwd, attn_bwd = modules._attention_bwd, ops.attn_bwd

        def owned(fwd, block=False):
            def forward_pm(layer, *a, **kw):
                if block:  # PixelSNAILBlock.forward_pm(geom, x_f, ...): the stream it reads, and its gradient
                    b = types.SimpleNamespace(owner=layer, x=a[1], grad=None)
                    self.blocks.append(b)
                    if b.x.requires_grad:
                        b.x.register_hook(lambda g: setattr(b, "grad", g))
                outer, self._owner = self._owner, layer
                try:
                    return fwd(layer, *a, **kw)
                finally:
                    self._owner = outer
            return forward_pm
        monkeypatch.setattr(gated_pixel_cnn.GatedPixelCNNLayer, "forward_pm",
                            owned(gated_pixel_cnn.GatedPixelCNNLayer.forward_pm))
        monkeypatch.setattr(pixel_snail.ResidualBlock, "forward_pm", owned(pixel_snail.ResidualBlock.forward_pm))
        monkeypatch.setattr(pixel_snail.PixelSNAILBlock, "forward_pm", owned(pixel_snail.PixelSNAILBlock.forward_pm,
                                                                             True))
        snail_fwd = pixel_snail.PixelSNAIL.forward

        def snail_forward(model, x):
            self.image = x
            return snail_fwd(model, x)
        monkeypatch.setattr(pixel_snail.PixelSNAIL, "forward", snail_forward)

        def vq_assign(x, emb, idx, *a, **kw):
            assign(x, emb, idx, *a, **kw)
            self._idx.append(idx)
        monkeypatch.setattr(_lib, "vq_assign", vq_assign)

        def dact(dy, ya, act, out):
            dact_from_out(dy, ya, act, out)
            self.dact[ya.data_ptr()] = out
        monkeypatch.setattr(_lib, "dact_from_out", dact)

        def attention_backward(ctx, dy_b):
            self._attn = self.records[ctx._stage_record]
            self._attn.dy_b = dy_b
            try:
                return attention_bwd(ctx, dy_b)
            finally:
                self._attn = None
        monkeypatch.setattr(modules, "_attention_bwd", attention_backward)

        def attn_backward(q, k, v, o, do, lse, dq, dk, dv, *a):
            out = attn_bwd(q, k, v, o, do, lse, dq, dk, dv, *a)
            if self._attn is not None:
                self._attn.attn = dict(do=do, dq=dq, dk=dk, dv=dv)
            return out
        monkeypatch.setattr(ops, "attn_bwd", attn_backward)
        for cls, kind in ((pm._Conv, "conv"), (pm._StridedConv, "strided"), (pm._TransposedConv, "transposed"),
                          (vq._Quantize, "quantizer"), (vae._Latent, "latent"), (losses._MSEMean, "mse"),
                          (pm._SmallConv, "small"), (pm._Gated, "gate"), (pm._GatedRes, "gated_res"),
                          (pm._ActCast, "act_cast"), (modules._AttentionPMFn, "attention")):
            self._wrap(monkeypatch, cls, kind)

    def _wrap(self, monkeypatch, cls, kind):
        fwd, bwd = cls.forward, cls.backward

        def forward(ctx, *args):
            r = types.SimpleNamespace(kind=kind, args=args, grads=None, res=None, owner=self._owner)
            if kind == "quantizer":
                r.emb = args[2].detach().clone()  # the codebook the loss uses, before the EMA update
            if kind == "attention":  # a_kv, q, kv, o, lse and the packed weights, as the forward saves them
                save = ctx.save_for_backward
                ctx.save_for_backward = lambda *t: (setattr(r, "saved", t), save(*t))[1]
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


def _conv_view(r, dact):
    """The record of a convolution in the reference's terms (input, operand, geometries, outputs, gradients, and the
    operand dact_from_out formed from its activated output's gradient)."""
    from pytorch_generative_b200.nn import pm

    a = r.args
    v = types.SimpleNamespace(x=a[0], xa=a[1], weight=a[2], bias=a[3], dact=None)
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
        v.dact = None if v.ya is None else dact.get(v.ya.data_ptr())
    else:
        rows, spatial, emit = a[4], a[5], a[9]
        v.in_geom, v.out_geom = (spatial, rows) if r.kind == "strided" else (rows, spatial)
        v.y, v.ya = (None, r.out) if emit is not None else (r.out, None)
        g = None if r.grads is None else r.grads[0]
        v.grads = None if r.grads is None else ((None, g) if emit is not None else (g, None))
        v.has_res, v.mode, v.dres = False, None, None
        v.bf16_partials = r.kind == "strided"
    return v


def _value(layer, r, v):
    """The tensor a recorded stage hands on: a convolution's activated output when it stands for y or is the output,
    else its main output; any other stage's output."""
    if v is not None:
        return v.ya if layer.act in ("post", "pre_grad") else v.y
    return r.out


def _incoming(layer, r, v):
    if v is not None:
        return None if v.grads is None else v.grads[1 if layer.act in ("post", "pre_grad") else 0]
    return None if r.grads is None else r.grads[0]


def _streams(T, rec, names, views):
    """{stream stage: (the fp32 stream it forms, the gradient that stream received)}: the input PixelSNAILBlock b + 1
    read and the gradient its hook saw; after the last block, `_output.0`'s input and input gradient."""
    nxt = {names[id(b.owner)]: b for b in rec.blocks}
    out = {}
    for name, layer in T.items():
        if layer.kind != "stream":
            continue
        i = int(name.split(":")[0].rsplit(".", 1)[1])
        b = nxt.get(f"_pixel_snail_blocks.{i + 1}")
        out[name] = (b.x, b.grad) if b is not None else (views["_output.0"].x, views["_output.0"].dx)
    return out


def replay(m, rec):
    """Every recorded stage against the stage table of m's state dict, and for a stage graph (GatedPixelCNN, PixelSNAIL)
    every hand-off between stages: (Checks, {record kind: count, a convolution's cast of its own input not counted},
    conv modes)."""
    state = m.state_dict()
    T = R.table(state)
    params = dict(m.named_parameters())
    by_weight = {id(p): k[: -len(".weight")] for k, p in params.items() if k.endswith(".weight")}
    names = {id(mod): k for k, mod in m.named_modules()}
    C = R.Checks()
    views, named, counts, modes = {}, {}, {}, set()
    # the casts a convolution makes of its own input (its `xa` when that is not its `x`), checked as its operand
    operands = {r.args[1].data_ptr() for r in rec.records
                if r.kind in ("conv", "strided", "transposed") and r.args[1].data_ptr() != r.args[0].data_ptr()}
    gates = {}
    for r in rec.records:
        if r.kind == "act_cast" and r.out.data_ptr() in operands:
            continue  # part of its convolution's stage
        counts[r.kind] = counts.get(r.kind, 0) + 1
        if r.kind in ("conv", "strided", "transposed"):
            name = by_weight[id(r.args[2])]
            assert name not in views, f"{name} recorded twice"
            views[name] = _conv_view(r, rec.dact)
        elif r.kind == "small":
            named[by_weight[id(r.args[1])]] = r
        elif r.kind == "gate":
            owner = names[id(r.owner)]
            i = gates.get(owner, 0)
            gates[owner] = i + 1
            named[f"{owner}:gate_{'vh'[i]}"] = r
        elif r.kind in ("act_cast", "gated_res"):
            named[f"{names[id(r.owner)]}:{r.kind}"] = r
        elif r.kind == "attention":
            named[by_weight[id(r.args[1])][: -len("._q")]] = r
    staged = {n for n, layer in T.items() if layer.kind != "stream"}
    assert not set(views) & set(named) and set(views) | set(named) == staged, sorted((set(views) | set(named)) ^ staged)
    streams = _streams(T, rec, names, views)
    values = {n: streams[n][0] if n in streams else _value(T[n], named.get(n), views.get(n)) for n in T}
    for name, layer in T.items():
        if name in views:
            v = views[name]
            modes.add(v.mode)
            res_in = res_dtype = None
            if layer.res:
                res_in = values[layer.res] if layer.res_of == "out" else views[layer.res].x
                res_dtype = R.out_dtype(T, layer.res) if layer.res_of == "out" else None
            given = len(layer.src or ()) == 1 and layer.src[0] in T and T[layer.src[0]].act == "pre_grad"
            R.conv_stage(C, name, layer, v, res_in, R.masked(layer, params[name + ".weight"]), params[name + ".bias"],
                         res_dtype, given)
        elif layer.kind == "image":
            R.small_stage(C, name, layer, named[name], R.masked(layer, params[name + ".weight"]),
                          params[name + ".bias"])
        elif layer.kind == "gate":
            R.gate_stage(C, name, named[name])
        elif layer.kind == "gated_res":
            R.gated_res_stage(C, name, named[name], values[layer.res])
        elif layer.kind == "attention":
            n, _, h, w = rec.image.shape
            R.attention_stage(C, name, layer, named[name], params, (n, h, w))
        elif layer.kind == "act_cast":
            R.act_cast_stage(C, name, named[name])
    if any(layer.src for layer in T.values()):
        inputs = {n: (views[n].x if n in views else named[n].args[0] if n in named else values[n]) for n in T}
        R.forward_handoffs(C, T, dict(values, image=rec.image), inputs)
        incoming = {n: streams[n][1] if n in streams else _incoming(T[n], named.get(n), views.get(n)) for n in T}
        returned = {}
        for n, layer in T.items():
            v, r = views.get(n), named.get(n)
            if incoming[n] is None:  # its backward did not run
                continue
            if layer.kind == "stream":  # a sum: each summand receives the sum's gradient
                dx, dres = incoming[n], None
            elif layer.kind == "attention":  # the features' columns of the operand's gradient
                dx, dres = r.res[0][:, 2: 2 + layer.attn.C], None
            else:
                dx = v.dx if v is not None else r.res[0]
                dres = v.dres if v is not None else (r.res[1] if layer.kind == "gated_res" else None)
            for s in layer.src or ():
                returned[(n, s)] = dx
            if layer.res and layer.res_of == "out":
                returned[(n, "res")] = dres
        R.backward_handoffs(C, T, incoming, returned)
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


def _mutate_fn(monkeypatch, owner, name, old, new, extra=None):
    """The plain function owner.name (a method or a module-level function) with `old` (once in its source) replaced by
    `new`, compiled in its module's namespace (plus the names in `extra`)."""
    import inspect
    import sys
    import textwrap

    fn = inspect.getattr_static(owner, name)
    src = textwrap.dedent(inspect.getsource(fn))
    assert src.count(old) == 1, old
    scope = sys.modules[fn.__module__].__dict__
    ns = {}
    exec(compile(src.replace(old, new), f"<mutated {name}>", "exec"), dict(scope, **extra) if extra else scope, ns)
    monkeypatch.setattr(owner, name, ns[fn.__name__])


def _mutate_layer(monkeypatch, old, new):
    """GatedPixelCNNLayer.forward_pm with `old` (once in its source) replaced by `new`."""
    from pytorch_generative_b200.models import gated_pixel_cnn

    _mutate_fn(monkeypatch, gated_pixel_cnn.GatedPixelCNNLayer, "forward_pm", old, new)


def bug_hstack_residual_from_bf16_copy(monkeypatch):
    """`_hstack_residual` adds the horizontal stream from its bf16 copy h_b instead of the fp32 stream h_f."""
    _mutate_layer(monkeypatch, "res=None if self._mask_center else h_f,", "res=None if self._mask_center else h_b,")


def bug_input_gate_reads_bf16_sum(monkeypatch):
    """The input layer's vertical gate reads bf16(v2 + 1x1(image)) instead of the fp32 sum (a no-op on later layers,
    whose gate input is bf16 already)."""
    _mutate_layer(monkeypatch, "v_out = pm.gated(vv, TANH)", "v_out = pm.gated(vv.to(torch.bfloat16), TANH)")


def bug_hs_gradient_from_skip_only(monkeypatch):
    """Of the two consumers of the horizontal gate's output, only `_hstack_skip`'s gradient reaches the gate:
    `_hstack_residual` reads a leaf copy of hs, so it still computes its input gradient, which then goes nowhere."""
    _mutate_layer(monkeypatch, "h_f, h_b = pm.conv(hs,", "h_f, h_b = pm.conv(hs.detach().requires_grad_(),")


def bug_input_hstack_sees_current_pixel(monkeypatch):
    """The input layer's horizontal image convolution is padded (0, p) instead of (0, p + 1): its 1 x (k // 2 + 1)
    window ends on the current pixel, which the causal layer must not see."""
    _mutate_layer(monkeypatch, "self._hstack_1xN.bias, (0, p + int(self._mask_center)))",
                  "self._hstack_1xN.bias, (0, p))")


def bug_small_conv_dw_from_bf16_dy(monkeypatch):
    """The direct image convolution's backward rounds its incoming gradient to bf16 before the weight gradient."""
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._SmallConv, "backward", "dy = dy.contiguous().float()",
               "dy = dy.contiguous().to(BF16).float()")


def bug_gated_res_dres_in_bf16(monkeypatch):
    """`_GatedRes.backward` hands the residual its incoming gradient rounded to bf16."""
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._GatedRes, "backward", "return dx, dy, None", "return dx, dy.to(BF16).float(), None")


def bug_residual_out_emits_pre_grad(monkeypatch):
    """`_residual_out` emits its ELU as PRE_GRAD instead of POST, so its backward never applies its own ELU'."""
    from pytorch_generative_b200.models import pixel_snail
    from pytorch_generative_b200.nn import pm

    conv = lambda *a, **kw: pm.conv(*a, **dict(kw, emit_mode=pm.PRE_GRAD))
    _mutate_fn(monkeypatch, pixel_snail.PixelSNAILBlock, "forward_pm", "_, r = pm.conv(res,", "_, r = _conv(res,",
               dict(_conv=conv))


def bug_post_backward_with_relu(monkeypatch):
    """The POST backward takes the activated output's derivative as ReLU's, whatever the emitted activation."""
    from pytorch_generative_b200.nn import pm

    BR._mutate(monkeypatch, pm._Conv, "backward", "L.dact_from_out(dya.contiguous(), ya, emit, d)",
               "L.dact_from_out(dya.contiguous(), ya, L.ACT_RELU, d)")


def bug_attention_not_strict(monkeypatch):
    """PixelSNAIL's attention lets each position see its own key."""
    from pytorch_generative_b200.nn import modules

    BR._mutate(monkeypatch, modules._AttentionPMFn, "forward", "n, h, w = geom", "n, h, w = geom; strict = False")


def bug_positions_rows_and_columns_swapped(monkeypatch):
    """The attention operand's position columns hold (column, row) instead of (row, column)."""
    from pytorch_generative_b200.models import pixel_snail

    _mutate_fn(monkeypatch, pixel_snail.PixelSNAIL, "forward", "._positions(x.shape, x.device)",
               "._positions(x.shape, x.device).flip(1)")


def bug_attention_da_without_q(monkeypatch):
    """The attention's input gradient leaves without the q projection's share."""
    from pytorch_generative_b200.nn import modules

    _mutate_fn(monkeypatch, modules, "_attention_bwd", "da_kv[:, :cin] += da_q[:, :cin]", "pass")


def bug_residual_out_reads_a_leaf(monkeypatch):
    """`_residual_out` reads a leaf copy of res: it still computes its input gradient, which then reaches no stream."""
    from pytorch_generative_b200.models import pixel_snail

    _mutate_fn(monkeypatch, pixel_snail.PixelSNAILBlock, "forward_pm", "_, r = pm.conv(res,",
               "_, r = pm.conv(res.detach().requires_grad_(),")


# name -> (apply(monkeypatch), the stage kind (R.kind_of) that must fail, the geometries that run the code it changes)
BUGS = {
    "fp32_dres_from_bf16_operand": (bug_fp32_dres_from_bf16_operand, "conv.dres", None),
    "transposed_bias_grad_before_emit": (bug_transposed_bias_grad_before_emit, "transposed.db", "stride4"),
    "pack_taps_t_kh_kw_swapped": (bug_pack_taps_t_kh_kw_swapped, "transposed.y", None),
    "commitment_scale_per_row": (bug_commitment_scale_per_row, "quantizer.dx", "vq"),
    "transposed_dx_without_in_act": (bug_transposed_dx_without_in_act, "transposed.dx", None),
    "gather_dx_without_in_act": (bug_gather_dx_without_in_act, "conv.dx", None),
    "hstack_residual_from_bf16_copy": (bug_hstack_residual_from_bf16_copy, "conv.y", "gated"),
    "input_gate_reads_bf16_sum": (bug_input_gate_reads_bf16_sum, "gate.x", "gated"),
    "hs_gradient_from_skip_only": (bug_hs_gradient_from_skip_only, "gate.dy", "gated"),
    "small_conv_dw_from_bf16_dy": (bug_small_conv_dw_from_bf16_dy, "small.dw", "gated"),
    "input_hstack_sees_current_pixel": (bug_input_hstack_sees_current_pixel, "small.y", "gated"),
    "gated_res_dres_in_bf16": (bug_gated_res_dres_in_bf16, "gated_res.dres", "snail"),
    "residual_out_emits_pre_grad": (bug_residual_out_emits_pre_grad, "conv.db", "snail"),
    # dw, db and dx are checked from the recorded dact_from_out operand, so a wrong derivative shows at that operand
    "post_backward_with_relu": (bug_post_backward_with_relu, "conv.dya", "snail"),
    "attention_not_strict": (bug_attention_not_strict, "attention.o", "snail"),
    "positions_rows_and_columns_swapped": (bug_positions_rows_and_columns_swapped, "attention.a_kv", "snail"),
    "attention_da_without_q": (bug_attention_da_without_q, "attention.da_kv", "snail"),
    "residual_out_reads_a_leaf": (bug_residual_out_reads_a_leaf, "gated_res.dy", "snail"),
}
