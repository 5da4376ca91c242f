"""Drives ImageGPT's fused stack (models/image_gpt.py) for the stage-replay tests: builds a model with parameters well
away from their initial values, records the backward intermediates the stack hands between its kernels, maps the
forward's saved activations and those records to the stage names of tests/_block_reference.py, and holds the bug models
the replay must reject.  Shared by tests/test_block_bounds_cpu.py and tests/test_block_kernels_gpu.py; not a test
module."""

import inspect
import sys
import textwrap

import torch

import _block_reference as R

BF16 = torch.bfloat16


def build(C, heads, shape, cout, n_blocks=2, seed=0, device="cpu"):
    """(model, x, G): an ImageGPT on `device` whose LayerNorm gammas are 1 + 0.5 N(0, 1), whose LayerNorm betas, biases
    and positional parameter are N(0, 0.5^2) (the other weights keep their initialisation), an image batch of `shape`
    in [0, 1) and a unit-scale cotangent of the logits."""
    from pytorch_generative_b200 import models

    n, cin, h, w = shape
    torch.manual_seed(seed)
    m = models.ImageGPT(in_channels=cin, out_channels=cout, in_size=max(h, w), n_transformer_blocks=n_blocks,
                        n_attention_heads=heads, n_embedding_channels=C)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            rn = torch.randn(p.shape, generator=g)
            if name.endswith("weight") and ("_ln" in name):
                p.copy_(1 + 0.5 * rn)
            elif name.endswith("bias") or name == "_pos":
                p.copy_(0.5 * rn)
    x = torch.rand(shape, generator=g)
    G = torch.randn(n, cout, h, w, generator=g)
    return m.to(device), x.to(device), G.to(device)


def geometry(m, x):
    n, cin, h, w = x.shape
    return R.geometry(n, cin, h, w, m._ln.weight.numel(), m._n_heads, m._out.weight.shape[0])


class Recorder:
    """Wraps ops.linear_dgrad, ops.layernorm_bwd, ops.attn_bwd, _lib.conv_small_bwd and GradArena.block.  A record is
    labelled by the identity of its weight (dgrad), of the tensor it normalises (LayerNorm) or of the attention output
    (attention), never by call order."""

    def __init__(self, monkeypatch):
        from pytorch_generative_b200 import _lib, ops
        from pytorch_generative_b200.models import image_gpt

        self.dgrad, self.ln, self.attn, self.conv, self.arena = {}, {}, {}, [], {}
        dgrad, ln_bwd, a_bwd, conv_bwd, block = (ops.linear_dgrad, ops.layernorm_bwd, ops.attn_bwd,
                                                 _lib.conv_small_bwd, image_gpt.GradArena.block)

        def linear_dgrad(dy, w, **kw):
            out = dgrad(dy, w, **kw)
            self.dgrad[id(w)] = dict(dy=dy, out=out)
            return out

        def layernorm_bwd(dy, x, *args, **kw):
            out = ln_bwd(dy, x, *args, **kw)
            self.ln[id(x)] = dict(dy=dy, out=out)
            return out

        def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, *args):
            out = a_bwd(q, k, v, o, do, lse, dq, dk, dv, *args)
            self.attn[id(o)] = dict(do=do, dq=dq, dk=dk, dv=dv)
            return out

        def conv_small_bwd(x, w, dy_pm, *args, **kw):
            self.conv.append(dy_pm)
            return conv_bwd(x, w, dy_pm, *args, **kw)

        def arena_block(arena, b):
            views = block(arena, b)
            self.arena[b] = views
            return views

        monkeypatch.setattr(ops, "linear_dgrad", linear_dgrad)
        monkeypatch.setattr(ops, "layernorm_bwd", layernorm_bwd)
        monkeypatch.setattr(ops, "attn_bwd", attn_bwd)
        monkeypatch.setattr(_lib, "conv_small_bwd", conv_small_bwd)
        monkeypatch.setattr(image_gpt.GradArena, "block", arena_block)


def forward_flat(m, x):
    """ImageGPT.forward's call of the fused node, without its CUDA check: the flat parameter list assembled as forward
    assembles it, every activation kept (the store path)."""
    from pytorch_generative_b200.models import image_gpt

    m._input.apply_mask()
    flat = [m._pos, m._input.weight, m._input.bias]
    for blk in m._transformer:
        flat.extend(blk.flat_params())
    flat.extend([m._ln.weight, m._ln.bias, m._out.weight, m._out.bias])
    return image_gpt._ImageGPTStack.apply(x.float(), m._n_heads, m._ln.eps, m._packed_training_weights(),
                                          dict(grad=True, hook=None, recompute=False), *flat)


def step(m, x, G, rec, forward):
    """One forward and backward; returns (logits, the node's saved dict, its per-block activations) as the forward left
    them (backward releases them from the node)."""
    for p in m.parameters():
        p.grad = None
    logits = forward(m, x)
    sv = dict(logits.grad_fn.saved)
    blocks = list(sv["blocks"])
    (logits * G).sum().backward()
    return logits, sv, blocks


def kernel_table(sv, blocks, rec, logits, g):
    """(stage name -> the product's tensor in true layout, stage name -> the pad that must be exactly zero)."""
    C, H, dk = g.C, g.H, g.dk
    T, Z = {}, {}

    def stream(name, t, width=C):
        T[name], Z[name] = t[:, :width], t[:, width:]

    def heads(name, t, slot):
        v = t.reshape(t.shape[0], H, slot)
        T[name], Z[name] = v[:, :, :dk].reshape(t.shape[0], H * dk), v[:, :, dk:]

    stream("stem.xs", blocks[0]["xs"])
    for b, blk in enumerate(blocks):
        s = f"b{b}."
        for k in ("mean1", "rstd1", "mean2", "rstd2", "lse"):
            T[s + k] = blk[k]
        for k in ("a1", "h", "a2"):
            stream(s + k, blk[k])
        nq = H * g.qk_slot
        qkv = blk["qkv"]
        parts = [(qkv[:, :nq], g.qk_slot), (qkv[:, nq: 2 * nq], g.qk_slot), (qkv[:, 2 * nq:], g.dv_slot)]
        for j, (t, slot) in enumerate(parts):
            heads(f"{s}qkv{j}", t, slot)
        T[s + "qkv"] = torch.cat([T.pop(f"{s}qkv{j}") for j in range(3)], dim=1)
        Z[s + "qkv"] = torch.cat([Z.pop(f"{s}qkv{j}").reshape(-1) for j in range(3)])
        heads(s + "o", blk["o"], g.dv_slot)
        stream(s + "g", blk["g"], 4 * C)
        T[s + "u"] = blk["u"][:, : 4 * C]  # u = GELU'(pre) is 0.5 in the pad, where it only meets zero gradients
        stream(s + "x_next", blocks[b + 1]["xs"] if b + 1 < len(blocks) else sv["xs_final"])
    T["head.mean"], T["head.rstd"] = sv["mean_f"], sv["rstd_f"]
    stream("head.af", sv["af"])
    T["head.logits"] = logits.detach().permute(0, 2, 3, 1).reshape(g.P, g.cout)

    r = rec.dgrad[id(sv["wo"])]
    T["head.dl"] = r["dy"]
    stream("head.daf", r["out"])
    r = rec.ln[id(sv["xs_final"])]["out"]
    stream("head.dx", r[0])
    stream("head.dx_b", r[1])
    for b, blk in enumerate(blocks):
        s = f"b{b}."
        stream(s + "du", rec.dgrad[id(blk["w2"])]["out"], 4 * C)
        stream(s + "da2", rec.dgrad[id(blk["w1"])]["out"])
        r = rec.ln[id(blk["h"])]["out"]
        stream(s + "dh", r[0])
        stream(s + "dh_b", r[1])
        heads(s + "do", rec.dgrad[id(blk["wp"])]["out"], g.dv_slot)
        r = rec.attn[id(blk["o"])]
        heads(s + "dq", r["dq"], g.qk_slot)
        heads(s + "dk", r["dk"], g.qk_slot)
        heads(s + "dv", r["dv"], g.dv_slot)
        stream(s + "da1", rec.dgrad[id(blk["wqkv"])]["out"])
        r = rec.ln[id(blk["xs"])]["out"]
        stream(s + "dx_in", r[0])
        stream(s + "dx_in_b", r[1])
    assert len(rec.conv) == 1
    stream("stem.dy", rec.conv[0])
    return T, Z


def arena_pads(views, g, dev):
    """The pad rows and columns of one block's packed gradients (GradArena.block), which must stay exactly zero."""
    from pytorch_generative_b200.nn.modules import head_layout

    C, H = g.C, g.H
    lay = head_layout(H, C, C, dev)

    def live(n, idx):
        m = torch.zeros(n, dtype=torch.bool, device=dev)
        m[idx] = True
        return m

    nq = H * g.qk_slot
    qkv_rows = torch.cat((live(nq, lay.rows_q), live(g.qkv_cols - nq, lay.rows_kv)))
    cols_v = live(H * g.dv_slot, lay.cols_v)
    c, f = live(g.c_p, slice(0, C)), live(g.f_p, slice(0, 4 * C))
    return dict(dw2=views.dw2[~c], dw2c=views.dw2[:, ~f], dw1=views.dw1[~f], dw1c=views.dw1[:, ~c],
                dwp=views.dwp[~c], dwpc=views.dwp[:, ~cols_v], dwqkv=views.dwqkv[~qkv_rows],
                dwqkvc=views.dwqkv[:, ~c], dbqkv=views.dbqkv[~qkv_rows], db1=views.db1[~f])


def replay(m, x, G, logits, sv, blocks, rec):
    """The stage replay of one step (tests/_block_reference.py): every stage and parameter gradient, every pad."""
    g = geometry(m, x)
    T, Z = kernel_table(sv, blocks, rec, logits, g)
    mode = R.Replay(T, dict(m.named_parameters()))
    W = R.weights(dict(m.named_parameters()), len(blocks), lambda t: t.to(BF16))
    pos = m._pos.detach()[:, :, : g.h, : g.w]
    x_in = (x.float() + pos).to(R.F64)
    R.run(W, g, x_in, G.permute(0, 2, 3, 1).reshape(g.P, g.cout), m._ln.eps, mode)
    for name, t in Z.items():
        mode.zero(name + ".pad", t)
    for b, views in rec.arena.items():
        for name, t in arena_pads(views, g, x.device).items():
            mode.zero(f"b{b}.arena.{name}", t)
    return mode


# ----------------------------------------------------------------------------------------------------------------------
# bug models: each changes only which valid tensor or argument the product passes, never a shape, pitch or pointer
# ----------------------------------------------------------------------------------------------------------------------
def _mutate(monkeypatch, cls, name, old, new):
    """Replaces the static method cls.name by a copy of its source with `old` (which must occur once) replaced by
    `new`, compiled in its module's namespace."""
    fn = inspect.getattr_static(cls, name).__func__
    src = textwrap.dedent(inspect.getsource(fn))
    assert src.count(old) == 1, (name, old)
    src = src.replace(old, new).replace("@staticmethod\n", "")
    ns = {}
    exec(compile(src, f"<mutated {name}>", "exec"), sys.modules[fn.__module__].__dict__, ns)
    monkeypatch.setattr(cls, name, staticmethod(ns[fn.__name__]))


def _wrap_scatter(monkeypatch, change):
    from pytorch_generative_b200.nn.modules import HeadLayout

    scatter = HeadLayout.scatter
    monkeypatch.setattr(HeadLayout, "scatter", lambda self, *a: change(self, *scatter(self, *a)))


def bug_qk_swapped(monkeypatch):
    def change(lay, wq, bq, wkv, bkv, wp):
        n = lay.n_heads * lay.qk_slot
        return (wkv[:n], bkv[:n], torch.cat((wq, wkv[n:])), torch.cat((bq, bkv[n:])), wp)
    _wrap_scatter(monkeypatch, change)


def bug_heads_rotated(monkeypatch):
    def change(lay, wq, bq, wkv, bkv, wp):
        n = lay.n_heads * lay.qk_slot
        kv = lambda t: torch.cat((t[:n].roll(lay.qk_slot, 0), t[n:].roll(lay.dv_slot, 0)))
        return wq.roll(lay.qk_slot, 0), bq.roll(lay.qk_slot, 0), kv(wkv), kv(bkv), wp
    _wrap_scatter(monkeypatch, change)


def bug_attention_scale_from_slot(monkeypatch):
    from pytorch_generative_b200 import ops

    fwd, bwd = ops.attn_fwd, ops.attn_bwd

    def attn_fwd(q, k, v, n_img, seq, heads, dk_true, qk_slot, dv_slot, strict):
        return fwd(q, k, v, n_img, seq, heads, qk_slot, qk_slot, dv_slot, strict)

    def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, n_img, seq, heads, dk_true, qk_slot, dv_slot, strict):
        return bwd(q, k, v, o, do, lse, dq, dk, dv, n_img, seq, heads, qk_slot, qk_slot, dv_slot, strict)
    monkeypatch.setattr(ops, "attn_fwd", attn_fwd)
    monkeypatch.setattr(ops, "attn_bwd", attn_bwd)


def _wrap_linear_fwd(monkeypatch, before=None, after=None):
    from pytorch_generative_b200 import ops

    fwd = ops.linear_fwd

    def linear_fwd(a, w, bias=None, **kw):
        if before:
            before(kw)
        out = fwd(a, w, bias, **kw)
        if after:
            after(kw, out)
        return out
    monkeypatch.setattr(ops, "linear_fwd", linear_fwd)


def bug_single_residual(monkeypatch):
    def before(kw):
        if kw.get("res1") is not None:  # fc2: x_next = h + fc2(...), the stream x left out
            kw["res0"], kw["res1"] = kw["res1"], None
    _wrap_linear_fwd(monkeypatch, before=before)


def bug_u_holds_gelu(monkeypatch):
    def after(kw, out):
        if kw.get("pre_deriv"):
            out[1].copy_(out[0])
    _wrap_linear_fwd(monkeypatch, after=after)


def _wrap_layernorm_bwd(monkeypatch, drop):
    from pytorch_generative_b200 import ops

    bwd = ops.layernorm_bwd

    def layernorm_bwd(dy, x, gamma, mean, rstd, dres0=None, dres1=None, **kw):
        if dres1 is not None:  # LN1: the only LayerNorm backward with two residual gradients
            dres0, dres1 = (None, dres1) if drop == "dres0" else (dres0, None)
        return bwd(dy, x, gamma, mean, rstd, dres0=dres0, dres1=dres1, **kw)
    monkeypatch.setattr(ops, "layernorm_bwd", layernorm_bwd)


def _wrap_block_bwd(monkeypatch, fn):
    from pytorch_generative_b200.models import image_gpt

    monkeypatch.setattr(image_gpt, "_block_bwd", lambda *a, _orig=image_gpt._block_bwd: fn(_orig, *a))


def bug_proj_bias_grad_from_dx_sum(monkeypatch):
    def fn(orig, *a):
        grads, dx, dx_b, dx_sum = orig(*a)
        return grads._replace(p_b=grads.f2_b), dx, dx_b, dx_sum
    _wrap_block_bwd(monkeypatch, fn)


def bug_fc1_wgrad_reads_a1(monkeypatch):
    _wrap_block_bwd(monkeypatch, lambda orig, blk, *a: orig(dict(blk, a2=blk["a1"]), *a))


def bug_kv_swapped_in_unpack_grads(monkeypatch):
    from pytorch_generative_b200.nn.modules import HeadLayout

    unpack = HeadLayout.unpack_grads

    def unpack_grads(self, *a):
        dq_w, dq_b, dkv_w, dkv_b, dp_w = unpack(self, *a)
        e = self.embed
        return dq_w, dq_b, torch.cat((dkv_w[e:], dkv_w[:e])), torch.cat((dkv_b[e:], dkv_b[:e])), dp_w
    monkeypatch.setattr(HeadLayout, "unpack_grads", unpack_grads)


def bug_ln2_stats_share_ln1_view(monkeypatch):
    from pytorch_generative_b200.models import image_gpt

    block = image_gpt.GradArena.block
    monkeypatch.setattr(image_gpt.GradArena, "block",
                        lambda self, b: (lambda v: v._replace(ln2_stats=v.ln1_stats))(block(self, b)))


def bug_stem_bias_grad_from_wrong_colsum(monkeypatch):
    from pytorch_generative_b200.models import image_gpt

    _mutate(monkeypatch, image_gpt._ImageGPTStack, "backward", "stem_grads = (dpos, din_w, dx_sum)",
            "stem_grads = (dpos, din_w, block_grads[0].f2_b)")


def bug_dpos_summed_over_channels_too(monkeypatch):
    from pytorch_generative_b200.models import image_gpt

    _mutate(monkeypatch, image_gpt._ImageGPTStack, "backward", "dx_in.sum(dim=0, keepdim=True)",
            "dx_in.sum(dim=(0, 1), keepdim=True)")


# name -> (apply(monkeypatch), the stage kind (R.kind) that must fail, True when it only reaches heads narrower than
# their kernel slots: the scatter packing path and a scale that differs from the slot's)
BUGS = {
    "qk_swapped_in_scatter": (bug_qk_swapped, "qkv", True),
    "heads_rotated_one_slot": (bug_heads_rotated, "qkv", True),
    "attention_scale_from_slot": (bug_attention_scale_from_slot, "o", True),
    "single_residual": (bug_single_residual, "x_next", False),
    "u_holds_gelu": (bug_u_holds_gelu, "u", False),
    "ln1_bwd_without_dres1": (lambda mp: _wrap_layernorm_bwd(mp, "dres1"), "dx_in", False),
    "ln1_bwd_without_dres0": (lambda mp: _wrap_layernorm_bwd(mp, "dres0"), "dx_in", False),
    "proj_bias_grad_from_dx_sum": (bug_proj_bias_grad_from_dx_sum, "grad _attn._proj.bias", False),
    "fc1_wgrad_reads_a1": (bug_fc1_wgrad_reads_a1, "grad _out.0.weight", False),
    "kv_swapped_in_unpack_grads": (bug_kv_swapped_in_unpack_grads, "grad _attn._kv.weight", False),
    "ln2_stats_share_ln1_view": (bug_ln2_stats_share_ln1_view, "grad _ln2.weight", False),
    "stem_bias_grad_from_wrong_colsum": (bug_stem_bias_grad_from_wrong_colsum, "grad _input.bias", False),
    "dpos_summed_over_channels_too": (bug_dpos_summed_over_channels_too, "grad _pos", False),
}
