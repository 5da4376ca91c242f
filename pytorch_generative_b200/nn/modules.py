"""Drop-in building blocks: same constructor signatures, parameter/buffer names and shapes as
`pytorch_generative.nn` (reference nn/convolution.py, nn/attention.py), arithmetic on the sm_90a kernels.

Each module takes and returns NCHW fp32 tensors like the reference (outputs are contiguous NCHW; the
reference's NCHWLayerNorm returns a channels-last-strided view, SURVEY.md §7.3-5).  Internally the data is
converted once to the pixel-major layout the kernels use.  The fused model stacks in `models/` bypass these
per-module conversions, but share the same `ops` primitives.
"""

import functools
import math

import torch
from torch import nn

from .. import _lib as L
from .. import ops

F32, BF16 = torch.float32, torch.bfloat16


def _require_cuda(x, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")


# --------------------------------------------------------------------------------------------------
# CausalConv2d
# --------------------------------------------------------------------------------------------------
class _SmallConvFn(torch.autograd.Function):
    """Direct conv for image-channel inputs (Cin*kh*kw <= 160): NCHW in, NCHW out."""

    @staticmethod
    def forward(ctx, x, weight, bias, padding, pre_act):
        x = x.contiguous().float()
        n, _, h, w = x.shape
        cout = weight.shape[0]
        out_pm = torch.empty(n * h * w, cout, dtype=F32, device=x.device)
        L.conv_small_fwd(x, weight.detach().contiguous(), None if bias is None else bias.detach(), padding,
                         out_f32=out_pm, pre_act=pre_act)
        ctx.save_for_backward(x, weight)
        ctx.padding, ctx.has_bias, ctx.pre_act = padding, bias is not None, pre_act
        return ops.pm_to_nchw(out_pm, n, cout, h, w)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        n, cout, h, w = dy.shape
        dy_pm = ops.nchw_to_pm(dy, F32)
        dw = torch.zeros_like(weight)
        db = torch.zeros(cout, dtype=F32, device=dy.device) if ctx.has_bias else None
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        L.conv_small_bwd(x, weight.detach().contiguous(), dy_pm, ctx.padding, dw=dw, dbias=db, dx=dx,
                         pre_act=ctx.pre_act)
        return dx, dw, db, None, None


class CausalConv2d(nn.Conv2d):
    """Conv2d masked so that a pixel only sees pixels above it and to its left (and itself unless
    `mask_center`) — API of reference nn/convolution.py:12-43.

    As in the reference, the 0/1 `mask` buffer has the weight's shape and `forward` zeroes the masked taps of
    the Parameter in place before convolving; the weight gradient is dense over all taps.
    """

    def __init__(self, mask_center, *args, **kwargs):
        super().__init__(*args, **kwargs)
        kh, kw = self.weight.shape[-2:]
        mask = torch.zeros_like(self.weight)
        mask[:, :, : kh // 2, :] = 1
        mask[:, :, kh // 2, : kw // 2 + (0 if mask_center else 1)] = 1
        self.register_buffer("mask", mask)

    def forward(self, x, pre_act=L.ACT_NONE):
        """`pre_act` (CUDA-path extension) fuses an activation applied to the conv's input."""
        _require_cuda(x, "CausalConv2d")
        self.weight.data *= self.mask
        cout, cin, kh, kw = self.weight.shape
        pad = self.padding if isinstance(self.padding, tuple) else (self.padding, self.padding)
        if self.stride != (1, 1) or self.dilation != (1, 1) or self.groups != 1 or self.padding_mode != "zeros":
            raise NotImplementedError("CausalConv2d: only stride 1, dilation 1, groups 1, zero padding are on the path")
        if pad != (kh // 2, kw // 2):
            raise NotImplementedError("CausalConv2d: only 'same' padding (k//2) is on the path")
        from .tapconv import small_conv_ok, tap_conv2d  # wide-channel masked convs run as a tap list on the wgmma GEMM

        if small_conv_ok(self.weight.shape):
            return _SmallConvFn.apply(x, self.weight, self.bias, pad, pre_act)

        return tap_conv2d(x, self.weight, self.bias, pad, pre_act=pre_act)


# --------------------------------------------------------------------------------------------------
# GatedActivation
# --------------------------------------------------------------------------------------------------
class _GatedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, act):
        n, c2, h, w = x.shape
        x_pm = ops.nchw_to_pm(x, F32)
        y_pm = torch.empty(n * h * w, c2 // 2, dtype=F32, device=x.device)
        L.gated_act_fwd(x_pm, y_pm, act)
        ctx.save_for_backward(x_pm)
        ctx.act, ctx.shape = act, (n, c2, h, w)
        return ops.pm_to_nchw(y_pm, n, c2 // 2, h, w)

    @staticmethod
    def backward(ctx, dy):
        (x_pm,) = ctx.saved_tensors
        n, c2, h, w = ctx.shape
        dy_pm = ops.nchw_to_pm(dy, F32)
        dx_pm = torch.empty_like(x_pm)
        L.gated_act_bwd(x_pm, dy_pm, dx_pm, ctx.act)
        return ops.pm_to_nchw(dx_pm, n, c2, h, w), None


def _activation_id(fn):
    if fn is torch.tanh or fn is torch.nn.functional.tanh or isinstance(fn, nn.Tanh):
        return L.ACT_TANH
    if fn is None or isinstance(fn, nn.Identity):
        return L.ACT_NONE
    raise NotImplementedError(
        f"GatedActivation: activation_fn {fn!r} is not on the CUDA path (torch.tanh and nn.Identity() are, "
        "the two the reference models use)"
    )


class GatedActivation(nn.Module):
    """activation_fn(x[:, :C/2]) * sigmoid(x[:, C/2:]) — API of reference nn/convolution.py:46-66."""

    def __init__(self, activation_fn=torch.tanh):
        super().__init__()
        self._activation_fn = activation_fn
        self._act_id = _activation_id(activation_fn)

    def forward(self, x):
        _require_cuda(x, "GatedActivation")
        c = x.shape[1]
        assert c % 2 == 0, "x must have an even number of channels."
        if (c // 2) % 8 != 0:
            raise NotImplementedError("GatedActivation: C/2 must be a multiple of 8 on the CUDA path")
        return _GatedFn.apply(x, self._act_id)


# --------------------------------------------------------------------------------------------------
# NCHWLayerNorm
# --------------------------------------------------------------------------------------------------
class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        n, c, h, w = x.shape
        x_pm = ops.nchw_to_pm(x, F32)
        _, y_pm, mean, rstd = ops.layernorm_fwd(x_pm, gamma.detach(), beta.detach(), eps, want_bf16=False,
                                                want_f32=True)
        ctx.save_for_backward(x_pm, gamma, mean, rstd)
        ctx.shape = (n, c, h, w)
        return ops.pm_to_nchw(y_pm, n, c, h, w)

    @staticmethod
    def backward(ctx, dy):
        x_pm, gamma, mean, rstd = ctx.saved_tensors
        n, c, h, w = ctx.shape
        dy_pm = ops.nchw_to_pm(dy, F32)
        dx_pm, _, dg, db = ops.layernorm_bwd(dy_pm, x_pm, gamma.detach(), mean, rstd, want_bf16=False)
        return ops.pm_to_nchw(dx_pm, n, c, h, w), dg, db, None


class NCHWLayerNorm(nn.LayerNorm):
    """LayerNorm over the channel dimension of NCHW tensors — API of reference nn/convolution.py:69-75."""

    def forward(self, x):
        _require_cuda(x, "NCHWLayerNorm")
        if not self.elementwise_affine:
            raise NotImplementedError("NCHWLayerNorm: elementwise_affine=False is not on the path")
        return _LayerNormFn.apply(x, self.weight, self.bias, self.eps)


# --------------------------------------------------------------------------------------------------
# image_positional_encoding
# --------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=32)
def image_positional_encoding(shape):
    """(N, 2, H, W) tensor of (row, col) coordinates scaled to [-.5, .5) — reference nn/attention.py:37-57.

    Built with the same float-step `arange` so the values are bit-identical to the reference's.
    """
    n, _, h, w = shape
    rows = torch.arange(-0.5, 0.5, 1 / h).view(1, 1, h, 1).expand(n, 1, h, w)
    cols = torch.arange(-0.5, 0.5, 1 / w).view(1, 1, 1, w).expand(n, 1, h, w)
    return torch.cat((rows, cols), dim=1)


# --------------------------------------------------------------------------------------------------
# CausalAttention
# --------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=64)
def head_slot_rows(n_heads, per_head, slot, device=None, offset=0):
    """Row indices that scatter `n_heads * per_head` projection rows into `slot`-wide head slots.  Cached per
    device: the index tensor is built once, so steady-state calls issue no host->device copy (graph-capturable)."""
    idx = torch.arange(n_heads * per_head)
    return ((idx // per_head) * slot + idx % per_head + offset).to(device)


def pack_qkv_weights(q_w, q_b, kv_w, kv_b, n_heads, embed, out_ch, cin_q_pad, cin_kv_pad):
    """Builds the slot-padded projection matrices used by the attention kernels.

    Returns (Wq [H*qk_slot, cin_q_pad] bf16, bq [H*qk_slot] fp32, Wkv [H*qk_slot + H*dv_slot, cin_kv_pad] bf16, bkv,
    meta), slot widths from ops.head_slots.  Rows of padded slots are zero, so padded q/k/v columns are exactly zero.
    """
    dk, dv = embed // n_heads, out_ch // n_heads
    qk_slot, dv_slot = ops.head_slots(dk, dv)
    dev = q_w.device
    if dk == qk_slot and dv == dv_slot and q_w[0].numel() == cin_q_pad and kv_w[0].numel() == cin_kv_pad:
        # heads already fill their slots (e.g. ImageGPT 512ch / 8 or 4 heads): no scatter, just cast
        meta = dict(dk=dk, dv=dv, qk_slot=qk_slot, dv_slot=dv_slot, rows_q=None, rows_v=None, identity=True)
        return (ops.to_bf16(q_w.detach().reshape(embed, -1)), q_b.detach(),
                ops.to_bf16(kv_w.detach().reshape(embed + out_ch, -1)), kv_b.detach(), meta)
    rows_q = head_slot_rows(n_heads, dk, qk_slot, dev)
    rows_v = head_slot_rows(n_heads, dv, dv_slot, dev, n_heads * qk_slot)
    wq = torch.zeros(n_heads * qk_slot, cin_q_pad, dtype=F32, device=dev)
    wq[rows_q, : q_w.shape[1]] = q_w.detach().reshape(q_w.shape[0], -1)
    bq = torch.zeros(n_heads * qk_slot, dtype=F32, device=dev)
    bq[rows_q] = q_b.detach()
    wkv = torch.zeros(n_heads * (qk_slot + dv_slot), cin_kv_pad, dtype=F32, device=dev)
    kv2 = kv_w.detach().reshape(kv_w.shape[0], -1)
    wkv[rows_q, : kv2.shape[1]] = kv2[:embed]
    wkv[rows_v, : kv2.shape[1]] = kv2[embed:]
    bkv = torch.zeros(n_heads * (qk_slot + dv_slot), dtype=F32, device=dev)
    bkv[rows_q] = kv_b.detach()[:embed]
    bkv[rows_v] = kv_b.detach()[embed:]
    meta = dict(dk=dk, dv=dv, qk_slot=qk_slot, dv_slot=dv_slot, rows_q=rows_q, rows_v=rows_v, identity=False)
    return ops.to_bf16(wq), bq, ops.to_bf16(wkv), bkv, meta


class _AttentionFn(torch.autograd.Function):
    """q/kv projections -> causal attention core -> output projection, all on pixel-major bf16."""

    @staticmethod
    def forward(ctx, x, extra, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, strict):
        n, cin, h, w = x.shape
        S, P, H = h * w, n * h * w, n_heads
        cin_p = ops.round_up(cin, 8)
        ce = 0 if extra is None else extra.shape[1]
        ckv_p = ops.round_up(cin + ce, 8)
        wq, bq, wkv, bkv, meta = pack_qkv_weights(q_w, q_b, kv_w, kv_b, H, embed, out_ch, cin_p, ckv_p)
        qk_slot, dv_slot = meta["qk_slot"], meta["dv_slot"]
        # A operand for the kv projection: [x | extra | 0-pad]; the q projection reads its first cin_p columns
        # (columns cin..cin_p of Wq are zero, so reading a few `extra` columns there is harmless).
        a_kv = torch.zeros(P, ckv_p, dtype=BF16, device=x.device)
        L.nchw_to_pm(x.contiguous().float(), a_kv[:, :cin])
        if extra is not None:
            L.nchw_to_pm(extra.contiguous().float(), a_kv[:, cin:cin + ce])
        q, _, _ = ops.linear_fwd(a_kv[:, :cin_p], wq, bq)
        kv, _, _ = ops.linear_fwd(a_kv, wkv, bkv)
        k, v = kv[:, : H * qk_slot], kv[:, H * qk_slot:]
        o, lse = ops.attn_fwd(q, k, v, n, S, H, meta["dk"], qk_slot, dv_slot, strict)
        # output projection reads the slot-padded o through a column-scattered weight
        if meta["identity"]:
            cols_v = None
            wp = ops.pack_weight(p_w)
        else:
            wp = torch.zeros(out_ch, H * dv_slot, dtype=F32, device=x.device)
            cols_v = meta["rows_v"] - H * qk_slot
            wp[:, cols_v] = p_w.detach().reshape(out_ch, -1)
            wp = ops.to_bf16(wp)
        _, _, y_pm = ops.linear_fwd(o, wp, p_b.detach(), want_bf16=False, want_f32=True)
        ctx.save_for_backward(a_kv, q, kv, o, lse, wq, wkv, wp)
        ctx.meta = dict(meta, n=n, h=h, w=w, cin=cin, ce=ce, cin_p=cin_p, H=H, embed=embed, out_ch=out_ch, strict=strict,
                        cols_v=cols_v)
        return ops.pm_to_nchw(y_pm, n, out_ch, h, w)

    @staticmethod
    def backward(ctx, dy):
        a_kv, q, kv, o, lse, wq, wkv, wp = ctx.saved_tensors
        m = ctx.meta
        n, h, w, H, qk_slot, dv_slot = m["n"], m["h"], m["w"], m["H"], m["qk_slot"], m["dv_slot"]
        S, P = h * w, n * h * w
        dev = dy.device
        dy_b = ops.nchw_to_pm(dy, BF16, width=ops.round_up(m["out_ch"], 8))
        # projection
        dp_b = ops.bias_grad(dy_b[:, : m["out_ch"]])
        dwp = torch.zeros(ops.round_up(m["out_ch"], 8), H * dv_slot, dtype=F32, device=dev)
        ops.linear_wgrad(dy_b, o, dwp)
        do = ops.linear_dgrad(dy_b[:, : m["out_ch"]], wp)
        # attention core
        k, v = kv[:, : H * qk_slot], kv[:, H * qk_slot:]
        dq = torch.empty_like(q)
        dkv = torch.empty_like(kv)
        ops.attn_bwd(q, k, v, o, do, lse, dq, dkv[:, : H * qk_slot], dkv[:, H * qk_slot:], n, S, H, m["dk"], qk_slot,
                     dv_slot, m["strict"])
        # projections q / kv
        dbq, dbkv = ops.bias_grad(dq), ops.bias_grad(dkv)
        dwq = torch.zeros(wq.shape, dtype=F32, device=dev)
        dwkv = torch.zeros(wkv.shape, dtype=F32, device=dev)
        ops.linear_wgrad(dq, a_kv[:, : m["cin_p"]], dwq)
        ops.linear_wgrad(dkv, a_kv, dwkv)
        _, da_kv = ops.linear_dgrad(dkv, wkv, want_f32=True)
        _, da_q = ops.linear_dgrad(dq, wq, want_f32=True)
        da_kv[:, : m["cin"]] += da_q[:, : m["cin"]]
        cin, ce, embed = m["cin"], m["ce"], m["embed"]
        dx = ops.pm_to_nchw(da_kv[:, :cin].contiguous(), n, cin, h, w)
        dextra = ops.pm_to_nchw(da_kv[:, cin:cin + ce].contiguous(), n, ce, h, w) if ce else None
        if m["identity"]:
            g_qw = dwq[:, :cin].reshape(embed, cin, 1, 1)
            g_kvw = dwkv[:, : cin + ce].reshape(embed + m["out_ch"], cin + ce, 1, 1)
            g_pw = dwp[: m["out_ch"]].reshape(m["out_ch"], m["out_ch"], 1, 1)
            return (dx, dextra, g_qw, dbq, g_kvw, dbkv, g_pw, dp_b, None, None, None, None)
        rq, rv = m["rows_q"], m["rows_v"]
        g_qw = dwq[rq, :cin].reshape(embed, cin, 1, 1)
        g_kvw = torch.cat((dwkv[rq, : cin + ce], dwkv[rv, : cin + ce])).reshape(embed + m["out_ch"], cin + ce, 1, 1)
        g_pw = dwp[: m["out_ch"], m["cols_v"]].reshape(m["out_ch"], m["out_ch"], 1, 1)
        return (dx, dextra, g_qw, dbq[rq], g_kvw, torch.cat((dbkv[rq], dbkv[rv])), g_pw, dp_b, None, None, None, None)


class _AttentionPMFn(torch.autograd.Function):
    """The same attention block on a pixel-major operand: a_kv = [x | extra | 0-pad] bf16 [P, ckv_p] in, fp32 [P, out] out
    (the fused conv stacks build a_kv once and never leave the pixel-major layout)."""

    @staticmethod
    def forward(ctx, a_kv, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, strict, geom, cin, ce):
        n, h, w = geom
        S, H = h * w, n_heads
        cin_p = ops.round_up(cin, 8)
        ckv_p = a_kv.shape[1]
        wq, bq, wkv, bkv, meta = pack_qkv_weights(q_w, q_b, kv_w, kv_b, H, embed, out_ch, cin_p, ckv_p)
        qk_slot, dv_slot = meta["qk_slot"], meta["dv_slot"]
        q, _, _ = ops.linear_fwd(a_kv[:, :cin_p], wq, bq)
        kv, _, _ = ops.linear_fwd(a_kv, wkv, bkv)
        k, v = kv[:, : H * qk_slot], kv[:, H * qk_slot:]
        o, lse = ops.attn_fwd(q, k, v, n, S, H, meta["dk"], qk_slot, dv_slot, strict)
        if meta["identity"]:
            cols_v = None
            wp = ops.pack_weight(p_w)
        else:
            wp = torch.zeros(out_ch, H * dv_slot, dtype=F32, device=a_kv.device)
            cols_v = meta["rows_v"] - H * qk_slot
            wp[:, cols_v] = p_w.detach().reshape(out_ch, -1)
            wp = ops.to_bf16(wp)
        _, _, y = ops.linear_fwd(o, wp, p_b.detach(), want_bf16=False, want_f32=True)
        ctx.save_for_backward(a_kv, q, kv, o, lse, wq, wkv, wp)
        ctx.meta = dict(meta, n=n, h=h, w=w, cin=cin, ce=ce, cin_p=cin_p, H=H, embed=embed, out_ch=out_ch, strict=strict,
                        cols_v=cols_v)
        return y

    @staticmethod
    def backward(ctx, dy):
        a_kv, q, kv, o, lse, wq, wkv, wp = ctx.saved_tensors
        m = ctx.meta
        n, h, w, H, qk_slot, dv_slot = m["n"], m["h"], m["w"], m["H"], m["qk_slot"], m["dv_slot"]
        S = h * w
        dev = dy.device
        out_p = ops.round_up(m["out_ch"], 8)
        dy = dy.contiguous()
        if out_p == m["out_ch"]:
            dy_b = torch.empty(dy.shape, dtype=BF16, device=dev)
            L.act_cast(dy.float() if dy.dtype != F32 else dy, L.ACT_NONE, dy_b)
        else:
            dy_b = torch.zeros(dy.shape[0], out_p, dtype=BF16, device=dev)
            dy_b[:, : m["out_ch"]] = dy
        dp_b = ops.bias_grad(dy_b[:, : m["out_ch"]])
        dwp = torch.zeros(out_p, H * dv_slot, dtype=F32, device=dev)
        ops.linear_wgrad(dy_b, o, dwp)
        do = ops.linear_dgrad(dy_b[:, : m["out_ch"]], wp)
        k, v = kv[:, : H * qk_slot], kv[:, H * qk_slot:]
        dq = torch.empty_like(q)
        dkv = torch.empty_like(kv)
        ops.attn_bwd(q, k, v, o, do, lse, dq, dkv[:, : H * qk_slot], dkv[:, H * qk_slot:], n, S, H, m["dk"], qk_slot,
                     dv_slot, m["strict"])
        dbq, dbkv = ops.bias_grad(dq), ops.bias_grad(dkv)
        dwq = torch.zeros(wq.shape, dtype=F32, device=dev)
        dwkv = torch.zeros(wkv.shape, dtype=F32, device=dev)
        ops.linear_wgrad(dq, a_kv[:, : m["cin_p"]], dwq)
        ops.linear_wgrad(dkv, a_kv, dwkv)
        _, da_kv = ops.linear_dgrad(dkv, wkv, want_f32=True)
        _, da_q = ops.linear_dgrad(dq, wq, want_f32=True)
        da_kv[:, : m["cin"]] += da_q[:, : m["cin"]]
        cin, ce, embed = m["cin"], m["ce"], m["embed"]
        tail = (None,) * 7
        if m["identity"]:
            g_qw = dwq[:, :cin].reshape(embed, cin, 1, 1)
            g_kvw = dwkv[:, : cin + ce].reshape(embed + m["out_ch"], cin + ce, 1, 1)
            g_pw = dwp[: m["out_ch"]].reshape(m["out_ch"], m["out_ch"], 1, 1)
            return (da_kv.to(BF16), g_qw, dbq, g_kvw, dbkv, g_pw, dp_b, *tail)
        rq, rv = m["rows_q"], m["rows_v"]
        g_qw = dwq[rq, :cin].reshape(embed, cin, 1, 1)
        g_kvw = torch.cat((dwkv[rq, : cin + ce], dwkv[rv, : cin + ce])).reshape(embed + m["out_ch"], cin + ce, 1, 1)
        g_pw = dwp[: m["out_ch"], m["cols_v"]].reshape(m["out_ch"], m["out_ch"], 1, 1)
        return (da_kv.to(BF16), g_qw, dbq[rq], g_kvw, torch.cat((dbkv[rq], dbkv[rv])), g_pw, dp_b, *tail)


class CausalAttention(nn.Module):
    """Autoregressively masked multi-head self-attention over image positions — API of reference
    nn/attention.py:66-161 (1x1-conv projections `_q`, `_kv`, `_proj`; heads are contiguous channel blocks;
    `mask_center=True` excludes the current position; `extra_input_channels` feed only keys/values)."""

    def __init__(self, in_channels, n_heads=1, embed_channels=None, out_channels=None, mask_center=False,
                 extra_input_channels=0):
        super().__init__()
        self._n_heads = n_heads
        self._embed_channels = embed_channels or in_channels
        self._out_channels = out_channels or in_channels
        self._mask_center = mask_center
        self._q = nn.Conv2d(in_channels=in_channels, out_channels=self._embed_channels, kernel_size=1)
        self._kv = nn.Conv2d(in_channels=in_channels + extra_input_channels,
                             out_channels=self._embed_channels + self._out_channels, kernel_size=1)
        self._proj = nn.Conv2d(in_channels=self._out_channels, out_channels=self._out_channels, kernel_size=1)

    def forward_pm(self, a_kv, geom, cin, ce):
        """Pixel-major entry of the fused stacks: a_kv = [x (cin) | extra_x (ce) | 0-pad] bf16 -> fp32 [P, out]."""
        return _AttentionPMFn.apply(a_kv, self._q.weight, self._q.bias, self._kv.weight, self._kv.bias, self._proj.weight,
                                    self._proj.bias, self._n_heads, self._embed_channels, self._out_channels,
                                    self._mask_center, geom, cin, ce)

    def forward(self, x, extra_x=None):
        _require_cuda(x, "CausalAttention")
        return _AttentionFn.apply(x, extra_x, self._q.weight, self._q.bias, self._kv.weight, self._kv.bias,
                                  self._proj.weight, self._proj.bias, self._n_heads, self._embed_channels,
                                  self._out_channels, self._mask_center)


def attention_scale(embed_channels, n_heads):
    """1/sqrt(dk) with dk = embed_channels / n_heads (reference nn/attention.py:152)."""
    return 1.0 / math.sqrt(embed_channels // n_heads)


# --------------------------------------------------------------------------------------------------
# LinearCausalAttention
# --------------------------------------------------------------------------------------------------
class _LinearAttnNumerator(torch.autograd.Function):
    """Unnormalised causal linear attention (reference nn/attention.py:168-200): out_i = Q_i . sum_{j<=i} K_j^T V_j.
    Q, K: [N, heads, L, d]; V: [N, heads, L, dv], any d and dv.  Chunked scan kernels (pg_linear_attn_fwd / _bwd)
    instead of a Python loop over L."""

    @staticmethod
    def forward(ctx, Q, K, V):
        n, h, l, d = Q.shape
        q, k, v = (t.contiguous().float().view(n * h, l, -1) for t in (Q, K, V))
        out = torch.empty_like(v)
        L.linear_attn_fwd(q, k, v, out)
        ctx.save_for_backward(q, k, v)
        ctx.shape = (n, h, l)
        return out.view(n, h, l, -1)

    @staticmethod
    def backward(ctx, G):
        q, k, v = ctx.saved_tensors
        n, h, l = ctx.shape
        g = G.contiguous().float().view(n * h, l, -1)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        L.linear_attn_bwd(q, k, v, g, dq, dk, dv)
        return dq.view(n, h, l, -1), dk.view(n, h, l, -1), dv.view(n, h, l, -1)


def _elu_plus_one(x):
    return torch.nn.functional.elu(x) + 1


class LinearCausalAttention(nn.Module):
    """O(N)-memory causal attention with a kernel feature map — API of reference nn/attention.py:209-275 (`_query`, `_kv`
    1x1-conv projections; `feature_fn` defaults to elu(x) + 1).

    The arithmetic follows the reference line by line, including its normaliser
    `1 / (einsum("nlhi,nlhi->nlh", Q, K.cumsum(1)) + 1e-10)`, whose cumulative sum runs over dimension 1 of the
    [N, heads, L, d] tensors (the heads).  The sequential part — the running K^T V state — runs on fp32 chunked-scan
    CUDA kernels (`pg_linear_attn_fwd/bwd`) instead of the reference's per-position Python loop, for heads of any
    width (d = embed_channels / n_heads, dv = out_channels / n_heads), deterministically."""

    def __init__(self, in_channels, feature_fn=_elu_plus_one, n_heads=1, embed_channels=None, out_channels=None):
        super().__init__()
        self._feature_fn = feature_fn
        self._n_heads = n_heads
        self._embed_channels = embed_channels or in_channels
        self._out_channels = out_channels or in_channels
        self._query = nn.Conv2d(in_channels=in_channels, out_channels=self._embed_channels, kernel_size=1)
        self._kv = nn.Conv2d(in_channels=in_channels, out_channels=self._embed_channels + self._out_channels, kernel_size=1)
        self._numerator = _LinearAttnNumerator.apply

    def forward(self, x):
        _require_cuda(x, "LinearCausalAttention")
        from .tapconv import tap_conv2d

        n, _, h, w = x.shape

        def to_multihead(t):  # (N, C, H, W) -> (N, heads, H*W, head_size)
            return t.view(n, self._n_heads, t.shape[1] // self._n_heads, -1).transpose(2, 3)

        q = to_multihead(tap_conv2d(x, self._query.weight, self._query.bias, (0, 0)))
        k, v = tap_conv2d(x, self._kv.weight, self._kv.bias, (0, 0)).split([self._embed_channels, self._out_channels], dim=1)
        k, v = to_multihead(k), to_multihead(v)
        q, k = self._feature_fn(q), self._feature_fn(k)
        den = 1 / (torch.einsum("nlhi,nlhi->nlh", q, k.cumsum(1)) + 1e-10)
        out = self._numerator(q, k, v) * torch.unsqueeze(den, -1)
        return out.transpose(2, 3).contiguous().view(n, -1, h, w)
