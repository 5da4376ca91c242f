"""Drop-in building blocks: same constructor signatures, parameter/buffer names and shapes as
`pytorch_generative.nn` (reference nn/convolution.py, nn/attention.py), arithmetic on the sm_90a kernels.

Each module takes and returns NCHW fp32 tensors like the reference (outputs are contiguous NCHW; the
reference's NCHWLayerNorm returns a channels-last-strided view, SURVEY.md §7.3-5).  Internally the data is
converted once to the pixel-major layout the kernels use: the convolutions and the gate are layout wrappers over the
ops of `nn/pm.py`, which the fused model stacks in `models/` call directly.
"""

import functools
import math
from typing import NamedTuple

import torch
from torch import nn

from .. import _lib as L
from .. import ops
from . import pm
from .tapconv import tap_conv2d

F32, BF16 = torch.float32, torch.bfloat16


def _require_cuda(x, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")


# --------------------------------------------------------------------------------------------------
# CausalConv2d
# --------------------------------------------------------------------------------------------------
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

    def apply_mask(self):
        """weight.data *= mask (reference nn/convolution.py:42), leaving the version counter as it is (ops.cached_copy)."""
        self.weight.data *= self.mask

    def forward(self, x, pre_act=L.ACT_NONE):
        """`pre_act` (CUDA-path extension) fuses an activation applied to the conv's input."""
        _require_cuda(x, "CausalConv2d")
        self.apply_mask()
        cout, cin, kh, kw = self.weight.shape
        pad = self.padding if isinstance(self.padding, tuple) else (self.padding, self.padding)
        if self.stride != (1, 1) or self.groups != 1 or self.padding_mode != "zeros":
            raise NotImplementedError("CausalConv2d: only stride 1, groups 1, zero padding are on the path")
        dh, dw = self.dilation
        if pad != (dh * (kh // 2), dw * (kw // 2)):
            raise NotImplementedError("CausalConv2d: only 'same' padding (dilation * (k//2)) is on the path")
        return tap_conv2d(x, self.weight, self.bias, pad, pre_act=pre_act, dilation=self.dilation)


# --------------------------------------------------------------------------------------------------
# GatedActivation
# --------------------------------------------------------------------------------------------------
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
        n, c, h, w = x.shape
        assert c % 2 == 0, "x must have an even number of channels."
        return pm.from_pm(pm.gated(pm.to_pm(x, F32), self._act_id, F32), pm.Geom(n, h, w), c // 2)


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
class HeadLayout(NamedTuple):
    """Where the attention kernels read each head: `n_heads` heads of dk = embed / n_heads query/key channels and
    dv = out_ch / n_heads value channels, in column slots qk_slot and dv_slot wide (`ops.head_slots`).  A head narrower
    than its slot sits in zero-padded weight rows.  This is the one owner of that layout: `pack` scatters the projection
    weights into it and `unpack_grads` gathers their gradients back to the shapes of `_q`, `_kv` and `_proj`.  Build it
    with `head_layout`."""

    n_heads: int
    embed: int
    out_ch: int
    dk: int
    dv: int
    qk_slot: int
    dv_slot: int
    identity: bool  # every head fills its slot: no row scatter, and the gathered gradients are views
    rows_q: torch.Tensor | slice  # slot row of each q (and k) projection row; slice(None) when identity
    rows_kv: torch.Tensor | slice  # ... of each kv projection row, in the [k slots | v slots] rows of the packed Wkv
    cols_v: torch.Tensor | slice  # ... of each v row, as a column of the packed output projection

    def scatter(self, q_w, q_b, kv_w, kv_b, p_w, cin_q_pad, cin_kv_pad):
        """The projections in slot layout, fp32: Wq [H*qk_slot, cin_q_pad], bq, Wkv [H*(qk_slot + dv_slot), cin_kv_pad],
        bkv, Wp [out_ch, H*dv_slot].  Rows of padded slots and padded input columns are zero, so padded q/k/v columns
        are exactly zero.  What needs no padding is the parameter itself (detached), not a copy."""
        H = self.n_heads
        n_q, n_kv = H * self.qk_slot, H * (self.qk_slot + self.dv_slot)
        wp = p_w.detach().reshape(self.out_ch, -1)
        if not self.identity:
            wp_slots = torch.zeros(self.out_ch, H * self.dv_slot, dtype=F32, device=wp.device)
            wp_slots[:, self.cols_v] = wp
            wp = wp_slots
        return (self._weight_rows(q_w, self.rows_q, n_q, cin_q_pad), self._bias_rows(q_b, self.rows_q, n_q),
                self._weight_rows(kv_w, self.rows_kv, n_kv, cin_kv_pad), self._bias_rows(kv_b, self.rows_kv, n_kv), wp)

    def pack(self, q_w, q_b, kv_w, kv_b, p_w, cin_q_pad, cin_kv_pad):
        """`scatter` with the matrices cast to bf16 for the tensor cores: (Wq, bq, Wkv, bkv, Wp), biases in fp32."""
        def build():
            wq, bq, wkv, bkv, wp = self.scatter(q_w, q_b, kv_w, kv_b, p_w, cin_q_pad, cin_kv_pad)
            return ops.to_bf16(wq), bq, ops.to_bf16(wkv), bkv, ops.to_bf16(wp)
        return ops.cached_copy((q_w, q_b, kv_w, kv_b, p_w), ("heads", self.n_heads, cin_q_pad, cin_kv_pad), build)

    def unpack_grads(self, dwq, dbq, dwkv, dbkv, dwp, cin_q, cin_kv):
        """Gradients of `scatter`'s five outputs (dwp may have padded rows below out_ch) -> the gradients of `_q.weight`,
        `_q.bias`, `_kv.weight`, `_kv.bias` and `_proj.weight` in their own shapes, for cin_q / cin_kv true input
        channels.  With identity they are views of the buffers passed in, so reducing those in place reduces them."""
        e, o = self.embed, self.out_ch
        return (dwq[self.rows_q, :cin_q].reshape(e, cin_q, 1, 1), dbq[self.rows_q],
                dwkv[self.rows_kv, :cin_kv].reshape(e + o, cin_kv, 1, 1), dbkv[self.rows_kv],
                dwp[:o, self.cols_v].reshape(o, o, 1, 1))

    def _weight_rows(self, w, rows, n_rows, n_cols):
        w = w.detach().reshape(w.shape[0], -1)
        if self.identity and w.shape == (n_rows, n_cols):
            return w
        out = torch.zeros(n_rows, n_cols, dtype=F32, device=w.device)
        out[rows, : w.shape[1]] = w
        return out

    def _bias_rows(self, b, rows, n_rows):
        if self.identity:
            return b.detach()
        out = torch.zeros(n_rows, dtype=F32, device=b.device)
        out[rows] = b.detach()
        return out


@functools.lru_cache(maxsize=64)
def head_layout(n_heads, embed, out_ch, device=None):
    """The HeadLayout of `n_heads` heads over `embed` query/key and `out_ch` value channels.  Cached per device: the
    index tensors are built once, so steady-state calls issue no host->device copy (graph-capturable)."""
    dk, dv = embed // n_heads, out_ch // n_heads
    qk_slot, dv_slot = ops.head_slots(dk, dv)
    if (dk, dv) == (qk_slot, dv_slot) and (embed, out_ch) == (n_heads * dk, n_heads * dv):
        every = slice(None)
        return HeadLayout(n_heads, embed, out_ch, dk, dv, qk_slot, dv_slot, True, every, every, every)

    def slot_rows(per_head, slot):
        idx = torch.arange(n_heads * per_head)
        return (idx // per_head) * slot + idx % per_head

    rows_q, rows_v = slot_rows(dk, qk_slot), slot_rows(dv, dv_slot)
    rows_kv = torch.cat((rows_q, rows_v + n_heads * qk_slot))
    return HeadLayout(n_heads, embed, out_ch, dk, dv, qk_slot, dv_slot, False, rows_q.to(device), rows_kv.to(device),
                      rows_v.to(device))


def _attention_fwd(ctx, a_kv, cin, ce, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, n, S, strict):
    """The attention block on a_kv = [x (cin) | extra (ce) | 0-pad] bf16 [P, ckv_p]: q/kv projections -> causal
    attention core -> output projection, fp32 [P, out_ch] out.  Shared by both autograd entries; saves what
    `_attention_bwd` reads on ctx."""
    lay = head_layout(n_heads, embed, out_ch, a_kv.device)
    cin_p = ops.round_up(cin, 8)
    wq, bq, wkv, bkv, wp = lay.pack(q_w, q_b, kv_w, kv_b, p_w, cin_p, a_kv.shape[1])
    # the q projection reads the first cin_p columns of a_kv (columns cin..cin_p of Wq are zero, so reading a few
    # `extra` columns there is harmless)
    q, _, _ = ops.linear_fwd(a_kv[:, :cin_p], wq, bq)
    kv, _, _ = ops.linear_fwd(a_kv, wkv, bkv)
    H, qk = n_heads, n_heads * lay.qk_slot
    o, lse = ops.attn_fwd(q, kv[:, :qk], kv[:, qk:], n, S, H, lay.dk, lay.qk_slot, lay.dv_slot, strict)
    # the output projection reads the slot-padded o through the column-scattered Wp
    _, _, y = ops.linear_fwd(o, wp, p_b.detach(), want_bf16=False, want_f32=True)
    ctx.save_for_backward(a_kv, q, kv, o, lse, wq, wkv, wp)
    ctx.layout, ctx.n, ctx.S, ctx.cin, ctx.ce, ctx.strict = lay, n, S, cin, ce, strict
    return y


def _attention_bwd(ctx, dy_b):
    """Backward of `_attention_fwd` from dy_b, bf16 [P, round_up(out_ch, 8)] with zero padded columns.  Returns
    (da_kv fp32 [P, ckv_p], gradients of q_w, q_b, kv_w, kv_b, p_w, p_b)."""
    a_kv, q, kv, o, lse, wq, wkv, wp = ctx.saved_tensors
    lay = ctx.layout
    H, out_ch, qk = lay.n_heads, lay.out_ch, lay.n_heads * lay.qk_slot
    dev = dy_b.device
    # projection
    dp_b = ops.bias_grad(dy_b[:, :out_ch])
    dwp = torch.zeros(dy_b.shape[1], H * lay.dv_slot, dtype=F32, device=dev)
    ops.linear_wgrad(dy_b, o, dwp)
    do = ops.linear_dgrad(dy_b[:, :out_ch], wp)
    # attention core
    dq = torch.empty_like(q)
    dkv = torch.empty_like(kv)
    ops.attn_bwd(q, kv[:, :qk], kv[:, qk:], o, do, lse, dq, dkv[:, :qk], dkv[:, qk:], ctx.n, ctx.S, H, lay.dk,
                 lay.qk_slot, lay.dv_slot, ctx.strict)
    # projections q / kv
    dbq, dbkv = ops.bias_grad(dq), ops.bias_grad(dkv)
    dwq = torch.zeros(wq.shape, dtype=F32, device=dev)
    dwkv = torch.zeros(wkv.shape, dtype=F32, device=dev)
    ops.linear_wgrad(dq, a_kv[:, : wq.shape[1]], dwq)
    ops.linear_wgrad(dkv, a_kv, dwkv)
    _, da_kv = ops.linear_dgrad(dkv, wkv, want_f32=True)
    _, da_q = ops.linear_dgrad(dq, wq, want_f32=True)
    cin = ctx.cin
    da_kv[:, :cin] += da_q[:, :cin]
    return da_kv, (*lay.unpack_grads(dwq, dbq, dwkv, dbkv, dwp, cin, cin + ctx.ce), dp_b)


class _AttentionFn(torch.autograd.Function):
    """The attention block on NCHW fp32 tensors: x and extra in, fp32 out; dx and dextra leave in fp32."""

    @staticmethod
    def forward(ctx, x, extra, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, strict):
        n, cin, h, w = x.shape
        ce = 0 if extra is None else extra.shape[1]
        a_kv = torch.zeros(n * h * w, ops.round_up(cin + ce, 8), dtype=BF16, device=x.device)
        L.nchw_to_pm(x.contiguous().float(), a_kv[:, :cin])
        if extra is not None:
            L.nchw_to_pm(extra.contiguous().float(), a_kv[:, cin:cin + ce])
        y_pm = _attention_fwd(ctx, a_kv, cin, ce, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, n, h * w,
                              strict)
        ctx.hw = (h, w)
        return ops.pm_to_nchw(y_pm, n, out_ch, h, w)

    @staticmethod
    def backward(ctx, dy):
        (h, w), n, cin, ce = ctx.hw, ctx.n, ctx.cin, ctx.ce
        da_kv, grads = _attention_bwd(ctx, ops.nchw_to_pm(dy, BF16, width=ops.round_up(ctx.layout.out_ch, 8)))
        dx = ops.pm_to_nchw(da_kv[:, :cin].contiguous(), n, cin, h, w)
        dextra = ops.pm_to_nchw(da_kv[:, cin:cin + ce].contiguous(), n, ce, h, w) if ce else None
        return (dx, dextra, *grads, None, None, None, None)


class _AttentionPMFn(torch.autograd.Function):
    """The same attention block on a pixel-major operand: a_kv = [x | extra | 0-pad] bf16 [P, ckv_p] in, fp32 [P, out] out,
    da_kv out in bf16 (the fused conv stacks build a_kv once and never leave the pixel-major layout)."""

    @staticmethod
    def forward(ctx, a_kv, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, strict, geom, cin, ce):
        n, h, w = geom
        return _attention_fwd(ctx, a_kv, cin, ce, q_w, q_b, kv_w, kv_b, p_w, p_b, n_heads, embed, out_ch, n, h * w,
                              strict)

    @staticmethod
    def backward(ctx, dy):
        out_ch = ctx.layout.out_ch
        out_p = ops.round_up(out_ch, 8)
        dy = dy.contiguous()
        if out_p == out_ch:
            dy_b = torch.empty(dy.shape, dtype=BF16, device=dy.device)
            L.act_cast(dy.float() if dy.dtype != F32 else dy, L.ACT_NONE, dy_b)
        else:
            dy_b = torch.zeros(dy.shape[0], out_p, dtype=BF16, device=dy.device)
            dy_b[:, :out_ch] = dy
        da_kv, grads = _attention_bwd(ctx, dy_b)
        return (da_kv.to(BF16), *grads, *(None,) * 7)


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
