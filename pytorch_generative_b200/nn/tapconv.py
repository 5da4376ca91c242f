"""Wide-channel convolutions as a tap list over the wgmma GEMM.

Every convolution on the path other than the image-channel input layers is evaluated as

    y[p] = bias + sum_t W_t . act_in(x[p + (dy_t, dx_t)])            (zero outside the image)

where the taps are all kernel positions `(i - pad_h, j - pad_w)` and the output is the input-sized front crop the
reference call sites take (`[:, :, :h, :w]`, reference gated_pixel_cnn.py:115,121, pixel_snail.py:54-55; for
'same' padding the crop is the identity).  `pg_tap_gather` lays the shifted inputs side by side, one
`pg_gemm_bf16` contracts over K = taps x channels, `pg_tap_scatter` folds the input gradient back.  A 1x1 conv
is the single tap (0, 0) and needs no gather.
"""

import torch
from torch import nn

from .. import _lib as L
from .. import ops

F32, BF16 = torch.float32, torch.bfloat16


SMALL_K = 160  # Cin*kh*kw at or below this goes to pg_conv_small_* (CUDA cores, fp32)


def small_conv_ok(wshape):
    """Shapes pg_conv_small_* handles: K = Cin*kh*kw <= 160 and the [K, Cout] fp32 weight tile of its dgrad kernel
    within 200 KB of shared memory."""
    cout, cin, kh, kw = wshape
    k = cin * kh * kw
    return k <= SMALL_K and k * cout * 4 <= 200 * 1024


def conv_taps(kh, kw, pad_h, pad_w):
    """Offsets (dy, dx) of every kernel position, row-major like the OIHW weight."""
    return tuple((i - pad_h, j - pad_w) for i in range(kh) for j in range(kw))


_PACK_CACHE = {}


def packed_tap_weight(weight, cin_p):
    """`ops.pack_taps` memoised on the Parameter's identity and version counter: the bf16 copy is rebuilt once per
    optimizer step, not once per forward (eval, sampling and gradient accumulation reuse it)."""
    if weight.is_cuda and torch.cuda.is_current_stream_capturing():
        return ops.pack_taps(weight, cin_p)  # inside a CUDA graph the cast must be a captured kernel of every replay
    key = (id(weight), cin_p)
    hit = _PACK_CACHE.get(key)
    sig = (weight._version, weight.data_ptr(), tuple(weight.shape))
    if hit is not None and hit[0] == sig and hit[2]() is weight:
        return hit[1]
    import weakref

    packed = ops.pack_taps(weight, cin_p)
    if len(_PACK_CACHE) > 4096:
        _PACK_CACHE.clear()
    _PACK_CACHE[key] = (sig, packed, weakref.ref(weight))
    return packed


class _TapConvFn(torch.autograd.Function):
    """NCHW fp32 in / out; bf16 tensor-core contraction in between."""

    @staticmethod
    def forward(ctx, x, weight, bias, taps, pre_act, post_act):
        n, cin, h, w = x.shape
        cout = weight.shape[0]
        cin_p = ops.round_up(cin, 8)
        T, P = len(taps), n * h * w
        x_pm = ops.nchw_to_pm(x, BF16, width=cin_p)  # pre-activation input, bf16
        if T == 1 and taps[0] == (0, 0) and pre_act == L.ACT_NONE:
            xcat = x_pm
        else:
            xcat = torch.empty(P, T * cin_p, dtype=BF16, device=x.device)
            L.tap_gather(x_pm, n, h, w, cin_p, taps, pre_act, xcat)
        wcat = ops.pack_taps(weight, cin_p)
        _, _, y_pm = ops.linear_fwd(xcat, wcat, None if bias is None else bias.detach(), want_bf16=False, want_f32=True)
        ctx.save_for_backward(x_pm if pre_act != L.ACT_NONE else None, xcat, wcat,
                              y_pm if post_act != L.ACT_NONE else None)
        ctx.meta = (n, cin, h, w, cout, cin_p, taps, pre_act, post_act, weight.shape, bias is not None)
        return ops.pm_to_nchw(y_pm, n, cout, h, w, act=post_act)

    @staticmethod
    def backward(ctx, dy):
        x_pre, xcat, wcat, y_pre = ctx.saved_tensors
        n, cin, h, w, cout, cin_p, taps, pre_act, post_act, wshape, has_bias = ctx.meta
        T, P = len(taps), n * h * w
        cout_p = ops.round_up(cout, 8)
        dy_b = ops.nchw_to_pm(dy, BF16, width=cout_p)
        if post_act != L.ACT_NONE:
            L.dact_mul(dy_b[:, :cout], y_pre, post_act, dy_b[:, :cout])
        db = ops.bias_grad(dy_b[:, :cout]) if has_bias else None
        dwcat = torch.zeros(cout_p, T * cin_p, dtype=F32, device=dy.device)
        ops.linear_wgrad(dy_b, xcat, dwcat)
        kh, kw = wshape[2], wshape[3]
        dw = dwcat[:cout].view(cout, kh, kw, cin_p)[..., :cin].permute(0, 3, 1, 2).contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            dxcat = ops.linear_dgrad(dy_b[:, :cout], wcat)  # [P, T*cin_p] bf16
            dx_pm = torch.empty(P, cin_p, dtype=F32, device=dy.device)
            L.tap_scatter(dxcat, n, h, w, cin_p, taps, pre_act, x_pre, dx_f32=dx_pm)
            dx = ops.pm_to_nchw(dx_pm, n, cin, h, w)
        return dx, dw, db, None, None, None


def tap_conv2d(x, weight, bias, padding, pre_act=L.ACT_NONE, post_act=L.ACT_NONE, live_mask=None):
    """conv2d(act_in(x), weight, bias, padding) cropped to x's H x W, then act_out."""
    if not x.is_cuda:
        raise RuntimeError("tap_conv2d: the CUDA path runs on CUDA tensors only (no CPU fallback)")
    kh, kw = weight.shape[-2:]
    if 2 * padding[0] < kh - 1 or 2 * padding[1] < kw - 1:
        raise NotImplementedError("tap_conv2d: padding too small for an input-sized output (not a shape on the path)")
    if small_conv_ok(weight.shape) and post_act == L.ACT_NONE:
        # a contraction this short (image-channel inputs, the 16/32-channel PixelCNN recipe) is not tensor-core work:
        # direct fp32 kernel, exact to 1e-3 (no bf16 rounding of the operands)
        from .modules import _SmallConvFn

        return _SmallConvFn.apply(x, weight, bias, tuple(padding), pre_act)
    taps = conv_taps(kh, kw, padding[0], padding[1])
    if len(taps) > 32:
        raise NotImplementedError(f"tap_conv2d: {len(taps)} taps exceed the 32-tap gather (kernel {kh}x{kw})")
    return _TapConvFn.apply(x.float(), weight, bias, taps, pre_act, post_act)


class TapConv2d(nn.Conv2d):
    """nn.Conv2d (same parameters / state-dict keys) evaluated on the CUDA path.  The output keeps the input's
    H x W: it is the front crop `[:h, :w]` of the padded convolution that every reference call site takes."""

    def forward(self, x, pre_act=L.ACT_NONE, post_act=L.ACT_NONE):
        if self.stride != (1, 1) or self.dilation != (1, 1) or self.groups != 1 or self.padding_mode != "zeros":
            raise NotImplementedError("TapConv2d: only stride 1, dilation 1, groups 1, zero padding are on the path")
        pad = self.padding if isinstance(self.padding, tuple) else (self.padding, self.padding)
        return tap_conv2d(x, self.weight, self.bias, pad, pre_act, post_act)
