"""Wide-channel convolutions as a tap list over the wgmma GEMM.

Every convolution on the path other than the image-channel input layers is evaluated as

    y[p] = bias + sum_t W_t . act_in(x[p + (dy_t, dx_t)])            (zero outside the image)

where the taps are all kernel positions `(i d_h - pad_h, j d_w - pad_w)` (d: the dilation) and the output is the
input-sized front crop the reference call sites take (`[:, :, :h, :w]`, reference gated_pixel_cnn.py:115,121,
pixel_snail.py:54-55; for 'same' padding the crop is the identity).  This file holds the tap list and the rule that sends short contractions to
the direct fp32 kernel; `pm.conv` picks how the taps are contracted, and `ops.pack_taps` packs the bf16 weights.
`TapConv2d` and `tap_conv2d` are the NCHW layout wrappers over `pm.image_conv`.
"""

from torch import nn

from .. import _lib as L


SMALL_K = 160  # Cin*kh*kw at or below this goes to pg_conv_small_* (CUDA cores, fp32)


def small_conv_ok(wshape):
    """Shapes pg_conv_small_* handles: K = Cin*kh*kw <= 160 and the [K, Cout] fp32 weight tile of its dgrad kernel
    within 200 KB of shared memory."""
    cout, cin, kh, kw = wshape
    k = cin * kh * kw
    return k <= SMALL_K and k * cout * 4 <= 200 * 1024


def conv_taps(kh, kw, pad_h, pad_w, dil_h=1, dil_w=1):
    """Offsets (dy, dx) of every kernel position, row-major like the OIHW weight."""
    return tuple((i * dil_h - pad_h, j * dil_w - pad_w) for i in range(kh) for j in range(kw))


def tap_conv2d(x, weight, bias, padding, pre_act=L.ACT_NONE, post_act=L.ACT_NONE, dilation=(1, 1)):
    """conv2d(act_in(x), weight, bias, padding, dilation) cropped to x's H x W, then act_out: NCHW fp32 in and out,
    computed by `pm.image_conv` on the pixel-major layout."""
    if not x.is_cuda:
        raise RuntimeError("tap_conv2d: the CUDA path runs on CUDA tensors only (no CPU fallback)")
    from . import pm  # imported here: pm imports this module

    n, _, h, w = x.shape
    return pm.from_pm(pm.image_conv(x, weight, bias, padding, pre_act, dilation), pm.Geom(n, h, w), weight.shape[0],
                      post_act)


class TapConv2d(nn.Conv2d):
    """nn.Conv2d (same parameters / state-dict keys) evaluated on the CUDA path.  The output keeps the input's
    H x W: it is the front crop `[:h, :w]` of the padded convolution that every reference call site takes."""

    def forward(self, x, pre_act=L.ACT_NONE, post_act=L.ACT_NONE):
        if self.stride != (1, 1) or self.dilation != (1, 1) or self.groups != 1 or self.padding_mode != "zeros":
            raise NotImplementedError("TapConv2d: only stride 1, dilation 1, groups 1, zero padding are on the path")
        pad = self.padding if isinstance(self.padding, tuple) else (self.padding, self.padding)
        return tap_conv2d(x, self.weight, self.bias, pad, pre_act, post_act)
