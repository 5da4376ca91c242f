"""PixelCNN on the CUDA path — API of reference models/autoregressive/pixel_cnn.py:23-110.

Same module tree and state-dict keys (`_input`, `_causal_layers.{i}._net.{1,3,5}`, `_head.{1,3}`).  The ReLUs of
the reference's `nn.Sequential`s are not separate ops here: each one is fused into the convolution that consumes it
(`pre_act`), so a block is three kernels-backed convs: 1x1, masked 3x3 (type B), 1x1.
"""

from torch import nn

from .. import _lib as L
from .. import nn as pg_nn
from . import base, incremental

RELU = L.ACT_RELU


class CausalResidualBlock(nn.Module):
    """x + net(x), net = ReLU-1x1-ReLU-causal3x3-ReLU-1x1 (reference pixel_cnn.py:23-53)."""

    def __init__(self, n_channels):
        super().__init__()
        self._net = nn.Sequential(  # container kept for the reference's parameter names; forward fuses the ReLUs
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=n_channels, out_channels=n_channels // 2, kernel_size=1),
            nn.ReLU(),
            pg_nn.CausalConv2d(mask_center=False, in_channels=n_channels // 2, out_channels=n_channels // 2,
                               kernel_size=3, padding=1),
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=n_channels // 2, out_channels=n_channels, kernel_size=1),
        )

    def forward(self, x):
        t = self._net[1](x, pre_act=RELU)
        t = self._net[3](t, pre_act=RELU)
        t = self._net[5](t, pre_act=RELU)
        return x + t


class PixelCNN(incremental.IncrementalSamplingMixin, base.AutoregressiveModel):
    """The PixelCNN model — constructor of reference pixel_cnn.py:59-104.  `sample()` evaluates one pixel at a time on
    line buffers (models/incremental.py) instead of one full forward per pixel."""

    def __init__(self, in_channels=1, out_channels=1, n_residual=15, residual_channels=128, head_channels=32,
                 sample_fn=None):
        super().__init__(sample_fn)
        self._input = pg_nn.CausalConv2d(mask_center=True, in_channels=in_channels,
                                         out_channels=2 * residual_channels, kernel_size=7, padding=3)
        self._causal_layers = nn.ModuleList(
            [CausalResidualBlock(n_channels=2 * residual_channels) for _ in range(n_residual)]
        )
        self._head = nn.Sequential(
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=2 * residual_channels, out_channels=head_channels, kernel_size=1),
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=head_channels, out_channels=out_channels, kernel_size=1),
        )

    # ---- per-pixel program of the incremental sampler ----
    # Every row block of the program (the fp32 stream x, t1, t2, the head's hidden layer) has its padded width
    # (incremental.pitch): zero weight rows and biases keep the pad columns at zero through the residuals and ReLUs.
    def _build_pixel_state(self, sp, c):
        half = self._input.weight.shape[0] // 2
        kh, kw = self._input.weight.shape[2:]
        self._taps_in = incremental.live_taps(self._input.mask[0, 0], kh // 2, kw // 2)
        self._taps_b = incremental.live_taps(self._causal_layers[0]._net[3].mask[0, 0], 1, 1) if len(self._causal_layers) else []
        image = sp.cache(c)
        t1 = [sp.cache(half) for _ in self._causal_layers]
        return dict(image=image, t1=t1, caches=[image, *t1], weights={})

    def _pack_pixel_weights(self):
        def conv(m, taps=None, logits=False):  # bf16 [Cout_p, taps * Cin_p] and the bias of one convolution
            positions = taps and [(i, j) for i, j, _, _ in taps]
            return incremental.pack(m, positions, out_parts=0 if logits else 1)

        self._input.apply_mask()
        w = {}
        w["in"], w["in_b"] = conv(self._input, self._taps_in)
        for i, blk in enumerate(self._causal_layers):
            n1, n3, n5 = blk._net[1], blk._net[3], blk._net[5]
            n3.apply_mask()
            w[f"b{i}_1"], w[f"b{i}_1b"] = conv(n1)
            w[f"b{i}_3"], w[f"b{i}_3b"] = conv(n3, self._taps_b)
            w[f"b{i}_5"], w[f"b{i}_5b"] = conv(n5)
        w["h1"], w["h1b"] = conv(self._head[1])
        w["h3"], w["h3b"] = conv(self._head[3], logits=True)
        return w

    def _pixel_program(self, sp, st):
        W = st["weights"]
        off_in = [(dy, dx) for _, _, dy, dx in self._taps_in]
        off_b = [(dy, dx) for _, _, dy, dx in self._taps_b]
        x = sp.linear(sp.gather(st["image"], off_in), W["in"], W["in_b"], f32=True)           # masked 7x7 on the image
        for i in range(len(self._causal_layers)):
            t1 = sp.linear(sp.act(x, RELU), W[f"b{i}_1"], W[f"b{i}_1b"], act=RELU)            # relu(1x1(relu(x)))
            sp.write(st["t1"][i], t1)
            t2 = sp.linear(sp.gather(st["t1"][i], off_b), W[f"b{i}_3"], W[f"b{i}_3b"], act=RELU)  # relu(causal 3x3)
            x = sp.linear(t2, W[f"b{i}_5"], W[f"b{i}_5b"], res0=x, res1=x, f32=True)           # x + (x + net(x))
        h1 = sp.linear(sp.act(x, RELU), W["h1"], W["h1b"], act=RELU)
        return sp.linear(h1, W["h3"], W["h3b"], f32=True)

    def forward(self, x):
        x = self._input(x)
        for layer in self._causal_layers:
            x = x + layer(x)  # the reference's second residual (pixel_cnn.py:109 on top of :53)
        x = self._head[1](x, pre_act=RELU)
        return self._head[3](x, pre_act=RELU)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference pixel_cnn.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_pixel_cnn(*args, **kwargs)
