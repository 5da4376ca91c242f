"""Gated PixelCNN on the CUDA path — API of reference models/autoregressive/gated_pixel_cnn.py:31-190.

Same module tree and state-dict keys (`_input` / `_gated_layers.{i}` with `_vstack_1xN, _vstack_Nx1, _vstack_1x1,
_link, _hstack_1xN, _hstack_residual, _hstack_skip`, `_head.{1,3}`).  The reference gets causality from plain
convolutions with extra padding followed by a front crop; here each such conv is a tap list whose offsets already
encode pad + crop (no padded rows are ever computed), contracted on the tensor cores.
"""

import torch
from torch import nn

from .. import _lib as L
from .. import nn as pg_nn
from .. import ops
from ..nn import pm
from . import base, incremental

RELU, TANH, NONE = L.ACT_RELU, L.ACT_TANH, L.ACT_NONE


class GatedPixelCNNLayer(nn.Module):
    """One two-stream layer (reference gated_pixel_cnn.py:31-130)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, mask_center=False):
        super().__init__()
        assert kernel_size % 2 == 1, "kernel_size cannot be even"
        self._in_channels, self._out_channels = in_channels, out_channels
        self._activation = pg_nn.GatedActivation()
        self._kernel_size = kernel_size
        self._padding = (kernel_size - 1) // 2
        self._mask_center = mask_center
        k, p = kernel_size, self._padding
        # vertical stack: 1xN over the row, then (N//2+1)x1 shifted down by the extra padding row
        self._vstack_1xN = pg_nn.TapConv2d(in_channels, out_channels, kernel_size=(1, k), padding=(0, p))
        self._vstack_Nx1 = pg_nn.TapConv2d(out_channels, 2 * out_channels, kernel_size=(k // 2 + 1, 1),
                                           padding=(p + 1, 0))
        self._vstack_1x1 = pg_nn.TapConv2d(in_channels, 2 * out_channels, kernel_size=1)
        self._link = pg_nn.TapConv2d(2 * out_channels, 2 * out_channels, kernel_size=1)
        # horizontal stack: 1x(N//2+1) looking left (excluding the centre when causal)
        self._hstack_1xN = pg_nn.TapConv2d(in_channels, 2 * out_channels, kernel_size=(1, k // 2 + 1),
                                           padding=(0, p + int(mask_center)))
        self._hstack_residual = pg_nn.TapConv2d(out_channels, out_channels, kernel_size=1)
        self._hstack_skip = pg_nn.TapConv2d(out_channels, out_channels, kernel_size=1)

    def forward_pm(self, geom, v_b, h_f, h_b, skips, image=None):
        """One layer on pixel-major tensors (the fused stack; same arithmetic as `forward`).

        v_b: vertical stack, bf16 [P, C];  h_f / h_b: horizontal stack as fp32 stream and its bf16 copy;  skips: running
        fp32 sum of the skip outputs (or None).  The causal input layer reads the NCHW `image` instead, through
        `pm.image_conv`.  Every `+` of the reference layer is a GEMM-epilogue residual:
        v + 1x1(v_in), link + 1xN(h_in), skips + skip, h + h_in."""
        p, c = self._padding, self._out_channels
        if image is not None:
            v1 = pm.act_cast(pm.image_conv(image, self._vstack_1xN.weight, self._vstack_1xN.bias, (0, p)))
        else:
            v1, _ = pm.conv(v_b, self._vstack_1xN.weight, self._vstack_1xN.bias, geom, (0, p))
        # Nx1(1xN(.)) and the link are short-lived sums, not streams: bf16 tensors, added in the consumer's epilogue as
        # bf16 residuals, so their gradients (the gate's bf16 output gradients) flow back without an fp32 round trip
        v2, _ = pm.conv(v1, self._vstack_Nx1.weight, self._vstack_Nx1.bias, geom, (p + 1, 0))
        link, _ = pm.conv(v2, self._link.weight, self._link.bias, geom)
        if image is not None:
            vv = v2 + pm.image_conv(image, self._vstack_1x1.weight, self._vstack_1x1.bias, (0, 0))
            hh = link + pm.image_conv(image, self._hstack_1xN.weight, self._hstack_1xN.bias, (0, p + int(self._mask_center)))
        else:
            vv, _ = pm.conv(v_b, self._vstack_1x1.weight, self._vstack_1x1.bias, geom, res=v2)
            hh, _ = pm.conv(h_f, self._hstack_1xN.weight, self._hstack_1xN.bias, geom, (0, p + int(self._mask_center)),
                            xa=h_b, res=link)
        v_out = pm.gated(vv, TANH)
        hs = pm.gated(hh, TANH)
        skips, _ = pm.conv(hs, self._hstack_skip.weight, self._hstack_skip.bias, geom, res=skips, out_f32=True)
        h_f, h_b = pm.conv(hs, self._hstack_residual.weight, self._hstack_residual.bias, geom,
                           res=None if self._mask_center else h_f, emit=NONE, out_f32=True)
        return v_out, h_f, h_b, skips

    def forward(self, vstack_input, hstack_input):
        """Standalone use of the layer on NCHW tensors (reference API); no model forward reaches it."""
        vstack = self._vstack_Nx1(self._vstack_1xN(vstack_input))  # TapConv2d output == the reference's [:h] crop
        link = self._link(vstack)
        vstack = self._activation(vstack + self._vstack_1x1(vstack_input))
        hstack = self._activation(link + self._hstack_1xN(hstack_input))  # == the reference's [:w] crop
        skip = self._hstack_skip(hstack)
        hstack = self._hstack_residual(hstack)
        if not self._mask_center:  # no residual on the causal layer: it would leak the current pixel
            hstack = hstack + hstack_input
        return vstack, hstack, skip


class GatedPixelCNN(incremental.IncrementalSamplingMixin, base.AutoregressiveModel):
    """The Gated PixelCNN model — constructor of reference gated_pixel_cnn.py:136-183.  `sample()` evaluates one pixel at a
    time on line buffers (models/incremental.py) instead of one full forward per pixel."""

    def __init__(self, in_channels=1, out_channels=1, n_gated=10, gated_channels=128, head_channels=32, sample_fn=None):
        super().__init__(sample_fn)
        self._input = GatedPixelCNNLayer(in_channels=in_channels, out_channels=gated_channels, kernel_size=7,
                                         mask_center=True)
        self._gated_layers = nn.ModuleList(
            [GatedPixelCNNLayer(in_channels=gated_channels, out_channels=gated_channels, kernel_size=3,
                                mask_center=False) for _ in range(n_gated)]
        )
        self._head = nn.Sequential(
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=gated_channels, out_channels=head_channels, kernel_size=1),
            nn.ReLU(),
            pg_nn.TapConv2d(in_channels=head_channels, out_channels=out_channels, kernel_size=1),
        )

    # ---- per-pixel program of the incremental sampler ----
    # The horizontal stack of pixel p is evaluated when p's logits are needed.  The vertical stack's OUTPUT at p also sees
    # image[p] (through `_vstack_1x1`; it only ever reaches pixels of later rows), so it is finished one step later, at
    # the start of the program of p + 1, from the `Nx1(1xN(.))` value saved at p.  `1xN` outputs are not cached: the
    # (k // 2 + 1) rows `Nx1` needs are recomputed from the layer's cached input (they are rows above p: complete).
    # Every row block has its padded width (incremental.pitch); the gates' 2C-wide inputs (v2, link, vv, hh) keep each
    # half at its own pitch, so the gates' outputs come out padded with zeros.
    def _layers(self):
        return [self._input, *self._gated_layers]

    def _incremental_ok(self, canvas):
        c = self._input._out_channels
        return super()._incremental_ok(canvas) and all(l._out_channels == c for l in self._gated_layers)

    def _build_pixel_state(self, sp, c):
        C = self._input._out_channels
        layers = self._layers()
        image = sp.cache(c)
        vc = [sp.cache(C) for _ in layers[:-1]]
        hc = [sp.cache(C) for _ in layers[:-1]]
        v2s = [torch.zeros(sp.n, incremental.pitch(2 * C, 2), dtype=torch.bfloat16, device=sp.device) for _ in layers]
        sp.prev = torch.zeros(1, dtype=torch.int64, device=sp.device)  # max(p - 1, 0): the pixel whose vertical stack is finished
        rows = torch.arange(sp.S) // sp.w
        valid = []
        for layer in layers:  # [S, R] 1 / 0: is row (r + i - pad - 1) of the 1xN output inside the image (else: zero padding)
            r_taps = layer._kernel_size // 2 + 1
            ok = (rows.view(-1, 1) + torch.arange(r_taps).view(1, -1) - layer._padding - 1) >= 0
            valid.append(ok.to(torch.bfloat16).to(sp.device))
        return dict(image=image, vc=vc, hc=hc, v2s=v2s, valid=valid, caches=[image, *vc, *hc, *v2s], weights={}, c=c)

    def _pack_pixel_weights(self):
        w = {}
        for i, layer in enumerate(self._layers()):
            # (key, convolution, parts of its input, parts of its output): 2 = a gate's [a | b] halves
            for key, conv, parts_in, parts_out in (
                    ("v1", layer._vstack_1xN, 1, 1), ("v2", layer._vstack_Nx1, 1, 2), ("vx", layer._vstack_1x1, 1, 2),
                    ("ln", layer._link, 2, 2), ("h", layer._hstack_1xN, 1, 2), ("hr", layer._hstack_residual, 1, 1),
                    ("hs", layer._hstack_skip, 1, 1)):
                w[f"{i}{key}"], w[f"{i}{key}b"] = incremental.pack(conv, in_parts=parts_in, out_parts=parts_out)
        w["h1"], w["h1b"] = incremental.pack(self._head[1])
        w["h3"], w["h3b"] = incremental.pack(self._head[3], out_parts=0)
        return w

    def _before_pixel(self, sp, st, canvas, row, col):
        sp.prev.fill_(max(row * canvas.shape[3] + col - 1, 0))

    def _pixel_program(self, sp, st):
        W, n = st["weights"], sp.n
        layers = self._layers()
        last = len(layers) - 1
        # (1) the previous pixel is final now: finish its vertical-stack outputs
        vin = st["image"].index_select(1, sp.prev)[:, 0]
        for i in range(last):
            vv = sp.linear(vin, W[f"{i}vx"], W[f"{i}vxb"], res0=st["v2s"][i])
            vin = pm.gated(vv, TANH)
            st["vc"][i].index_copy_(1, sp.prev, vin.unsqueeze(1))
        # (2) position p
        h_f = skips = None
        for i, layer in enumerate(layers):
            k, pd, mc = layer._kernel_size, layer._padding, int(layer._mask_center)
            r_taps = k // 2 + 1
            v_src = st["image"] if i == 0 else st["vc"][i - 1]
            h_src = st["image"] if i == 0 else st["hc"][i - 1]
            offs_v = [(ii - pd - 1, j - pd) for ii in range(r_taps) for j in range(k)]
            a = sp.gather(v_src, offs_v).view(n * r_taps, -1)
            v1 = sp.linear(a, W[f"{i}v1"], W[f"{i}v1b"]).view(n, r_taps, -1)
            v1 = v1 * st["valid"][i].index_select(0, sp.pos).view(1, r_taps, 1)   # rows above the image are zero padding
            v2 = sp.linear(v1.view(n, -1), W[f"{i}v2"], W[f"{i}v2b"])
            st["v2s"][i].copy_(v2)
            link = sp.linear(v2, W[f"{i}ln"], W[f"{i}lnb"])
            offs_h = [(0, j - pd - mc) for j in range(r_taps)]
            hh = sp.linear(sp.gather(h_src, offs_h), W[f"{i}h"], W[f"{i}hb"], res0=link)
            hs = pm.gated(hh, TANH)
            skips = sp.linear(hs, W[f"{i}hs"], W[f"{i}hsb"], res0=skips, f32=True)
            h_b, _, h_f = ops.linear_fwd(hs, W[f"{i}hr"], W[f"{i}hrb"], res0=None if mc else h_f, want_f32=True, skinny=True)
            if i < last:
                sp.write(st["hc"][i], h_b)
        t = sp.linear(sp.act(skips, RELU), W["h1"], W["h1b"], act=RELU)
        return sp.linear(t, W["h3"], W["h3b"], f32=True)

    def forward(self, x):
        """The whole network on pixel-major tensors: NCHW only at the image and at the logits."""
        n, _, h, w = x.shape
        geom = pm.Geom(n, h, w)
        v_b, h_f, h_b, skips = self._input.forward_pm(geom, None, None, None, None, image=x)
        for layer in self._gated_layers:
            v_b, h_f, h_b, skips = layer.forward_pm(geom, v_b, h_f, h_b, skips)
        t, t_a = pm.conv(skips, self._head[1].weight, self._head[1].bias, geom, in_act=RELU, emit=RELU,
                         emit_mode=pm.PRE_GRAD, want_main=False)
        logits, _ = pm.conv(t_a, self._head[3].weight, self._head[3].bias, geom, in_act=RELU, xa=t_a, out_f32=True)
        return pm.from_pm(logits, geom, self._head[3].weight.shape[0])


def reproduce(*args, **kwargs):
    """The recipe of this model (reference gated_pixel_cnn.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_gated_pixel_cnn(*args, **kwargs)
