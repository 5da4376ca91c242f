"""PixelSNAIL on the CUDA path — API of reference models/autoregressive/pixel_snail.py:27-187.

Same module tree and state-dict keys (`_input`, `_pixel_snail_blocks.{i}` with `_residual.{j}.{_input_conv,
_output_conv}`, `_attention.{_q,_kv,_proj}`, `_residual_out`, `_attention_out`, `_out`; `_output.{0,1}`).  The 2x2
convolutions with pad 1 + crop are tap lists {(-1,-1),(-1,0),(0,-1),(0,0)} on the tensor-core GEMM; every ELU is
fused into the conv that consumes or produces it (`pre_act` / `post_act`); the gate uses the identity activation.
"""

import torch
from torch import nn

from .. import _lib as L
from .. import nn as pg_nn
from .. import ops
from ..nn import pm
from ..nn.modules import head_layout
from . import base, incremental

ELU, NONE = L.ACT_ELU, L.ACT_NONE


class ResidualBlock(nn.Module):
    """x + gate(conv2x2(elu(conv2x2(elu(x))))) (reference pixel_snail.py:31-56)."""

    def __init__(self, n_channels):
        super().__init__()
        self._input_conv = pg_nn.TapConv2d(n_channels, n_channels, kernel_size=2, padding=1)
        self._output_conv = pg_nn.TapConv2d(n_channels, 2 * n_channels, kernel_size=2, padding=1)
        self._activation = pg_nn.GatedActivation(activation_fn=nn.Identity())

    def forward_pm(self, geom, x_f, x_e=None):
        """Pixel-major: x_f fp32 stream [P, C] (x_e = bf16 elu(x_f) when a producer already emitted it) -> fp32 stream.
        conv -> elu -> conv runs as two tap-loop GEMMs: the first one's epilogue writes elu(.) only, the second one's
        dgrad epilogue applies elu'."""
        _, t = pm.conv(x_f, self._input_conv.weight, self._input_conv.bias, geom, (1, 1), in_act=ELU, xa=x_e, emit=ELU,
                       emit_mode=pm.PRE_GRAD, want_main=False)
        u, _ = pm.conv(t, self._output_conv.weight, self._output_conv.bias, geom, (1, 1), in_act=ELU, xa=t)
        return pm.gated_res(u, x_f, NONE)

    def forward(self, x):
        """Standalone use of the block on NCHW tensors (reference API); no model forward reaches it."""
        out = self._input_conv(x, pre_act=ELU)       # conv(elu(x)), cropped to h x w
        out = self._output_conv(out, pre_act=ELU)    # conv(elu(.)), cropped
        return x + self._activation(out)


class PixelSNAILBlock(nn.Module):
    """Residual blocks + causal attention over (position, features | image) (reference pixel_snail.py:59-119)."""

    def __init__(self, n_channels, input_img_channels=1, n_residual_blocks=2, attention_key_channels=4,
                 attention_value_channels=32):
        super().__init__()

        def conv(in_channels):
            return pg_nn.TapConv2d(in_channels, out_channels=n_channels, kernel_size=1)

        self._residual = nn.Sequential(*[ResidualBlock(n_channels) for _ in range(n_residual_blocks)])
        self._attention = pg_nn.CausalAttention(in_channels=n_channels + 2, embed_channels=attention_key_channels,
                                                out_channels=attention_value_channels, mask_center=True,
                                                extra_input_channels=input_img_channels)
        self._residual_out = conv(n_channels)
        self._attention_out = conv(attention_value_channels)
        self._out = conv(n_channels)
        self._pos_cache = {}

    def _positions(self, shape, device):
        key = (tuple(shape), str(device))
        if key not in self._pos_cache:  # same values as the reference's image_positional_encoding, kept on device
            self._pos_cache[key] = pg_nn.image_positional_encoding(tuple(shape)).to(device)
        return self._pos_cache[key]

    def forward_pm(self, geom, x_f, img_b, pos_b, pad_b, c_img):
        """Pixel-major block: x_f fp32 stream [P, C]; img_b / pos_b bf16 [P, c_img] / [P, 2]; returns the block output
        (to be added to the stream)."""
        res = x_f
        for rb in self._residual:
            res = rb.forward_pm(geom, res)
        c = res.shape[1]
        a_kv = torch.cat((pos_b, pm.act_cast(res), img_b, pad_b), dim=1)  # [pos | features | image | 0-pad], bf16
        attn = self._attention.forward_pm(a_kv, geom, c + 2, c_img)       # fp32 [P, value channels]
        _, r = pm.conv(res, self._residual_out.weight, self._residual_out.bias, geom, in_act=ELU, emit=ELU,
                       emit_mode=pm.POST, want_main=False)
        _, a = pm.conv(attn, self._attention_out.weight, self._attention_out.bias, geom, in_act=ELU, emit=ELU,
                       emit_mode=pm.POST, want_main=False)
        _, out = pm.conv(r + a, self._out.weight, self._out.bias, geom, in_act=ELU, emit=ELU, emit_mode=pm.POST,
                         want_main=False)
        return out

    def forward(self, x, input_img):
        """Standalone use of the block on NCHW tensors (reference API); no model forward reaches it."""
        res = self._residual(x)
        pos = self._positions(input_img.shape, res.device)
        attn = self._attention(torch.cat((pos, res), dim=1), input_img)
        res = self._residual_out(res, pre_act=ELU, post_act=ELU)
        attn = self._attention_out(attn, pre_act=ELU, post_act=ELU)
        return self._out(res + attn, pre_act=ELU, post_act=ELU)


TAPS_2X2 = [(-1, -1), (-1, 0), (0, -1), (0, 0)]  # the live window of "2x2 conv, pad 1, crop to h x w", row-major like the weight


class PixelSNAIL(incremental.IncrementalSamplingMixin, base.AutoregressiveModel):
    """The PixelSNAIL model — constructor of reference pixel_snail.py:130-180.  `sample()` evaluates one pixel at a time
    on line buffers and K/V caches (models/incremental.py) instead of one full forward per pixel."""

    # the positional encoding is a function of the image height (arange(-.5, .5, 1/h)), so a pixel cannot be evaluated
    # on a truncated canvas: the fallback sample() runs the full forward per pixel, exactly like the reference
    _row_truncated_sampling = False

    def __init__(self, in_channels=1, out_channels=1, n_channels=64, n_pixel_snail_blocks=8, n_residual_blocks=2,
                 attention_key_channels=4, attention_value_channels=32, sample_fn=None):
        super().__init__(sample_fn)
        self._input = pg_nn.CausalConv2d(mask_center=True, in_channels=in_channels, out_channels=n_channels,
                                         kernel_size=3, padding=1)
        self._pixel_snail_blocks = nn.ModuleList(
            [PixelSNAILBlock(n_channels=n_channels, input_img_channels=in_channels,
                             n_residual_blocks=n_residual_blocks, attention_key_channels=attention_key_channels,
                             attention_value_channels=attention_value_channels)
             for _ in range(n_pixel_snail_blocks)]
        )
        self._output = nn.Sequential(
            pg_nn.TapConv2d(in_channels=n_channels, out_channels=n_channels // 2, kernel_size=1),
            pg_nn.TapConv2d(in_channels=n_channels // 2, out_channels=out_channels, kernel_size=1),
        )

    # ---- per-pixel program of the incremental sampler ----
    # Every row block has its padded width (incremental.pitch): the stream x and res (C), the residual blocks' gate
    # inputs (2C, each half at its own pitch), the attention output (value channels) and the output layer's hidden
    # row (C // 2).  The attention operand keeps the training layout [position | features | image | 0-pad].
    def _incremental_ok(self, canvas):
        att = self._pixel_snail_blocks[0]._attention if len(self._pixel_snail_blocks) else None
        ok = att is None or (att._n_heads == 1 and att._embed_channels <= ops.KERNEL_SLOTS[-1])
        return super()._incremental_ok(canvas) and ok

    def _build_pixel_state(self, sp, c):
        C = self._input.weight.shape[0]
        kh, kw = self._input.weight.shape[2:]
        self._taps_in = incremental.live_taps(self._input.mask[0, 0], kh // 2, kw // 2)
        image = sp.cache(c)
        caches, blocks = [image], []
        ckv_p = ops.round_up(2 + C + c, 8)
        pos_tab = None
        for blk in self._pixel_snail_blocks:
            att = blk._attention
            lay = head_layout(att._n_heads, att._embed_channels, att._out_channels)
            qk_slot, dv_slot = lay.qk_slot, lay.dv_slot
            b = dict(ea=[sp.cache(C) for _ in blk._residual], eb=[sp.cache(C) for _ in blk._residual],
                     kc=torch.zeros(sp.n * sp.S, qk_slot, dtype=torch.bfloat16, device=sp.device),
                     vc=torch.zeros(sp.n * sp.S, dv_slot, dtype=torch.bfloat16, device=sp.device),
                     akv=torch.zeros(sp.n, ckv_p, dtype=torch.bfloat16, device=sp.device), qk_slot=qk_slot,
                     dv_slot=dv_slot)
            caches += [*b["ea"], *b["eb"], b["kc"], b["vc"], b["akv"]]
            blocks.append(b)
            if pos_tab is None:  # [S, 2] bf16: the positional encoding of every pixel (same values as the full forward)
                enc = blk._positions((1, c, sp.h, sp.w), sp.device)
                pos_tab = enc[0].reshape(2, sp.S).t().contiguous().to(torch.bfloat16)
        sp.prev = torch.zeros(1, dtype=torch.int64, device=sp.device)   # max(p - 1, 0): the row of the K/V fix-up
        return dict(image=image, caches=caches, blocks=blocks, weights={}, pos_tab=pos_tab, c=c, ckv_p=ckv_p)

    def _pack_pixel_weights(self):
        conv = incremental.pack  # bf16 [Cout_p, taps * Cin_p] and the bias of one convolution, padded layout
        self._input.apply_mask()
        C, c = self._input.weight.shape[:2]
        w = {}
        w["in"], w["in_b"] = conv(self._input, [(i, j) for i, j, _, _ in self._taps_in])
        for bi, blk in enumerate(self._pixel_snail_blocks):
            for j, rb in enumerate(blk._residual):
                w[f"{bi}r{j}i"], w[f"{bi}r{j}ib"] = conv(rb._input_conv)
                w[f"{bi}r{j}o"], w[f"{bi}r{j}ob"] = conv(rb._output_conv, out_parts=2)   # the identity gate's input
            att = blk._attention
            cin_p, ckv_p = ops.round_up(C + 2, 8), ops.round_up(2 + C + c, 8)
            lay = head_layout(att._n_heads, att._embed_channels, att._out_channels, att._q.weight.device)
            w[f"{bi}q"], w[f"{bi}qb"], w[f"{bi}kv"], w[f"{bi}kvb"], wp = lay.pack(
                att._q.weight, att._q.bias, att._kv.weight, att._kv.bias, att._proj.weight, cin_p, ckv_p)
            w[f"{bi}p"], w[f"{bi}pb"] = incremental.pad_rows(wp, att._proj.bias)
            for name, m in (("ro", blk._residual_out), ("ao", blk._attention_out), ("out", blk._out)):
                w[f"{bi}{name}"], w[f"{bi}{name}b"] = conv(m)
        w["o0"], w["o0b"] = conv(self._output[0])
        w["o1"], w["o1b"] = conv(self._output[1], out_parts=0)
        return w

    def _before_pixel(self, sp, st, canvas, row, col):
        sp.prev.fill_(max(row * canvas.shape[3] + col - 1, 0))

    def _pixel_program(self, sp, st):
        W, c, n = st["weights"], st["c"], sp.n
        C = self._input.weight.shape[0]
        cin_p = ops.round_up(C + 2, 8)
        bf16 = torch.bfloat16
        # (1) the previous pixel is final now: recompute its key / value rows, whose kv input holds the image value
        prev_img = st["image"].index_select(1, sp.prev)[:, 0, :c]
        for bi, b in enumerate(st["blocks"]):
            b["akv"][:, 2 + C: 2 + C + c] = prev_img
            kv = sp.linear(b["akv"], W[f"{bi}kv"], W[f"{bi}kvb"])
            qks = b["qk_slot"]
            b["kc"].view(n, sp.S, -1).index_copy_(1, sp.prev, kv[:, :qks].unsqueeze(1))
            b["vc"].view(n, sp.S, -1).index_copy_(1, sp.prev, kv[:, qks:].unsqueeze(1))
        # (2) position p through the stack
        off_in = [(dy, dx) for _, _, dy, dx in self._taps_in]
        x = sp.linear(sp.gather(st["image"], off_in), W["in"], W["in_b"], f32=True)
        pos_row = st["pos_tab"].index_select(0, sp.pos).expand(n, 2)
        img_row = st["image"].index_select(1, sp.pos)[:, 0, :c]
        for bi, (blk, b) in enumerate(zip(self._pixel_snail_blocks, st["blocks"])):
            res = x
            for j in range(len(blk._residual)):
                sp.write(b["ea"][j], sp.act(res, ELU))
                t = sp.linear(sp.gather(b["ea"][j], TAPS_2X2), W[f"{bi}r{j}i"], W[f"{bi}r{j}ib"], act=ELU)
                sp.write(b["eb"][j], t)
                u = sp.linear(sp.gather(b["eb"][j], TAPS_2X2), W[f"{bi}r{j}o"], W[f"{bi}r{j}ob"])
                res = pm.gated_res(u, res, NONE)
            akv = b["akv"]
            akv[:, :2] = pos_row
            akv[:, 2: 2 + C] = res[:, :C].to(bf16)
            akv[:, 2 + C: 2 + C + c] = img_row          # placeholder: the strict mask hides position p's own key / value
            q = sp.linear(akv[:, :cin_p], W[f"{bi}q"], W[f"{bi}qb"])
            kv = sp.linear(akv, W[f"{bi}kv"], W[f"{bi}kvb"])
            o = torch.empty(n, b["dv_slot"], dtype=bf16, device=sp.device)
            qks = b["qk_slot"]
            L.attn_decode(q, kv[:, :qks], kv[:, qks:], b["kc"], b["vc"], o, sp.pos32, n, sp.S, 1, qks, b["dv_slot"],
                          True, dk_true=blk._attention._embed_channels)
            attn = sp.linear(o, W[f"{bi}p"], W[f"{bi}pb"], f32=True)
            r = sp.linear(sp.act(res, ELU), W[f"{bi}ro"], W[f"{bi}rob"], act=ELU)
            a = sp.linear(sp.act(attn, ELU), W[f"{bi}ao"], W[f"{bi}aob"], act=ELU)
            out = sp.linear(sp.act(r.float() + a.float(), ELU), W[f"{bi}out"], W[f"{bi}outb"], act=ELU)
            x = x + out.float()
        t = sp.linear(x.to(bf16), W["o0"], W["o0b"])
        return sp.linear(t, W["o1"], W["o1b"], f32=True)

    def forward(self, x):
        """The whole network on pixel-major tensors: NCHW only at the image and at the logits."""
        n, c_img, h, w = x.shape
        geom = pm.Geom(n, h, w)
        self._input.apply_mask()
        kh, kw = self._input.weight.shape[2:]
        s = pm.image_conv(x, self._input.weight, self._input.bias, (kh // 2, kw // 2))  # fp32 stream [P, C]
        if len(self._pixel_snail_blocks):  # the attention operands besides the features, shared by every block
            pos_b = ops.nchw_to_pm(self._pixel_snail_blocks[0]._positions(x.shape, x.device), torch.bfloat16)
            img_b = ops.nchw_to_pm(x, torch.bfloat16)
            width = ops.round_up(2 + s.shape[1] + c_img, 8)
            pad_b = torch.zeros(n * h * w, width - (2 + s.shape[1] + c_img), dtype=torch.bfloat16, device=x.device)
        for block in self._pixel_snail_blocks:
            s = s + block.forward_pm(geom, s, img_b, pos_b, pad_b, c_img)
        t, _ = pm.conv(s, self._output[0].weight, self._output[0].bias, geom)
        logits, _ = pm.conv(t, self._output[1].weight, self._output[1].bias, geom, out_f32=True)
        return pm.from_pm(logits, geom, self._output[1].weight.shape[0])


def reproduce(*args, **kwargs):
    """The recipe of this model (reference pixel_snail.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_pixel_snail(*args, **kwargs)
