"""ImageGPT on the CUDA path — API of reference models/autoregressive/image_gpt.py:21-109.

Module tree, parameter names and shapes are the reference's (`_pos`, `_input`, `_transformer.{i}.{_ln1,_ln2,
_attn.{_q,_kv,_proj},_out.{0,2}}`, `_ln`, `_out`), so checkpoints are interchangeable.  `forward` does not walk
that tree: the whole stack runs as ONE autograd node over pixel-major tensors —

    stream x (fp32 [P, C])  --LN-->  bf16  --GEMM(q|k|v)-->  causal attention  --GEMM(proj)+x--> h (fp32)
    h --LN--> bf16 --GEMM(4C)+GELU--> bf16 --GEMM(C) + x + h--> next stream      (x <- x + h + mlp, the
                                                                                  reference's double residual)

with every bias / activation / residual folded into a GEMM epilogue, the residual stream and all summed
gradients kept in fp32, and bf16 used only for tensor-core operands (SURVEY.md §7.3-2).

A stream of C channels lives in round_up(C, 8) columns with exactly-zero pad columns (`StreamLayout`), so every bf16
GEMM operand keeps the 16-byte pitch TMA needs at any C.

Training keeps every block's activations until backward when they fit into the memory the process can still get;
otherwise it keeps only each block's input stream, attention output and lse and rebuilds the rest block by block in
backward (`activation_memory`, `recompute_activations`).  Both paths compute the same bits.
"""

import math
import os
from typing import NamedTuple

import torch
from torch import nn

from .. import _lib as L
from .. import nn as pg_nn
from .. import ops
from ..nn.modules import head_layout
from . import base, incremental

F32, BF16 = torch.float32, torch.bfloat16
PARAMS_PER_BLOCK = 14


class TransformerBlock(nn.Module):
    """Holds the parameters of one block (reference image_gpt.py:21-52); standalone `forward` composes the
    drop-in nn modules, the fused model path reads the parameters directly."""

    def __init__(self, n_channels, n_attention_heads):
        super().__init__()
        self._ln1 = pg_nn.NCHWLayerNorm(n_channels)
        self._ln2 = pg_nn.NCHWLayerNorm(n_channels)
        self._attn = pg_nn.CausalAttention(in_channels=n_channels, n_heads=n_attention_heads,
                                           embed_channels=n_channels, out_channels=n_channels)
        self._out = nn.Sequential(
            nn.Conv2d(in_channels=n_channels, out_channels=4 * n_channels, kernel_size=1),
            nn.GELU(),
            nn.Conv2d(in_channels=4 * n_channels, out_channels=n_channels, kernel_size=1),
        )

    def forward(self, x):
        """Standalone use of one block on an NCHW tensor (reference image_gpt.py:50-52), composed of the drop-in
        modules; `ImageGPT.forward` does not come through here (it runs the fused stack)."""
        from ..nn.tapconv import tap_conv2d

        h = x + self._attn(self._ln1(x))
        t = tap_conv2d(self._ln2(h), self._out[0].weight, self._out[0].bias, (0, 0), post_act=L.ACT_GELU)
        return h + tap_conv2d(t, self._out[2].weight, self._out[2].bias, (0, 0))

    def flat_params(self):
        a = self._attn
        return [self._ln1.weight, self._ln1.bias, a._q.weight, a._q.bias, a._kv.weight, a._kv.bias, a._proj.weight,
                a._proj.bias, self._ln2.weight, self._ln2.bias, self._out[0].weight, self._out[0].bias,
                self._out[2].weight, self._out[2].bias]


class StreamLayout(NamedTuple):
    """Where the fused stack keeps its channels: the stream's c channels in c_p = round_up(c, 8) columns and the MLP's
    4c hidden channels in f_p = round_up(4c, 8), so every bf16 GEMM operand has a 16-byte pitch.  The pad columns are
    exactly zero in every activation and gradient: the packed weights are zero in the pad rows and columns and the
    packed biases in the pad entries, LayerNorm writes zeros past c (`pg_layernorm_fwd_ld` / `_bwd_ld`) and GELU(0) = 0.
    This is the one owner of that layout: `pack` pads a parameter into it and `unpack` crops a gradient back to the
    parameter's shape.  With c % 8 == 0 (`identity`) both hand back their argument (detached / as a view).  Build it
    with `stream_layout`."""

    c: int
    c_p: int
    f_p: int

    @property
    def identity(self):
        return self.c_p == self.c

    @staticmethod
    def pack(t, rows, cols=None):
        """fp32 [rows, cols] (a bias when cols is None: [rows]) holding t, detached and flattened to 2-D, in its top-left
        corner and zeros elsewhere; t's own data when it has that shape already."""
        t = t.detach()
        t = t.reshape(t.shape[0], -1) if cols is not None else t
        shape = (rows,) if cols is None else (rows, cols)
        if tuple(t.shape) == shape:
            return t
        out = torch.zeros(shape, dtype=F32, device=t.device)
        out[tuple(slice(0, n) for n in t.shape)] = t
        return out

    @staticmethod
    def unpack(g, shape):
        """The gradient of a parameter of `shape` from g, its gradient in packed layout: a view of g when nothing was
        padded, else a cropped copy."""
        rows = shape[0]
        if g.dim() == 1:
            return g if g.shape[0] == rows else g[:rows].clone()
        cols = math.prod(shape[1:])
        if tuple(g.shape) == (rows, cols):
            return g.view(shape)
        return g[:rows, :cols].reshape(shape)


def stream_layout(c):
    return StreamLayout(c, ops.round_up(c, 8), ops.round_up(4 * c, 8))


class ActivationMemory(NamedTuple):
    """Bytes of the fused stack's training memory for one batch, estimated from the shapes (`activation_memory`)."""
    store_block: int      # activations one block keeps until backward when everything is kept
    recompute_block: int  # ... when only its input stream, attention output and lse are kept
    store: int            # everything the stack keeps until backward, every block's activations kept
    recompute: int        # ... with the recompute path
    backward: int         # the widest point of one block's backward (gradient transients) plus the gradient arena


def activation_memory(n_pixels, channels, n_heads, qk_slot, dv_slot, n_blocks):
    """Estimates, from the shapes alone, what the fused stack keeps from forward to backward on either path and what
    one block's backward needs on top.  Pure: no device is queried.  n_pixels = batch x height x width; q/k/v and the
    attention output are counted at their head-slot widths (`head_layout`), padding included."""
    C, H = channels, n_heads
    qkv_cols, o_cols = H * (2 * qk_slot + dv_slot), H * dv_slot
    # per pixel and block: xs and h (fp32), a1 and a2 (bf16), qkv and o (bf16), lse (fp32 per head), u and g (bf16, 4C),
    # two LayerNorms' mean and rstd (fp32)
    store_px = 4 * C + 4 * C + 2 * C + 2 * C + 2 * qkv_cols + 2 * o_cols + 4 * H + 2 * 4 * C + 2 * 4 * C + 16
    recompute_px = 4 * C + 2 * o_cols + 4 * H
    head_px = 4 * C + 2 * C + 8  # both paths: the final stream, its LayerNorm output and statistics
    # a block's backward holds the incoming and outgoing stream gradients and dh (fp32 + bf16 each: 12C) plus, at its
    # widest, either du and da2 / da1 (8C) or do, dqkv and the softmax row sums
    bwd_px = 12 * C + max(8 * C, 2 * o_cols + 2 * qkv_cols + 4 * H)
    arena = 4 * n_blocks * (8 * C * C + C * o_cols + qkv_cols * C + 10 * C + qkv_cols)  # fp32 weight gradients
    P = n_pixels
    return ActivationMemory(store_block=P * store_px, recompute_block=P * recompute_px,
                            store=P * (n_blocks * store_px + head_px), recompute=P * (n_blocks * recompute_px + head_px),
                            backward=P * bwd_px + arena)


def recompute_activations(mem, available):
    """The stack's memory policy: keep every block's activations when they and one block's backward fit into
    `available` bytes; otherwise (True) keep only each block's input stream, attention output and lse, and rebuild the
    rest of a block's activations just before its backward.  Either path computes the same bits."""
    return mem.store + mem.backward > available


# what the recompute path keeps of each block, and the packed weights every saved block refers to
_KEPT = ("xs", "o", "lse")
_WEIGHTS = ("wqkv", "bqkv", "wp", "bp", "w1", "b1", "w2", "b2", "layout")


def _block_fwd(xs, p, pk, n, S, H, eps, attn=None):
    """One transformer block on the fp32 stream xs [P, C]; p = its 14 parameters, pk = its packed weights.  Returns
    (next stream, every activation the block's backward reads).  Given attn = (o, lse) of an earlier forward, it rebuilds
    those activations for the backward instead, without the attention forward or fc2 (next stream None): the same
    kernels on the same inputs in the same order, so the same bits as the forward's."""
    (ln1_w, ln1_b, _, _, _, _, _, _, ln2_w, ln2_b, _, _, _, _) = p
    lay = pk["layout"]
    dv_slot, slot = lay.dv_slot, lay.qk_slot
    a1, _, mean1, rstd1 = ops.layernorm_fwd(xs, ln1_w.detach(), ln1_b.detach(), eps)
    qkv, _, _ = ops.linear_fwd(a1, pk["wqkv"], pk["bqkv"])
    if attn is None:
        q, k, v = qkv[:, : H * slot], qkv[:, H * slot: 2 * H * slot], qkv[:, 2 * H * slot:]
        o, lse = ops.attn_fwd(q, k, v, n, S, H, lay.dk, slot, dv_slot, False)
    else:
        o, lse = attn
    _, _, hres = ops.linear_fwd(o, pk["wp"], pk["bp"], res0=xs, want_bf16=False, want_f32=True)
    a2, _, mean2, rstd2 = ops.layernorm_fwd(hres, ln2_w.detach(), ln2_b.detach(), eps)
    g, u, _ = ops.linear_fwd(a2, pk["w1"], pk["b1"], act=L.ACT_GELU, want_pre=True, pre_deriv=True)  # u = GELU'(pre)
    acts = dict(xs=xs, a1=a1, qkv=qkv, o=o, lse=lse, h=hres, a2=a2, u=u, g=g, mean1=mean1, rstd1=rstd1, mean2=mean2,
                rstd2=rstd2, **{k: pk[k] for k in _WEIGHTS})
    if attn is not None:
        return None, acts
    _, _, xs_new = ops.linear_fwd(g, pk["w2"], pk["b2"], res0=xs, res1=hres, want_bf16=False, want_f32=True)
    return xs_new, acts


class _ImageGPTStack(torch.autograd.Function):
    """forward(x_nchw, params...) -> logits_nchw; one node for the whole network."""

    @staticmethod
    def forward(ctx, x, n_heads, eps, packed, opts, *params):
        pos, in_w, in_b = params[0], params[1], params[2]
        n_blocks = (len(params) - 7) // PARAMS_PER_BLOCK
        ln_w, ln_b, out_w, out_b = params[-4:]
        n, cin, h, w = x.shape
        S, P, H = h * w, n * h * w, n_heads
        C, c_p = in_w.shape[0], packed["in_w"].shape[0]
        # needs_input_grad ignores torch.no_grad(): eval / sampling must not retain every block's activations
        keep = any(ctx.needs_input_grad) and opts["grad"]
        recompute = keep and opts["recompute"]

        x_in = (x + pos[:, :, : h, : w]).contiguous()  # sampling evaluates the top rows of the canvas only
        xs = torch.empty(P, c_p, dtype=F32, device=x.device)
        L.conv_small_fwd(x_in, packed["in_w"], packed["in_b"], (in_w.shape[2] // 2, in_w.shape[3] // 2), out_f32=xs)
        saved = []
        for b in range(n_blocks):
            xs_new, acts = _block_fwd(xs, params[3 + b * PARAMS_PER_BLOCK: 3 + (b + 1) * PARAMS_PER_BLOCK],
                                      packed["blocks"][b], n, S, H, eps)
            if keep:
                saved.append({k: acts[k] for k in _KEPT + _WEIGHTS} if recompute else acts)
            del acts  # what is not saved goes before the next block allocates its own
            xs = xs_new
        af, _, mean_f, rstd_f = ops.layernorm_fwd(xs, ln_w.detach(), ln_b.detach(), eps)
        cout = out_w.shape[0]
        wo = packed["wo"]
        _, _, logits_pm = ops.linear_fwd(af, wo, out_b.detach(), want_bf16=False, want_f32=True)
        if keep:
            ctx.saved = dict(blocks=saved, x_in=x_in, xs_final=xs, af=af, mean_f=mean_f, rstd_f=rstd_f, wo=wo,
                             in_w=packed["in_w"], sl=packed["stream"], params=params, dims=(n, cin, h, w, C, H, cout),
                             eps=eps, hook=opts.get("hook"), recompute=recompute)
        return ops.pm_to_nchw(logits_pm, n, cout, h, w)

    @staticmethod
    def backward(ctx, dlogits):
        sv = getattr(ctx, "saved", None)
        if sv is None:
            raise RuntimeError("ImageGPT: the activations of this forward were already consumed by a backward pass "
                               "(retain_graph is not supported by the fused stack)")
        params = sv["params"]
        n, cin, h, w, C, H, cout = sv["dims"]
        S, P = h * w, n * h * w
        dev = dlogits.device
        n_blocks = len(sv["blocks"])
        grads = [None] * len(params)
        ln_w = params[-4]
        sl = sv["sl"]
        c_p, f_p = sl.c_p, sl.f_p

        # head: logits = 1x1(LN(x))
        dl = ops.nchw_to_pm(dlogits, BF16, width=ops.round_up(cout, 8))
        grads[-1] = ops.bias_grad(dl[:, :cout])
        dwo = torch.zeros(ops.round_up(cout, 8), c_p, dtype=F32, device=dev)
        ops.linear_wgrad(dl, sv["af"], dwo)
        grads[-2] = dwo[:cout, :C].reshape(cout, C, 1, 1)
        daf = ops.linear_dgrad(dl[:, :cout], sv["wo"])
        # every LayerNorm backward also emits the column sums of the gradient it writes = the bias gradient of the
        # linear layer that produced its input (fc2 of the block above / the attention projection)
        dx, dx_b, grads[-4], grads[-3], dx_sum = ops.layernorm_bwd(daf, sv["xs_final"], ln_w.detach(), sv["mean_f"],
                                                                    sv["rstd_f"], want_colsum=True)
        del daf

        # one zero-filled fp32 arena for every weight gradient of the stack (the wgrad GEMMs accumulate into it with
        # TMA reduce-adds): a single memset instead of four per block
        qkv_rows = sv["blocks"][0]["wqkv"].shape[0] if n_blocks else 0
        dvs = sv["blocks"][0]["layout"].dv_slot if n_blocks else 0
        per_block = 2 * f_p * c_p + c_p * H * dvs + qkv_rows * c_p
        # ... followed by the small per-block gradients (LayerNorm dgamma / dbeta / column sums, bias gradients of the qkv
        # and fc1 layers), which their kernels accumulate with atomics: they share the one memset too
        per_small = 6 * C + qkv_rows + f_p
        arena = torch.zeros(n_blocks * (per_block + per_small), dtype=F32, device=dev)
        small_base = n_blocks * per_block

        def carve_small(b, off, n):
            start = small_base + b * per_small + off
            return arena[start: start + n]

        def carve(b, off, rows, cols):
            start = b * per_block + off
            return arena[start: start + rows * cols].view(rows, cols)

        # data parallelism: each block's slice of the arena is handed to the bucket hook (an asynchronous all-reduce)
        # as soon as its last wgrad GEMM is queued; see parallel.OverlappedGradAverager
        bucket_hook = sv["hook"] if _arena_views_are_grads(sv) else None
        # transformer blocks per all-reduce; 0 = the whole stack in one bucket, issued when block 0's last wgrad is queued
        # (overlaps the input convolution's backward and the small-gradient bucket only).  Finer buckets overlap more, but
        # every NCCL kernel that runs next to the GEMMs competes with them for SMs.
        bucket_blocks = int(os.environ.get("PG_DP_BUCKET_BLOCKS", "0"))
        if bucket_blocks <= 0:
            bucket_blocks = n_blocks
        pending = []

        for b in reversed(range(n_blocks)):
            blk = sv["blocks"][b]
            base_i = 3 + b * PARAMS_PER_BLOCK
            if sv["recompute"]:  # rebuild what the forward did not keep, from what it did
                _, blk = _block_fwd(blk["xs"], params[base_i: base_i + PARAMS_PER_BLOCK], blk, n, S, H, sv["eps"],
                                    attn=(blk["o"], blk["lse"]))
            (ln1_w, _, q_w, _, kv_w, _, p_w, _, ln2_w, _, f1_w, _, f2_w, _) = params[base_i: base_i + PARAMS_PER_BLOCK]
            lay = blk["layout"]
            dv_slot, slot = lay.dv_slot, lay.qk_slot
            # x_new = x + h + fc2(gelu(fc1(ln2(h))))
            grads[base_i + 13] = dx_sum
            dw2 = carve(b, 0, c_p, f_p)
            ops.linear_wgrad(dx_b, blk["g"], dw2)
            grads[base_i + 12] = sl.unpack(dw2, f2_w.shape)
            du = ops.linear_dgrad(dx_b, blk["w2"], aux=blk["u"], dact=L.ACT_GIVEN)
            # the bias gradient (column sums of du) is reduced by the wgrad launch from the du tiles it stages
            db1 = carve_small(b, 6 * C + qkv_rows, f_p)
            dw1 = carve(b, f_p * c_p, f_p, c_p)
            ops.linear_wgrad(du, blk["a2"], dw1, db_out=db1)
            grads[base_i + 10], grads[base_i + 11] = sl.unpack(dw1, f1_w.shape), sl.unpack(db1, (4 * C,))
            da2 = ops.linear_dgrad(du, blk["w1"])
            del du
            # h receives: LN2 path + direct (x_new = ... + h)
            dh, dh_b, grads[base_i + 8], grads[base_i + 9], grads[base_i + 7] = ops.layernorm_bwd(
                da2, blk["h"], ln2_w.detach(), blk["mean2"], blk["rstd2"], dres0=dx, want_colsum=True,
                stats=carve_small(b, 3 * C, 3 * C).view(3, C))
            del da2
            # h = x + proj(attn)
            dwp = carve(b, 2 * f_p * c_p, c_p, H * dv_slot)
            ops.linear_wgrad(dh_b, blk["o"], dwp)
            do = ops.linear_dgrad(dh_b, blk["wp"])
            qkv = blk["qkv"]
            q, k, v = qkv[:, : H * slot], qkv[:, H * slot: 2 * H * slot], qkv[:, 2 * H * slot:]
            dqkv = torch.empty_like(qkv)
            ops.attn_bwd(q, k, v, blk["o"], do, blk["lse"], dqkv[:, : H * slot], dqkv[:, H * slot: 2 * H * slot],
                         dqkv[:, 2 * H * slot:], n, S, H, lay.dk, slot, dv_slot, False)
            del do
            dbqkv = carve_small(b, 6 * C, qkv_rows)
            dwqkv = carve(b, 2 * f_p * c_p + c_p * H * dv_slot, qkv_rows, c_p)
            ops.linear_wgrad(dqkv, blk["a1"], dwqkv, db_out=dbqkv)
            # q_w, q_b, kv_w, kv_b, p_w: views of the arena when heads fill their slots
            grads[base_i + 2: base_i + 7] = lay.unpack_grads(dwqkv[: H * slot], dbqkv[: H * slot], dwqkv[H * slot:],
                                                              dbqkv[H * slot:], dwp, C, C)
            da1 = ops.linear_dgrad(dqkv, blk["wqkv"])
            del dqkv
            # x receives: LN1 path + direct from h (dh) + direct from x_new (dx)
            dx, dx_b, grads[base_i + 0], grads[base_i + 1], dx_sum = ops.layernorm_bwd(
                da1, blk["xs"], ln1_w.detach(), blk["mean1"], blk["rstd1"], dres0=dx, dres1=dh, want_colsum=True,
                stats=carve_small(b, 0, 3 * C).view(3, C))
            del da1, dh, dh_b
            if bucket_hook is not None and b % bucket_blocks == 0:
                # blocks b .. b + bucket_blocks - 1 are complete: one contiguous slice of the arena
                hi = min(b + bucket_blocks, n_blocks)
                pending.append(bucket_hook(arena[b * per_block: hi * per_block]))
            sv["blocks"][b] = None  # release this block's activations
            del blk, qkv, q, k, v  # (rebuilt ones too) before the next block rebuilds its own

        in_w = params[1]
        dw_in = torch.zeros_like(sv["in_w"])
        db_in = dx_sum  # bias gradient of the input conv = column sums of the stream gradient
        dx_in = torch.empty(n, cin, h, w, dtype=F32, device=dev)
        L.conv_small_bwd(sv["x_in"], sv["in_w"], dx, (in_w.shape[2] // 2, in_w.shape[3] // 2), dw=dw_in, dbias=None,
                         dx=dx_in)
        grads[1], grads[2] = sl.unpack(dw_in.view(dw_in.shape[0], -1), in_w.shape), db_in
        dpos = torch.zeros_like(params[0])
        dpos[:, :, : h, : w] = dx_in.sum(dim=0, keepdim=True)
        grads[0] = dpos
        ctx.saved = None
        for handle in pending:  # the gradients leave this node averaged
            handle.wait()
        return (dx_in if ctx.needs_input_grad[0] else None, None, None, None, None, *grads)


def _arena_views_are_grads(sv):
    """True when every block's weight gradients are plain views of the gradient arena (heads fill their kernel slots,
    e.g. 512 channels / 8 or 4 heads, and the stream needs no pad columns): only then can the arena slice be averaged in
    place."""
    return bool(sv["blocks"]) and sv["sl"].identity and all(blk["layout"].identity for blk in sv["blocks"])




class ImageGPT(incremental.IncrementalSamplingMixin, base.AutoregressiveModel):
    """The (convolutional) ImageGPT model — constructor of reference image_gpt.py:64-103."""

    def __init__(self, in_channels=1, out_channels=1, in_size=28, n_transformer_blocks=8, n_attention_heads=4,
                 n_embedding_channels=16, sample_fn=None):
        super().__init__(sample_fn)
        self._pos = nn.Parameter(torch.zeros(1, in_channels, in_size, in_size))
        self._input = pg_nn.CausalConv2d(mask_center=True, in_channels=in_channels,
                                         out_channels=n_embedding_channels, kernel_size=3, padding=1)
        self._transformer = nn.ModuleList(
            TransformerBlock(n_channels=n_embedding_channels, n_attention_heads=n_attention_heads)
            for _ in range(n_transformer_blocks)
        )
        self._ln = pg_nn.NCHWLayerNorm(n_embedding_channels)
        self._out = nn.Conv2d(in_channels=n_embedding_channels, out_channels=out_channels, kernel_size=1)
        self._n_heads = n_attention_heads

    # ------------------------------------------------------------------------------------------------------------
    # bf16 tensor-core copies of the weight matrices.  The fp32 Parameters stay the master weights (reference
    # semantics: the optimizer updates them in place); `ops.cached_copy` rebuilds the copies.  With heads that fill
    # their slots that is ONE multi-tensor cast into a fresh bf16 arena (q | kv adjacent: the fused qkv projection needs
    # no torch.cat) and one concatenation of the q / kv biases; a refresh captured in a CUDA graph casts into its own.
    # ------------------------------------------------------------------------------------------------------------
    def _packed_training_weights(self):
        blocks = list(self._transformer)
        mats = [w for blk in blocks for w in (blk._attn._q.weight, blk._attn._kv.weight, blk._attn._proj.weight,
                                              blk._out[0].weight, blk._out[2].weight)] + [self._out.weight]
        biases = [b for blk in blocks for b in (blk._attn._q.bias, blk._attn._kv.bias)]
        sl = stream_layout(self._input.weight.shape[0])
        # in the padded layout the remaining biases and the input convolution are packed copies too
        padded = [] if sl.identity else [self._input.weight, self._input.bias] + [
            b for blk in blocks for b in (blk._attn._proj.bias, blk._out[0].bias, blk._out[2].bias)]
        return ops.cached_copy(mats + biases + padded, "image_gpt",
                               lambda: self._pack_training_weights(blocks, mats, biases))

    def _pack_training_weights(self, blocks, mats, biases):
        C, H = self._input.weight.shape[0], self._n_heads
        dev = mats[0].device
        cout = self._out.weight.shape[0]
        lay = head_layout(H, C, C, dev)
        sl = stream_layout(C)
        c_p, f_p = sl.c_p, sl.f_p
        in_w = self._input.weight
        packed = {"blocks": [], "stream": sl, "in_w": sl.pack(in_w, c_p, in_w[0].numel()).view(c_p, *in_w.shape[1:]),
                  "in_b": sl.pack(self._input.bias, c_p)}

        def biases_of(blk):  # the projection and MLP biases, padded
            return dict(bp=sl.pack(blk._attn._proj.bias, c_p), b1=sl.pack(blk._out[0].bias, f_p),
                        b2=sl.pack(blk._out[2].bias, c_p))

        if lay.identity and blocks:
            per_block = 12 * C * C
            arena = torch.empty(len(blocks) * per_block + cout * C, dtype=BF16, device=dev)
            views, dsts = [], []
            for b in range(len(blocks)):
                base = b * per_block
                wqkv = arena[base: base + 3 * C * C].view(3 * C, C)
                wp = arena[base + 3 * C * C: base + 4 * C * C].view(C, C)
                w1 = arena[base + 4 * C * C: base + 8 * C * C].view(4 * C, C)
                w2 = arena[base + 8 * C * C: base + 12 * C * C].view(C, 4 * C)
                views.append((wqkv, wp, w1, w2))
                dsts += [wqkv[:C], wqkv[C:], wp, w1, w2]
            wo = arena[len(blocks) * per_block:].view(cout, C)
            dsts.append(wo)
            plan = self.__dict__.get("_cast_plan")
            if plan is None or plan["src_key"] != tuple(p.data_ptr() for p in mats):
                from .. import optim

                numel = [p.numel() for p in mats]
                chunks = [(t, c) for t, n in enumerate(numel) for c in range((n + optim.CHUNK - 1) // optim.CHUNK)]
                plan = dict(src_key=tuple(p.data_ptr() for p in mats), n_chunks=len(chunks), chunk=optim.CHUNK,
                            numel=torch.tensor(numel, dtype=torch.int64, device=dev),
                            chunks=torch.tensor(chunks, dtype=torch.int32, device=dev).contiguous(),
                            src=torch.tensor([p.data_ptr() for p in mats], dtype=torch.int64, device=dev),
                            dst_bytes=torch.tensor([d.data_ptr() - arena.data_ptr() for d in dsts], device=dev))
                self.__dict__["_cast_plan"] = plan
            dst = plan["dst_bytes"] + arena.data_ptr()  # every arena has the same layout; only its base differs
            L.cast_multi(plan["src"], dst, plan["numel"], plan["chunks"], plan["n_chunks"], plan["chunk"])
            ball = torch.cat([b.detach() for b in biases])  # [blocks * 3C]: q | kv biases of every block
            for b, (wqkv, wp, w1, w2) in enumerate(views):
                packed["blocks"].append(dict(wqkv=wqkv, bqkv=ball[b * 3 * C: (b + 1) * 3 * C], wp=wp, w1=w1, w2=w2,
                                             layout=lay, **biases_of(blocks[b])))
            packed["wo"], packed["arena"] = wo, arena
        else:  # other heads live in zero-padded 64- or 128-wide slots, other streams in padded columns: pack per block
            for blk in blocks:
                a = blk._attn
                if sl.identity:
                    wq, bq, wkv, bkv, wp = lay.pack(a._q.weight, a._q.bias, a._kv.weight, a._kv.bias, a._proj.weight, C, C)
                    w1, w2 = ops.pack_taps(blk._out[0].weight, C), ops.pack_taps(blk._out[2].weight, 4 * C)
                else:
                    wq, bq, wkv, bkv, wp = lay.scatter(a._q.weight, a._q.bias, a._kv.weight, a._kv.bias, a._proj.weight,
                                                       c_p, c_p)
                    wq, wkv, wp = ops.to_bf16(wq), ops.to_bf16(wkv), ops.to_bf16(sl.pack(wp, c_p, wp.shape[1]))
                    w1 = ops.to_bf16(sl.pack(blk._out[0].weight, f_p, c_p))
                    w2 = ops.to_bf16(sl.pack(blk._out[2].weight, c_p, f_p))
                packed["blocks"].append(dict(wqkv=torch.cat((wq, wkv)), bqkv=torch.cat((bq, bkv)), wp=wp, w1=w1, w2=w2,
                                             layout=lay, **biases_of(blk)))
            packed["wo"] = ops.pack_taps(self._out.weight, c_p)
        return packed

    # ------------------------------------------------------------------------------------------------------------
    # Incremental sampling (models/incremental.py).  The model is exactly causal, so the logits of pixel p only need p's
    # own row through the stack plus the keys / values of the pixels before it.  Per pixel: input conv on the 3x3
    # window of (x + pos) around p, and per block LN -> q|k|v GEMM (M = batch rows) -> pg_attn_decode over the K/V
    # caches -> proj / MLP GEMMs with the same fused epilogues as training.
    # ------------------------------------------------------------------------------------------------------------
    def _incremental_ok(self, canvas):  # any batch: the 32-row limit is the convolutional programs'
        h, w = canvas.shape[2:]
        return self._incremental_sampling and canvas.is_cuda and h <= self._pos.shape[2] and w <= self._pos.shape[3]

    def _build_pixel_state(self, sp, c):
        C, H = self._input.weight.shape[0], self._n_heads
        kh, kw = self._input.weight.shape[2:]
        lay = head_layout(H, C, C, sp.device)
        # the K/V caches need no reset per call: the decode writes row p before it reads rows <= p
        kc = [torch.zeros(sp.n * sp.S, H * lay.qk_slot, dtype=BF16, device=sp.device) for _ in self._transformer]
        vc = [torch.zeros(sp.n * sp.S, H * lay.dv_slot, dtype=BF16, device=sp.device) for _ in self._transformer]
        return dict(layout=lay, kc=kc, vc=vc, weights={},
                    xin=torch.zeros(sp.n, c, sp.h + kh - 1, sp.w + kw - 1, dtype=F32, device=sp.device),  # padded x + pos
                    patch=torch.zeros(sp.n, c, kh, kw, dtype=F32, device=sp.device))

    def _pack_pixel_weights(self):
        self._input.apply_mask()
        packed = self._packed_training_weights()
        w = {"wo": packed["wo"], "in_w": packed["in_w"], "in_b": packed["in_b"]}
        for b, pb in enumerate(packed["blocks"]):
            w.update({f"{b}{k}": pb[k] for k in ("wqkv", "bqkv", "wp", "bp", "w1", "b1", "w2", "b2")})
        return w

    def _start_pixels(self, st, canvas):
        h, w = canvas.shape[2:]
        kh, kw = self._input.weight.shape[2:]
        st["xin"][:, :, kh // 2: kh // 2 + h, kw // 2: kw // 2 + w] = canvas + self._pos[:, :, :h, :w]

    def _before_pixel(self, sp, st, canvas, row, col):
        kh, kw = self._input.weight.shape[2:]
        st["patch"].copy_(st["xin"][:, :, row: row + kh, col: col + kw])

    def _after_pixel(self, sp, st, new, row, col):
        kh, kw = self._input.weight.shape[2:]
        st["xin"][:, :, row + kh // 2, col + kw // 2] = new + self._pos[0, :, row, col]

    def _pixel_program(self, sp, st):
        """One position for every image of the batch: st["patch"] (window of x + pos around the pixel) -> logits."""
        W, lay, n, C, H, eps = st["weights"], st["layout"], sp.n, self._input.weight.shape[0], self._n_heads, self._ln.eps
        kh, kw = self._input.weight.shape[2:]
        slot = lay.qk_slot
        c_p = W["in_w"].shape[0]
        taps_out = torch.empty(n * kh * kw, c_p, dtype=F32, device=sp.device)
        L.conv_small_fwd(st["patch"], W["in_w"], W["in_b"], (kh // 2, kw // 2), out_f32=taps_out)
        xs = taps_out.view(n, kh * kw, c_p)[:, (kh // 2) * kw + kw // 2].contiguous()  # the window's centre pixel
        for b, blk in enumerate(self._transformer):
            a1, _, _, _ = ops.layernorm_fwd(xs, blk._ln1.weight.detach(), blk._ln1.bias.detach(), eps)
            qkv = sp.linear(a1, W[f"{b}wqkv"], W[f"{b}bqkv"])
            q, k, v = qkv[:, : H * slot], qkv[:, H * slot: 2 * H * slot], qkv[:, 2 * H * slot:]
            o = torch.empty(n, H * lay.dv_slot, dtype=BF16, device=sp.device)
            L.attn_decode(q, k, v, st["kc"][b], st["vc"][b], o, sp.pos32, n, sp.S, H, slot, lay.dv_slot, False,
                          dk_true=lay.dk)
            hres = sp.linear(o, W[f"{b}wp"], W[f"{b}bp"], res0=xs, f32=True)
            a2, _, _, _ = ops.layernorm_fwd(hres, blk._ln2.weight.detach(), blk._ln2.bias.detach(), eps)
            g = sp.linear(a2, W[f"{b}w1"], W[f"{b}b1"], act=L.ACT_GELU)
            xs = sp.linear(g, W[f"{b}w2"], W[f"{b}b2"], res0=xs, res1=hres, f32=True)
        af, _, _, _ = ops.layernorm_fwd(xs, self._ln.weight.detach(), self._ln.bias.detach(), eps)
        return sp.linear(af, W["wo"], self._out.bias.detach(), f32=True)

    # ---- data-parallel bucket protocol (parallel.OverlappedGradAverager) ----
    def set_grad_bucket_hook(self, fn):
        """fn(flat_fp32_bucket) -> handle with wait(); called once per transformer block during backward."""
        self.__dict__["_grad_bucket_hook"] = fn  # per model instance; None removes it

    def bucketed_parameters(self):
        """Parameters whose gradients are averaged by the bucket hook (the block weight matrices), or [] when the
        head geometry needs slot padding (their gradients are then gathered copies, averaged by the flat bucket)."""
        c = self._ln.weight.numel()
        if not head_layout(self._n_heads, c, c).identity:
            return []
        out = []
        for blk in self._transformer:
            a = blk._attn
            out += [a._q.weight, a._kv.weight, a._proj.weight, blk._out[0].weight, blk._out[2].weight]
        return out

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("ImageGPT (CUDA path) needs CUDA tensors; there is no CPU fallback")
        self._input.apply_mask()  # same in-place side effect as the reference's CausalConv2d
        flat = [self._pos, self._input.weight, self._input.bias]
        for blk in self._transformer:
            flat.extend(blk.flat_params())
        flat.extend([self._ln.weight, self._ln.bias, self._out.weight, self._out.bias])
        grad = torch.is_grad_enabled()
        return _ImageGPTStack.apply(x.float(), self._n_heads, self._ln.eps, self._packed_training_weights(),
                                    dict(grad=grad, hook=self.__dict__.get("_grad_bucket_hook"),
                                         recompute=grad and self._recompute_for(x)), *flat)

    def _recompute_for(self, x):
        """recompute_activations for a training forward of this batch shape, on the memory this process can still get:
        the driver's free memory plus what the caching allocator holds unallocated.  That memory is read at the first
        training forward of each batch shape and device only: read every step, the queries made a C5 step about 1 ms
        (0.5 %) slower on an H100 80GB HBM3 at 400 W.  Under CUDA-graph capture, where the driver must not be queried, the decision of the last eager
        forward of the same shape (GraphedTrainStep's warm-up), or recompute when there was none."""
        n, _, h, w = x.shape
        seen = self.__dict__.setdefault("_memory_by_shape", {})  # (n, h, w, device) -> [available bytes, decision]
        key = (n, h, w, x.device)
        if torch.cuda.is_current_stream_capturing():
            return seen[key][1] if key in seen else True
        if key not in seen:
            free, _ = torch.cuda.mem_get_info(x.device)
            seen[key] = [free + torch.cuda.memory_reserved(x.device) - torch.cuda.memory_allocated(x.device), None]
        C, H = self._ln.weight.numel(), self._n_heads
        lay = head_layout(H, C, C)
        mem = activation_memory(n * h * w, stream_layout(C).c_p, H, lay.qk_slot, lay.dv_slot, len(self._transformer))
        seen[key][1] = recompute_activations(mem, seen[key][0])
        return seen[key][1]


def reproduce(*args, **kwargs):
    """The recipe of this model (reference image_gpt.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_image_gpt(*args, **kwargs)
