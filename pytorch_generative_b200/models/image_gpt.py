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

Three layouts, each with one owner: `BlockParams` names a block's 14 parameters in the order of the node's flat
argument list (and of the gradients it returns), `StreamLayout` is the padded stream, and `GradArena` is the one fp32
buffer every block's weight gradients accumulate into.  `_block_fwd` and `_block_bwd` are one block's forward and
backward; `_ImageGPTStack` strings them together between the input convolution and the head.
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


# one transformer block's parameters, or their gradients, in the order `_ImageGPTStack` takes and returns them
BlockParams = NamedTuple("BlockParams", [(name, torch.Tensor) for name in (
    "ln1_w", "ln1_b", "q_w", "q_b", "kv_w", "kv_b", "p_w", "p_b", "ln2_w", "ln2_b", "f1_w", "f1_b", "f2_w", "f2_b")])
PARAMS_PER_BLOCK = len(BlockParams._fields)


def _split_params(params):
    """The stack's flat parameter list as ((pos, in_w, in_b), [BlockParams per block], (ln_w, ln_b, out_w, out_b))."""
    stem, head = params[:3], params[-4:]
    blocks = [BlockParams(*params[i: i + PARAMS_PER_BLOCK]) for i in range(3, len(params) - 4, PARAMS_PER_BLOCK)]
    return stem, blocks, head


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
        return BlockParams(ln1_w=self._ln1.weight, ln1_b=self._ln1.bias, q_w=a._q.weight, q_b=a._q.bias,
                           kv_w=a._kv.weight, kv_b=a._kv.bias, p_w=a._proj.weight, p_b=a._proj.bias,
                           ln2_w=self._ln2.weight, ln2_b=self._ln2.bias, f1_w=self._out[0].weight,
                           f1_b=self._out[0].bias, f2_w=self._out[2].weight, f2_b=self._out[2].bias)


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


# one block's views of the `GradArena`, in the order they lie in it (shapes: `GradArena._shapes`); the LayerNorm
# statistics are dgamma, dbeta and the column sums of the gradient that LayerNorm's backward writes
BlockGradViews = NamedTuple("BlockGradViews", [(name, torch.Tensor) for name in (
    "dw2", "dw1", "dwp", "dwqkv", "ln1_stats", "ln2_stats", "dbqkv", "db1")])


class GradArena:
    """The one zero-filled fp32 buffer behind every per-block gradient of the stack, in packed layout (`StreamLayout`,
    `HeadLayout`): a single memset instead of eight per block.  The four weight matrices of block 0, of block 1, ...
    come first (the wgrad GEMMs accumulate into them with TMA reduce-adds), so the matrices of consecutive blocks are
    one contiguous slice (`bucket`), which data parallelism averages in place.  The small gradients of every block
    follow: LayerNorm dgamma / dbeta / column sums and the bias gradients of the qkv and fc1 layers, which their kernels
    accumulate with atomics."""

    def __init__(self, n_blocks, sl, lay, device):
        self.n_blocks = n_blocks
        self._mats, self._vecs = self._shapes(sl, lay)
        self._per_block, self._per_small = (sum(math.prod(s) for s in shapes) for shapes in (self._mats, self._vecs))
        self.buf = torch.zeros(self.numel(n_blocks, sl, lay), dtype=F32, device=device)
        # True when every weight gradient of a block is a plain view of `buf` (heads fill their kernel slots, e.g. 512
        # channels / 8 or 4 heads, and the stream needs no pad columns): only then can a bucket be averaged in place
        self.views_are_grads = n_blocks > 0 and sl.identity and lay.identity
        # transformer blocks per all-reduce; 0 = the whole stack in one bucket, issued when block 0's last wgrad is
        # queued (overlaps the input convolution's backward and the small-gradient bucket only).  Finer buckets overlap
        # more, but every NCCL kernel that runs next to the GEMMs competes with them for SMs.
        bucket_blocks = int(os.environ.get("PG_DP_BUCKET_BLOCKS", "0"))
        self.bucket_blocks = bucket_blocks if bucket_blocks > 0 else n_blocks

    @staticmethod
    def _shapes(sl, lay):
        """(the four matrices' shapes, the four small gradients' shapes) of one block, in `BlockGradViews` order."""
        H, (C, c_p, f_p) = lay.n_heads, sl
        qkv_rows = H * (2 * lay.qk_slot + lay.dv_slot)
        return ((c_p, f_p), (f_p, c_p), (c_p, H * lay.dv_slot), (qkv_rows, c_p)), ((3, C), (3, C), (qkv_rows,), (f_p,))

    @classmethod
    def numel(cls, n_blocks, sl, lay):
        """Elements of the buffer; pure (no device)."""
        return n_blocks * sum(math.prod(s) for shapes in cls._shapes(sl, lay) for s in shapes)

    def block(self, b):
        views = []
        for start, shapes in ((b * self._per_block, self._mats),
                              (self.n_blocks * self._per_block + b * self._per_small, self._vecs)):
            for shape in shapes:
                views.append(self.buf[start: start + math.prod(shape)].view(shape))
                start += math.prod(shape)
        return BlockGradViews(*views)

    def bucket(self, lo, hi):
        """The weight matrices of blocks lo .. hi - 1: one contiguous slice."""
        return self.buf[lo * self._per_block: hi * self._per_block]


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
    # fp32 weight gradients: 4 * GradArena.numel when the stream needs no pad columns; with pad columns this counts 4C
    # where the arena has round_up(4 * true C, 8), and C = c_p small gradients where it has true C: a little over
    arena = 4 * n_blocks * (8 * C * C + C * o_cols + qkv_cols * C + 10 * C + qkv_cols)
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
    """One transformer block on the fp32 stream xs [P, C]; p = its BlockParams, pk = its packed weights.  Returns
    (next stream, every activation the block's backward reads).  Given attn = (o, lse) of an earlier forward, it rebuilds
    those activations for the backward instead, without the attention forward or fc2 (next stream None): the same
    kernels on the same inputs in the same order, so the same bits as the forward's."""
    lay = pk["layout"]
    dv_slot, slot = lay.dv_slot, lay.qk_slot
    a1, _, mean1, rstd1 = ops.layernorm_fwd(xs, p.ln1_w.detach(), p.ln1_b.detach(), eps)
    qkv, _, _ = ops.linear_fwd(a1, pk["wqkv"], pk["bqkv"])
    if attn is None:
        q, k, v = qkv[:, : H * slot], qkv[:, H * slot: 2 * H * slot], qkv[:, 2 * H * slot:]
        o, lse = ops.attn_fwd(q, k, v, n, S, H, lay.dk, slot, dv_slot, False)
    else:
        o, lse = attn
    _, _, hres = ops.linear_fwd(o, pk["wp"], pk["bp"], res0=xs, want_bf16=False, want_f32=True)
    a2, _, mean2, rstd2 = ops.layernorm_fwd(hres, p.ln2_w.detach(), p.ln2_b.detach(), eps)
    g, u, _ = ops.linear_fwd(a2, pk["w1"], pk["b1"], act=L.ACT_GELU, want_pre=True, pre_deriv=True)  # u = GELU'(pre)
    acts = dict(xs=xs, a1=a1, qkv=qkv, o=o, lse=lse, h=hres, a2=a2, u=u, g=g, mean1=mean1, rstd1=rstd1, mean2=mean2,
                rstd2=rstd2, **{k: pk[k] for k in _WEIGHTS})
    if attn is not None:
        return None, acts
    _, _, xs_new = ops.linear_fwd(g, pk["w2"], pk["b2"], res0=xs, res1=hres, want_bf16=False, want_f32=True)
    return xs_new, acts


def _block_bwd(blk, p, g, sl, dx, dx_b, dx_sum, n, S, H):
    """Backward of `_block_fwd`.  blk = the block's activations and packed weights, p = its BlockParams, g = its
    BlockGradViews; dx (fp32), dx_b (bf16) = the gradient of the block's output stream and dx_sum its column sums.
    Returns (the parameters' gradients as BlockParams, then the same three for the block's input stream).  Every
    LayerNorm backward also emits the column sums of the gradient it writes = the bias gradient of the linear layer that
    produced its input (fc2 of the block above / the attention projection)."""
    lay = blk["layout"]
    dv_slot, slot, C = lay.dv_slot, lay.qk_slot, sl.c
    # x_new = x + h + fc2(gelu(fc1(ln2(h))))
    ops.linear_wgrad(dx_b, blk["g"], g.dw2)
    df2_w = sl.unpack(g.dw2, p.f2_w.shape)
    du = ops.linear_dgrad(dx_b, blk["w2"], aux=blk["u"], dact=L.ACT_GIVEN)
    # the bias gradient (column sums of du) is reduced by the wgrad launch from the du tiles it stages
    ops.linear_wgrad(du, blk["a2"], g.dw1, db_out=g.db1)
    df1_w, df1_b = sl.unpack(g.dw1, p.f1_w.shape), sl.unpack(g.db1, (4 * C,))
    da2 = ops.linear_dgrad(du, blk["w1"])
    del du
    # h receives: LN2 path + direct (x_new = ... + h)
    dh, dh_b, dln2_w, dln2_b, dp_b = ops.layernorm_bwd(da2, blk["h"], p.ln2_w.detach(), blk["mean2"], blk["rstd2"],
                                                       dres0=dx, want_colsum=True, stats=g.ln2_stats)
    del da2
    # h = x + proj(attn)
    ops.linear_wgrad(dh_b, blk["o"], g.dwp)
    do = ops.linear_dgrad(dh_b, blk["wp"])
    qkv = blk["qkv"]
    q, k, v = qkv[:, : H * slot], qkv[:, H * slot: 2 * H * slot], qkv[:, 2 * H * slot:]
    dqkv = torch.empty_like(qkv)
    ops.attn_bwd(q, k, v, blk["o"], do, blk["lse"], dqkv[:, : H * slot], dqkv[:, H * slot: 2 * H * slot],
                 dqkv[:, 2 * H * slot:], n, S, H, lay.dk, slot, dv_slot, False)
    del do
    ops.linear_wgrad(dqkv, blk["a1"], g.dwqkv, db_out=g.dbqkv)
    # views of the arena when heads fill their slots
    dq_w, dq_b, dkv_w, dkv_b, dp_w = lay.unpack_grads(g.dwqkv[: H * slot], g.dbqkv[: H * slot], g.dwqkv[H * slot:],
                                                      g.dbqkv[H * slot:], g.dwp, C, C)
    da1 = ops.linear_dgrad(dqkv, blk["wqkv"])
    del dqkv
    # x receives: LN1 path + direct from h (dh) + direct from x_new (dx)
    dx_in, dx_in_b, dln1_w, dln1_b, dx_in_sum = ops.layernorm_bwd(
        da1, blk["xs"], p.ln1_w.detach(), blk["mean1"], blk["rstd1"], dres0=dx, dres1=dh, want_colsum=True,
        stats=g.ln1_stats)
    grads = BlockParams(ln1_w=dln1_w, ln1_b=dln1_b, q_w=dq_w, q_b=dq_b, kv_w=dkv_w, kv_b=dkv_b, p_w=dp_w, p_b=dp_b,
                        ln2_w=dln2_w, ln2_b=dln2_b, f1_w=df1_w, f1_b=df1_b, f2_w=df2_w, f2_b=dx_sum)
    return grads, dx_in, dx_in_b, dx_in_sum


class _ImageGPTStack(torch.autograd.Function):
    """forward(x_nchw, params...) -> logits_nchw; one node for the whole network."""

    @staticmethod
    def forward(ctx, x, n_heads, eps, packed, opts, *params):
        split = _split_params(params)
        (pos, in_w, in_b), blocks, (ln_w, ln_b, out_w, out_b) = split
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
        for p, pk in zip(blocks, packed["blocks"]):
            xs_new, acts = _block_fwd(xs, p, pk, n, S, H, eps)
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
                             in_w=packed["in_w"], sl=packed["stream"], lay=packed["layout"], params=split,
                             dims=(n, cin, h, w, C, H, cout), eps=eps, hook=opts.get("hook"), recompute=recompute)
        return ops.pm_to_nchw(logits_pm, n, cout, h, w)

    @staticmethod
    def backward(ctx, dlogits):
        sv = getattr(ctx, "saved", None)
        if sv is None:
            raise RuntimeError("ImageGPT: the activations of this forward were already consumed by a backward pass "
                               "(retain_graph is not supported by the fused stack)")
        (pos, in_w, _), blocks, (ln_w, _, _, _) = sv["params"]
        n, cin, h, w, C, H, cout = sv["dims"]
        S = h * w
        dev = dlogits.device
        n_blocks = len(blocks)
        sl = sv["sl"]

        # head: logits = 1x1(LN(x))
        dl = ops.nchw_to_pm(dlogits, BF16, width=ops.round_up(cout, 8))
        dout_b = ops.bias_grad(dl[:, :cout])
        dwo = torch.zeros(ops.round_up(cout, 8), sl.c_p, dtype=F32, device=dev)
        ops.linear_wgrad(dl, sv["af"], dwo)
        dout_w = dwo[:cout, :C].reshape(cout, C, 1, 1)
        daf = ops.linear_dgrad(dl[:, :cout], sv["wo"])
        dx, dx_b, dln_w, dln_b, dx_sum = ops.layernorm_bwd(daf, sv["xs_final"], ln_w.detach(), sv["mean_f"],
                                                           sv["rstd_f"], want_colsum=True)
        del daf
        head_grads = (dln_w, dln_b, dout_w, dout_b)

        arena = GradArena(n_blocks, sl, sv["lay"], dev)
        # data parallelism: each bucket of the arena is handed to the bucket hook (an asynchronous all-reduce) as soon
        # as the last wgrad GEMM of its blocks is queued; see parallel.OverlappedGradAverager
        bucket_hook = sv["hook"] if arena.views_are_grads else None
        pending = []
        block_grads = [None] * n_blocks
        for b in reversed(range(n_blocks)):
            blk = sv["blocks"][b]
            if sv["recompute"]:  # rebuild what the forward did not keep, from what it did
                _, blk = _block_fwd(blk["xs"], blocks[b], blk, n, S, H, sv["eps"], attn=(blk["o"], blk["lse"]))
            block_grads[b], dx, dx_b, dx_sum = _block_bwd(blk, blocks[b], arena.block(b), sl, dx, dx_b, dx_sum, n, S, H)
            if bucket_hook is not None and b % arena.bucket_blocks == 0:  # this bucket's blocks are complete
                pending.append(bucket_hook(arena.bucket(b, min(b + arena.bucket_blocks, n_blocks))))
            sv["blocks"][b] = None  # release this block's activations
            del blk  # (rebuilt ones too) before the next block rebuilds its own

        dw_in = torch.zeros_like(sv["in_w"])
        dx_in = torch.empty(n, cin, h, w, dtype=F32, device=dev)
        L.conv_small_bwd(sv["x_in"], sv["in_w"], dx, (in_w.shape[2] // 2, in_w.shape[3] // 2), dw=dw_in, dbias=None,
                         dx=dx_in)
        din_w = sl.unpack(dw_in.view(dw_in.shape[0], -1), in_w.shape)
        dpos = torch.zeros_like(pos)
        dpos[:, :, : h, : w] = dx_in.sum(dim=0, keepdim=True)
        stem_grads = (dpos, din_w, dx_sum)  # the input conv's bias gradient = column sums of the stream gradient
        ctx.saved = None
        for handle in pending:  # the gradients leave this node averaged
            handle.wait()
        return (dx_in if ctx.needs_input_grad[0] else None, None, None, None, None, *stem_grads,
                *(g for grads in block_grads for g in grads), *head_grads)


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
        packed = {"blocks": [], "stream": sl, "layout": lay,
                  "in_w": sl.pack(in_w, c_p, in_w[0].numel()).view(c_p, *in_w.shape[1:]),
                  "in_b": sl.pack(self._input.bias, c_p)}

        def biases_of(blk):  # the projection and MLP biases, padded
            return dict(bp=sl.pack(blk._attn._proj.bias, c_p), b1=sl.pack(blk._out[0].bias, f_p),
                        b2=sl.pack(blk._out[2].bias, c_p))

        if lay.identity and blocks:
            per_block = 12 * C * C
            arena = torch.empty(len(blocks) * per_block + cout * C, dtype=BF16, device=dev)

            def views_of(b):  # (wqkv, wp, w1, w2) of block b, adjacent in that order; q | kv rows adjacent in wqkv
                views, start = [], b * per_block
                for rows, cols in ((3 * C, C), (C, C), (4 * C, C), (C, 4 * C)):
                    views.append(arena[start: start + rows * cols].view(rows, cols))
                    start += rows * cols
                return views

            views = [views_of(b) for b in range(len(blocks))]
            wo = arena[len(blocks) * per_block:].view(cout, C)
            dsts = [d for wqkv, wp, w1, w2 in views for d in (wqkv[:C], wqkv[C:], wp, w1, w2)] + [wo]
            plan = self.__dict__.get("_cast_plan")
            if plan is None or plan["src_key"] != tuple(p.data_ptr() for p in mats):
                from .. import optim

                numel, chunks, n_chunks = optim.chunk_table([p.numel() for p in mats], dev)
                plan = dict(src_key=tuple(p.data_ptr() for p in mats), n_chunks=n_chunks, chunk=optim.CHUNK,
                            numel=numel, chunks=chunks,
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
