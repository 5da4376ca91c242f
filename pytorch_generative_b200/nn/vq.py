"""VectorQuantizer on the CUDA path — API of reference nn/utils.py `VectorQuantizer`.

Same constructor, buffers (`_embedding`, `_cluster_size`, `_embedding_avg` with EMA) or Parameter (`_embedding`
without), state-dict keys and init bits under a seed as the reference, so checkpoints interchange.

One autograd Function carries the quantizer over pixel-major rows ([P, d] fp32, the reference's flat_x):
  * `pg_vq_assign` picks each row's nearest code in fp32 on the CUDA cores (the first minimal index on ties, as
    torch.argmin), writes the straight-through value x + (q - x) as its consumer's operand (bf16 for a decoder, at a
    column offset when the operand is a concatenation) and adds up sum (x - q)^2 in a fixed order on the device;
  * in training with EMA, `pg_vq_code_sums` and `pg_vq_ema_update` update the three buffers in place after the loss
    has used the old codebook, and their version counters are bumped (no host synchronisation anywhere, so a training
    step captures as a CUDA graph);
  * the backward is one `pg_vq_bwd` launch (dx = dq + g 2 (x - q) / numel) and, without EMA, the codebook gradient
    `pg_vq_code_sums` of g 2 (q - x) / numel.
"""

import torch
from torch import nn
from torch.nn import init

from .. import _lib as L
from .. import ops
from . import pm

F32, BF16 = torch.float32, torch.bfloat16


class _Quantize(torch.autograd.Function):
    """(z_grad, z [P, >=d] fp32, embedding, left) -> (out [P, width], loss).  out holds `left` (if any) in its first
    columns, then x + (q - x) in d columns and zeros up to `width`.  z carries the values and is passed detached; the
    gradient of z leaves through `z_grad` in its dtype (the bf16 copy a convolution's epilogue wrote beside z, whose
    backward reads a bf16 operand anyway, or z itself)."""

    @staticmethod
    def forward(ctx, z_grad, z, embedding, left, vq, width, out_dtype):
        P = z.shape[0]
        d, K = vq.embedding_dim, vq.n_embeddings
        c0 = 0 if left is None else left.shape[1]
        out = torch.empty(P, width, dtype=out_dtype, device=z.device)
        if left is not None:
            out[:, :c0].copy_(left)
        idx = torch.empty(P, dtype=torch.int32, device=z.device)
        acc = torch.zeros(1, dtype=F32, device=z.device)
        emb = embedding.detach()
        L.vq_assign(z, emb, idx, out, c0, width - c0, acc)
        numel = P * d
        loss = (acc / numel).reshape(())
        if vq._use_ema and vq.training:
            emb = emb.clone()  # the backward's q is the codebook the loss used
            counts = torch.empty(K, dtype=F32, device=z.device)
            sums = torch.empty(K, d, dtype=F32, device=z.device)
            L.vq_code_sums(z, idx, K, sums, counts)
            L.vq_ema_update(counts, sums, vq._decay, vq._cluster_size, vq._embedding_avg, vq._embedding)
            # written behind autograd's back: every version-keyed cache and saved-tensor check must see it
            torch.autograd.graph.increment_version([vq._cluster_size, vq._embedding_avg, vq._embedding])
        elif not vq._use_ema:
            loss = loss + loss  # the reference adds mse(q, x), equal in value, whose gradient reaches the codebook
        ctx.save_for_backward(z, emb, idx)
        ctx.meta = (c0, numel, K, z_grad.shape[1], z_grad.dtype)
        ctx.set_materialize_grads(False)
        return out, loss

    @staticmethod
    def backward(ctx, dout, dloss):
        z, emb, idx = ctx.saved_tensors
        c0, numel, K, zw, z_dtype = ctx.meta
        d = emb.shape[1]
        g = None if dloss is None else dloss.reshape(1).float().contiguous()
        dz = demb = dleft = None
        if ctx.needs_input_grad[0]:
            width = ops.round_up(d, 8) if z_dtype == BF16 else zw  # a bf16 operand keeps the 16-byte pitch
            dx = torch.empty(z.shape[0], width, dtype=z_dtype, device=z.device)
            dq = None if dout is None else dout.to(z_dtype).contiguous()
            L.vq_bwd(z, emb, idx, dq, c0, g, 2.0 / numel, dx)
            dz = dx if width == zw else dx[:, :zw]
        if ctx.needs_input_grad[2] and g is not None:
            demb = torch.empty(K, d, dtype=F32, device=z.device)
            L.vq_code_sums(z, idx, K, demb, emb=emb, g=g, scale=2.0 / numel)
        if ctx.needs_input_grad[3] and dout is not None:
            dleft = dout[:, :c0]
        return dz, None, demb, dleft, None, None, None


class VectorQuantizer(nn.Module):
    """A vector quantizer (reference nn/utils.py VectorQuantizer): inputs are quantized to the nearest embedding in
    Euclidean distance; the embeddings are updated by exponential moving averages (use_ema) or by gradient descent."""

    def __init__(self, n_embeddings, embedding_dim, use_ema=True, ema_decay=0.99):
        super().__init__()
        self.n_embeddings = n_embeddings
        self.embedding_dim = embedding_dim
        self._use_ema = use_ema
        self._decay = ema_decay

        embedding = torch.zeros(n_embeddings, embedding_dim)
        init.kaiming_uniform_(embedding, nonlinearity="linear")
        if self._use_ema:
            self.register_buffer("_embedding", embedding)
            self.register_buffer("_cluster_size", torch.zeros(n_embeddings))
            self.register_buffer("_embedding_avg", embedding.clone())
        else:
            self._embedding = nn.Parameter(embedding)

    def _check(self, z):
        if not z.is_cuda:
            raise RuntimeError(f"VectorQuantizer: the CUDA path runs on CUDA tensors only (no CPU fallback); got {z.device}")
        for name in ("_embedding", "_cluster_size", "_embedding_avg"):
            t = getattr(self, name, None)
            if t is not None and (t.dtype != F32 or not t.is_cuda or not t.is_contiguous()):
                raise RuntimeError(f"VectorQuantizer: the CUDA path needs a contiguous fp32 CUDA {name}; got {t.dtype} on "
                                   f"{t.device}")
        if z.dtype != F32:
            raise RuntimeError(f"VectorQuantizer: the CUDA path takes fp32 inputs; got {z.dtype}")

    def _pm(self, z_grad, z, width, left=None, out_dtype=BF16):
        """Pixel-major entry: z fp32 [P, >=d] (values; detached), z_grad the tensor its gradient leaves through.
        Returns (out [P, width] in out_dtype: `left`'s columns, then x + (q - x), zeros to `width`; the loss)."""
        self._check(z)
        return _Quantize.apply(z_grad, z, self._embedding, left, self, width, out_dtype)

    def forward(self, x):
        """(x + (q - x), loss) on NCHW fp32, as the reference's module."""
        n, c, h, w = x.shape
        assert c == self.embedding_dim, "Input channels must equal embedding_dim."
        self._check(x)
        z = pm.to_pm(x, F32)
        q, loss = self._pm(z, z.detach(), c, out_dtype=F32)
        return pm.from_pm(q, pm.Geom(n, h, w), c), loss
