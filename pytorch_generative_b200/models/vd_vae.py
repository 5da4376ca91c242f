"""VeryDeepVAE on the CUDA path — API of reference models/vae/vd_vae.py (`StackConfig`, `DEFAULT_MODEL`,
`BottleneckBlock`, `TopDownBlock`, `EncoderStack`, `DecoderStack`, `VeryDeepVAE`, `reproduce`).

Same constructors, module tree, state-dict keys, parameter order and init bits under a seed as the reference, so
checkpoints interchange; that includes the reference's decoder kernel size (every DecoderStack gets the encoder loop's
last `bottleneck_kernel_size`, see DESIGN §2).  `VeryDeepVAE.forward(x)` returns `(logits [n, out, H, W] fp32, kl [n])`.

Activations stay pixel-major ([N*H*W, C] matrices, fp32 streams) from `_input` (`pm.image_conv`) to the logits:
  * a BottleneckBlock is four `pm.conv` calls with GELU inputs.  GELU's derivative does not follow from its output, so
    each GELU operand travels with its bf16 derivative (`pm.GeluOperand`): the three inner convolutions emit GELU and
    GELU' from their epilogues (PRE_GRAD), and each dgrad multiplies by the stored derivative (ACT_GIVEN);
  * a residual block's last convolution adds the stream in its epilogue and, when the next block follows in the same
    stack, also emits the next block's GeluOperand; so does each `_latents` convolution for its `_out` block;
  * `pg_gelu_cast` makes the GeluOperands no epilogue produces: the input of each stack's first block (after `_input`,
    a pooling or a bias / unpool) and the posterior's operand [GELU(x) | GELU(mixin)], whose mixin half is computed
    once per decoder stack and whose x half is written in place of each block's copy;
  * the prior and posterior write fp32 outputs (the latent kernel's values) and bf16 copies through which their
    gradients return as the GEMM operands of their backward: `pg_vd_latent_bwd` writes [dp_mean | dp_log_std |
    bf16(dsum)] and [dq_mean | dq_log_std] directly;
  * `pg_vd_latent_fwd` also writes s = x + p_h (the reference's order), which the `_latents` epilogue adds as one fp32
    residual: the GEMM epilogue's two residuals share one pitch, and p_h is a column view of the prior's output
    (pitch 2L + C);
  * pooling and bias + unpooling are `pg_avg_pool2_*` and `pg_bias_unpool_*`.
The forward and backward never synchronise with the host, so a training step captures as a CUDA graph.
"""

import math
from dataclasses import dataclass

import torch
from torch import nn

from .. import _lib as L
from .. import ops
from ..nn import pm
from . import base

BF16, F32 = torch.bfloat16, torch.float32
GELU = L.ACT_GELU


@dataclass
class StackConfig:
    """Encoder and decoder blocks at one resolution (reference vd_vae.py StackConfig)."""

    n_encoder_blocks: int
    n_decoder_blocks: int


DEFAULT_MODEL = [StackConfig(n_encoder_blocks=1, n_decoder_blocks=1) for _ in range(6)]


def draw_noise(shape, device):
    """A TopDownBlock's reparameterisation noise: one torch.randn of the latent's NCHW shape (the reference's
    randn_like), drawn once per block in decoder order."""
    return torch.randn(shape, device=device)


def _require(x, module, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")
    for p in module.parameters():
        if p.dtype != F32 or not p.is_cuda or not p.is_contiguous():
            raise RuntimeError(f"{who}: the CUDA path needs contiguous fp32 CUDA parameters; got {p.dtype} on {p.device}")
    if x.dtype != F32:
        raise RuntimeError(f"{who}: the CUDA path takes fp32 inputs; got {x.dtype}")


class BottleneckBlock(nn.Module):
    """GELU, 1x1, GELU, kxk, GELU, kxk, GELU, 1x1 (+ x when residual) (reference vd_vae.py BottleneckBlock)."""

    def __init__(self, in_channels, out_channels, bottleneck_channels, bottleneck_kernel_size=3, is_residual=True):
        super().__init__()
        self._is_residual = is_residual
        padding = 1 if bottleneck_kernel_size == 3 else 0
        self._net = nn.Sequential(
            nn.GELU(),
            nn.Conv2d(in_channels=in_channels, out_channels=bottleneck_channels, kernel_size=1),
            nn.GELU(),
            nn.Conv2d(in_channels=bottleneck_channels, out_channels=bottleneck_channels,
                      kernel_size=bottleneck_kernel_size, padding=padding),
            nn.GELU(),
            nn.Conv2d(in_channels=bottleneck_channels, out_channels=bottleneck_channels,
                      kernel_size=bottleneck_kernel_size, padding=padding),
            nn.GELU(),
            nn.Conv2d(in_channels=bottleneck_channels, out_channels=out_channels, kernel_size=1),
        )

    def _pm(self, x, geom, xa=None, emit=None, emit_mode=pm.COMPANION):
        """x: the block's input before its GELU (an fp32 stream [P, Cin]); xa: its GeluOperand, or None to build one.
        Returns (y fp32 [P, Cout], ya) with ya what the last convolution's epilogue emits (`pm.conv`)."""
        convs = self._net[1::2]
        h, ha = x, xa
        for conv in convs[:-1]:
            _, ha = pm.conv(h, conv.weight, conv.bias, geom, conv.padding, in_act=GELU, xa=ha, emit=GELU,
                            emit_mode=pm.PRE_GRAD, want_main=False)
            h = ha.a
        last = convs[-1]
        return pm.conv(h, last.weight, last.bias, geom, in_act=GELU, xa=ha, res=x if self._is_residual else None,
                       out_f32=True, emit=emit, emit_mode=emit_mode)

    def forward(self, x):
        raise NotImplementedError("BottleneckBlock runs inside VeryDeepVAE on the CUDA path (its pixel-major stream); "
                                  "call the model")


class _CatGrad(torch.autograd.Function):
    """Stands for cat(x, mixin) [P, width] in the graph without materialising it: the posterior's operand is written
    by pg_gelu_cast, and this node hands the two halves of its input gradient back to x and mixin."""

    @staticmethod
    def forward(ctx, x, mixin, width):
        ctx.c = x.shape[1]
        return x.new_zeros(()).expand(x.shape[0], width)

    @staticmethod
    def backward(ctx, d):
        c = ctx.c
        return d[:, :c], d[:, c:2 * c], None


class _Latent(torch.autograd.Function):
    """A TopDownBlock's latent (pg_vd_latent_fwd / _bwd).  prior_b / post_b: the bf16 copies of the prior's and the
    posterior's outputs, through which their gradients leave as the bf16 operands of those convolutions' backward;
    prior / post: the fp32 values (detached); post None samples from the prior.  Returns (z bf16 [P, round_up(L, 8)],
    s = x + p_h fp32 [P, C], kl_in + KL [n] or None)."""

    @staticmethod
    def forward(ctx, prior_b, post_b, x, prior, post, eps, kl_in, L_):
        P, C = x.shape
        z = torch.empty(P, ops.round_up(L_, 8), dtype=BF16, device=x.device)
        s = torch.empty(P, C, dtype=F32, device=x.device)
        kl = None if post is None else torch.empty(eps.shape[0], dtype=F32, device=x.device)
        L.vd_latent_fwd(prior, post, x.detach(), eps, z, s, None if kl_in is None else kl_in.detach(), kl)
        ctx.save_for_backward(prior, post, eps)
        ctx.dims = (L_, C, kl_in is not None)
        ctx.set_materialize_grads(False)
        return z, s, kl

    @staticmethod
    def backward(ctx, dz, ds, dkl):
        prior, post, eps = ctx.saved_tensors
        L_, C, has_kl_in = ctx.dims
        P = prior.shape[0]
        if ds is None:
            ds = torch.zeros(P, C, dtype=F32, device=prior.device)
        dprior = torch.empty(P, ops.round_up(2 * L_ + C, 8), dtype=BF16, device=prior.device)
        dpost = None if post is None else torch.empty(P, ops.round_up(2 * L_, 8), dtype=BF16, device=prior.device)
        L.vd_latent_bwd(prior, post, eps, None if dz is None else dz.contiguous(),
                        None if dkl is None else dkl.contiguous(), ds.contiguous(), dprior, dpost)
        return (dprior[:, : 2 * L_ + C], None if dpost is None else dpost[:, : 2 * L_], ds, None, None, None,
                dkl if has_kl_in else None, None)


class TopDownBlock(nn.Module):
    """Prior, posterior, latent projection and a residual BottleneckBlock (reference vd_vae.py TopDownBlock)."""

    def __init__(self, n_channels, latent_channels, bottleneck_channels, bottleneck_kernel_size):
        super().__init__()
        self._n_channels = n_channels
        self._latent_channels = latent_channels
        self._prior = BottleneckBlock(in_channels=self._n_channels,
                                      out_channels=2 * self._latent_channels + self._n_channels,
                                      bottleneck_channels=bottleneck_channels, is_residual=False)
        self._posterior = BottleneckBlock(in_channels=2 * self._n_channels, out_channels=2 * self._latent_channels,
                                          bottleneck_channels=bottleneck_channels, is_residual=False)
        self._latents = nn.Conv2d(in_channels=self._latent_channels, out_channels=self._n_channels, kernel_size=1)
        self._out = BottleneckBlock(in_channels=self._n_channels, out_channels=self._n_channels,
                                    bottleneck_channels=bottleneck_channels,
                                    bottleneck_kernel_size=bottleneck_kernel_size, is_residual=True)

    def _pm(self, x, xa, geom, mixin, mixin_op, kl, emit):
        """x: the stream [P, C] fp32, xa its GeluOperand or None; mixin: the encoder features at this resolution and
        mixin_op the posterior's operand with GELU(mixin) in columns [C, 2C), or both None to sample from the prior.
        Returns (stream, its GeluOperand or bf16 copy per `emit`, kl)."""
        C, L_ = self._n_channels, self._latent_channels
        prior, prior_b = self._prior._pm(x, geom, xa, emit=L.ACT_NONE, emit_mode=pm.POST)
        post = post_b = None
        if mixin is not None:
            op = pm.GeluOperand(mixin_op.a.clone(), mixin_op.d.clone())
            L.gelu_cast(x.detach(), op.a[:, :C], op.d[:, :C])
            cat = _CatGrad.apply(x, mixin, op.a.shape[1])
            post, post_b = self._posterior._pm(cat, geom, op, emit=L.ACT_NONE, emit_mode=pm.POST)
            post = post.detach()
        eps = draw_noise((geom.n, L_, geom.h, geom.w), x.device)
        z, s, kl = _Latent.apply(prior_b, post_b, x, prior.detach(), post, eps, kl, L_)
        lat = self._latents
        y, ya = pm.conv(z, lat.weight, lat.bias, geom, res=s, out_f32=True, emit=GELU)
        y, ya = self._out._pm(y, geom, ya, emit)
        return y, ya, kl

    def forward(self, x, mixin=None):
        raise NotImplementedError("TopDownBlock runs inside VeryDeepVAE on the CUDA path (its pixel-major stream); "
                                  "call the model")


class EncoderStack(nn.Module):
    """Residual BottleneckBlocks, then 2x2 average pooling unless last (reference vd_vae.py EncoderStack)."""

    def __init__(self, n_residual_blocks, pool, n_channels, bottleneck_channels, bottleneck_kernel_size):
        super().__init__()
        residuals = [BottleneckBlock(in_channels=n_channels, out_channels=n_channels,
                                     bottleneck_channels=bottleneck_channels,
                                     bottleneck_kernel_size=bottleneck_kernel_size, is_residual=True)
                     for _ in range(n_residual_blocks)]
        self._residuals = nn.Sequential(*residuals)
        self._pool = nn.AvgPool2d(kernel_size=2, stride=2) if pool else None

    def forward(self, x):
        raise NotImplementedError("EncoderStack runs inside VeryDeepVAE on the CUDA path (its pixel-major stream); "
                                  "call the model")


class DecoderStack(nn.Module):
    """Nearest-neighbour unpooling unless first, then TopDownBlocks (reference vd_vae.py DecoderStack)."""

    def __init__(self, n_topdown_blocks, unpool, n_channels, latent_channels, bottleneck_channels,
                 bottleneck_kernel_size):
        super().__init__()
        self._unpool = nn.Upsample(scale_factor=2, mode="nearest") if unpool else None
        topdowns = [TopDownBlock(n_channels, latent_channels, bottleneck_channels, bottleneck_kernel_size)
                    for _ in range(n_topdown_blocks)]
        self._topdowns = nn.ModuleList(topdowns)

    def forward(self, x, mixin=None):
        raise NotImplementedError("DecoderStack runs inside VeryDeepVAE on the CUDA path (its pixel-major stream); "
                                  "call the model")


class _Pool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, geom):
        y = torch.empty(geom.n * (geom.h // 2) * (geom.w // 2), x.shape[1], dtype=F32, device=x.device)
        L.avg_pool2_fwd(x, geom.n, geom.h, geom.w, y)
        ctx.geom = geom
        return y

    @staticmethod
    def backward(ctx, dy):
        g = ctx.geom
        dx = torch.empty(g.n * g.h * g.w, dy.shape[1], dtype=F32, device=dy.device)
        L.avg_pool2_bwd(dy.contiguous(), g.n, g.h, g.w, dx)
        return dx, None


class _BiasUnpool(torch.autograd.Function):
    """up_f(x + bias) of the decoder stream (x None: the zeros the decoder starts from)."""

    @staticmethod
    def forward(ctx, x, bias, n, f):
        _, C, s, _ = bias.shape
        y = torch.empty(n * s * s * f * f, C, dtype=F32, device=bias.device)
        L.bias_unpool_fwd(None if x is None else x.detach(), bias.detach(), n, f, y)
        ctx.dims = (n, f, x is not None)
        ctx.bias_shape = bias.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        n, f, has_x = ctx.dims
        _, C, s, _ = ctx.bias_shape
        dx = torch.empty(n * s * s, C, dtype=F32, device=dy.device) if has_x and ctx.needs_input_grad[0] else None
        dbias = torch.empty(ctx.bias_shape, dtype=F32, device=dy.device)
        L.bias_unpool_bwd(dy.contiguous(), n, f, dx, dbias)
        return dx, dbias, None, None


class VeryDeepVAE(base.VariationalAutoEncoder):
    """The Very Deep VAE (reference vd_vae.py VeryDeepVAE)."""

    def __init__(self, in_channels=1, out_channels=1, input_resolution=32, stack_configs=DEFAULT_MODEL,
                 latent_channels=4, hidden_channels=16, bottleneck_channels=8, sample_fn=None):
        super().__init__(sample_fn)
        self._input = nn.Conv2d(in_channels, out_channels=hidden_channels, kernel_size=3, padding=1)
        self._encoder = nn.ModuleList()
        resolutions = [input_resolution // 2**i for i in range(len(stack_configs))]
        self._resolutions = resolutions
        encoder_blocks = [conf.n_encoder_blocks for conf in stack_configs]
        total_encoder_blocks = sum(encoder_blocks)
        for i, (res, n_blocks) in enumerate(zip(resolutions, encoder_blocks)):
            pool = i < len(stack_configs) - 1
            bottleneck_kernel_size = 3 if res >= 3 else 1
            stack = EncoderStack(n_residual_blocks=n_blocks, pool=pool, n_channels=hidden_channels,
                                 bottleneck_channels=bottleneck_channels, bottleneck_kernel_size=bottleneck_kernel_size)
            for block in stack._residuals:
                block._net[-1].weight.data /= math.sqrt(total_encoder_blocks)
            self._encoder.append(stack)

        biases = [nn.Parameter(torch.zeros(1, hidden_channels, size, size))
                  for size in resolutions[1:] + [resolutions[-1]]]
        self._biases = nn.ParameterList(biases)

        self._decoder = nn.ModuleList()
        decoder_blocks = [conf.n_decoder_blocks for conf in stack_configs]
        total_decoder_blocks = sum(decoder_blocks)
        for i, (res, n_blocks) in enumerate(zip(reversed(resolutions), reversed(decoder_blocks))):
            # As in the reference: the kernel size computed here is never used; every DecoderStack gets the encoder
            # loop's last `bottleneck_kernel_size` (DESIGN §2).
            stack = DecoderStack(n_topdown_blocks=n_blocks, unpool=i > 0, n_channels=hidden_channels,
                                 latent_channels=latent_channels, bottleneck_channels=bottleneck_channels,
                                 bottleneck_kernel_size=bottleneck_kernel_size)
            for block in stack._topdowns:
                block._out._net[-1].weight.data /= math.sqrt(total_decoder_blocks)
                block._latents.weight.data /= math.sqrt(total_decoder_blocks)
            self._decoder.append(stack)
        self._output = nn.Conv2d(in_channels=hidden_channels, out_channels=out_channels, kernel_size=1)

    def _check_resolutions(self):
        """Raises before any launch on the shapes the reference cannot run: each pooled side must be even, so that
        unpooling restores it, and the last side at least 1."""
        res = self._resolutions
        if res[-1] < 1 or any(r % 2 for r in res[:-1]):
            raise ValueError(f"VeryDeepVAE: stack resolutions {res} cannot run: every pooled side must be even (its "
                             f"unpooled decoder stream must match the encoder's) and the last at least 1")

    def _decode(self, n, mixins, device):
        """The decoder stream from the biases: (fp32 stream [n*R*R, C], its geometry, kl [n] or None)."""
        x, kl, geom = None, None, None
        last_stack = len(self._decoder) - 1
        for i, (stack, bias) in enumerate(zip(self._decoder, reversed(self._biases))):
            f = 1 if stack._unpool is None else 2
            s = bias.shape[-1]
            x = _BiasUnpool.apply(x, bias, n, f)
            geom = pm.Geom(n, s * f, s * f)
            xa = None
            mixin = mixin_op = None
            if mixins is not None:
                mixin = mixins[len(mixins) - 1 - i]
                c = mixin.shape[1]
                w = ops.round_up(2 * c, 8)
                mixin_op = pm.GeluOperand(torch.empty(mixin.shape[0], w, dtype=BF16, device=device),
                                          torch.empty(mixin.shape[0], w, dtype=BF16, device=device))
                L.gelu_cast(mixin.detach(), mixin_op.a[:, c:], mixin_op.d[:, c:])
            for j, block in enumerate(stack._topdowns):
                if j < len(stack._topdowns) - 1:
                    emit = GELU
                else:  # the output convolution reads a plain bf16 copy of the last stream
                    emit = L.ACT_NONE if i == last_stack else None
                x, xa, kl = block._pm(x, xa, geom, mixin, mixin_op, kl, emit)
        return x, xa, geom, kl

    def _logits(self, x, xa, geom):
        out = self._output
        y, _ = pm.conv(x, out.weight, out.bias, geom, xa=xa, out_f32=True)
        return pm.from_pm(y, geom, out.out_channels)

    def forward(self, x):
        """(logits, kl): the decoder's output for latents drawn from the posteriors, and each image's KL divergence
        summed over the blocks in decoder order (not normalised by the input's size), as in the reference."""
        _require(x, self, type(self).__name__)
        self._check_resolutions()
        n, c, h, w = x.shape
        r = self._resolutions[0]
        if c != self._input.in_channels or h != r or w != r:
            raise ValueError(f"VeryDeepVAE: expected [n, {self._input.in_channels}, {r}, {r}] inputs (the biases are "
                             f"built for input_resolution {r}); got {list(x.shape)}")
        inp = self._input
        geom = pm.Geom(n, h, w)
        x = pm.image_conv(x.contiguous(), inp.weight, inp.bias, inp.padding)
        mixins = []
        for stack in self._encoder:
            xa = None
            blocks = list(stack._residuals)
            for j, block in enumerate(blocks):
                x, xa = block._pm(x, geom, xa, GELU if j < len(blocks) - 1 else None)
            mixins.append(x)
            if stack._pool is not None:
                x = _Pool.apply(x, geom)
                geom = pm.Geom(n, geom.h // 2, geom.w // 2)
        y, ya, geom, kl = self._decode(n, mixins, x.device)
        if kl is None:
            kl = torch.zeros(n, dtype=F32, device=x.device)
        return self._logits(y, ya, geom), kl

    def _sample(self, n_samples):
        """The decoder's output with every latent drawn from its prior, in decoder order."""
        _require(self._biases[0], self, type(self).__name__)
        self._check_resolutions()
        y, ya, geom, _ = self._decode(n_samples, None, self.device)
        return self._logits(y, ya, geom)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference vd_vae.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_vd_vae(*args, **kwargs)
