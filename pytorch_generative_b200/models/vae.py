"""VAE on the CUDA path — API of reference models/vae/vae.py (`VAE`, `reproduce`) and the parts of models/vae/vaes.py
that it uses (`ResidualBlock`, `ResidualStack`, `Encoder`, `Decoder`, `unit_gaussian_kl_div`, `sample_from_gaussian`).

Same constructors, module tree (`nn.Conv2d` / `nn.ConvTranspose2d` / `nn.ReLU` holders), state-dict keys
(`_encoder.{i}._net.{j}...`), parameter order and init bits under a seed as the reference, so checkpoints interchange.
`VAE.forward(x)` returns `(logits [n, out, H', W'] fp32, kl [n])`.

Activations stay pixel-major ([N*H*W, C] matrices) from the input layer to the logits:
  * the stride-2 `Conv2d(4, 2, 1)` layers are `pm.conv_strided` (gather -> GEMM) and write bf16 ReLU(y), the operand
    of their consumer;
  * a residual block is `pm.conv` 3x3 with `in_act=ReLU` whose epilogue writes bf16 ReLU(h), then `pm.conv` 1x1 with the
    stream as `res`; the stack's trailing ReLU is the next layer's `in_act`;
  * the stream after an encoder's last strided convolution is a post-ReLU value, and the GEMM epilogue writes no
    fp32-activated output.  Rather than spend a pass on an fp32 copy, the first residual block adds the bf16 ReLU(y)
    its 3x3 convolution reads anyway as a bf16 `res`: the stream's first term carries bf16 rounding (2^-9 relative),
    every later block adds to an fp32 stream;
  * the `ConvTranspose2d(4, 2, 1)` layers are `pm.conv_transposed` (GEMM -> scatter with the bias and the next ReLU);
  * the latent is one `pg_vae_latent_fwd` launch (z as the decoder's bf16 operand and the per-image KL), and its
    backward one `pg_vae_latent_bwd` launch, whose bf16 dh reaches the encoder's last convolution as its GEMM operand
    (through the bf16 copy of h that the convolution's epilogue writes beside the fp32 h).
The forward and backward never synchronise with the host, so a training step captures as a CUDA graph.
"""

import torch
from torch import nn

from .. import _lib as L
from .. import ops
from ..nn import pm
from ..nn.vq import VectorQuantizer
from . import base

BF16, F32 = torch.bfloat16, torch.float32
RELU = L.ACT_RELU


def draw_noise(shape, device):
    """The reparameterisation's noise: one torch.randn of the latent's NCHW shape (the reference's randn_like)."""
    return torch.randn(shape, device=device)


def _require(x, module, who):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: the CUDA path runs on CUDA tensors only (no CPU fallback); got {x.device}")
    for p in module.parameters():
        if p.dtype != F32 or not p.is_cuda or not p.is_contiguous():
            raise RuntimeError(f"{who}: the CUDA path needs contiguous fp32 CUDA parameters; got {p.dtype} on {p.device}")
    if x.dtype != F32:
        raise RuntimeError(f"{who}: the CUDA path takes fp32 inputs; got {x.dtype}")


class ResidualBlock(nn.Module):
    """x + conv1x1(relu(conv3x3(relu(x)))) (reference vaes.py ResidualBlock)."""

    def __init__(self, n_channels, hidden_channels):
        super().__init__()
        self._net = nn.Sequential(
            nn.ReLU(),
            nn.Conv2d(in_channels=n_channels, out_channels=hidden_channels, kernel_size=3, padding=1),
            nn.ReLU(),
            nn.Conv2d(in_channels=hidden_channels, out_channels=n_channels, kernel_size=1),
        )

    def _pm(self, x, geom, post_act=False):
        """x: fp32 stream [P, C] (the block's input before its ReLU), or with post_act the bf16 ReLU(y) of a strided
        convolution [P, C_p] (ReLU is then the identity on it, and it enters the sum as a bf16 residual)."""
        c3, c1 = self._net[1], self._net[3]
        res = x[:, : c1.out_channels] if post_act else x
        _, h = pm.conv(x, c3.weight, c3.bias, geom, c3.padding, in_act=L.ACT_NONE if post_act else RELU,
                       xa=x if post_act else None, emit=RELU, emit_mode=pm.PRE_GRAD, want_main=False)
        y, _ = pm.conv(h, c1.weight, c1.bias, geom, in_act=RELU, xa=h, res=res, out_f32=True)
        return y

    def forward(self, x):
        raise NotImplementedError("ResidualBlock runs inside Encoder / Decoder on the CUDA path (their pixel-major "
                                  "stream); call the Encoder or Decoder")


class ResidualStack(nn.Module):
    """ResidualBlocks followed by a ReLU (reference vaes.py ResidualStack)."""

    def __init__(self, n_channels, hidden_channels, n_residual_blocks=1):
        super().__init__()
        self._net = nn.Sequential(*[ResidualBlock(n_channels, hidden_channels) for _ in range(n_residual_blocks)]
                                  + [nn.ReLU()])

    def _pm(self, x, geom, post_act=False):
        """The stack WITHOUT its trailing ReLU (the consumer's in_act): fp32 stream [P, C]."""
        for i, block in enumerate(self._net[:-1]):
            x = block._pm(x, geom, post_act and i == 0)
        return x

    def forward(self, x):
        raise NotImplementedError("ResidualStack runs inside Encoder / Decoder on the CUDA path (its trailing ReLU is "
                                  "the next convolution's input activation); call the Encoder or Decoder")


class Encoder(nn.Module):
    """Stride-2 Conv2d(4, 2, 1) + ReLU layers, a ResidualStack and a 3x3 Conv2d (reference vaes.py Encoder)."""

    def __init__(self, in_channels, out_channels, hidden_channels, n_residual_blocks, residual_channels, stride):
        super().__init__()
        assert stride % 2 == 0, '"stride" must be even.'
        net = []
        for i in range(stride // 2):
            first, last = 0, stride // 2 - 1
            in_c = in_channels if i == first else hidden_channels // 2
            out_c = hidden_channels // 2 if i < last else hidden_channels
            net.append(nn.Conv2d(in_channels=in_c, out_channels=out_c, kernel_size=4, stride=2, padding=1))
            net.append(nn.ReLU())
        net.append(ResidualStack(n_channels=hidden_channels, hidden_channels=residual_channels,
                                 n_residual_blocks=n_residual_blocks))
        net.append(nn.Conv2d(in_channels=hidden_channels, out_channels=out_channels, kernel_size=3, padding=1))
        self._net = nn.Sequential(*net)

    def _geoms(self, geom):
        """Geometry after each strided convolution; raises before any launch when the input is too small."""
        for conv in self._net[:-2:2]:
            geom = pm.strided_geom(conv, geom)
        return geom

    def _pm(self, x, geom, out_f32, bf16_copy=False):
        """x [P, C(_p)] (bf16 or fp32, the encoder's input as is) -> (y [P', C_out] fp32 or bf16, geom').  bf16_copy:
        also a bf16 copy of y from the same epilogue, an ordinary output through which y's gradient may arrive in
        bf16 (the operand the convolution's backward reads): returns (y, y_bf16, geom')."""
        for conv in self._net[:-2:2]:
            x, geom = pm.conv_strided(x, conv, geom, emit=RELU)
        x = self._net[-2]._pm(x, geom, post_act=True)
        last = self._net[-1]
        y, yb = pm.conv(x, last.weight, last.bias, geom, last.padding, in_act=RELU, out_f32=out_f32,
                        emit=L.ACT_NONE if bf16_copy else None, emit_mode=pm.POST)
        return (y, yb, geom) if bf16_copy else (y, geom)

    def forward(self, x):
        """NCHW fp32 in and out, as the reference's module."""
        return _nchw(self, x, self._net[-1].out_channels)


class Decoder(nn.Module):
    """A 3x3 Conv2d, a ResidualStack and ConvTranspose2d(4, 2, 1) layers with ReLUs between them (reference vaes.py
    Decoder)."""

    def __init__(self, in_channels, out_channels, hidden_channels, n_residual_blocks, residual_channels, stride):
        super().__init__()
        assert stride % 2 == 0, '"stride" must be even.'
        net = [
            nn.Conv2d(in_channels=in_channels, out_channels=hidden_channels, kernel_size=3, padding=1),
            ResidualStack(n_channels=hidden_channels, hidden_channels=residual_channels,
                          n_residual_blocks=n_residual_blocks),
        ]
        for i in range(stride // 2):
            first, last = 0, stride // 2 - 1
            in_c = hidden_channels if i == first else hidden_channels // 2
            out_c = hidden_channels // 2 if i < last else out_channels
            net.append(nn.ConvTranspose2d(in_channels=in_c, out_channels=out_c, kernel_size=4, stride=2, padding=1))
            if i < last:
                net.append(nn.ReLU())
        self._net = nn.Sequential(*net)

    def _geoms(self, geom):
        for conv in self._transposed():
            geom = pm.strided_geom(conv, geom)
        return geom

    def _transposed(self):
        return [m for m in self._net[2:] if isinstance(m, nn.ConvTranspose2d)]

    def _pm(self, x, geom, out_f32):
        """x [P, C(_p)] (bf16 or fp32) -> (y [P', round_up(C_out, 8)] fp32 or bf16, geom')."""
        first = self._net[0]
        x, _ = pm.conv(x, first.weight, first.bias, geom, first.padding, out_f32=True)
        x = self._net[1]._pm(x, geom)
        convs = self._transposed()
        in_act = RELU
        for i, conv in enumerate(convs):
            last = i == len(convs) - 1
            x, geom = pm.conv_transposed(x, conv, geom, in_act=in_act, emit=None if last else RELU, out_f32=out_f32)
            in_act = L.ACT_NONE
        return x, geom

    def forward(self, x):
        """NCHW fp32 in and out, as the reference's module."""
        return _nchw(self, x, self._transposed()[-1].out_channels)


def _nchw(stage, x, c_out):
    """An Encoder / Decoder on an NCHW fp32 tensor: to pixel-major, the stage, back to NCHW."""
    _require(x, stage, type(stage).__name__)
    n, c, h, w = x.shape
    geom = pm.Geom(n, h, w)
    stage._geoms(geom)
    y, geom = stage._pm(pm.to_pm(x, F32, ops.round_up(c, 8)), geom, True)
    return pm.from_pm(y, geom, c_out)


class Quantizer(nn.Module):
    """A 1x1 Conv2d into a VectorQuantizer (reference vaes.py Quantizer)."""

    def __init__(self, in_channels, n_embeddings, embedding_dim):
        super().__init__()
        self._net = nn.Sequential(
            nn.Conv2d(in_channels=in_channels, out_channels=embedding_dim, kernel_size=1),
            VectorQuantizer(n_embeddings, embedding_dim),
        )

    def _pm(self, x, geom, left=None):
        """x [P, C(_p)] (bf16, or an fp32 stream) -> (the decoder's bf16 operand [P, round_up(c0 + d, 8)], vq_loss).  With
        `left` (bf16 [P, c0]) the operand is cat(left, quantized) along channels, the quantizer writing its columns in
        place.  The 1x1 convolution writes z in fp32 (the distances) and a bf16 copy through which z's gradient
        returns as the operand its backward reads."""
        conv, vq = self._net
        z, z_bf16 = pm.conv(x, conv.weight, conv.bias, geom, out_f32=True, emit=L.ACT_NONE, emit_mode=pm.POST)
        c0 = 0 if left is None else left.shape[1]
        return vq._pm(z_bf16, z.detach(), ops.round_up(c0 + vq.embedding_dim, 8), left)

    def forward(self, x):
        """(x + (q - x), vq_loss) on NCHW fp32, as the reference's module."""
        _require(x, self, type(self).__name__)
        conv, vq = self._net
        n, c, h, w = x.shape
        geom = pm.Geom(n, h, w)
        z, _ = pm.conv(pm.to_pm(x, F32, ops.round_up(c, 8)), conv.weight, conv.bias, geom, out_f32=True)
        q, loss = vq._pm(z, z.detach(), vq.embedding_dim, out_dtype=F32)
        return pm.from_pm(q, geom, vq.embedding_dim), loss


class _Latent(torch.autograd.Function):
    """h [P, 2L] fp32 (mean | log_std), eps [n, L, h, w] -> (z bf16 [P, round_up(L, 8)], kl [n]).  The gradient leaves
    through `h_bf16`, the encoder convolution's bf16 copy of h: autograd casts a gradient to its input's dtype, so
    through the fp32 h (passed detached, for its values) the bf16 dh would come back as fp32 and be cast again."""

    @staticmethod
    def forward(ctx, h_bf16, h, eps, L_):
        n = eps.shape[0]
        z = torch.empty(h.shape[0], ops.round_up(L_, 8), dtype=BF16, device=h.device)
        kl = torch.empty(n, dtype=F32, device=h.device)
        L.vae_latent_fwd(h, eps, z, kl)
        ctx.save_for_backward(h, eps)
        ctx.set_materialize_grads(False)
        return z, kl

    @staticmethod
    def backward(ctx, dz, dkl):
        h, eps = ctx.saved_tensors
        if dz is None:
            dz = torch.zeros(h.shape[0], ops.round_up(eps.shape[1], 8), dtype=BF16, device=h.device)
        elif dz.dtype != BF16:
            dz = dz.to(BF16)
        c = h.shape[1]
        cp = ops.round_up(c, 8)
        dh = torch.empty(h.shape[0], cp, dtype=BF16, device=h.device)
        L.vae_latent_bwd(h, eps, dz.contiguous(), None if dkl is None else dkl.contiguous().float(), dh)
        return (dh if cp == c else dh[:, :c]), None, None, None


class VAE(base.VariationalAutoEncoder):
    """The Variational Autoencoder (reference vae.py VAE)."""

    def __init__(self, in_channels=1, out_channels=1, latent_channels=16, strides=[4], hidden_channels=64,
                 residual_channels=32, sample_fn=None):
        super().__init__(sample_fn)
        self._latent_channels = latent_channels
        self._total_stride = sum(strides)

        encoder = []
        for i, stride in enumerate(strides):
            in_c = in_channels if i == 0 else hidden_channels
            out_c = hidden_channels if i < len(strides) - 1 else 2 * self._latent_channels
            encoder.append(Encoder(in_channels=in_c, out_channels=out_c, hidden_channels=hidden_channels,
                                   residual_channels=residual_channels, n_residual_blocks=2, stride=stride))
        self._encoder = nn.Sequential(*encoder)

        decoder = []
        for i, stride in enumerate(reversed(strides)):
            in_c = self._latent_channels if i == 0 else hidden_channels
            out_c = hidden_channels if i < len(strides) - 1 else out_channels
            decoder.append(Decoder(in_channels=in_c, out_channels=out_c, hidden_channels=hidden_channels,
                                   residual_channels=residual_channels, n_residual_blocks=2, stride=stride))
        self._decoder = nn.Sequential(*decoder)

    def _decode(self, z, geom):
        """Pixel-major latent operand -> fp32 logits [P, round_up(out, 8)] and their geometry."""
        for i, dec in enumerate(self._decoder):
            z, geom = dec._pm(z, geom, out_f32=i == len(self._decoder) - 1)
        return z, geom

    def forward(self, x):
        """(logits, kl): the decoder's output for latents drawn from the posterior, and each image's KL divergence from
        the unit Gaussian prior (not normalised by the input's size), as in the reference."""
        _require(x, self, type(self).__name__)
        n, c, h, w = x.shape
        geom = pm.Geom(n, h, w)
        for enc in self._encoder:
            geom = enc._geoms(geom)
        geom = pm.Geom(n, h, w)
        y = pm.to_pm(x, BF16, ops.round_up(c, 8))
        for enc in self._encoder[:-1]:
            y, geom = enc._pm(y, geom, out_f32=False)
        h, h_bf16, geom = self._encoder[-1]._pm(y, geom, out_f32=True, bf16_copy=True)
        L_ = self._latent_channels
        eps = draw_noise((n, L_, geom.h, geom.w), x.device)
        z, kl = _Latent.apply(h_bf16, h.detach(), eps, L_)
        logits, geom = self._decode(z, geom)
        return pm.from_pm(logits, geom, self._decoder[-1]._transposed()[-1].out_channels), kl

    def _sample(self, n_samples):
        """The decoder's output for latents from the unit Gaussian, drawn as the reference draws them."""
        latent_size = self._h // 2 ** (self._total_stride // 2)
        shape = (n_samples, self._latent_channels, latent_size, latent_size)
        latents = torch.randn(shape, device=self.device)
        _require(latents, self, type(self).__name__)
        n, c, h, w = latents.shape
        geom = pm.Geom(n, int(h), int(w))
        logits, geom = self._decode(pm.to_pm(latents, BF16, ops.round_up(c, 8)), geom)
        return pm.from_pm(logits, geom, self._decoder[-1]._transposed()[-1].out_channels)


def reproduce(*args, **kwargs):
    """The recipe of this model (reference vae.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_vae(*args, **kwargs)
