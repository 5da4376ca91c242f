"""VQ-VAE-2 on the CUDA path — API of reference models/vae/vq_vae_2.py (`VectorQuantizedVAE2`, `reproduce`).

Same constructor, module tree, state-dict keys, parameter and buffer order and init bits under a seed as the reference,
so checkpoints interchange.  `forward(x)` returns `(x_hat, 0.5 (vq_b + vq_t) + mse(decoded_t, encoded_b))`.

Pixel-major throughout.  encoded_b stays an fp32 stream with three consumers (encoder_t, quantizer_b and the MSE), whose
gradients autograd adds.  decoder_b's input cat(_conv(decoded_t), quantized_b) is one bf16 operand: `_conv` writes its
columns and quantizer_b writes its own in place, with the pad columns zero.
"""

from torch import nn

from .. import losses, ops
from ..nn import pm
from . import base
from .vae import BF16, Decoder, Encoder, Quantizer, _require


class VectorQuantizedVAE2(base.VariationalAutoEncoder):
    """The VQ-VAE-2 model with a latent hierarchy of depth 2 (reference vq_vae_2.py VectorQuantizedVAE2)."""

    def __init__(self, in_channels=1, out_channels=1, hidden_channels=128, n_residual_blocks=2, residual_channels=32,
                 n_embeddings=128, embedding_dim=16, sample_fn=None):
        super().__init__(sample_fn)
        stage = dict(hidden_channels=hidden_channels, n_residual_blocks=n_residual_blocks,
                     residual_channels=residual_channels, stride=2)
        self._encoder_b = Encoder(in_channels=in_channels, out_channels=hidden_channels, **stage)
        self._encoder_t = Encoder(in_channels=hidden_channels, out_channels=hidden_channels, **stage)
        self._quantizer_t = Quantizer(in_channels=hidden_channels, n_embeddings=n_embeddings,
                                      embedding_dim=embedding_dim)
        self._quantizer_b = Quantizer(in_channels=hidden_channels, n_embeddings=n_embeddings,
                                      embedding_dim=embedding_dim)
        self._decoder_t = Decoder(in_channels=embedding_dim, out_channels=hidden_channels, **stage)
        self._conv = nn.Conv2d(in_channels=hidden_channels, out_channels=embedding_dim, kernel_size=1)
        self._decoder_b = Decoder(in_channels=2 * embedding_dim, out_channels=out_channels, **stage)

    def forward(self, x):
        """(x_hat, loss): the bottom decoder's output and 0.5 (vq_loss_b + vq_loss_t) + mse(decoded_t, encoded_b)."""
        _require(x, self, type(self).__name__)
        n, c, h, w = x.shape
        geom = pm.Geom(n, h, w)
        geom_b = self._encoder_b._geoms(geom)  # raises before any launch when x is too small
        geom_t = self._encoder_t._geoms(geom_b)
        if self._decoder_t._geoms(geom_t) != geom_b:
            raise ValueError(f"VectorQuantizedVAE2: a {h}x{w} input gives a top level of {geom_t.h}x{geom_t.w} whose "
                             f"decoding does not match the bottom level's {geom_b.h}x{geom_b.w}")
        self._decoder_b._geoms(geom_b)
        encoded_b, _ = self._encoder_b._pm(pm.to_pm(x, BF16, ops.round_up(c, 8)), geom, out_f32=True)
        encoded_t, _ = self._encoder_t._pm(encoded_b, geom_b, out_f32=False)
        quantized_t, vq_loss_t = self._quantizer_t._pm(encoded_t, geom_t)
        decoded_t, _ = self._decoder_t._pm(quantized_t, geom_t, out_f32=True)
        left, _ = pm.conv(decoded_t, self._conv.weight, self._conv.bias, geom_b)
        cat, vq_loss_b = self._quantizer_b._pm(encoded_b, geom_b, left=left)
        x_hat, geom = self._decoder_b._pm(cat, geom_b, out_f32=True)
        hidden = self._conv.in_channels
        loss = 0.5 * (vq_loss_b + vq_loss_t) + losses.mse_loss_pm(decoded_t, encoded_b, hidden)
        return pm.from_pm(x_hat, geom, self._decoder_b._transposed()[-1].out_channels), loss

    def _sample(self, n_samples):
        raise NotImplementedError("VQ-VAE-2 does not support sampling.")


def reproduce(*args, **kwargs):
    """The recipe of this model (reference vq_vae_2.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_vq_vae_2(*args, **kwargs)
