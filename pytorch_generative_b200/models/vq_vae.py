"""VQ-VAE on the CUDA path — API of reference models/vae/vq_vae.py (`VectorQuantizedVAE`, `reproduce`).

Same constructor, module tree (`_encoder`, `_quantizer`, `_decoder` of `models/vae.py`), state-dict keys, parameter and
buffer order and init bits under a seed as the reference, so checkpoints interchange.  `forward(x)` returns
`(x_hat, vq_loss)`.  Activations stay pixel-major from the input to x_hat: the encoder's bf16 output is the operand of
the quantizer's 1x1 convolution, and the quantizer writes the decoder's bf16 operand.
"""

from .. import ops
from ..nn import pm
from . import base
from .vae import BF16, Decoder, Encoder, Quantizer, _require


class VectorQuantizedVAE(base.VariationalAutoEncoder):
    """The Vector Quantized Variational Autoencoder (reference vq_vae.py VectorQuantizedVAE)."""

    def __init__(self, in_channels=1, out_channels=1, hidden_channels=128, n_residual_blocks=2, residual_channels=32,
                 n_embeddings=128, embedding_dim=16, sample_fn=None):
        super().__init__(sample_fn)
        self._encoder = Encoder(in_channels=in_channels, out_channels=hidden_channels, hidden_channels=hidden_channels,
                                n_residual_blocks=n_residual_blocks, residual_channels=residual_channels, stride=4)
        self._quantizer = Quantizer(in_channels=hidden_channels, n_embeddings=n_embeddings, embedding_dim=embedding_dim)
        self._decoder = Decoder(in_channels=embedding_dim, out_channels=out_channels, hidden_channels=hidden_channels,
                                n_residual_blocks=n_residual_blocks, residual_channels=residual_channels, stride=4)

    def forward(self, x):
        """(x_hat, vq_loss): the decoder's output for the quantized encoding of x, and the quantizer's loss."""
        _require(x, self, type(self).__name__)
        n, c, h, w = x.shape
        geom = pm.Geom(n, h, w)
        self._decoder._geoms(self._encoder._geoms(geom))  # raises before any launch when x is too small
        y, geom = self._encoder._pm(pm.to_pm(x, BF16, ops.round_up(c, 8)), geom, out_f32=False)
        q, vq_loss = self._quantizer._pm(y, geom)
        x_hat, geom = self._decoder._pm(q, geom, out_f32=True)
        return pm.from_pm(x_hat, geom, self._decoder._transposed()[-1].out_channels), vq_loss

    def _sample(self, n_samples):
        raise NotImplementedError("VQ-VAE does not support sampling.")


def reproduce(*args, **kwargs):
    """The recipe of this model (reference vq_vae.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_vq_vae(*args, **kwargs)
