"""BetaVAE on the CUDA path — API of reference models/vae/beta_vae.py: the VAE with its KL divergence scaled by
`beta`."""

from . import vae


class BetaVAE(vae.VAE):
    """The Beta-VAE model (reference beta_vae.py BetaVAE)."""

    def __init__(self, in_channels=1, out_channels=1, beta=4.0, latent_channels=16, strides=[4], hidden_channels=64,
                 residual_channels=32, sample_fn=None):
        super().__init__(in_channels, out_channels, latent_channels, strides, hidden_channels, residual_channels,
                         sample_fn)
        self._beta = beta

    def forward(self, x):
        out, kl_div = super().forward(x)
        return out, self._beta * kl_div


def reproduce(*args, **kwargs):
    """The recipe of this model (reference beta_vae.py `reproduce`); see `pytorch_generative_b200.recipes`."""
    from .. import recipes

    return recipes.reproduce_beta_vae(*args, **kwargs)
