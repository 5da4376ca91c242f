"""Drop-in equivalents of `pytorch_generative.models` for the autoregressive-image path
(reference models/__init__.py:4-9)."""

from .base import (AutoregressiveModel, CategoricalSampleFn, GenerativeModel, LogisticMixtureSampleFn, VariationalAutoEncoder,
                   categorical_sample_fn, logistic_mixture_sample_fn)
from .beta_vae import BetaVAE
from .fvbn import FullyVisibleBeliefNetwork
from .gated_pixel_cnn import GatedPixelCNN
from .gaussian_process import GaussianProcess
from .image_gpt import ImageGPT
from .kde import GaussianKernel, KernelDensityEstimator, ParzenWindowKernel
from .made import MADE
from .mixture_models import BernoulliMixtureModel, GaussianMixtureModel
from .nade import NADE
from .nice import NICE
from .pixel_cnn import PixelCNN
from .pixel_snail import PixelSNAIL
from .vae import VAE
from .vd_vae import VeryDeepVAE
from .vq_vae import VectorQuantizedVAE
from .vq_vae_2 import VectorQuantizedVAE2

__all__ = ["AutoregressiveModel", "CategoricalSampleFn", "categorical_sample_fn", "LogisticMixtureSampleFn", "logistic_mixture_sample_fn", "GenerativeModel", "VariationalAutoEncoder", "BernoulliMixtureModel", "BetaVAE", "FullyVisibleBeliefNetwork", "GatedPixelCNN", "GaussianKernel",
           "GaussianProcess",
           "GaussianMixtureModel", "ImageGPT", "KernelDensityEstimator", "MADE", "NADE", "NICE", "ParzenWindowKernel", "PixelCNN", "PixelSNAIL", "VAE",
           "VectorQuantizedVAE", "VectorQuantizedVAE2", "VeryDeepVAE"]
