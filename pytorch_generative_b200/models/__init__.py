"""Drop-in equivalents of `pytorch_generative.models` for the autoregressive-image path
(reference models/__init__.py:4-9)."""

from .base import AutoregressiveModel, GenerativeModel
from .fvbn import FullyVisibleBeliefNetwork
from .gated_pixel_cnn import GatedPixelCNN
from .image_gpt import ImageGPT
from .made import MADE
from .nade import NADE
from .nice import NICE
from .pixel_cnn import PixelCNN
from .pixel_snail import PixelSNAIL

__all__ = ["AutoregressiveModel", "GenerativeModel", "FullyVisibleBeliefNetwork", "GatedPixelCNN", "ImageGPT", "MADE", "NADE", "NICE", "PixelCNN", "PixelSNAIL"]
