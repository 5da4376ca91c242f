"""Drop-in equivalents of `pytorch_generative.nn` for the classes on the hot path (reference nn/__init__.py:3-13)."""

from .modules import (
    CausalAttention,
    CausalConv2d,
    GatedActivation,
    LinearCausalAttention,
    NCHWLayerNorm,
    image_positional_encoding,
)

from .tapconv import TapConv2d, tap_conv2d
from .vq import VectorQuantizer

__all__ = ["CausalAttention", "LinearCausalAttention", "CausalConv2d", "GatedActivation", "NCHWLayerNorm", "image_positional_encoding",
           "TapConv2d", "tap_conv2d", "VectorQuantizer"]
