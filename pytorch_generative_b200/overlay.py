"""Overlay onto an importable reference package (SURVEY.md §8b): `install()` rebinds the hot-path names of
`pytorch_generative` to this package's classes so that the reference's own `train.py` / `reproduce()` / `Trainer` drive them
unmodified; every other model of the reference keeps running on its own code.

The reference's `train.py:10-24` dereferences 13 model modules at import, so shadowing the whole package is not an
option; rebinding is.  `reproduce()` of each recipe constructs its model as `models.<Name>(...)`
(e.g. image_gpt.py:140-148), i.e. through the attribute this function replaces.
"""

import importlib
import importlib.util

_NN_NAMES = ("CausalConv2d", "GatedActivation", "NCHWLayerNorm", "CausalAttention", "LinearCausalAttention",
             "image_positional_encoding")
_MODEL_NAMES = {"PixelCNN": "pixel_cnn", "GatedPixelCNN": "gated_pixel_cnn", "PixelSNAIL": "pixel_snail",
                "ImageGPT": "image_gpt"}
# Bound only where the reference package has the module (releases without MADE, NADE, FVBN, NICE, the VAEs, the mixture
# models or the KDE keep the four names above); the modules are named under pytorch_generative.models (`vae` is a
# namespace package there).
_OPTIONAL_MODEL_NAMES = {"MADE": "autoregressive.made", "NADE": "autoregressive.nade",
                         "FullyVisibleBeliefNetwork": "autoregressive.fvbn", "NICE": "flow.nice", "VAE": "vae.vae",
                         "BetaVAE": "vae.beta_vae", "VectorQuantizedVAE": "vae.vq_vae",
                         "VectorQuantizedVAE2": "vae.vq_vae_2", "VeryDeepVAE": "vae.vd_vae",
                         "GaussianMixtureModel": "mixture_models",
                         "BernoulliMixtureModel": "mixture_models", "KernelDensityEstimator": "kde",
                         "GaussianKernel": "kde", "ParzenWindowKernel": "kde"}
# Bound in their own module only, where the reference package has it: the reference's models/__init__.py does not export
# these names, so pytorch_generative.models gains none.
_MODULE_ONLY_MODEL_NAMES = {"GaussianProcess": "gaussian_process"}
# Bound only where the reference's nn package exports it (and in nn/utils.py, where it is defined, when that module has it)
_OPTIONAL_NN_NAMES = ("VectorQuantizer",)
_saved = {}


def install():
    """Rebinds pytorch_generative.nn.* / pytorch_generative.models.* (hot-path names only).  Returns the names bound."""
    import pytorch_generative as ref  # the reference must be importable (pip-installed or on sys.path)

    from . import models as our_models
    from . import nn as our_nn

    bound = []

    def bind(obj, name, value):
        _saved.setdefault((obj, name), getattr(obj, name))
        setattr(obj, name, value)
        bound.append(f"{obj.__name__}.{name}")

    for name in _NN_NAMES:
        bind(ref.nn, name, getattr(our_nn, name))
    for cls, mod in _MODEL_NAMES.items():
        bind(ref.models, cls, getattr(our_models, cls))
        bind(importlib.import_module(f"pytorch_generative.models.autoregressive.{mod}"), cls, getattr(our_models, cls))
    for name in _OPTIONAL_NN_NAMES:
        if not hasattr(ref.nn, name):
            continue
        bind(ref.nn, name, getattr(our_nn, name))
        if _has_module("pytorch_generative.nn.utils"):
            utils = importlib.import_module("pytorch_generative.nn.utils")
            if hasattr(utils, name):
                bind(utils, name, getattr(our_nn, name))
    for cls, mod in _OPTIONAL_MODEL_NAMES.items():
        if not _has_module(f"pytorch_generative.models.{mod}"):
            continue
        bind(ref.models, cls, getattr(our_models, cls))
        bind(importlib.import_module(f"pytorch_generative.models.{mod}"), cls, getattr(our_models, cls))
    for cls, mod in _MODULE_ONLY_MODEL_NAMES.items():
        if _has_module(f"pytorch_generative.models.{mod}"):
            bind(importlib.import_module(f"pytorch_generative.models.{mod}"), cls, getattr(our_models, cls))
    return bound


def _has_module(name):
    """Whether `name` can be imported; find_spec raises instead of returning None when a parent package is missing."""
    try:
        return importlib.util.find_spec(name) is not None
    except ModuleNotFoundError:
        return False


def uninstall():
    """Restores every name `install()` replaced."""
    for (obj, name), value in _saved.items():
        setattr(obj, name, value)
    _saved.clear()
