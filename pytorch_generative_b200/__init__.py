"""H100-native drop-in for the autoregressive-image hot path of pytorch-generative.

`nn` and `models` mirror `pytorch_generative.nn` / `pytorch_generative.models` for the classes on the
path (SURVEY.md §8); the arithmetic runs in hand-written sm_90a kernels behind the C ABI in
include/pg_b200.h (see `_lib`).  Importing this package does not load the native library; the first
kernel call does, and raises if it is missing — there is no CPU fallback.
"""

__version__ = "0.1.0"
