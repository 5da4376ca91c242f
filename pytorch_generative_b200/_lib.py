"""ctypes binding of libpg_b200.so (the C ABI declared in include/pg_b200.h).

This is the only place Python touches the native library.  Tensors cross the boundary as raw device
pointers plus sizes; the current torch CUDA stream is passed explicitly to every call, so the kernels
are ordered with the rest of the autograd graph (forward on the main thread, backward on autograd's
device thread).  There is deliberately NO CPU fallback: if the shared library is missing or the inputs
are not CUDA tensors, the call raises.
"""

import ctypes
import functools
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# PG_B200_LIB: developer knob to load an alternative build of the same ABI (kernel A/B experiments)
LIB_PATH = os.environ.get("PG_B200_LIB") or os.path.join(_HERE, "libpg_b200.so")

ACT_NONE, ACT_RELU, ACT_GELU, ACT_ELU, ACT_TANH = 0, 1, 2, 3, 4
ACT_GIVEN = 5  # dact only: aux already holds the derivative
ACT_RELU_OUT, ACT_ELU_OUT = 6, 7  # dact only: aux holds the activated value
DACT_FROM_OUT = {ACT_RELU: ACT_RELU_OUT, ACT_ELU: ACT_ELU_OUT}
ACT_STORE_DERIV = 0x100  # OR-ed into act: out_pre receives act'(pre)
ACT_RES_BF16 = 0x200  # OR-ed into act: res0 / res1 are bf16 matrices (set by _epilogue from the tensors' dtype)
ACT_BY_NAME = {None: ACT_NONE, "none": ACT_NONE, "relu": ACT_RELU, "gelu": ACT_GELU, "elu": ACT_ELU, "tanh": ACT_TANH}

_vp, _i32, _i64, _f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float


class GemmEpilogue(ctypes.Structure):
    """Mirror of `pg_gemm_epilogue` (include/pg_b200.h)."""

    _fields_ = [
        ("bias", _vp), ("aux", _vp), ("res0", _vp), ("res1", _vp),
        ("out_bf16", _vp), ("out_pre", _vp), ("out_f32", _vp),
        ("ld_aux", _i64), ("ld_res", _i64), ("ld_out_bf16", _i64), ("ld_out_pre", _i64), ("ld_out_f32", _i64),
        ("act", ctypes.c_int32), ("dact", ctypes.c_int32), ("accumulate", ctypes.c_int32), ("alpha", _f32),
        ("bias_grad", _vp),
    ]


class ConvGeom(ctypes.Structure):
    """Mirror of `pg_conv_geom` (include/pg_b200.h)."""

    _fields_ = [("mode", ctypes.c_int32), ("N", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("C", ctypes.c_int32), ("n_taps", ctypes.c_int32), ("dy", ctypes.c_int32 * 32), ("dx", ctypes.c_int32 * 32)]


CONV_FWD, CONV_DGRAD, CONV_WGRAD = 1, 2, 3
MAX_TAPS = 225          # taps of pg_gemm_bf16_conv_taps and the tap gathers / scatters: a 15 x 15 kernel
MAX_TAP_OFFSET = 64     # |dy|, |dx| of a tap on the TMA tap loop (int8 in the kernel parameters)
NADE_CHUNK = 16         # PG_NADE_CHUNK: dimensions between two checkpoints of NADE's hidden pre-activation
REZERO_CHUNK = 8192     # PG_REZERO_CHUNK: elements per block of pg_rezero_bwd's partial sums

# name -> argtypes (restype is always int unless listed in _SPECIAL)
_SIGNATURES = {
    "pg_gemm_bf16": [_vp, _i32, _i64, _vp, _i32, _i64, _i32, _i32, _i32, _i32, ctypes.POINTER(GemmEpilogue), _i32, _vp],
    "pg_gemm_bf16_conv": [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, ctypes.POINTER(GemmEpilogue), ctypes.POINTER(ConvGeom), _vp],
    "pg_gemm_bf16_conv_taps": [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, ctypes.POINTER(GemmEpilogue), _i32, _i32, _i32,
                               _i32, _i32, _i32, _vp, _vp, _vp],
    "pg_colsum_bf16": [_vp, _i64, _i32, _i32, _vp, _i32, _vp],
    "pg_colsum_f32": [_vp, _i64, _i32, _i32, _vp, _i32, _vp],
    "pg_layernorm_fwd": [_vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp],
    "pg_layernorm_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "pg_layernorm_fwd_ld": [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp],
    "pg_layernorm_bwd_ld": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "pg_gated_act_fwd": [_vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp],
    "pg_gated_act_bwd": [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp],
    "pg_gated_res_fwd": [_vp, _i32, _vp, _i32, _i32, _i32, _vp, _vp],
    "pg_dact_from_out": [_vp, _i32, _vp, _i64, _i32, _vp, _vp],
    "pg_bce_logits_fwd_bwd": [_vp, _vp, _i64, _f32, _vp, _vp, _vp],
    "pg_nchw_to_pm": [_vp, _i32, _i32, _i32, _vp, _i32, _i64, _vp],
    "pg_pm_to_nchw": [_vp, _i32, _i64, _i32, _i32, _i32, _i32, _vp, _vp],
    "pg_dact_mul": [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_cast_f32_to_bf16": [_vp, _vp, _i64, _vp],
    "pg_act_cast_bf16": [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_causal_attn_fwd": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _vp],
    "pg_causal_attn_bwd": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _i64,
                           _vp, _i64, _i32, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _vp],
    "pg_conv_small_fwd": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp],
    "pg_conv_small_bwd": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp],
    "pg_conv_small_fwd_d": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp,
                            _i32, _vp],
    "pg_conv_small_bwd_d": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp,
                            _vp, _vp],
    "pg_attn_decode": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32,
                       _f32, _i32, _vp],
    "pg_linear_attn_fwd": [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp],
    "pg_linear_attn_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp],
    "pg_cast_multi_bf16": [_vp, _vp, _vp, _vp, _i32, _i32, _vp],
    "pg_grad_sqnorm": [_vp, _vp, _vp, _i32, _i32, _vp, _vp],
    "pg_adam_step": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _f32, _f32, ctypes.c_double, ctypes.c_double,
                     ctypes.c_double, ctypes.c_double, _i32, _vp, _vp],
    "pg_adabelief_step": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _f32, _f32, ctypes.c_double,
                          ctypes.c_double, ctypes.c_double, _i32, _vp, _vp],
    "pg_rezero_fwd": [_vp, _vp, _vp, _i64, _vp, _vp],
    "pg_rezero_bwd": [_vp, _vp, _vp, _i64, _vp, _vp, _vp],
    "pg_tap_gather": [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _vp],
    "pg_tap_scatter": [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _i64, _vp, _vp, _i64, _vp],
    "pg_made_mask_cast": [_vp, _i32, _i32, _vp, _vp, _i32, _vp, _i32, _i64, _vp, _vp],
    "pg_made_sample_step": [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _i32, _vp,
                            _vp, _vp],
    "pg_nade_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp],
    "pg_nade_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp],
    "pg_fvbn_fwd": [_vp, _vp, _i32, _i32, _vp, _vp],
    "pg_fvbn_bwd": [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp],
    "pg_fvbn_sample_step": [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp],
    "pg_nice_split": [_vp, _i32, _i32, _vp, _f32, _vp, _vp, _i64, _i32, _vp, _vp],
    "pg_nice_join": [_vp, _vp, _i64, _i32, _i32, _vp, _f32, _vp, _vp, _vp],
    "pg_nice_scale_bwd": [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i64, _i32, _vp, _vp, _vp],
    "pg_logistic_prior_fwd_bwd": [_vp, _i32, _i32, _f32, _vp, _vp, _vp],
    "pg_strided_gather": [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp],
    "pg_strided_scatter": [_vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32,
                           _vp, _i64, _vp, _vp, _i64, _vp],
    "pg_vae_latent_fwd": [_vp, _i64, _vp, _i32, _i32, _i32, _vp, _i64, _vp, _vp],
    "pg_vae_latent_bwd": [_vp, _i64, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_gelu_cast": [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp],
    "pg_vd_latent_fwd": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _vp, _vp,
                         _vp],
    "pg_vd_latent_bwd": [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp,
                         _i64, _vp],
    "pg_avg_pool2_fwd": [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_avg_pool2_bwd": [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_bias_unpool_fwd": [_vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp],
    "pg_bias_unpool_bwd": [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _vp],
    "pg_vq_assign": [_vp, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _i64, _i32, _i32, _vp, _vp],
    "pg_vq_code_sums": [_vp, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _f32, _vp, _vp, _vp],
    "pg_vq_ema_update": [_vp, _vp, _i32, _i32, _f32, _f32, _vp, _vp, _vp, _vp],
    "pg_vq_bwd": [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _i64, _i32, _vp, _f32, _i32, _vp, _i64, _vp],
    "pg_mse_mean": [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _f32, _vp, _vp, _i64, _vp, _i64, _vp],
    "pg_kde_gauss_fwd": [_vp, _i32, _vp, _i32, _i32, _f32, _f32, _vp, _vp, _vp],
    "pg_kde_gauss_bwd": [_vp, _i32, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp],
    "pg_kde_parzen_count": [_vp, _i32, _vp, _i32, _i32, ctypes.c_double, _vp, _vp, _vp],
    "pg_mixture_fwd": [_i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp],
    "pg_mixture_bwd": [_i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "pg_gemm_f64": [_i32, _i32, _i32, _i32, _i32, ctypes.c_double, _vp, _i64, _vp, _i64, ctypes.c_double, _vp, _i64, _i32,
                    _vp],
    "pg_gp_potrf": [_vp, _i32, _i64, ctypes.c_double, _vp, _vp],
    "pg_gp_trsm": [_vp, _i32, _vp, _i32, _i32, _vp],
}
EXPORTED_SYMBOLS = sorted(list(_SIGNATURES) + ["pg_abi_version", "pg_last_error", "pg_sm_count", "pg_launch_count",
                                                 "pg_reserve_sms"])

_lib = None


def load():
    """Loads libpg_b200.so (raises if it has not been built: there is no fallback path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m pytorch_generative_b200._build` "
            "(or __graft_entry__.build()); the CUDA path has no CPU fallback"
        )
    lib = ctypes.CDLL(LIB_PATH)
    lib.pg_last_error.restype = ctypes.c_char_p
    lib.pg_last_error.argtypes = []
    lib.pg_abi_version.restype = ctypes.c_int
    lib.pg_abi_version.argtypes = []
    lib.pg_sm_count.restype = ctypes.c_int
    lib.pg_sm_count.argtypes = []
    lib.pg_launch_count.restype = ctypes.c_ulonglong
    lib.pg_launch_count.argtypes = []
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = ctypes.c_int
    if lib.pg_abi_version() != 1:
        raise RuntimeError(f"libpg_b200.so ABI version {lib.pg_abi_version()} != 1")
    _lib = lib
    return lib


def _check(rc, name):
    if rc != 0:
        raise RuntimeError(f"{name} failed: {_lib.pg_last_error().decode(errors='replace')}")


def _ptr(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("pytorch_generative_b200 kernels need CUDA tensors (there is no CPU fallback)")
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _device_guarded(fn):
    """Runs a binding on the device its tensors live on: every operand must share one CUDA device; when that is not
    the current device the call (stream lookup, TMA descriptor encode, launch) happens under `torch.cuda.device(idx)`,
    like torch's own ops do."""

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        idx = None
        for a in (*args, *kwargs.values()):
            if torch.is_tensor(a) and a.is_cuda:
                if idx is None:
                    idx = a.device.index
                elif a.device.index != idx:
                    raise RuntimeError(f"{fn.__name__}: operands live on different CUDA devices ({idx} and {a.device.index})")
        if idx is None or idx == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(idx):
            return fn(*args, **kwargs)

    return wrapper


def _pm(t):
    """Checks a pixel-major 2-D view (unit inner stride) and returns (ptr, pitch)."""
    assert t.dim() == 2 and t.stride(1) == 1, f"expected a [P, C] matrix with unit inner stride, got {t.shape} {t.stride()}"
    return _ptr(t), t.stride(0)


def launch_count():
    """Kernels launched by libpg_b200.so so far in this process."""
    return int(load().pg_launch_count())


# Optional per-call timing hook used by bench.py: when set, gemm() brackets its launch with CUDA events on
# the launching stream and reports (flops, start_event, end_event, algorithmic_bytes).
gemm_timing_hook = None

_sm_count = None


def sm_count():
    global _sm_count
    if _sm_count is None:
        _sm_count = load().pg_sm_count()
    return _sm_count


def reserve_sms(n):
    """SMs left out of the persistent grids (see pg_reserve_sms); returns the previous setting."""
    global _sm_count
    lib = load()
    lib.pg_reserve_sms.restype = ctypes.c_int
    lib.pg_reserve_sms.argtypes = [ctypes.c_int]
    old = lib.pg_reserve_sms(int(n))
    _sm_count = None
    return old


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
@_device_guarded
def gemm(A, B, M, N, K, *, a_mn=False, b_mn=False, bias=None, aux=None, dact=ACT_NONE, res0=None, res1=None,
         out_bf16=None, out_pre=None, out_f32=None, act=ACT_NONE, accumulate=False, alpha=1.0, split_k=1, impl=0,
         bias_grad=None):
    """acc = A·Bᵀ (see pg_gemm_bf16 in include/pg_b200.h); all tensors are 2-D bf16/fp32 CUDA views.
    bias_grad (weight-gradient GEMMs, a_mn=True): fp32 [M] += sum_k A(m, k), reduced from the staged A tiles."""
    lib = load()
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    a_ptr, lda = _pm(A)
    b_ptr, ldb = _pm(B)
    e = _epilogue(M, N, bias, aux, dact, res0, res1, out_bf16, out_pre, out_f32, act, accumulate, alpha, bias_grad)
    hook = gemm_timing_hook
    if hook is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    _check(lib.pg_gemm_bf16(a_ptr, int(a_mn), lda, b_ptr, int(b_mn), ldb, M, N, K, split_k, ctypes.byref(e), impl,
                            _stream()), "pg_gemm_bf16")
    if hook is not None:
        ev1.record()
        hook(2.0 * M * N * K, ev0, ev1, _gemm_io(M, N, K, out_bf16, out_pre, out_f32, aux, res0, res1))


def _gemm_io(M, N, K, out_bf16, out_pre, out_f32, aux, res0, res1):
    """Algorithmic HBM bytes of one contraction: both operands once, every epilogue tensor once."""
    return 2 * (M * K + N * K) + M * N * (2 * (out_bf16 is not None) + 2 * (out_pre is not None) + 4 * (out_f32 is not None)
                                          + 2 * (aux is not None) + sum(r.element_size() for r in (res0, res1) if r is not None))


@_device_guarded
def gemm_conv(A, B, M, N, K, mode, n_img, H, W, C, taps, *, bias=None, aux=None, dact=ACT_NONE, res0=None, res1=None,
              out_bf16=None, out_pre=None, out_f32=None, act=ACT_NONE, accumulate=False, alpha=1.0, split_k=1,
              bias_grad=None):
    """Tap-loop convolution on the GEMM kernel (pg_gemm_bf16_conv); `taps` = [(dy, dx), ...] as the kernel applies them
    (the caller negates them for dgrad)."""
    lib = load()
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    a_ptr, lda = _pm(A)
    b_ptr, ldb = _pm(B)
    e = _epilogue(M, N, bias, aux, dact, res0, res1, out_bf16, out_pre, out_f32, act, accumulate, alpha, bias_grad)
    dy, dx = _int_array([t[0] for t in taps]), _int_array([t[1] for t in taps])
    hook = gemm_timing_hook
    if hook is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    _check(lib.pg_gemm_bf16_conv_taps(a_ptr, lda, b_ptr, ldb, M, N, K, split_k, ctypes.byref(e), mode, n_img, H, W, C,
                                      len(taps), ctypes.cast(dy, ctypes.c_void_p), ctypes.cast(dx, ctypes.c_void_p),
                                      _stream()), "pg_gemm_bf16_conv_taps")
    if hook is not None:
        ev1.record()
        # the shifted operand is read once per tap from L2 but only once from HBM
        io = _gemm_io(M, N, K, out_bf16, out_pre, out_f32, aux, res0, res1)
        if mode == CONV_WGRAD:
            io -= 2 * K * (N - C)
        else:
            io -= 2 * M * (K - C)
        hook(2.0 * M * N * K, ev0, ev1, io)


def conv_gemm_supported(H, W, C, taps=()):
    """Geometry the TMA tap loop handles (pg_gemm_bf16_conv_taps): the image, the channel count and every tap offset
    within MAX_TAP_OFFSET; other convolutions go through pg_tap_gather."""
    return (C % 64 == 0 and 1 <= W <= 64 and 64 % W == 0 and (H * W) % 128 == 0
            and all(abs(dy) <= MAX_TAP_OFFSET and abs(dx) <= MAX_TAP_OFFSET for dy, dx in taps))


def _epilogue(M, N, bias, aux, dact, res0, res1, out_bf16, out_pre, out_f32, act, accumulate, alpha, bias_grad=None):
    e = GemmEpilogue()
    if bias_grad is not None:
        assert bias_grad.dtype == torch.float32 and bias_grad.numel() >= M and bias_grad.is_contiguous()
    e.bias_grad = _ptr(bias_grad)
    e.bias = _ptr(bias)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() >= N and bias.is_contiguous()
    ld_res, res_dtype = 0, None
    for r in (res0, res1):
        if r is not None:
            assert r.dtype in (torch.float32, torch.bfloat16) and r.shape[0] >= M
            assert res_dtype in (None, r.dtype), "res0/res1 must share a dtype"
            p, ld = _pm(r)
            assert ld_res in (0, ld), "res0/res1 must share a pitch"
            ld_res, res_dtype = ld, r.dtype
    e.res0, e.res1, e.ld_res = _ptr(res0), _ptr(res1), ld_res
    if res_dtype == torch.bfloat16:
        act = act | ACT_RES_BF16
    if aux is not None:
        assert aux.dtype == torch.bfloat16
        e.aux, e.ld_aux = _pm(aux)
    if out_bf16 is not None:
        assert out_bf16.dtype == torch.bfloat16 and out_bf16.shape[0] >= M
        e.out_bf16, e.ld_out_bf16 = _pm(out_bf16)
    if out_pre is not None:
        assert out_pre.dtype == torch.bfloat16 and out_pre.shape[0] >= M
        e.out_pre, e.ld_out_pre = _pm(out_pre)
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.shape[0] >= M
        e.out_f32, e.ld_out_f32 = _pm(out_f32)
    e.act, e.dact, e.accumulate, e.alpha = act, dact, int(accumulate), alpha
    return e


@_device_guarded
def colsum(x, out, accumulate=False):
    lib = load()
    p, ld = _pm(x)
    P, C = x.shape
    assert out.dtype == torch.float32 and out.numel() >= C
    fn = lib.pg_colsum_bf16 if x.dtype == torch.bfloat16 else lib.pg_colsum_f32
    _check(fn(p, ld, P, C, _ptr(out), int(accumulate), _stream()), "pg_colsum")


# ------------------------------------------------------------------------------------------------
# LayerNorm / gated activation / loss / converters
# ------------------------------------------------------------------------------------------------
@_device_guarded
def layernorm_fwd(x, gamma, beta, eps, y_bf16=None, y_f32=None, mean=None, rstd=None):
    """LayerNorm over the gamma.numel() = C first columns of x [P, ld >= C]; columns C..ld of the outputs become zero."""
    lib = load()
    P, ld = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    _check(lib.pg_layernorm_fwd_ld(_ptr(x), _ptr(gamma), _ptr(beta), P, gamma.numel(), ld, eps, _ptr(y_bf16), _ptr(y_f32),
                                   _ptr(mean), _ptr(rstd), _stream()), "pg_layernorm_fwd")


@_device_guarded
def layernorm_bwd(dy, x, gamma, mean, rstd, dres0=None, dres1=None, dx_f32=None, dx_bf16=None, dgamma=None,
                  dbeta=None, dx_colsum=None):
    """Backward of layernorm_fwd on rows of pitch x.shape[1] (every [P, *] tensor shares it); statistics over C."""
    lib = load()
    P, ld = x.shape
    assert dy.is_contiguous() and x.is_contiguous()
    dy_b = _ptr(dy) if dy.dtype == torch.bfloat16 else None
    dy_f = _ptr(dy) if dy.dtype == torch.float32 else None
    _check(lib.pg_layernorm_bwd_ld(dy_b, dy_f, _ptr(x), _ptr(gamma), _ptr(mean), _ptr(rstd), P, gamma.numel(), ld,
                                   _ptr(dres0), _ptr(dres1), _ptr(dx_f32), _ptr(dx_bf16), _ptr(dgamma), _ptr(dbeta),
                                   _ptr(dx_colsum), _stream()),
           "pg_layernorm_bwd")


@_device_guarded
def gated_act_fwd(x, y, act):
    lib = load()
    P, C2 = x.shape
    assert x.is_contiguous() and y.is_contiguous() and y.shape == (P, C2 // 2)
    _check(lib.pg_gated_act_fwd(_ptr(x), int(x.dtype == torch.float32), P, C2 // 2, act, _ptr(y),
                                int(y.dtype == torch.float32), _stream()), "pg_gated_act_fwd")


@_device_guarded
def gated_res_fwd(x, res, y, act):
    """y = res + act(x[:, :C]) * sigmoid(x[:, C:]); res, y fp32 [P, C]."""
    P, C2 = x.shape
    assert x.is_contiguous() and res.is_contiguous() and y.is_contiguous() and res.dtype == y.dtype == torch.float32
    _check(load().pg_gated_res_fwd(_ptr(x), int(x.dtype == torch.float32), _ptr(res), P, C2 // 2, act, _ptr(y), _stream()),
           "pg_gated_res_fwd")


@_device_guarded
def dact_from_out(dy, ya, act, out):
    """out = bf16(dy * act'(pre)) with ya = act(pre) (relu / elu)."""
    assert dy.is_contiguous() and ya.is_contiguous() and out.is_contiguous() and ya.dtype == out.dtype == torch.bfloat16
    _check(load().pg_dact_from_out(_ptr(dy), int(dy.dtype == torch.float32), _ptr(ya), dy.numel(), act, _ptr(out), _stream()),
           "pg_dact_from_out")


@_device_guarded
def gated_act_bwd(x, dy, dx, act):
    lib = load()
    P, C2 = x.shape
    assert x.is_contiguous() and dy.is_contiguous() and dx.is_contiguous()
    _check(lib.pg_gated_act_bwd(_ptr(x), int(x.dtype == torch.float32), _ptr(dy), int(dy.dtype == torch.float32), P,
                                C2 // 2, act, _ptr(dx), int(dx.dtype == torch.float32), _stream()), "pg_gated_act_bwd")


@_device_guarded
def bce_logits(logits, target, grad_scale, loss_sum, dlogits=None):
    lib = load()
    assert logits.dtype == torch.float32 and target.dtype == torch.float32
    assert logits.is_contiguous() and target.is_contiguous() and logits.numel() == target.numel()
    _check(lib.pg_bce_logits_fwd_bwd(_ptr(logits), _ptr(target), logits.numel(), grad_scale, _ptr(loss_sum),
                                     _ptr(dlogits), _stream()), "pg_bce_logits_fwd_bwd")


@_device_guarded
def nchw_to_pm(x, out):
    """x: [N, C, H, W] fp32 contiguous -> out: [N*H*W, >=C] bf16/fp32 (pixel-major)."""
    lib = load()
    N, C, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    p, ld = _pm(out)
    _check(lib.pg_nchw_to_pm(_ptr(x), N, C, H * W, p, int(out.dtype == torch.float32), ld, _stream()), "pg_nchw_to_pm")


@_device_guarded
def pm_to_nchw(x_pm, out, act=ACT_NONE):
    lib = load()
    N, C, H, W = out.shape
    assert out.dtype == torch.float32 and out.is_contiguous()
    p, ld = _pm(x_pm)
    _check(lib.pg_pm_to_nchw(p, int(x_pm.dtype == torch.float32), ld, N, C, H * W, act, _ptr(out), _stream()),
           "pg_pm_to_nchw")


@_device_guarded
def dact_mul(dy, pre, act, out):
    """out = bf16(dy * act'(pre)); dy/out bf16 [P, C] views, pre fp32."""
    lib = load()
    (dp, ldd), (pp, ldp), (op, ldo) = _pm(dy), _pm(pre), _pm(out)
    P, C = dy.shape
    assert dy.dtype == torch.bfloat16 and pre.dtype == torch.float32 and out.dtype == torch.bfloat16
    _check(lib.pg_dact_mul(dp, ldd, pp, ldp, P, C, act, op, ldo, _stream()), "pg_dact_mul")


@_device_guarded
def act_cast(x, act, out):
    """out = bf16(act(x)); x: [P, C] fp32 or bf16 view, out: [P, C] bf16 view."""
    lib = load()
    (xp, ldx), (op, ldo) = _pm(x), _pm(out)
    P, C = x.shape
    assert out.dtype == torch.bfloat16 and out.shape == x.shape and x.dtype in (torch.float32, torch.bfloat16)
    _check(lib.pg_act_cast_bf16(xp, int(x.dtype == torch.float32), ldx, P, C, act, op, ldo, _stream()), "pg_act_cast_bf16")


@_device_guarded
def cast_bf16(x, y):
    lib = load()
    assert x.dtype == torch.float32 and y.dtype == torch.bfloat16 and x.is_contiguous() and y.is_contiguous()
    _check(lib.pg_cast_f32_to_bf16(_ptr(x), _ptr(y), x.numel(), _stream()), "pg_cast_f32_to_bf16")


# ------------------------------------------------------------------------------------------------
# Attention / small conv
# ------------------------------------------------------------------------------------------------
@_device_guarded
def causal_attn_fwd(q, k, v, o, lse, N, S, H, dk, dv, strict, impl=0, dk_true=None):
    """dk is the column width of a head slot; dk_true (default dk) sets the 1/sqrt(dk) scale."""
    lib = load()
    (qp, ldq), (kp, ldk), (vp, ldv), (op, ldo) = _pm(q), _pm(k), _pm(v), _pm(o)
    scale = 1.0 / math.sqrt(dk_true or dk)
    _check(lib.pg_causal_attn_fwd(qp, ldq, kp, ldk, vp, ldv, op, ldo, _ptr(lse), N, S, H, dk, dv, scale, int(strict),
                                  impl, _stream()), "pg_causal_attn_fwd")


@_device_guarded
def causal_attn_bwd(q, k, v, o, do, lse, delta, dq_accum, dq, dk_, dv_, N, S, H, dk, dv, strict, impl=0, dk_true=None):
    lib = load()
    (qp, ldq), (kp, ldk), (vp, ldv), (op, ldo), (dop, lddo) = _pm(q), _pm(k), _pm(v), _pm(o), _pm(do)
    (dqp, lddq), (dkp, lddk), (dvp, lddv) = _pm(dq), _pm(dk_), _pm(dv_)
    scale = 1.0 / math.sqrt(dk_true or dk)
    _check(lib.pg_causal_attn_bwd(qp, ldq, kp, ldk, vp, ldv, op, ldo, dop, lddo, _ptr(lse), _ptr(delta),
                                  _ptr(dq_accum), dqp, lddq, dkp, lddk, dvp, lddv, N, S, H, dk, dv, scale, int(strict),
                                  impl, _stream()), "pg_causal_attn_bwd")


@_device_guarded
def conv_small_fwd(x, w, bias, pad, out_f32=None, out_bf16=None, act_bf16=ACT_NONE, pre_act=ACT_NONE, dilation=(1, 1)):
    lib = load()
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = w.shape
    assert x.is_contiguous() and w.is_contiguous() and x.dtype == torch.float32 and w.dtype == torch.float32
    _check(lib.pg_conv_small_fwd_d(_ptr(x), _ptr(w), _ptr(bias), N, Cin, H, W, Cout, kh, kw, pad[0], pad[1], dilation[0],
                                   dilation[1], pre_act, _ptr(out_f32), _ptr(out_bf16), act_bf16, _stream()),
           "pg_conv_small_fwd")


@_device_guarded
def conv_small_bwd(x, w, dy_pm, pad, dw=None, dbias=None, dx=None, pre_act=ACT_NONE, dilation=(1, 1)):
    lib = load()
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = w.shape
    assert dy_pm.dtype == torch.float32 and dy_pm.is_contiguous()
    _check(lib.pg_conv_small_bwd_d(_ptr(x), _ptr(w), _ptr(dy_pm), N, Cin, H, W, Cout, kh, kw, pad[0], pad[1], dilation[0],
                                   dilation[1], pre_act, _ptr(dw), _ptr(dbias), _ptr(dx), _stream()), "pg_conv_small_bwd")


@_device_guarded
def linear_attn_fwd(q, k, v, out):
    """q, k: [B, L, d]; v, out: [B, L, dv]; fp32 contiguous."""
    B, Lq, d = q.shape
    for t in (q, k, v, out):
        assert t.dtype == torch.float32 and t.is_contiguous()
    _check(load().pg_linear_attn_fwd(_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, Lq, d, v.shape[2], _stream()), "pg_linear_attn_fwd")


@_device_guarded
def linear_attn_bwd(q, k, v, g, dq, dk, dv):
    B, Lq, d = q.shape
    for t in (q, k, v, g, dq, dk, dv):
        assert t.dtype == torch.float32 and t.is_contiguous()
    _check(load().pg_linear_attn_bwd(_ptr(q), _ptr(k), _ptr(v), _ptr(g), _ptr(dq), _ptr(dk), _ptr(dv), B, Lq, d, v.shape[2],
                                     _stream()), "pg_linear_attn_bwd")


@_device_guarded
def cast_multi(src_ptrs, dst_ptrs, numel, chunks, n_chunks, chunk_elems):
    _check(load().pg_cast_multi_bf16(_ptr(src_ptrs), _ptr(dst_ptrs), _ptr(numel), _ptr(chunks), n_chunks, chunk_elems,
                                     _stream()), "pg_cast_multi_bf16")


@_device_guarded
def grad_sqnorm(grad_ptrs, numel, chunks, n_chunks, chunk_elems, partials):
    _check(load().pg_grad_sqnorm(_ptr(grad_ptrs), _ptr(numel), _ptr(chunks), n_chunks, chunk_elems, _ptr(partials),
                                 _stream()), "pg_grad_sqnorm")


@_device_guarded
def adam_step(param_ptrs, grad_ptrs, m_ptrs, v_ptrs, numel, chunks, n_chunks, chunk_elems, partials, max_norm, skip_above,
              lr, beta1, beta2, eps, step, norm_out):
    _check(load().pg_adam_step(_ptr(param_ptrs), _ptr(grad_ptrs), _ptr(m_ptrs), _ptr(v_ptrs), _ptr(numel), _ptr(chunks),
                               n_chunks, chunk_elems, _ptr(partials), max_norm, skip_above, lr, beta1, beta2, eps, step,
                               _ptr(norm_out), _stream()), "pg_adam_step")


@_device_guarded
def adabelief_step(param_ptrs, grad_ptrs, m_ptrs, v_ptrs, numel, chunks, n_chunks, chunk_elems, partials, n_partials,
                   max_norm, skip_above, lr, beta1, beta2, step, norm_out):
    """One parameter group's AdaBelief update: `chunks` holds its n_chunks rows of the chunk table, `partials` the
    n_partials norm partials of every group (see pg_adabelief_step)."""
    _check(load().pg_adabelief_step(_ptr(param_ptrs), _ptr(grad_ptrs), _ptr(m_ptrs), _ptr(v_ptrs), _ptr(numel),
                                    _ptr(chunks), n_chunks, chunk_elems, _ptr(partials), n_partials, max_norm,
                                    skip_above, lr, beta1, beta2, step, _ptr(norm_out), _stream()), "pg_adabelief_step")


def _rezero_operands(*tensors):
    for t in tensors:
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous(), "ReZero operands are contiguous fp32 tensors"


@_device_guarded
def rezero_fwd(x, f, alpha, y):
    """y = x + alpha f elementwise (alpha a one-element fp32 tensor on the device)."""
    _rezero_operands(x, f, alpha, y)
    assert x.numel() == f.numel() == y.numel() and alpha.numel() == 1
    _check(load().pg_rezero_fwd(_ptr(x), _ptr(f), _ptr(alpha), x.numel(), _ptr(y), _stream()), "pg_rezero_fwd")


@_device_guarded
def rezero_bwd(dy, f, alpha, df=None, dalpha=None):
    """df = alpha dy and / or dalpha[0] = sum(dy f) (fixed order); either may be None."""
    _rezero_operands(dy, f, alpha, df, dalpha)
    assert (df is None or df.numel() == dy.numel()) and (dalpha is None or (dalpha.numel() == 1 and f.numel() == dy.numel()))
    _check(load().pg_rezero_bwd(_ptr(dy), _ptr(f), _ptr(alpha), dy.numel(), _ptr(df), _ptr(dalpha), _stream()),
           "pg_rezero_bwd")


def _int_array(vals):
    arr = (ctypes.c_int * len(vals))(*[int(v) for v in vals])
    return arr


@_device_guarded
def tap_gather(x_pm, N, H, W, C, taps, act, out):
    """x_pm: [P, >=C] bf16; taps: list of (dy, dx); out: [P, T*C] bf16 contiguous."""
    lib = load()
    p, ld = _pm(x_pm)
    dy, dx = _int_array([t[0] for t in taps]), _int_array([t[1] for t in taps])
    assert out.is_contiguous() and out.dtype == torch.bfloat16 and x_pm.dtype == torch.bfloat16
    _check(lib.pg_tap_gather(p, ld, N, H, W, C, len(taps), ctypes.cast(dy, ctypes.c_void_p), ctypes.cast(dx, ctypes.c_void_p),
                             act, _ptr(out), _stream()), "pg_tap_gather")


@_device_guarded
def tap_scatter(dxcat, N, H, W, C, taps, act, x_pre, dx_f32=None, dx_bf16=None):
    lib = load()
    assert dxcat.is_contiguous() and dxcat.dtype == torch.bfloat16
    dy, dx = _int_array([t[0] for t in taps]), _int_array([t[1] for t in taps])
    pre_p, pre_ld = (None, 0) if x_pre is None else _pm(x_pre)
    tgt = dx_f32 if dx_f32 is not None else dx_bf16
    _, ld_dx = _pm(tgt)
    if dx_f32 is not None and dx_bf16 is not None:
        assert dx_bf16.stride(0) == ld_dx
    _check(lib.pg_tap_scatter(_ptr(dxcat), N, H, W, C, len(taps), ctypes.cast(dy, ctypes.c_void_p),
                              ctypes.cast(dx, ctypes.c_void_p), act, pre_p, pre_ld, _ptr(dx_f32), _ptr(dx_bf16), ld_dx,
                              _stream()), "pg_tap_scatter")


@_device_guarded
def made_mask_cast(w, conn_in, conn_out, strict, w_bf16, mask=None):
    """w *= mask (in place, through the raw pointer) and w_bf16 = bf16(w * mask) for the connectivity mask of one MADE
    layer (see pg_made_mask_cast); mask: the layer's fp32 `mask` buffer to rewrite, or None."""
    rows, cols = w.shape
    assert w.dtype == torch.float32 and w.is_contiguous()
    assert conn_in.dtype == conn_out.dtype == torch.int32 and conn_in.numel() == cols and conn_out.numel() == rows
    assert w_bf16.dtype == torch.bfloat16 and w_bf16.is_contiguous()
    if mask is not None:
        assert mask.dtype == torch.float32 and mask.is_contiguous() and mask.shape == w.shape
    _check(load().pg_made_mask_cast(_ptr(w), rows, cols, _ptr(conn_in), _ptr(conn_out), int(strict), _ptr(w_bf16),
                                    w_bf16.shape[0], w_bf16.shape[1], _ptr(mask), _stream()), "pg_made_mask_cast")


@_device_guarded
def made_sample_step(pos, order, n, canvas, x_in, w1t, h1, update, w_out, b_out, logits, a1=None, hl=None):
    """One step of MADE's incremental sampler (see pg_made_sample_step).  pos: int64 device scalar; order: int32 [D];
    canvas, x_in: fp32 [n, D]; w1t: fp32 [D, H]; h1: fp32 [n, H]; w_out: fp32 [D, K]; a1, hl: bf16 [n, >= H / K]."""
    D = order.numel()
    assert pos.dtype == torch.int64 and order.dtype == torch.int32
    for t in (canvas, x_in, w1t, h1, w_out, b_out, logits):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous())
    H = h1.shape[1] if h1 is not None else 0
    a1_p, ld_a1 = _pm(a1) if a1 is not None else (None, 0)
    hl_p, ld_hl = _pm(hl) if hl is not None else (None, 0)
    K = w_out.shape[1] if w_out is not None else 0
    _check(load().pg_made_sample_step(_ptr(pos), _ptr(order), D, n, _ptr(canvas), _ptr(x_in), _ptr(w1t), _ptr(h1), H,
                                      update, a1_p, ld_a1, hl_p, ld_hl, _ptr(w_out), K, _ptr(b_out), _ptr(logits),
                                      _stream()), "pg_made_sample_step")


def _fp32_contiguous(*tensors):
    for t in tensors:
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous()), "expected contiguous fp32 tensors"


@_device_guarded
def nade_fwd(x, u, in_w, in_b, h_w, h_b, p, xt, ckpt=None):
    """NADE's scan (see pg_nade_fwd): x, u, p, xt [n, D]; in_w [H, D]; in_b [H]; h_w [D, H]; h_b [D];
    ckpt [n, ceil(D / NADE_CHUNK), H] or None.  p may be None (sampling)."""
    n, D = x.shape
    H = in_b.numel()
    _fp32_contiguous(x, u, in_w, in_b, h_w, h_b, p, xt, ckpt)
    assert u.shape == xt.shape == (n, D) and in_w.shape == (H, D) and h_w.shape == (D, H) and h_b.numel() == D
    assert p is None or p.shape == (n, D)
    assert ckpt is None or ckpt.shape == (n, -(-D // NADE_CHUNK), H)
    _check(load().pg_nade_fwd(_ptr(x), _ptr(u), _ptr(in_w), _ptr(in_b), _ptr(h_w), _ptr(h_b), n, D, H, _ptr(p), _ptr(xt),
                              _ptr(ckpt), _stream()), "pg_nade_fwd")


@_device_guarded
def nade_bwd(x, xt, p, g, ckpt, in_w, h_w, d_in_w, d_in_b, d_h_w, d_h_b, dx=None):
    """Adds the gradients of one NADE forward (see pg_nade_bwd) to d_in_w [H, D], d_in_b [H], d_h_w [D, H], d_h_b [D]
    and, when given, dx [n, D]."""
    n, D = x.shape
    H = in_w.shape[0]
    _fp32_contiguous(x, xt, p, g, ckpt, in_w, h_w, d_in_w, d_in_b, d_h_w, d_h_b, dx)
    assert xt.shape == p.shape == g.shape == (n, D) and ckpt.shape == (n, -(-D // NADE_CHUNK), H)
    assert d_in_w.shape == in_w.shape == (H, D) and d_h_w.shape == h_w.shape == (D, H)
    assert d_in_b.numel() == H and d_h_b.numel() == D and (dx is None or dx.shape == (n, D))
    _check(load().pg_nade_bwd(_ptr(x), _ptr(xt), _ptr(p), _ptr(g), _ptr(ckpt), _ptr(in_w), _ptr(h_w), n, D, H,
                              _ptr(d_in_w), _ptr(d_in_b), _ptr(d_h_w), _ptr(d_h_b), _ptr(dx), _stream()), "pg_nade_bwd")


def _fvbn_table(params, D):
    assert params.dtype == torch.int64 and params.is_contiguous() and params.numel() == 2 * D, \
        "expected the int64 table of the 2 * D parameter addresses"


@_device_guarded
def fvbn_fwd(params, x, logits):
    """FVBN's logits (see pg_fvbn_fwd): params int64 [2 * D] (row weights, then biases); x, logits fp32 [n, D]."""
    n, D = x.shape
    _fvbn_table(params, D)
    _fp32_contiguous(x, logits)
    assert logits.shape == (n, D)
    _check(load().pg_fvbn_fwd(_ptr(params), _ptr(x), n, D, _ptr(logits), _stream()), "pg_fvbn_fwd")


@_device_guarded
def fvbn_bwd(params, x, g, dw, db, dx=None):
    """Adds FVBN's weight gradients to dw (packed, [1 + D (D - 1) / 2]) and db [D]; writes dx [n, D] when given (see
    pg_fvbn_bwd)."""
    n, D = x.shape
    _fvbn_table(params, D)
    _fp32_contiguous(x, g, dw, db, dx)
    assert g.shape == (n, D) and dw.numel() == 1 + D * (D - 1) // 2 and db.numel() == D
    assert dx is None or dx.shape == (n, D)
    _check(load().pg_fvbn_bwd(_ptr(params), _ptr(x), _ptr(g), n, D, _ptr(dw), _ptr(db), _ptr(dx), _stream()),
           "pg_fvbn_bwd")


@_device_guarded
def fvbn_sample_step(params, pos, canvas, logits):
    """The [n, c] logits of pixel *pos of the canvas [n, c, h, w] (see pg_fvbn_sample_step); pos: int64 device scalar."""
    n, c, h, w = canvas.shape
    _fvbn_table(params, c * h * w)
    _fp32_contiguous(canvas, logits)
    assert pos.dtype == torch.int64 and logits.shape == (n, c)
    _check(load().pg_fvbn_sample_step(_ptr(params), _ptr(pos), _ptr(canvas), n, c, h * w, _ptr(logits), _stream()),
           "pg_fvbn_sample_step")


def _nice_halves(n, D, *halves):
    """Checks fp32 [n, ld] half buffers of one pitch ld >= D - D/2 (bf16 ones too, for the operand copies); returns ld."""
    ld = None
    for t in halves:
        if t is None:
            continue
        assert t.dim() == 2 and t.is_contiguous() and t.shape[0] == n and t.dtype in (torch.float32, torch.bfloat16)
        assert ld in (None, t.shape[1]), "the halves must share a pitch"
        ld = t.shape[1]
    assert ld is not None and ld >= D - D // 2
    return ld


@_device_guarded
def nice_split(x, lo, hi, log_scale=None, sign=1.0, out_bf16=None, bf16_half=0):
    """x [n, D] -> the halves lo, hi [n, ld] (see pg_nice_split); optionally scaled by exp(sign * log_scale) and with a
    bf16 copy of half `bf16_half` (0 = lo, 1 = hi)."""
    n, D = x.shape
    _fp32_contiguous(x, lo, hi, log_scale)
    ld = _nice_halves(n, D, lo, hi, out_bf16)
    assert log_scale is None or log_scale.numel() == D
    _check(load().pg_nice_split(_ptr(x), n, D, _ptr(log_scale), float(sign), _ptr(lo), _ptr(hi), ld, int(bf16_half),
                                _ptr(out_bf16), _stream()), "pg_nice_split")


@_device_guarded
def nice_join(lo, hi, z, log_scale=None, sign=1.0, log_det=None):
    """z [n, D] = [lo | hi] (* exp(sign * log_scale)); log_det (fp32 device scalar) = sum(log_scale) (see pg_nice_join)."""
    n, D = z.shape
    _fp32_contiguous(lo, hi, z, log_scale, log_det)
    ld = _nice_halves(n, D, lo, hi)
    assert log_scale is None or log_scale.numel() == D
    _check(load().pg_nice_join(_ptr(lo), _ptr(hi), ld, n, D, _ptr(log_scale), float(sign), _ptr(z), _ptr(log_det),
                               _stream()), "pg_nice_join")


@_device_guarded
def nice_scale_bwd(dz, z, log_scale, g_log_det, d_lo, d_hi, d_log_scale, dm_bf16=None, bf16_half=0):
    """The scaling layer's backward (see pg_nice_scale_bwd): d_lo, d_hi = dz * exp(log_scale) as halves, optionally a bf16
    copy of one half, and d_log_scale = g_log_det + sum over images of dz * z (g_log_det: device scalar or None)."""
    n, D = dz.shape
    _fp32_contiguous(dz, z, log_scale, g_log_det, d_lo, d_hi, d_log_scale)
    ld = _nice_halves(n, D, d_lo, d_hi, dm_bf16)
    assert z.shape == (n, D) and log_scale.numel() == D and d_log_scale.numel() == D
    _check(load().pg_nice_scale_bwd(_ptr(dz), _ptr(z), _ptr(log_scale), _ptr(g_log_det), n, D, _ptr(d_lo), _ptr(d_hi),
                                    ld, int(bf16_half), _ptr(dm_bf16), _ptr(d_log_scale), _stream()),
           "pg_nice_scale_bwd")


@_device_guarded
def logistic_prior_fwd_bwd(z, log_prob, dz=None, grad_scale=1.0):
    """log_prob [n] = -sum_j softplus(z) + softplus(-z) over the rows of z [n, D]; dz = grad_scale * tanh(z / 2) when
    given (see pg_logistic_prior_fwd_bwd)."""
    n, D = z.shape
    _fp32_contiguous(z, log_prob, dz)
    assert log_prob.numel() == n and (dz is None or dz.shape == z.shape)
    _check(load().pg_logistic_prior_fwd_bwd(_ptr(z), n, D, float(grad_scale), _ptr(log_prob), _ptr(dz), _stream()),
           "pg_logistic_prior_fwd_bwd")


@_device_guarded
def attn_decode(q, k_new, v_new, k_cache, v_cache, o, pos_dev, N, S, H, dk, dv, strict, dk_true=None):
    """One new position per image against the KV caches (see pg_attn_decode); pos_dev: int32 device scalar."""
    lib = load()
    (qp, ldq), (knp, ldkn), (vnp, ldvn) = _pm(q), _pm(k_new), _pm(v_new)
    (kcp, ldkc), (vcp, ldvc), (op, ldo) = _pm(k_cache), _pm(v_cache), _pm(o)
    assert pos_dev.dtype == torch.int32 and pos_dev.is_cuda
    scale = 1.0 / math.sqrt(dk_true or dk)
    _check(lib.pg_attn_decode(qp, ldq, knp, ldkn, vnp, ldvn, kcp, ldkc, vcp, ldvc, op, ldo, _ptr(pos_dev), N, S, H, dk, dv,
                              scale, int(strict), _stream()), "pg_attn_decode")


@_device_guarded
def strided_gather(x_pm, rows, spatial, C, taps, stride, out):
    """X_cat [N*Hg*Wg, T*C] bf16 of x_pm [N*Hs*Ws, >=C] bf16 (see pg_strided_gather); rows = (N, Hg, Wg), spatial =
    (N, Hs, Ws)."""
    p, ld = _pm(x_pm)
    n, hg, wg = rows
    _, hs, ws = spatial
    assert x_pm.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and out.is_contiguous()
    assert x_pm.shape[0] == n * hs * ws and out.shape == (n * hg * wg, len(taps) * C)
    dy, dx = _int_array([t[0] for t in taps]), _int_array([t[1] for t in taps])
    _check(load().pg_strided_gather(p, ld, n, hg, wg, hs, ws, C, len(taps), stride, ctypes.cast(dy, ctypes.c_void_p),
                                    ctypes.cast(dx, ctypes.c_void_p), _ptr(out), _stream()), "pg_strided_gather")


@_device_guarded
def strided_scatter(ycat, rows, spatial, C, taps, stride, *, bias=None, act=ACT_NONE, dact=ACT_NONE, x_pre=None,
                    out_f32=None, out_bf16=None):
    """The adjoint of strided_gather: out [N*Hs*Ws, C] = sum of Y_cat's taps (+ bias, * dact'(x_pre)); out_f32 gets the
    sum, out_bf16 act(sum) (see pg_strided_scatter)."""
    n, hg, wg = rows
    _, hs, ws = spatial
    assert ycat.dtype in (torch.float32, torch.bfloat16) and ycat.is_contiguous()
    assert ycat.shape == (n * hg * wg, len(taps) * C)
    assert bias is None or (bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() <= C)
    outs = [o for o in (out_f32, out_bf16) if o is not None]
    _, ld = _pm(outs[0])
    for o in outs:
        assert o.shape[0] == n * hs * ws and o.stride(0) == ld
    assert out_f32 is None or out_f32.dtype == torch.float32
    assert out_bf16 is None or out_bf16.dtype == torch.bfloat16
    pre_p, pre_ld = (None, 0) if x_pre is None else _pm(x_pre)
    assert x_pre is None or x_pre.dtype == torch.bfloat16
    dy, dx = _int_array([t[0] for t in taps]), _int_array([t[1] for t in taps])
    _check(load().pg_strided_scatter(_ptr(ycat), int(ycat.dtype == torch.float32), n, hg, wg, hs, ws, C, len(taps),
                                     stride, ctypes.cast(dy, ctypes.c_void_p), ctypes.cast(dx, ctypes.c_void_p),
                                     _ptr(bias), 0 if bias is None else bias.numel(), act, dact, pre_p, pre_ld,
                                     _ptr(out_f32), _ptr(out_bf16), ld, _stream()), "pg_strided_scatter")


@_device_guarded
def vae_latent_fwd(h, eps, z, kl):
    """z (bf16 [n*hw, ld_z]) and kl (fp32 [n]) from h (fp32 [n*hw, >=2L]) and eps (fp32 [n, L, h, w]); see
    pg_vae_latent_fwd."""
    n, L = eps.shape[:2]
    hw = eps[0, 0].numel()
    hp, ld_h = _pm(h)
    zp, ld_z = _pm(z)
    _fp32_contiguous(eps, kl)
    assert h.dtype == torch.float32 and z.dtype == torch.bfloat16 and kl.numel() == n
    assert h.shape[0] == n * hw and z.shape[0] == n * hw
    assert z.shape[1] == ld_z, "vae_latent_fwd writes every column of z's pitch: z must be a whole matrix, not a view"
    _check(load().pg_vae_latent_fwd(hp, ld_h, _ptr(eps), n, L, hw, zp, ld_z, _ptr(kl), _stream()), "pg_vae_latent_fwd")


@_device_guarded
def vae_latent_bwd(h, eps, dz, g_kl, dh):
    """dh (bf16 [n*hw, ld_dh]) from dz (bf16 [n*hw, >=L]) and g_kl (fp32 [n] or None); see pg_vae_latent_bwd."""
    n, L = eps.shape[:2]
    hw = eps[0, 0].numel()
    hp, ld_h = _pm(h)
    dzp, ld_dz = _pm(dz)
    dhp, ld_dh = _pm(dh)
    _fp32_contiguous(eps, g_kl)
    assert h.dtype == torch.float32 and dz.dtype == torch.bfloat16 and dh.dtype == torch.bfloat16
    assert h.shape[0] == dz.shape[0] == dh.shape[0] == n * hw and (g_kl is None or g_kl.numel() == n)
    assert dh.shape[1] == ld_dh, "vae_latent_bwd writes every column of dh's pitch: dh must be a whole matrix, not a view"
    _check(load().pg_vae_latent_bwd(hp, ld_h, _ptr(eps), dzp, ld_dz, _ptr(g_kl), n, L, hw, dhp, ld_dh, _stream()),
           "pg_vae_latent_bwd")


# ------------------------------------------------------------------------------------------------
# VeryDeepVAE (scalar kernels: any pitch, column views welcome)
# ------------------------------------------------------------------------------------------------
def _f32_pm(t):
    assert t.dtype == torch.float32, f"expected an fp32 pixel-major matrix, got {t.dtype}"
    return _pm(t)


@_device_guarded
def gelu_cast(x, g, d):
    """g = bf16(GELU(x)), d = bf16(GELU'(x)) for x fp32 [P, C]; g and d are bf16 [P, width >= C] views with one pitch,
    zero in their columns >= C (see pg_gelu_cast)."""
    xp, ldx = _f32_pm(x)
    (gp, ld), (dp, ldd) = _pm(g), _pm(d)
    P, C = x.shape
    assert g.dtype == d.dtype == torch.bfloat16 and g.shape == d.shape and g.shape[0] == P and ld == ldd
    _check(load().pg_gelu_cast(xp, ldx, P, C, g.shape[1], gp, dp, ld, _stream()), "pg_gelu_cast")


@_device_guarded
def vd_latent_fwd(prior, post, x, eps, z, s, kl_in, kl_out):
    """z (bf16 [P, ld_z], whole), s = x + p_h (fp32 [P, C]) and kl_out = kl_in + KL (when post is given); see
    pg_vd_latent_fwd."""
    n, L = eps.shape[:2]
    hw = eps[0, 0].numel()
    C = x.shape[1]
    (pp, ldp), (xp, ldx), (zp, ldz), (sp, lds) = _f32_pm(prior), _f32_pm(x), _pm(z), _f32_pm(s)
    qp, ldq = (None, 0) if post is None else _f32_pm(post)
    _fp32_contiguous(eps, kl_in, kl_out)
    assert z.dtype == torch.bfloat16 and z.shape[1] == ldz, "z must be a whole bf16 matrix: every column is written"
    assert prior.shape[0] == x.shape[0] == z.shape[0] == s.shape[0] == n * hw and s.shape[1] == C
    assert post is None or (post.shape[0] == n * hw and kl_out is not None and kl_out.numel() == n)
    _check(load().pg_vd_latent_fwd(pp, ldp, qp, ldq, xp, ldx, _ptr(eps), n, L, C, hw, zp, ldz, sp, lds, _ptr(kl_in),
                                   _ptr(kl_out), _stream()), "pg_vd_latent_fwd")


@_device_guarded
def vd_latent_bwd(prior, post, eps, dz, g_kl, dsum, dprior, dpost):
    """dprior (bf16 [P, >= 2L + C], whole) and dpost (bf16 [P, >= 2L], whole, or None without post); see
    pg_vd_latent_bwd."""
    n, L = eps.shape[:2]
    hw = eps[0, 0].numel()
    C = dsum.shape[1]
    (pp, ldp), (sp, lds), (dpp, lddp) = _f32_pm(prior), _f32_pm(dsum), _pm(dprior)
    qp, ldq = (None, 0) if post is None else _f32_pm(post)
    dqp, lddq = (None, 0) if dpost is None else _pm(dpost)
    zp, ldz = (None, 0) if dz is None else _pm(dz)
    _fp32_contiguous(eps, g_kl)
    assert dprior.dtype == torch.bfloat16 and dprior.shape[1] == lddp
    assert dpost is None or (dpost.dtype == torch.bfloat16 and dpost.shape[1] == lddq)
    assert dz is None or dz.dtype == torch.bfloat16
    _check(load().pg_vd_latent_bwd(pp, ldp, qp, ldq, _ptr(eps), zp, ldz, _ptr(g_kl), sp, lds, n, L, C, hw, dpp, lddp,
                                   dqp, lddq, _stream()), "pg_vd_latent_bwd")


@_device_guarded
def avg_pool2_fwd(x, n, h, w, y):
    """nn.AvgPool2d(2, 2) of fp32 x [n*h*w, C] into fp32 y [n*(h//2)*(w//2), C]."""
    (xp, ldx), (yp, ldy) = _f32_pm(x), _f32_pm(y)
    assert x.shape[0] == n * h * w and y.shape == (n * (h // 2) * (w // 2), x.shape[1])
    _check(load().pg_avg_pool2_fwd(xp, ldx, n, h, w, x.shape[1], yp, ldy, _stream()), "pg_avg_pool2_fwd")


@_device_guarded
def avg_pool2_bwd(dy, n, h, w, dx):
    (dyp, lddy), (dxp, lddx) = _f32_pm(dy), _f32_pm(dx)
    assert dx.shape[0] == n * h * w and dy.shape == (n * (h // 2) * (w // 2), dx.shape[1])
    _check(load().pg_avg_pool2_bwd(dyp, lddy, n, h, w, dx.shape[1], dxp, lddx, _stream()), "pg_avg_pool2_bwd")


@_device_guarded
def bias_unpool_fwd(x, bias, n, f, y):
    """y = up_f(x + bias) (x fp32 [n*s*s, C] or None, bias fp32 [1, C, s, s]) into fp32 y [n*(f s)^2, C]."""
    _, C, s, _ = bias.shape
    _fp32_contiguous(bias)
    xp, ldx = (None, 0) if x is None else _f32_pm(x)
    yp, ldy = _f32_pm(y)
    assert x is None or x.shape == (n * s * s, C)
    assert y.shape == (n * s * s * f * f, C)
    _check(load().pg_bias_unpool_fwd(xp, ldx, _ptr(bias), n, s, C, f, yp, ldy, _stream()), "pg_bias_unpool_fwd")


@_device_guarded
def bias_unpool_bwd(dy, n, f, dx, dbias):
    """dx (fp32 [n*s*s, C] or None) and dbias (fp32 [1, C, s, s], overwritten) from dy [n*(f s)^2, C]."""
    _, C, s, _ = dbias.shape
    _fp32_contiguous(dbias)
    dyp, lddy = _f32_pm(dy)
    dxp, lddx = (None, 0) if dx is None else _f32_pm(dx)
    assert dy.shape == (n * s * s * f * f, C) and (dx is None or dx.shape == (n * s * s, C))
    _check(load().pg_bias_unpool_bwd(dyp, lddy, n, s, C, f, dxp, lddx, _ptr(dbias), _stream()), "pg_bias_unpool_bwd")


def _codebook(emb, d):
    assert emb.dtype == torch.float32 and emb.is_contiguous() and emb.dim() == 2 and emb.shape[1] == d, \
        "expected a contiguous fp32 [K, d] codebook"
    return emb.shape[0]


@_device_guarded
def vq_assign(x, emb, idx, out=None, col0=0, out_cols=None, loss_sum=None):
    """idx (int32 [P]) = the nearest code of each row of x (fp32 [P, >=d]); out (bf16 or fp32 [P, ld]) gets
    x + (q - x) in columns [col0, col0 + d) and zeros up to col0 + out_cols; loss_sum (fp32 [1]) += sum (x - q)^2.
    See pg_vq_assign."""
    d = emb.shape[1]
    xp, ld_x = _pm(x)
    K = _codebook(emb, d)
    assert x.dtype == torch.float32 and idx.dtype == torch.int32 and idx.is_contiguous() and idx.numel() == x.shape[0]
    op, ld_out = (None, 0) if out is None else _pm(out)
    assert out is None or (out.dtype in (torch.float32, torch.bfloat16) and out.shape[0] == x.shape[0])
    out_cols = d if out_cols is None else out_cols
    assert loss_sum is None or (loss_sum.dtype == torch.float32 and loss_sum.numel() == 1)
    _check(load().pg_vq_assign(xp, ld_x, x.shape[0], d, _ptr(emb), K, _ptr(idx), op,
                               int(out is not None and out.dtype == torch.float32), ld_out, col0, out_cols,
                               _ptr(loss_sum), _stream()), "pg_vq_assign")


@_device_guarded
def vq_code_sums(x, idx, K, sums, counts=None, emb=None, g=None, scale=0.0):
    """sums (fp32 [K, d]) = per-code sums of the rows of x (fp32 [P, >=d]) assigned by idx, in ascending row order, or
    of ((q - x) scale) g when emb is given; counts (fp32 [K]) = rows per code.  See pg_vq_code_sums."""
    d = sums.shape[1]
    xp, ld_x = _pm(x)
    _fp32_contiguous(sums, counts, g)
    assert emb is None or _codebook(emb, d) == K
    assert idx.dtype == torch.int32 and idx.numel() == x.shape[0] and sums.shape[0] == K
    assert (emb is None) == (g is None)
    _check(load().pg_vq_code_sums(xp, ld_x, x.shape[0], d, _ptr(idx), K, _ptr(emb), _ptr(g), scale, _ptr(counts),
                                  _ptr(sums), _stream()), "pg_vq_code_sums")


@_device_guarded
def vq_ema_update(counts, sums, decay, cluster_size, embedding_avg, embedding):
    """The EMA codebook update of reference nn/utils.py, in place (see pg_vq_ema_update)."""
    K, d = embedding.shape
    _fp32_contiguous(counts, sums, cluster_size, embedding_avg, embedding)
    assert counts.numel() == cluster_size.numel() == K and sums.shape == embedding_avg.shape == (K, d)
    _check(load().pg_vq_ema_update(_ptr(counts), _ptr(sums), K, d, float(decay), float(1 - decay), _ptr(cluster_size),
                                   _ptr(embedding_avg), _ptr(embedding), _stream()), "pg_vq_ema_update")


@_device_guarded
def vq_bwd(x, emb, idx, dq, col0, g, scale, dx):
    """dx [P, ld] = dq[:, col0:col0 + d] + ((x - q) scale) g, zero beyond d; dq / dx both bf16 or both fp32 (see
    pg_vq_bwd)."""
    d = emb.shape[1]
    xp, ld_x = _pm(x)
    _codebook(emb, d)
    dqp, ld_dq = (None, 0) if dq is None else _pm(dq)
    dxp, ld_dx = _pm(dx)
    assert dx.shape[1] == ld_dx, "vq_bwd writes every column of dx's pitch: dx must be a whole matrix, not a view"
    assert dq is None or dq.dtype == dx.dtype
    assert idx.dtype == torch.int32 and idx.numel() == x.shape[0] == dx.shape[0]
    _fp32_contiguous(g)
    _check(load().pg_vq_bwd(xp, ld_x, x.shape[0], d, _ptr(emb), _ptr(idx), dqp, ld_dq, col0, _ptr(g), scale,
                            int(dx.dtype == torch.float32), dxp, ld_dx, _stream()), "pg_vq_bwd")


@_device_guarded
def mse_mean(a, b, cols, *, loss_sum=None, g=None, scale=0.0, da=None, db=None):
    """Forward (loss_sum): loss_sum += sum over the first `cols` columns of (a - b)^2; backward (g): da = ((a - b) scale)
    g, db = -da, zero in their pad columns.  a, b, da, db: fp32 [rows, pitch] (see pg_mse_mean)."""
    ap, ld_a = _pm(a)
    bp, ld_b = _pm(b)
    assert a.dtype == b.dtype == torch.float32 and a.shape[0] == b.shape[0]
    dap, ld_da = (None, 0) if da is None else _pm(da)
    dbp, ld_db = (None, 0) if db is None else _pm(db)
    for t in (da, db):
        assert t is None or (t.dtype == torch.float32 and t.shape[0] == a.shape[0] and t.shape[1] == t.stride(0))
    _fp32_contiguous(loss_sum, g)
    _check(load().pg_mse_mean(ap, ld_a, bp, ld_b, a.shape[0], cols, _ptr(g), scale, _ptr(loss_sum), dap, ld_da, dbp,
                              ld_db, _stream()), "pg_mse_mean")


MIXTURE_GAUSSIAN, MIXTURE_BERNOULLI = 0, 1  # PG_MIXTURE_* (include/pg_b200.h)


def _rows(x, t):
    """Checks queries x [N, D] and training points t [M, D] (contiguous fp32); returns (N, M, D)."""
    _fp32_contiguous(x, t)
    assert x.dim() == 2 and t.dim() == 2 and x.shape[1] == t.shape[1], (x.shape, t.shape)
    return x.shape[0], t.shape[0], t.shape[1]


@_device_guarded
def kde_gauss_fwd(x, t, bandwidth, Z, out, lse=None):
    """out [N] = logsumexp_m(-0.5 |x_n - t_m|^2 / h^2) - Z, lse [N] the logsumexp (see pg_kde_gauss_fwd)."""
    N, M, D = _rows(x, t)
    _fp32_contiguous(out, lse)
    assert out.numel() == N and (lse is None or lse.numel() == N)
    _check(load().pg_kde_gauss_fwd(_ptr(x), N, _ptr(t), M, D, float(bandwidth), float(Z), _ptr(lse), _ptr(out),
                                   _stream()), "pg_kde_gauss_fwd")


@_device_guarded
def kde_gauss_bwd(x, t, bandwidth, lse, g, dx):
    """dx [N, D] += -(g_n / h^2) sum_m w_nm (x_n - t_m), w = exp(s - lse) (see pg_kde_gauss_bwd)."""
    N, M, D = _rows(x, t)
    _fp32_contiguous(lse, g, dx)
    assert lse.numel() == N and g.numel() == N and dx.shape == x.shape
    _check(load().pg_kde_gauss_bwd(_ptr(x), N, _ptr(t), M, D, float(bandwidth), _ptr(lse), _ptr(g), _ptr(dx), _stream()),
           "pg_kde_gauss_bwd")


@_device_guarded
def kde_parzen_count(x, t, bandwidth, count=None, out=None):
    """count [N] (int32) = training rows whose every |x_d - t_d| / h <= 0.5; out [N] = log(count / M) - D log h (see
    pg_kde_parzen_count)."""
    N, M, D = _rows(x, t)
    _fp32_contiguous(out)
    assert count is None or (count.dtype == torch.int32 and count.is_contiguous() and count.numel() == N)
    assert out is None or out.numel() == N
    _check(load().pg_kde_parzen_count(_ptr(x), N, _ptr(t), M, D, float(bandwidth), _ptr(count), _ptr(out), _stream()),
           "pg_kde_parzen_count")


def _mixture_args(kind, x, mixture_logits, p0, p1):
    N, D = x.shape
    K = mixture_logits.numel()
    _fp32_contiguous(x, mixture_logits, p0, p1)
    assert kind in (MIXTURE_GAUSSIAN, MIXTURE_BERNOULLI) and p0.shape == (K, D)
    assert (p1 is not None and p1.shape == (K, D)) if kind == MIXTURE_GAUSSIAN else p1 is None
    return N, D, K


@_device_guarded
def mixture_fwd(kind, x, mixture_logits, p0, p1, a, out):
    """a [N, K] = log_softmax(mixture_logits) + sum_d term, out [N] = logsumexp_k a (see pg_mixture_fwd)."""
    N, D, K = _mixture_args(kind, x, mixture_logits, p0, p1)
    _fp32_contiguous(a, out)
    assert a.shape == (N, K) and out.numel() == N
    _check(load().pg_mixture_fwd(kind, _ptr(x), N, D, K, _ptr(mixture_logits), _ptr(p0), _ptr(p1), _ptr(a), _ptr(out),
                                 _stream()), "pg_mixture_fwd")


@_device_guarded
def mixture_bwd(kind, x, mixture_logits, p0, p1, a, out, g, dparams, dx=None):
    """dparams (flat fp32, added to) = the parameter gradients in the order of pg_mixture_bwd; dx [N, D] written when
    given."""
    N, D, K = _mixture_args(kind, x, mixture_logits, p0, p1)
    _fp32_contiguous(a, out, g, dparams, dx)
    P = 2 if kind == MIXTURE_GAUSSIAN else 1
    assert a.shape == (N, K) and out.numel() == N and g.numel() == N and dparams.numel() == P * K * D + K
    assert dx is None or dx.shape == (N, D)
    _check(load().pg_mixture_bwd(kind, _ptr(x), N, D, K, _ptr(mixture_logits), _ptr(p0), _ptr(p1), _ptr(a), _ptr(out),
                                 _ptr(g), _ptr(dparams), _ptr(dx), _stream()), "pg_mixture_bwd")


# ------------------------------------------------------------------------------------------------
# Gaussian process: fp64 GEMM, Cholesky and triangular solves
# ------------------------------------------------------------------------------------------------
GP_NB = 64  # block size of pg_gp_potrf / pg_gp_trsm


def _f64_rows(t):
    """Checks a 2-D fp64 CUDA matrix with unit inner stride; returns (ptr, pitch)."""
    if not t.is_cuda:
        raise RuntimeError("pytorch_generative_b200 kernels need CUDA tensors (there is no CPU fallback)")
    assert t.dtype == torch.float64 and t.dim() == 2 and t.stride(1) == 1, (t.dtype, t.shape, t.stride())
    return t.data_ptr(), max(t.stride(0), 1)


@_device_guarded
def gemm_f64(A, B, C, *, trans_a=False, trans_b=False, alpha=1.0, beta=0.0, lower_only=False):
    """C = alpha op(A) op(B) + beta C on fp64 [rows, cols] matrices with unit inner stride (see pg_gemm_f64)."""
    m, n = C.shape
    k = A.shape[0] if trans_a else A.shape[1]
    assert (A.shape[1] if trans_a else A.shape[0]) == m and (B.shape[1] if trans_b else B.shape[0]) == k, \
        (A.shape, B.shape, C.shape, trans_a, trans_b)
    assert (B.shape[0] if trans_b else B.shape[1]) == n, (B.shape, C.shape)
    ap, lda = _f64_rows(A)
    bp, ldb = _f64_rows(B)
    cp, ldc = _f64_rows(C)
    lda, ldb, ldc = max(lda, A.shape[1]), max(ldb, B.shape[1]), max(ldc, n)
    _check(load().pg_gemm_f64(int(trans_a), int(trans_b), m, n, k, float(alpha), ap, lda, bp, ldb, float(beta), cp, ldc,
                              int(lower_only), _stream()), "pg_gemm_f64")
    return C


@_device_guarded
def gp_potrf(A, noise, dropped):
    """A [n, n] fp64 (unit inner stride) := the lower Cholesky factor of A + noise I with the semi-definite pivot rule;
    dropped: a CUDA int32 [1] receiving the number of dropped pivots (see pg_gp_potrf)."""
    n = A.shape[0]
    assert A.shape == (n, n)
    assert dropped.dtype == torch.int32 and dropped.is_cuda and dropped.numel() >= 1
    ap, lda = _f64_rows(A)
    _check(load().pg_gp_potrf(ap, n, max(lda, n), float(noise), dropped.data_ptr(), _stream()), "pg_gp_potrf")
    return A


@_device_guarded
def gp_trsm(L, B, transpose=False):
    """B [n, ncols] (contiguous fp64) := L^-1 B or L^-T B, L [n, n] contiguous lower (see pg_gp_trsm)."""
    n = L.shape[0]
    assert L.shape == (n, n) and B.shape[0] == n and B.dim() == 2 and L.is_contiguous() and B.is_contiguous()
    lp, _ = _f64_rows(L)
    bp, _ = _f64_rows(B)
    _check(load().pg_gp_trsm(lp, n, bp, B.shape[1], int(transpose), _stream()), "pg_gp_trsm")
    return B
