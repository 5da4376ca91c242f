"""Activations in float64 and the documented error of the kernels' fp32 versions (pg_act_fwd / pg_act_bwd in
csrc/pg_common.cuh).  Shared by tests/test_conv_path_kernels_gpu.py and tests/_step_reference.py; not a test module."""

import math

import torch

U24 = 2.0 ** -24  # fp32 unit roundoff
U23 = 2.0 ** -23  # one fp32 ulp relative to the leading bit
F64 = torch.float64

NONE, RELU, GELU, ELU, TANH, GIVEN, RELU_OUT, ELU_OUT = 0, 1, 2, 3, 4, 5, 6, 7
ACT_NAMES = {NONE: "none", RELU: "relu", GELU: "gelu", ELU: "elu", TANH: "tanh", GIVEN: "given", RELU_OUT: "relu_out",
             ELU_OUT: "elu_out"}


def act64(act, x):
    x = x.to(F64)
    if act == RELU:
        return x.clamp_min(0)
    if act == GELU:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    if act == ELU:
        return torch.where(x > 0, x, torch.expm1(x))
    if act == TANH:
        return torch.tanh(x)
    assert act == NONE
    return x


def dact64(act, x):
    """act'(pre) at x = pre; for GIVEN / *_OUT the operand semantics of pg_gemm_epilogue.dact."""
    x = x.to(F64)
    one = torch.ones_like(x)
    if act in (RELU, RELU_OUT):
        return (x > 0).to(F64)
    if act == GELU:
        return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    if act == ELU:
        return torch.where(x > 0, one, torch.exp(x))
    if act == TANH:
        return 1 - torch.tanh(x) ** 2
    if act == GIVEN:
        return x
    if act == ELU_OUT:
        return torch.where(x > 0, one, x + 1)
    assert act == NONE
    return one


def _gelu_fit_tanh(x):
    """The kernels' GELU fit (pg_common.cuh): q(x) and t = tanh(q(x)) in float64, with q's clamp to [-8, 8]."""
    xc = x.clamp(-8, 8)
    x2 = xc * xc
    q = xc * ((x2 * -0.0003563930330798993 + 0.037032072878891306) * x2 + 0.7974856909542073)
    qp = (x2 * -0.0017819651653994965 + 0.11109621863667392) * x2 + 0.7974856909542073
    return xc, qp, torch.tanh(q)


def act_err(act, x):
    """(r, a): |kernel act(x) - act(x)| <= r |act(x)| + a for the fp32 pg_act_fwd at x.
    GELU = 0.5 x (1 + tanh(q(x))) with q fitted: the fit itself is within 2.8e-5 of erf-GELU (2.77e-5 at its worst,
    x = -1.31), and tanh.approx is within 2^-11 of tanh relative (PTX ISA), which moves the result by up to
    0.5 |x t| 2^-11.  (The fit's 2.8e-5 alone does not hold on the device: an H100 run reached 3.2e-5.)  ELU: expm1f,
    1 ulp; TANH: tanhf, 2 ulp (CUDA math API accuracy tables): 2 ulp = 2^-22 relative covers both."""
    if act == GELU:
        x = x.to(F64)
        _, _, t = _gelu_fit_tanh(x)
        return 0.0, 2.8e-5 + 0.5 * (x * t).abs() * 2.0 ** -11
    return {NONE: (0.0, 0.0), RELU: (0.0, 0.0), ELU: (2 * U23, 0.0), TANH: (2 * U23, 0.0)}[act]


def deriv_err(act, x):
    """(r, a) of the fp32 pg_act_bwd at x (x is the operand the kernel reads: pre, the derivative, or the activated value).
    GELU': the derivative of the same fit, d = x q' (1 - t^2) / 2 + (1 + t) / 2, is within 1.2e-4 of erf-GELU's with an
    exact tanh; tanh.approx's 2^-11 |t| moves it by |dd/dt| = |1/2 - x q' t| times that.  ELU': __expf,
    (2 + 1.173 |x|) ulp (CUDA math API), taken as (3 + 1.2 |x|) 2^-23 relative.  TANH': 1 - t^2 with t = tanhf(x) within
    2 ulp (<= 2^-23 absolute for |t| < 1) and one rounding of t^2: |err| <= 2 |t| 2^-23 + 2^-24 < 2^-21.  ELU_OUT: x + 1
    rounded once (<= 2^-24, the result is <= 1).  RELU / RELU_OUT / GIVEN / NONE are exact."""
    x = x.to(F64)
    if act == GELU:
        xc, qp, t = _gelu_fit_tanh(x)
        return 0.0, 1.2e-4 + (0.5 - xc * qp * t).abs() * t.abs() * 2.0 ** -11
    if act == ELU:
        return (3 + 1.2 * x.abs()) * U23, 0.0
    if act == TANH:
        return 0.0, 2.0 ** -21
    if act == ELU_OUT:
        return 0.0, U24
    return 0.0, 0.0
