"""Activations and the gate in float64 and the documented error of the kernels' fp32 versions (pg_act_fwd / pg_act_bwd in
csrc/pg_common.cuh, the gated kernels of csrc/pg_elementwise.cu).  Shared by tests/test_conv_path_kernels_gpu.py,
tests/_step_reference.py and tests/_conv_stack_reference.py; not a test module."""

import math

import torch

U24 = 2.0 ** -24  # fp32 unit roundoff
U23 = 2.0 ** -23  # one fp32 ulp relative to the leading bit
U8 = 2.0 ** -8    # bf16 unit roundoff
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


def gate_ref(x64, C, act):
    """(act(f), sigmoid(g), tanh(g / 2)) in float64 of a gate input x = [f | g] (GatedActivation)."""
    f, g = x64[:, :C], x64[:, C:]
    a = torch.tanh(f) if act == TANH else f
    return a, torch.sigmoid(g), torch.tanh(0.5 * g)


def gate_fwd_err(x, C, act):
    """Absolute error of the kernel's fp32 gate act(f) sigmoid(g), before any output rounding.
    fp32 x (exact functions): tanhf 2 ulp (2^-22), sigmoid = 1 / (1 + __expf(-g)) within (3 + 1.2 |g|) 2^-23 + 2 U24
      relative, one rounding of the product.
    bf16 x (the fused stacks, one MUFU each): tanh.approx within 2^-11 relative (PTX ISA), sigmoid = 0.5 tanh.approx(g / 2)
      + 0.5 within 2^-12 |tanh(g / 2)| + U24 absolute; second-order terms are below 2^-22 |a| and covered by the 2 U24."""
    a, s, th = gate_ref(x.to(F64), C, act)
    g = x.to(F64)[:, C:]
    if x.dtype == torch.float32:
        ra = 2 * U23 if act == TANH else 0.0
        rs = (3 + 1.2 * g.abs()) * U23 + 2 * U24
        return (a * s).abs() * (ra + rs + U24)
    ra = 2.0 ** -11 if act == TANH else 0.0
    return (a * s).abs() * (ra + U24) + a.abs() * (2.0 ** -12 * th.abs() + 2 * U24)


def gate_bwd(x, dy, C, act, out_dtype):
    """(ref_f, tol_f, ref_g, tol_g): float64 d f = dy s act'(f) and d g = dy act(f) s (1 - s) of the gate backward
    (pg_gated_act_bwd) at x, and their element-wise tolerances for a result stored in out_dtype.
    With es the sigmoid's absolute error, ea act's, eda that of act' (0 for none):
      bf16 x (one MUFU each): es = 2^-12 |tanh(g/2)| + U24, ea = 2^-11 |a|, act' = 1 - a^2 from that a: eda = 2 |a| ea + 2 U24;
      fp32 x (exact functions): es = s ((3 + 1.2 |g|) 2^-23 + 2 U24), ea = 2 U23 |a|, eda = 2^-21 (deriv_err);
      d f: |dy| (es |act'| + s eda) (1 + U8) + (3 U24 + r_out) |ref|;
      d g: |dy| (ea s (1 - s) + |a| es (1 + es)) (1 + U8) + (4 U24 + r_out) |ref|;
    r_out = U8 for a bf16 result (its rounding), 0 for fp32."""
    a, s, th = gate_ref(x.to(F64), C, act)
    d = dy.to(F64)
    g = x.to(F64)[:, C:]
    tanh = act == TANH
    if x.dtype == torch.float32:
        es = s * ((3 + 1.2 * g.abs()) * U23 + 2 * U24)
        ea = 2 * U23 * a.abs() if tanh else torch.zeros_like(a)
        eda = torch.full_like(a, 2.0 ** -21) if tanh else torch.zeros_like(a)
    else:
        es = 2.0 ** -12 * th.abs() + U24
        ea = 2.0 ** -11 * a.abs() if tanh else torch.zeros_like(a)
        eda = 2 * a.abs() * ea + 2 * U24 if tanh else torch.zeros_like(a)
    da = 1 - a * a if tanh else torch.ones_like(a)
    r_out = U8 if out_dtype == torch.bfloat16 else 0.0
    ref_f, ref_g = d * s * da, d * a * s * (1 - s)
    tol_f = (r_out + 3 * U24) * ref_f.abs() + d.abs() * (es * da.abs() + s * eda) * (1 + U8)
    tol_g = (r_out + 4 * U24) * ref_g.abs() + d.abs() * (ea * s * (1 - s) + a.abs() * es * (1 + es)) * (1 + U8)
    return ref_f, tol_f, ref_g, tol_g
