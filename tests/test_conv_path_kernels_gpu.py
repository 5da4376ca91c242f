"""Kernel tests for the conv-model path (PixelCNN, GatedPixelCNN, PixelSNAIL): every activation of the GEMM epilogue on
its vector and scalar branches, the conv GEMM with the stacks' epilogues, tap gather / scatter, the elementwise ops and
the linear-attention numerator.

Every test rounds its inputs to bf16 first and computes the reference in float64 on the GPU from the same rounded
values.  Results are compared element by element, |got - ref| <= r |ref| + a, with r and a derived from
  * the output dtype: a bf16 result carries its rounding, U8 = 2^-8 relative (8 significant bits, round to nearest);
  * the documented error of the activation the kernel evaluates (act_err / deriv_err in tests/_act_reference.py);
  * an fp32 accumulation bound n U24 sum|terms| (U24 = 2^-24, n the number of roundings along the longest chain),
    computed in float64 from the absolute values of the terms: the classic worst-case bound of recursive summation,
    which holds in any summation order.
A bound on the largest element only (rtol * max|ref|) would hide errors on small entries: the negative ELU branch,
derivatives near zero, gate derivatives.  Copies and casts must match bit for bit.  A failure names the worst element
(largest error / bound), its index, the value the kernel produced and the reference value."""

import math
import random

import pytest
import torch

from _act_reference import (ACT_NAMES, ELU, ELU_OUT, GELU, GIVEN, NONE, RELU, RELU_OUT, TANH, U23, U24, act64,
                            act_err, dact64, deriv_err)

pytestmark = pytest.mark.gpu

U8 = 2.0 ** -8    # bf16 unit roundoff
F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64

FWD_ACTS = [NONE, RELU, GELU, ELU, TANH]
DACTS = [RELU, GELU, ELU, TANH, GIVEN, RELU_OUT, ELU_OUT]


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _dev():
    return torch.device("cuda:0")


def _randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(_dev())


def _pitched(P, C, ld, dtype, fill=float("nan")):
    """[P, C] view of a [P, ld] buffer (unit inner stride, row pitch ld), the rest of the buffer set to `fill`."""
    return torch.full((P, ld), fill, dtype=dtype, device=_dev())[:, :C]


def _copy_into(src, ld):
    out = _pitched(src.shape[0], src.shape[1], ld, src.dtype)
    out.copy_(src)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# comparison helpers
# ----------------------------------------------------------------------------------------------------------------------
def _worst(got, ref, err, tol, bad):
    ratio = torch.where(bad, (err / tol).nan_to_num(nan=math.inf, posinf=math.inf), torch.zeros_like(err))
    flat = int(ratio.reshape(-1).argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), got.shape))
    return idx, got[idx].item(), ref[idx].item(), tol[idx].item()


def check(name, got, ref, r=0.0, a=0.0):
    """|got - ref| <= r |ref| + a element by element (r, a: numbers or tensors broadcasting to ref); NaN fails."""
    g = got.to(F64)
    ref = ref.to(F64)
    tol = (r * ref.abs() + a) * torch.ones_like(ref)
    err = (g - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        idx, gv, rv, tv = _worst(g, ref, err, tol, bad)
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound; worst at {idx}: "
                             f"got {gv!r}, ref {rv!r}, |err| {abs(gv - rv):.3e} > bound {tv:.3e}")


def _within(got, ref, r=0.0, a=0.0):
    ref = ref.to(F64)
    return bool(((got.to(F64) - ref).abs() <= r * ref.abs() + a).all())


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def check_equal(name, got, ref):
    """Bit-for-bit equality (NaN payloads included)."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
    bad = _bits(got.contiguous()) != _bits(ref.contiguous())
    if bad.any():
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements differ; first at {idx}: "
                             f"got {got[idx].item()!r}, ref {ref[idx].item()!r}")


def check_bf16_ulps(name, got, ref, ulps):
    """bf16 results at most `ulps` units in the last place from the bf16 reference (same sign)."""
    gb, rb = _bits(got.contiguous()).int(), _bits(ref.contiguous()).int()
    same_sign = (gb < 0) == (rb < 0)
    bad = ~same_sign | ((gb - rb).abs() > ulps)
    bad &= ~((got == 0) & (ref == 0))
    if bad.any():
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements more than {ulps} ulp off; first at {idx}: "
                             f"got {got[idx].item()!r}, ref {ref[idx].item()!r}")


# ----------------------------------------------------------------------------------------------------------------------
# A. GEMM epilogue matrix
# ----------------------------------------------------------------------------------------------------------------------
# branch -> (M, N, K, pitched).  "vec": N % 32 == 0, fresh aligned tensors: every 32-column segment takes the vector
# branch.  "tail": N = 200 leaves an 8-column segment per row on the scalar branch.  "scalar": every epilogue tensor has a
# row pitch of N + 12 = 204 (not a multiple of 8 for bf16) and the bias starts one float into its allocation, so vec_ok is 0
# and every segment is scalar.
BRANCHES = {"vec": (640, 256, 256, False), "tail": (1000, 200, 72, False), "scalar": (640, 192, 256, True)}


def _gemm_inputs(M, N, K, seed):
    """A [M, K] and B [N, K] bf16; B scaled so that pre ~ N(0, 4): both branches of ELU / GELU / TANH are well populated."""
    A = _randn((M, K), seed).to(BF16)
    B = _randn((N, K), seed + 1, 2 / math.sqrt(K)).to(BF16)
    A64, B64 = A.to(F64), B.to(F64)
    return A, B, A64 @ B64.t(), A64.abs() @ B64.abs().t()


def _epi_tensor(src, pitched):
    return _copy_into(src, src.shape[1] + 12) if pitched else src.contiguous()


def _bias(N, seed, pitched):
    b = _randn((N,), seed)
    if not pitched:
        return b
    buf = torch.zeros(N + 1, device=_dev())
    buf[1:] = b
    return buf[1:]  # 4 bytes past a 16-byte boundary


def _epi_out(M, N, dtype, pitched):
    return _pitched(M, N, N + 12 if pitched else N, dtype)


def _forward_epilogue_case(L, impl, M, N, K, pitched, act, res_dtype, seed):
    """One forward GEMM with every output and a second with PG_ACT_STORE_DERIV, both checked against float64.

    out_f32 = alpha acc + bias + res0 + res1: K products accumulated, then 4 more roundings (alpha, bias, res0, res1), so
      |err| <= (K + 4) U24 (alpha sum_k |a||b| + |bias| + |res0| + |res1|).
    out_pre = bf16(out_f32) bit for bit (the same fp32 value, rounded to nearest even).
    out_bf16 = bf16(act(pre)) against act applied in float64 to the kernel's own fp32 pre (activation error kept apart
      from accumulation error): |err| <= U8 |ref| + (r_act |ref| + a_act)(1 + U8).
    out_pre with STORE_DERIV = bf16(act'(pre)), likewise with the derivative's error."""
    A, B, acc, acc_abs = _gemm_inputs(M, N, K, seed)
    alpha = 0.75
    bias = _bias(N, seed + 2, pitched)
    r0 = _epi_tensor(_randn((M, N), seed + 3).to(res_dtype), pitched)
    r1 = _epi_tensor(_randn((M, N), seed + 4).to(res_dtype), pitched)
    of, op, ob = _epi_out(M, N, F32, pitched), _epi_out(M, N, BF16, pitched), _epi_out(M, N, BF16, pitched)
    L.gemm(A, B, M, N, K, bias=bias, res0=r0, res1=r1, out_f32=of, out_pre=op, out_bf16=ob, act=act, alpha=alpha,
           impl=impl)
    of2, od, ob2 = _epi_out(M, N, F32, pitched), _epi_out(M, N, BF16, pitched), _epi_out(M, N, BF16, pitched)
    L.gemm(A, B, M, N, K, bias=bias, res0=r0, res1=r1, out_f32=of2, out_pre=od, out_bf16=ob2,
           act=act | L.ACT_STORE_DERIV, alpha=alpha, impl=impl)
    torch.cuda.synchronize()
    b64, r064, r164 = bias.to(F64), r0.to(F64), r1.to(F64)
    pre = alpha * acc + b64 + r064 + r164
    bound = (K + 4) * U24 * (alpha * acc_abs + b64.abs() + r064.abs() + r164.abs())
    tag = f"impl {impl} act {ACT_NAMES[act]} res {res_dtype}"
    check(f"{tag}: out_f32", of, pre, a=bound)
    check_equal(f"{tag}: out_pre = bf16(out_f32)", op, of.to(BF16))
    pre_k = of.to(F64)
    ra, aa = act_err(act, pre_k)
    check(f"{tag}: out_bf16 = bf16(act(pre))", ob, act64(act, pre_k), r=U8 + ra * (1 + U8), a=aa * (1 + U8))
    check_equal(f"{tag}: out_f32 of the STORE_DERIV launch", of2, of)
    rd, ad = deriv_err(act, pre_k)
    check(f"{tag}: out_pre = bf16(act'(pre))", od, dact64(act, pre_k), r=U8 + rd * (1 + U8), a=ad * (1 + U8))
    check_equal(f"{tag}: out_bf16 of the STORE_DERIV launch", ob2, ob)


@pytest.mark.parametrize("res_dtype", [F32, BF16], ids=["res_f32", "res_bf16"])
@pytest.mark.parametrize("act", FWD_ACTS, ids=[ACT_NAMES[a] for a in FWD_ACTS])
@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_epilogue_act_forward(L, impl, branch, act, res_dtype):
    """Forward epilogue, every activation, tensor-core kernel (impl 0) and SIMT kernel (impl 1), on the vector branch, with
    a scalar tail segment, and with every segment scalar.  Bounds: see _forward_epilogue_case."""
    M, N, K, pitched = BRANCHES[branch]
    _forward_epilogue_case(L, impl, M, N, K, pitched, act, res_dtype, seed=100 + act)


@pytest.mark.parametrize("res_dtype", [F32, BF16], ids=["res_f32", "res_bf16"])
@pytest.mark.parametrize("act", FWD_ACTS, ids=[ACT_NAMES[a] for a in FWD_ACTS])
def test_gemm_epilogue_act_forward_skinny(L, act, res_dtype):
    """The same forward epilogue on the skinny kernel (impl 2, M <= 32 rows: incremental sampling), one element per lane,
    with a pitched layout and an offset bias.  Bounds: see _forward_epilogue_case."""
    _forward_epilogue_case(L, 2, 24, 200, 72, True, act, res_dtype, seed=200 + act)


@pytest.mark.parametrize("dact", DACTS, ids=[ACT_NAMES[a] for a in DACTS])
@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("impl", [0, 1])
def test_gemm_epilogue_dact(L, impl, branch, dact):
    """Backward epilogue (dgrad layout, B read MN-major): out = acc * act'(aux) + res0.

    aux is bf16: the pre-activation z for RELU / GELU / ELU / TANH, gelu'(z) for GIVEN, and the ACTIVATED value
    relu(z) / elu(z) for RELU_OUT / ELU_OUT.  With g = act'(aux) in float64 and (r_g, a_g) its documented error:
      out_f32: |err| <= (K + 2) U24 (sum_k |a||b| |g| + |res0|) + sum_k |a||b| (r_g |g| + a_g)
        (K products, one multiply, one add; the derivative's own error scales |acc| <= sum_k |a||b|);
      out_bf16 = bf16(out_f32) bit for bit.
    *_OUT, second check: the factor the kernel derives from the bf16 ya must also be the true derivative e^z (z <= 0) to
    within 2^-8 absolute.  ya + 1 = bf16(e^z - 1) + 1 and e^z - 1 lies in (-1, 0], where bf16 values are spaced at most
    2^-8 apart (spacing 2^-8 on [-1, -1/2)): rounding to nearest moves it by at most half that, so the bound adds
    2^-8 |acc|.  For RELU_OUT the factor is exact: relu(z) rounds to a positive bf16 exactly when z > 0."""
    M, N, K, pitched = BRANCHES[branch]
    seed = 300 + dact
    A, B, acc, acc_abs = _gemm_inputs(M, N, K, seed)
    Bt = B.t().contiguous()  # [K, N]: the dgrad operand layout
    z = _randn((M, N), seed + 5, 2.0)
    if dact == RELU_OUT:
        aux_src = act64(RELU, z)
    elif dact == ELU_OUT:
        aux_src = act64(ELU, z)
    elif dact == GIVEN:
        aux_src = dact64(GELU, z)
    else:
        aux_src = z
    aux = _epi_tensor(aux_src.to(BF16), pitched)
    r0 = _epi_tensor(_randn((M, N), seed + 6), pitched)
    of, ob = _epi_out(M, N, F32, pitched), _epi_out(M, N, BF16, pitched)
    L.gemm(A, Bt, M, N, K, b_mn=True, aux=aux, dact=dact, res0=r0, out_f32=of, out_bf16=ob, impl=impl)
    torch.cuda.synchronize()
    g = dact64(dact, aux)
    rg, ag = deriv_err(dact, aux.to(F64))
    r064 = r0.to(F64)
    bound = (K + 2) * U24 * (acc_abs * g.abs() + r064.abs()) + acc_abs * (rg * g.abs() + ag)
    tag = f"impl {impl} dact {ACT_NAMES[dact]}"
    check(f"{tag}: out_f32 = acc act'(aux) + res0", of, acc * g + r064, a=bound)
    check_equal(f"{tag}: out_bf16 = bf16(out_f32)", ob, of.to(BF16))
    if dact in (RELU_OUT, ELU_OUT):
        z64 = z.to(F64)
        true_g = (z64 > 0).to(F64) if dact == RELU_OUT else torch.where(z64 > 0, torch.ones_like(z64), torch.exp(z64))
        extra = 0.0 if dact == RELU_OUT else U8 * acc.abs()
        check(f"{tag}: factor vs the true derivative e^pre", of, acc * true_g + r064, a=bound + extra)


# ----------------------------------------------------------------------------------------------------------------------
# B. conv GEMM (pg_gemm_bf16_conv) with the stacks' epilogues
# ----------------------------------------------------------------------------------------------------------------------
def _shift(x, dy, dx):
    """out[n, h, w] = x[n, h + dy, w + dx], zero outside the image (x: [N, H, W, C])."""
    N, H, W, C = x.shape
    out = torch.zeros_like(x)
    h0, h1 = max(0, -dy), min(H, H - dy)
    w0, w1 = max(0, -dx), min(W, W - dx)
    if h1 > h0 and w1 > w0:
        out[:, h0:h1, w0:w1] = x[:, h0 + dy:h1 + dy, w0 + dx:w1 + dx]
    return out


def _tap_sum(x_pm, w_cat, geom, taps, sign=1):
    """sum_t shift(x, sign * off_t) @ W_t^T  with W_t = w_cat[:, t C:(t + 1) C]  (float64, [P, Cout])."""
    n, h, w = geom
    C = x_pm.shape[1]
    x4 = x_pm.reshape(n, h, w, C)
    return sum(_shift(x4, sign * a, sign * b).reshape(-1, C) @ w_cat[:, t * C:(t + 1) * C].t()
               for t, (a, b) in enumerate(taps))


def _tap_sum_t(dy64, w64, geom, taps):
    """Dgrad of the tap sum: dx[p] = sum_t W_t^T dy[p - off_t]  (float64, [P, Cin])."""
    n, h, w = geom
    Cout = dy64.shape[1]
    Cin = w64.shape[1] // len(taps)
    d4 = dy64.reshape(n, h, w, Cout)
    return sum(_shift(d4, -a, -b).reshape(-1, Cout) @ w64[:, t * Cin:(t + 1) * Cin] for t, (a, b) in enumerate(taps))


CONV_CASES = {
    # name: (N, H, W, Cin, Cout, taps)
    "w8": (2, 16, 8, 64, 64, [(0, 0), (-1, 0), (0, -1), (-1, -1), (-16, 0), (3, -9)]),     # TMA box of 16 rows
    "w64_h2": (3, 2, 64, 192, 128, [(0, 0), (-1, -1), (-1, 0), (-2, 0), (1, 5), (0, -64)]),  # boxes of 2 rows; |dy| >= H
    "w64_h4": (1, 4, 64, 64, 192, [(-1, -1), (-1, 0), (0, -1), (0, 0), (-4, 3), (5, 0)]),
    "cout8": (2, 16, 8, 192, 8, [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 0)]),             # a padded logits conv
}


@pytest.mark.parametrize("res_dtype", [F32, BF16], ids=["res_f32", "res_bf16"])
@pytest.mark.parametrize("act", [RELU, ELU], ids=["relu", "elu"])
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_gemm_epilogues(L, case, act, res_dtype):
    """ops.conv_fwd / conv_dgrad / conv_wgrad with the epilogues of nn/pm.py's stacks, against explicit shifted sums.

    Forward, y = sum_t W_t x[p + off_t] + bias + res0 with act into out_bf16, plus out_pre and out_f32:
      out_f32 within (T C + 3) U24 (sum |w||x| + |bias| + |res0|); out_pre = bf16(out_f32) bit for bit;
      out_bf16 against act(out_f32) in float64: U8 |ref| + act error (see act_err).
    Dgrad, dx = (sum_t W_t^T dy[p - off_t]) * act'(aux) + res0, aux = bf16(act(z)) (RELU_OUT / ELU_OUT): out_f32 within
      (T Cout + 3) U24 (sum |w||dy| |g| + |res0|) + sum |w||dy| a_g; out_bf16 = bf16(out_f32) bit for bit.
    Wgrad, dW[:, t C + c] = sum_p dy[p] x[p + off_t, c] within (P + 2) U24 sum_p |dy||x|, and the bias gradient riding on
      the same launch within (P + 2) U24 (sum_p |dy| + |db0|).  Dgrad and wgrad run twice: identical bits."""
    from pytorch_generative_b200 import ops

    N, H, W, Cin, Cout, taps = CONV_CASES[case]
    T, P = len(taps), N * H * W
    seed = 400 + act
    x = _randn((P, Cin), seed).to(BF16)
    wcat = _randn((Cout, T * Cin), seed + 1, 2 / math.sqrt(T * Cin)).to(BF16)
    bias = _randn((Cout,), seed + 2)
    res = _randn((P, Cout), seed + 3).to(res_dtype)
    x64, w64 = x.to(F64), wcat.to(F64)
    geom = (N, H, W)
    tag = f"{case} {ACT_NAMES[act]} res {res_dtype}"

    ya, yp, yf = ops.conv_fwd(x, wcat, bias, N, H, W, taps, act=act, res0=res, want_bf16=True, want_pre=True,
                              want_f32=True)
    torch.cuda.synchronize()
    ref = _tap_sum(x64, w64, geom, taps) + bias.to(F64) + res.to(F64)
    bound = (T * Cin + 3) * U24 * (_tap_sum(x64.abs(), w64.abs(), geom, taps) + bias.to(F64).abs() + res.to(F64).abs())
    check(f"{tag}: fwd out_f32", yf, ref, a=bound)
    check_equal(f"{tag}: fwd out_pre = bf16(out_f32)", yp, yf.to(BF16))
    ra, aa = act_err(act, yf)
    check(f"{tag}: fwd out_bf16 = bf16(act(pre))", ya, act64(act, yf), r=U8 + ra * (1 + U8), a=aa * (1 + U8))

    if Cout % 64 == 0:  # the dgrad operand (dy) is the shifted tensor: C % 64 (a logits conv is pointwise in the stacks)
        dy = _randn((P, Cout), seed + 4).to(BF16)
        aux = act64(act, _randn((P, Cin), seed + 5, 2.0)).to(BF16)
        rd = _randn((P, Cin), seed + 6).to(res_dtype)
        dact = L.DACT_FROM_OUT[act]
        outs = [ops.conv_dgrad(dy, wcat, Cin, N, H, W, taps, aux=aux, dact=dact, want_f32=True, want_bf16=True, res0=rd)
                for _ in range(2)]
        torch.cuda.synchronize()
        (dxb, dxf), (dxb2, dxf2) = outs
        g = dact64(dact, aux)
        _, ag = deriv_err(dact, aux)
        dy64 = dy.to(F64)
        s = _tap_sum_t(dy64, w64, geom, taps)
        s_abs = _tap_sum_t(dy64.abs(), w64.abs(), geom, taps)
        bound = (T * Cout + 3) * U24 * (s_abs * g.abs() + rd.to(F64).abs()) + s_abs * ag
        check(f"{tag}: dgrad out_f32", dxf, s * g + rd.to(F64), a=bound)
        check_equal(f"{tag}: dgrad out_bf16 = bf16(out_f32)", dxb, dxf.to(BF16))
        check_equal(f"{tag}: dgrad repeated", dxf2, dxf)

    dy = _randn((P, Cout), seed + 7).to(BF16)
    dws, dbs = [], []
    for _ in range(2):
        dw = torch.zeros(Cout, T * Cin, device=_dev())
        db = torch.full((Cout,), 0.5, device=_dev())
        ops.conv_wgrad(dy, x, dw, N, H, W, taps, db_out=db)
        dws.append(dw)
        dbs.append(db)
    torch.cuda.synchronize()
    dy64 = dy.to(F64)
    x4 = x64.reshape(N, H, W, Cin)
    xs = torch.cat([_shift(x4, a, b).reshape(P, Cin) for a, b in taps], dim=1)
    check(f"{tag}: wgrad dW", dws[0], dy64.t() @ xs, a=(P + 2) * U24 * (dy64.abs().t() @ xs.abs()))
    check(f"{tag}: wgrad bias gradient", dbs[0], dy64.sum(0) + 0.5, a=(P + 2) * U24 * (dy64.abs().sum(0) + 0.5))
    check_equal(f"{tag}: wgrad repeated", dws[1], dws[0])
    check_equal(f"{tag}: bias gradient repeated", dbs[1], dbs[0])


# ----------------------------------------------------------------------------------------------------------------------
# C. tap gather / scatter
# ----------------------------------------------------------------------------------------------------------------------
GATHER_GEOMS = {"28x28": (2, 28, 28), "7x9": (3, 7, 9), "1x5": (4, 1, 5)}


def _taps(T, H, W, seed):
    """(0, 0) and T - 1 offsets drawn from [-(H + 2), H + 2] x [-(W + 2), W + 2]: some taps lie wholly outside the image."""
    rng = random.Random(seed)
    return [(0, 0)] + [(rng.randint(-H - 2, H + 2), rng.randint(-W - 2, W + 2)) for _ in range(T - 1)]


def _gathered(x_pm, geom, taps):
    n, h, w = geom
    C = x_pm.shape[1]
    x4 = x_pm.reshape(n, h, w, C)
    return torch.cat([_shift(x4, a, b).reshape(-1, C) for a, b in taps], dim=1)


def _scattered(dxcat, geom, taps, C):
    """sum_t dxcat[p - off_t, t C:(t + 1) C]."""
    n, h, w = geom
    return sum(_shift(dxcat[:, t * C:(t + 1) * C].reshape(n, h, w, C), -a, -b).reshape(-1, C)
               for t, (a, b) in enumerate(taps))


@pytest.mark.parametrize("T", [1, 4, 9, 25, 32])
@pytest.mark.parametrize("C", [8, 136])
@pytest.mark.parametrize("geom", list(GATHER_GEOMS))
def test_tap_gather(L, geom, C, T):
    """X_cat[p, t C + c] = act(x[p + off_t, c]), zero outside the image, from a pitched x (ld = C + 8).
    NONE and RELU are copies (relu of a bf16 value is a bf16 value): bit for bit.  ELU is expm1f in fp32, then rounded to
    bf16: within 1 bf16 ulp of the float64 ELU rounded to bf16 (the two roundings may straddle a midpoint)."""
    n, h, w = GATHER_GEOMS[geom]
    P = n * h * w
    taps = _taps(T, h, w, seed=T * 1000 + C)
    x = _copy_into(_randn((P, C), 500 + T).to(BF16), C + 8)
    for act in (NONE, RELU, ELU):
        out = torch.full((P, T * C), float("nan"), dtype=BF16, device=_dev())
        L.tap_gather(x, n, h, w, C, taps, act, out)
        torch.cuda.synchronize()
        ref = _gathered(act64(act, x.to(F64)), (n, h, w), taps).to(BF16)
        if act == ELU:
            check_bf16_ulps(f"gather {ACT_NAMES[act]}", out, ref, 1)
        else:
            check_equal(f"gather {ACT_NAMES[act]}", out, ref)


@pytest.mark.parametrize("T", [1, 4, 9, 25, 32])
@pytest.mark.parametrize("C", [8, 136])
@pytest.mark.parametrize("geom", list(GATHER_GEOMS))
def test_tap_scatter(L, geom, C, T):
    """dx[p, c] = act'(x_pre[p, c]) sum_t dX_cat[p - off_t, t C + c], dx_f32 and dx_bf16 written by one call through one
    pitch (C + 8), x_pre pitched as well.  The fp32 sum of at most T bf16 terms and one multiply by the derivative:
    |err| <= (T + 2) U24 sum_t |terms| |g| + sum_t |terms| (r_g |g| + a_g).  dx_bf16 = bf16(dx_f32) bit for bit; the
    columns past C stay untouched; a second run gives the same bits."""
    n, h, w = GATHER_GEOMS[geom]
    P = n * h * w
    taps = _taps(T, h, w, seed=T * 1000 + C + 1)
    dxcat = _randn((P, T * C), 600 + T).to(BF16)
    x_pre = _copy_into(_randn((P, C), 601 + T, 2.0).to(BF16), C + 8)
    s = _scattered(dxcat.to(F64), (n, h, w), taps, C)
    s_abs = _scattered(dxcat.to(F64).abs(), (n, h, w), taps, C)
    for act in (NONE, RELU, ELU):
        runs = []
        for _ in range(2):
            dxf_buf = torch.full((P, C + 8), 7.0, device=_dev())
            dxb_buf = torch.full((P, C + 8), 7.0, dtype=BF16, device=_dev())
            L.tap_scatter(dxcat, n, h, w, C, taps, act, x_pre, dx_f32=dxf_buf[:, :C], dx_bf16=dxb_buf[:, :C])
            runs.append((dxf_buf, dxb_buf))
        torch.cuda.synchronize()
        (dxf_buf, dxb_buf), (dxf2, _) = runs
        dxf, dxb = dxf_buf[:, :C], dxb_buf[:, :C]
        g = dact64(act, x_pre)
        rg, ag = deriv_err(act, x_pre)
        tag = f"scatter {ACT_NAMES[act]}"
        check(f"{tag}: dx_f32", dxf, s * g, a=(T + 2) * U24 * s_abs * g.abs() + s_abs * (rg * g.abs() + ag))
        check_equal(f"{tag}: dx_bf16 = bf16(dx_f32)", dxb, dxf.to(BF16))
        assert bool((dxf_buf[:, C:] == 7.0).all()) and bool((dxb_buf[:, C:] == 7.0).all()), f"{tag}: wrote past C"
        check_equal(f"{tag}: repeated", dxf2, dxf_buf)


@pytest.mark.parametrize("act", [NONE, ELU], ids=["none", "elu"])
def test_tap_conv_round_trip(L, act):
    """gather -> ops.linear_fwd and ops.linear_dgrad -> scatter is conv2d(act(x), w, padding (1, 1)) cropped to the input
    size (GatedPixelCNN's 2x3 vertical-stack conv at 28 x 28), and its input gradient, computed here with float64 conv2d
    and autograd.
    Forward: gathered operands are bf16(act(x)): exact for NONE, within U8 relative for ELU (plus expm1f's 2^-22); the GEMM
      sums T C products: |err| <= ((T C + 2) U24 + e_op) conv(|act(x)|, |w|) with e_op = 0 (NONE), U8 + 2^-22 (ELU).
    Backward: dX_cat = bf16(dy W) rounds every per-tap term (U8) after Cout + 1 fp32 roundings; the scatter adds T terms
      and multiplies by act'(x): |err| <= ((Cout + T + 3) U24 + U8) D |g| + D (r_g |g| + a_g), D = sum_t |dy||W_t| shifted
      (the same tap sum on absolute values)."""
    from pytorch_generative_b200 import ops
    from pytorch_generative_b200.nn.tapconv import conv_taps

    n, cin, h, w, cout, kh, kw = 2, 64, 28, 28, 128, 2, 3
    P = n * h * w
    taps = conv_taps(kh, kw, 1, 1)
    T = len(taps)
    x_pm = _randn((P, cin), 700).to(BF16)
    wt = _randn((cout, cin, kh, kw), 701, 1 / math.sqrt(cin * kh * kw)).to(BF16)
    wcat = wt.permute(0, 2, 3, 1).reshape(cout, T * cin).contiguous()
    bias = _randn((cout,), 702)
    dy = _randn((P, cout), 703).to(BF16)

    xcat = torch.empty(P, T * cin, dtype=BF16, device=_dev())
    L.tap_gather(x_pm, n, h, w, cin, taps, act, xcat)
    _, _, y = ops.linear_fwd(xcat, wcat, bias, want_bf16=False, want_f32=True)
    dxcat = ops.linear_dgrad(dy, wcat)
    dx = torch.empty(P, cin, device=_dev())
    L.tap_scatter(dxcat, n, h, w, cin, taps, act, x_pm, dx_f32=dx)
    torch.cuda.synchronize()

    def nchw(t):
        return t.to(F64).reshape(n, h, w, -1).permute(0, 3, 1, 2)

    def pm(t):
        return t.permute(0, 2, 3, 1).reshape(P, -1)

    x64 = nchw(x_pm).requires_grad_(True)
    w64 = wt.to(F64)
    conv = torch.nn.functional.conv2d
    y64 = conv(act64(act, x64), w64, bias.to(F64), padding=(1, 1))[:, :, :h, :w]
    y64.backward(nchw(dy))
    y_abs = conv(act64(act, x64.detach()).abs(), w64.abs(), padding=(1, 1))[:, :, :h, :w]
    e_op = 0.0 if act == NONE else U8 + 2 * U23
    check(f"round trip {ACT_NAMES[act]}: forward", y, pm(y64.detach()),
          a=((T * cin + 2) * U24 + e_op) * pm(y_abs) + (T * cin + 2) * U24 * bias.to(F64).abs())
    D = _scattered(dy.to(F64).abs() @ wcat.to(F64).abs(), (n, h, w), taps, cin)
    g = dact64(act, x_pm)
    rg, ag = deriv_err(act, x_pm)
    check(f"round trip {ACT_NAMES[act]}: input gradient", dx, pm(x64.grad),
          a=((cout + T + 3) * U24 + U8) * D * g.abs() + D * (rg * g.abs() + ag))


# ----------------------------------------------------------------------------------------------------------------------
# D. elementwise ops
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("act", FWD_ACTS, ids=[ACT_NAMES[a] for a in FWD_ACTS])
def test_act_cast(L, act, in_dtype):
    """out = bf16(act(x)) between pitched views (x: ld = C + 8, out: ld = C + 16).  NONE and RELU match torch's
    round-to-nearest-even cast bit for bit; GELU / ELU / TANH are within U8 |ref| + act error (act_err).  The columns past
    C stay untouched."""
    P, C = 300, 136
    x = _copy_into(_randn((P, C), 800 + act, 2.0).to(BF16).to(in_dtype), C + 8)
    out_buf = torch.full((P, C + 16), 7.0, dtype=BF16, device=_dev())
    out = out_buf[:, :C]
    L.act_cast(x, act, out)
    torch.cuda.synchronize()
    tag = f"act_cast {ACT_NAMES[act]} from {in_dtype}"
    if act in (NONE, RELU):
        check_equal(tag, out, (x.float().clamp_min(0) if act == RELU else x.float()).to(BF16))
    else:
        ra, aa = act_err(act, x)
        check(tag, out, act64(act, x), r=U8 + ra * (1 + U8), a=aa * (1 + U8))
    assert bool((out_buf[:, C:] == 7.0).all()), f"{tag}: wrote past C"


@pytest.mark.parametrize("act", FWD_ACTS, ids=[ACT_NAMES[a] for a in FWD_ACTS])
def test_dact_mul(L, act):
    """out = bf16(dy act'(pre)), dy / out bf16 and pre fp32 pitched views; also in place (dy and out the same view, as
    nn/tapconv.py's backward calls it).  One fp32 multiply then the bf16 rounding:
    |err| <= (U8 + 2 U24) |ref| + |dy| (r_g |g| + a_g)(1 + U8).  In place gives the same bits."""
    P, C = 500, 72
    dy = _copy_into(_randn((P, C), 900 + act).to(BF16), C + 8)
    pre = _copy_into(_randn((P, C), 901 + act, 2.0).to(BF16).float(), C + 4)
    out_buf = torch.full((P, C + 8), 7.0, dtype=BF16, device=_dev())
    out = out_buf[:, :C]
    L.dact_mul(dy, pre, act, out)
    inplace = dy.clone()
    L.dact_mul(inplace, pre, act, inplace)
    torch.cuda.synchronize()
    g = dact64(act, pre)
    rg, ag = deriv_err(act, pre)
    tag = f"dact_mul {ACT_NAMES[act]}"
    check(tag, out, dy.to(F64) * g, r=U8 + 2 * U24, a=dy.to(F64).abs() * (rg * g.abs() + ag) * (1 + U8))
    check_equal(f"{tag}: in place", inplace, out)
    assert bool((out_buf[:, C:] == 7.0).all()), f"{tag}: wrote past C"


@pytest.mark.parametrize("shape", [(37, 24), (1000, 136)], ids=["888", "136000"])
@pytest.mark.parametrize("dy_dtype", [F32, BF16], ids=["dy_f32", "dy_bf16"])
@pytest.mark.parametrize("act", [RELU, ELU], ids=["relu", "elu"])
def test_dact_from_out(L, act, dy_dtype, shape):
    """out = bf16(dy act'(pre)) from the activated value ya = bf16(act(pre)): relu' = [ya > 0], elu' = ya + 1 for ya <= 0.
    numel is a multiple of 8 but not of 2048 (a partial last block).  The factor from the same bf16 ya is exact in fp32
    (ya + 1 needs no more than 24 bits for ya in (-1, 0]); one fp32 multiply and the bf16 rounding:
    |err| <= (U8 + 2 U24) |ref|."""
    ya = act64(act, _randn(shape, 1000 + act, 2.0)).to(BF16)
    dy = _randn(shape, 1001 + act).to(BF16).to(dy_dtype)
    out = torch.full(shape, float("nan"), dtype=BF16, device=_dev())
    L.dact_from_out(dy, ya, act, out)
    torch.cuda.synchronize()
    g = dact64(L.DACT_FROM_OUT[act], ya)
    check(f"dact_from_out {ACT_NAMES[act]} dy {dy_dtype}", out, dy.to(F64) * g, r=U8 + 2 * U24)


def _gate_ref(x64, C, act):
    f, g = x64[:, :C], x64[:, C:]
    a = torch.tanh(f) if act == TANH else f
    return a, torch.sigmoid(g), torch.tanh(0.5 * g)


def _gate_fwd_err(x, C, act):
    """Absolute error of the kernel's fp32 gate act(f) sigmoid(g), before any output rounding.
    fp32 x (exact functions): tanhf 2 ulp (2^-22), sigmoid = 1 / (1 + __expf(-g)) within (3 + 1.2 |g|) 2^-23 + 2 U24
      relative, one rounding of the product.
    bf16 x (the fused stacks, one MUFU each): tanh.approx within 2^-11 relative (PTX ISA), sigmoid = 0.5 tanh.approx(g / 2)
      + 0.5 within 2^-12 |tanh(g / 2)| + U24 absolute; second-order terms are below 2^-22 |a| and covered by the 2 U24."""
    a, s, th = _gate_ref(x.to(F64), C, act)
    g = x.to(F64)[:, C:]
    if x.dtype == F32:
        ra = 2 * U23 if act == TANH else 0.0
        rs = (3 + 1.2 * g.abs()) * U23 + 2 * U24
        return (a * s).abs() * (ra + rs + U24)
    ra = 2.0 ** -11 if act == TANH else 0.0
    return (a * s).abs() * (ra + U24) + a.abs() * (2.0 ** -12 * th.abs() + 2 * U24)


@pytest.mark.parametrize("act", [TANH, NONE], ids=["tanh", "none"])
@pytest.mark.parametrize("x_dtype", [F32, BF16], ids=["x_f32", "x_bf16"])
def test_gated_res_fwd(L, x_dtype, act):
    """y = res + act(x[:, :C]) sigmoid(x[:, C:]) (PixelSNAIL's gated residual block), fp32 res / y:
    |err| <= gate error (_gate_fwd_err) + U24 |ref| (the add)."""
    P, C = 700, 136
    x = _randn((P, 2 * C), 1100 + act, 2.0).to(BF16).to(x_dtype)
    res = _randn((P, C), 1101)
    y = torch.full((P, C), float("nan"), device=_dev())
    L.gated_res_fwd(x, res, y, act)
    torch.cuda.synchronize()
    a, s, _ = _gate_ref(x.to(F64), C, act)
    ref = res.to(F64) + a * s
    check(f"gated_res_fwd {x_dtype} {ACT_NAMES[act]}", y, ref, r=U24, a=_gate_fwd_err(x, C, act))


@pytest.mark.parametrize("act", [TANH, NONE], ids=["tanh", "none"])
def test_gated_mixed_dtypes(L, act):
    """The mixed-dtype gated combinations: forward fp32 x -> bf16 y and bf16 x -> fp32 y; backward bf16 x with fp32 dy ->
    bf16 dx (what the gated residual block's backward runs).
    Forward: gate error (_gate_fwd_err), plus U8 |ref| (1 + ...) for the bf16 output.
    Backward on bf16 x (one MUFU per function), with es = 2^-12 |tanh(g/2)| + U24 the sigmoid's absolute error, ea =
    2^-11 |a| tanh's (0 for none), eda = 2 |a| ea + 2 U24 that of 1 - a^2:
      d f: |dy| (es |act'| + s eda) (1 + U8) + U8 |ref| + 3 U24 |ref|;
      d g: |dy| (ea s (1 - s) + |a| es (1 + es)) (1 + U8) + U8 |ref| + 4 U24 |ref|."""
    P, C = 600, 72
    xf = _randn((P, 2 * C), 1200 + act, 2.0).to(BF16).float()
    xb = xf.to(BF16)
    y_b = torch.empty(P, C, dtype=BF16, device=_dev())
    y_f = torch.empty(P, C, device=_dev())
    L.gated_act_fwd(xf, y_b, act)
    L.gated_act_fwd(xb, y_f, act)
    dy = _randn((P, C), 1201)
    dx = torch.full((P, 2 * C), float("nan"), dtype=BF16, device=_dev())
    L.gated_act_bwd(xb, dy, dx, act)
    torch.cuda.synchronize()
    a, s, th = _gate_ref(xf.to(F64), C, act)
    tag = f"gated {ACT_NAMES[act]}"
    check(f"{tag}: fwd fp32 -> bf16", y_b, a * s, r=U8, a=_gate_fwd_err(xf, C, act) * (1 + U8))
    check(f"{tag}: fwd bf16 -> fp32", y_f, a * s, a=_gate_fwd_err(xb, C, act))
    d = dy.to(F64)
    es = 2.0 ** -12 * th.abs() + U24
    ea = 2.0 ** -11 * a.abs() if act == TANH else torch.zeros_like(a)
    da = 1 - a * a if act == TANH else torch.ones_like(a)
    eda = 2 * a.abs() * ea + 2 * U24 if act == TANH else torch.zeros_like(a)
    ref_f = d * s * da
    ref_g = d * a * s * (1 - s)
    check(f"{tag}: bwd d f (bf16 x, fp32 dy)", dx[:, :C], ref_f, r=U8 + 3 * U24,
          a=d.abs() * (es * da.abs() + s * eda) * (1 + U8))
    check(f"{tag}: bwd d g (bf16 x, fp32 dy)", dx[:, C:], ref_g, r=U8 + 4 * U24,
          a=d.abs() * (ea * s * (1 - s) + a.abs() * es * (1 + es)) * (1 + U8))


def _special_f32():
    """fp32 values whose bf16 rounding is easy to get wrong, as bit patterns: signed zeros, infinities, the largest
    finite value (rounds to inf), subnormals (including a subnormal halfway case), halfway cases with an even and with an
    odd upper half (ties to even), just above and below a halfway case, and quiet / signalling NaNs."""
    pats = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F7FFF,
            0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x00007FFF, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x00408000,
            0x3F808000, 0x3F818000, 0x3F808001, 0x3F807FFF, 0xBF808000, 0xBF818000, 0x4B7F8000, 0x4B7E8000,
            0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FBFFFFF]
    return torch.tensor([p - (1 << 32) if p >= 1 << 31 else p for p in pats], dtype=torch.int32).view(F32)


def test_cast_f32_to_bf16(L):
    """pg_cast_f32_to_bf16 against round to nearest even done on the bit patterns, bit for bit, over the special values and
    random ones across the exponent range, numel not a multiple of 8; for NaN inputs only NaN-ness is compared (payloads
    are not specified)."""
    g = torch.Generator().manual_seed(1300)
    rnd = torch.randn(1000, generator=g) * torch.exp2(torch.randint(-140, 120, (1000,), generator=g).float())
    x_cpu = torch.cat([_special_f32(), rnd, torch.tensor([1.0, -2.5, 3.0])])
    assert x_cpu.numel() % 8 != 0
    u = x_cpu.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    ref = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF)  # round to nearest even on the bit pattern
    ref = torch.where(ref >= 1 << 15, ref - (1 << 16), ref).to(torch.int16).view(BF16)
    x = x_cpu.to(_dev())
    y = torch.empty(x.numel(), dtype=BF16, device=_dev())
    L.cast_bf16(x, y)
    torch.cuda.synchronize()
    y = y.cpu()
    nan = torch.isnan(x_cpu)
    assert torch.equal(torch.isnan(y), nan), "NaN-ness differs"
    check_equal("cast_f32_to_bf16", y[~nan], ref[~nan])


def test_cast_multi_bf16(L):
    """pg_cast_multi_bf16 (per-step refresh of the bf16 weight copies) over several tensors in one launch: numels not a
    multiple of 8 (the scalar tail after the 16-byte loop), and one source / destination pair whose bases sit one
    element into their allocations, so that the kernel's alignment test sends that tensor down the scalar loop.  Every
    destination must equal torch's cast bit for bit, and nothing next to the offset destination may be written."""
    chunk = 256
    numel = [1001, 64, 37, 2050]
    srcs = [_randn((n,), 1400 + i) * 10 for i, n in enumerate(numel)]
    big_src = torch.zeros(numel[2] + 2, device=_dev())
    big_dst = torch.full((numel[2] + 2,), 7.0, dtype=BF16, device=_dev())
    big_src[1:1 + numel[2]] = srcs[2]
    srcs[2] = big_src[1:1 + numel[2]]
    dsts = [torch.full((n,), float("nan"), dtype=BF16, device=_dev()) for n in numel]
    dsts[2] = big_dst[1:1 + numel[2]]
    chunks = [(t, c) for t, n in enumerate(numel) for c in range((n + chunk - 1) // chunk)]
    i64 = dict(dtype=torch.int64, device=_dev())
    src_ptrs = torch.tensor([s.data_ptr() for s in srcs], **i64)
    dst_ptrs = torch.tensor([d.data_ptr() for d in dsts], **i64)
    L.cast_multi(src_ptrs, dst_ptrs, torch.tensor(numel, **i64), torch.tensor(chunks, dtype=torch.int32, device=_dev()),
                 len(chunks), chunk)
    torch.cuda.synchronize()
    for i, (s, d) in enumerate(zip(srcs, dsts)):
        check_equal(f"cast_multi tensor {i}", d, s.to(BF16))
    assert big_dst[0].item() == 7.0 and big_dst[-1].item() == 7.0, "cast_multi wrote outside the offset destination"


@pytest.mark.parametrize("src", ["f32", "bf16"])
@pytest.mark.parametrize("act", FWD_ACTS, ids=[ACT_NAMES[a] for a in FWD_ACTS])
def test_pm_to_nchw_act(L, act, src):
    """pg_pm_to_nchw with an activation on the way out (conv outputs followed by an activation, nn/tapconv.py), from a
    pitched pixel-major view (ld = C + 10).  NONE / RELU are exact; the others are fp32 results within act_err."""
    N, C, H, W = 2, 70, 7, 9
    x = _copy_into(_randn((N * H * W, C), 1500 + act, 2.0).to(BF16).to(F32 if src == "f32" else BF16), C + 10)
    out = torch.empty(N, C, H, W, device=_dev())
    L.pm_to_nchw(x, out, act=act)
    torch.cuda.synchronize()
    x_nchw = x.to(F64).reshape(N, H, W, C).permute(0, 3, 1, 2)
    ref = act64(act, x_nchw)
    if act in (NONE, RELU):
        check_equal(f"pm_to_nchw {ACT_NAMES[act]}", out, ref.to(F32))
    else:
        ra, aa = act_err(act, x_nchw)
        check(f"pm_to_nchw {ACT_NAMES[act]}", out, ref, r=ra + U24, a=aa)


# ----------------------------------------------------------------------------------------------------------------------
# F. linear attention numerator
# ----------------------------------------------------------------------------------------------------------------------
def _linear_attn64(q, k, v):
    mask = torch.tril(torch.ones(q.shape[1], q.shape[1], dtype=F64, device=q.device))
    return torch.einsum("bij,bjc->bic", torch.einsum("bia,bja->bij", q, k) * mask, v)


@pytest.mark.parametrize("B", [1, 6])
@pytest.mark.parametrize("d,dv", [(1, 1), (16, 32), (64, 128), (64, 1), (7, 100)])
@pytest.mark.parametrize("Lseq", [1, 31, 32, 33, 784])
def test_linear_attention(L, Lseq, d, dv, B):
    """out_i = sum_{j <= i} (q_i . k_j) v_j and its gradients (fp64 autograd of the masked einsum).  The kernel keeps the
    state S_i = sum_{j <= i} k_j^T v_j (a chain of up to L fp32 fmas) and contracts it with q_i (d more), so
      |err| <= (n + 2) U24 (tril(|q| |k|^T) |v|)_ic,  n = L + max(d, dv),
    and the same with absolute values for dq = tril(g v^T) k, dk = tril(g v^T)^T q, dv = tril(q k^T)^T g.  The same bound
    rejects a causal mask off by one (j < i).  The backward runs twice: identical bits."""
    seed = 1600 + Lseq + 7 * d + dv
    q, k, v, g = (_randn((B, Lseq, n_), seed + i).to(BF16).float() for i, n_ in enumerate((d, d, dv, dv)))
    out = torch.full((B, Lseq, dv), float("nan"), device=_dev())
    L.linear_attn_fwd(q, k, v, out)
    grads = []
    for _ in range(2):
        dq, dk, dvv = (torch.full(t.shape, float("nan"), device=_dev()) for t in (q, k, v))
        L.linear_attn_bwd(q, k, v, g, dq, dk, dvv)
        grads.append((dq, dk, dvv))
    torch.cuda.synchronize()
    q64, k64, v64 = (t.to(F64).requires_grad_(True) for t in (q, k, v))
    ref = _linear_attn64(q64, k64, v64)
    ref.backward(g.to(F64))
    qa, ka, va, ga = (t.to(F64).abs() for t in (q, k, v, g))
    mask = torch.tril(torch.ones(Lseq, Lseq, dtype=F64, device=_dev()))
    c = (Lseq + max(d, dv) + 2) * U24
    qk = torch.einsum("bia,bja->bij", qa, ka) * mask
    gv = torch.einsum("bic,bjc->bij", ga, va) * mask
    bound = c * qk @ va
    tag = f"linear attention B={B} L={Lseq} d={d} dv={dv}"
    check(f"{tag}: out", out, ref.detach(), a=bound)
    strict = _linear_attn64(q.to(F64), k.to(F64), v.to(F64)) - torch.einsum("bia,bia->bi", q.to(F64), k.to(F64))[..., None] * v.to(F64)
    assert not _within(strict, ref.detach(), a=bound), f"{tag}: the bound does not separate j <= i from j < i"
    dq, dk, dvv = grads[0]
    check(f"{tag}: dq", dq, q64.grad, a=c * gv @ ka)
    check(f"{tag}: dk", dk, k64.grad, a=c * gv.transpose(1, 2) @ qa)
    check(f"{tag}: dv", dvv, v64.grad, a=c * qk.transpose(1, 2) @ ga)
    for name, a_, b_ in zip(("dq", "dk", "dv"), grads[0], grads[1]):
        check_equal(f"{tag}: {name} repeated", b_, a_)
