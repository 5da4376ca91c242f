"""Per-kernel numerics on the GPU: every C-ABI entry point against a plain torch restatement of the
same op on the same (bf16-rounded) inputs.  These are floating-point kernels, so the bar is a stated
tolerance: fp32 accumulation of bf16 products must match an fp32 matmul of the same bf16 values to
~1e-5 relative (summation order only); bf16 outputs to one bf16 ulp (2^-8 relative).

This file covers the GEMM main loop, split-K and the bias gradient, softmax attention (full and KV-cached), column
sums, LayerNorm, the gated activation, the BCE loss, the layout converters, the tap-loop conv GEMM and the small-Cin
conv.  tests/test_conv_path_kernels_gpu.py checks the entry points of the conv-model path with float64 references and
element-wise bounds: every GEMM epilogue activation and derivative on the vector and scalar branches, the conv GEMM with
the stacks' epilogues, pg_tap_gather / pg_tap_scatter, pg_act_cast_bf16, pg_dact_mul, pg_dact_from_out,
pg_gated_res_fwd, the mixed-dtype gated combinations, pg_cast_f32_to_bf16, pg_cast_multi_bf16 and
pg_linear_attn_fwd / _bwd.  tests/test_gemm_kernels_gpu.py checks pg_gemm_bf16's main loop (every operand layout and tile
edge, NaN-padded views), its schedule invariance, split-K through pg_sum_partials with the bias gradient, and the
skinny kernel against float64 with element-wise bounds.  tests/test_attention_kernels_gpu.py checks
pg_causal_attn_fwd / _bwd (every tensor-core instance and the SIMT kernels, both delta kernels) and pg_attn_decode
(one-block and split paths) against float64 with element-wise bounds, in every input regime, layout and edge shape.  tests/test_wide_heads_gpu.py checks attention with
128-wide heads.  tests/test_step_kernels_gpu.py checks LayerNorm (the fast, generic and pitched _ld paths), the small-Cin
conv, the BCE loss, column sums and pg_grad_sqnorm / pg_adam_step against float64 with element-wise bounds, in large-mean,
constant and wide-range regimes, on shrunk persistent grids and NaN-padded buffers; pg_grad_sqnorm / pg_adam_step are
also checked against torch.optim.Adam in tests/test_parity_full_gpu.py."""

import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

# The torch restatements are the fp32 yardstick: no TF32 shortcuts in cuDNN/cuBLAS.
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _dev():
    return torch.device("cuda:0")


def _report_mismatch(name, got, ref, tol):
    err = (got.float() - ref.float()).abs()
    bad = err > tol
    msg = [f"{name}: max err {err.max().item():.4e} tol {tol:.3e}; mismatched {bad.sum().item()}/{bad.numel()}"]
    if bad.any() and got.dim() == 2:
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        msg.append(f"  bad rows: n={rows.numel()} first={rows[:12].tolist()} last={rows[-4:].tolist()}")
        msg.append(f"  bad cols: n={cols.numel()} first={cols[:12].tolist()} last={cols[-4:].tolist()}")
        r, c = rows[0].item(), cols[0].item()
        msg.append(f"  got[{r},{c}:{c + 6}]={got[r, c:c + 6].float().tolist()}")
        msg.append(f"  ref[{r},{c}:{c + 6}]={ref[r, c:c + 6].float().tolist()}")
        msg.append(f"  frac zeros in got: {(got == 0).float().mean().item():.3f}; nan: {torch.isnan(got.float()).any().item()}")
    return "\n".join(msg)


def assert_close(name, got, ref, rtol, atol=0.0):
    ref = ref.float()
    tol = atol + rtol * ref.abs().max().item()
    err = (got.float() - ref).abs().max().item()
    assert err <= tol and not torch.isnan(got.float()).any(), _report_mismatch(name, got, ref, tol)


# --------------------------------------------------------------------------------------------------
# GEMM
# --------------------------------------------------------------------------------------------------
GEMM_SHAPES = [
    (128, 128, 64), (128, 256, 64), (256, 256, 128), (384, 64, 192), (1000, 200, 72), (130, 24, 512),
    (4096, 512, 512), (2048, 1536, 512), (1024, 2048, 512), (2048, 512, 2048), (4096, 3, 512), (777, 136, 264),
    # more work items (128-row tiles) than SMs, so each persistent CTA runs several and its two consumer warpgroups take
    # turns, with M / N / K tails
    (16384, 512, 512), (8192, 1536, 256), (10000, 768, 320), (19000, 264, 72),
]


def _operands(M, N, K, a_mn, b_mn, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(_dev()).bfloat16()
    B = torch.randn(N, K, generator=g).to(_dev()).bfloat16()
    ref = A.float() @ B.float().t()
    # MN-major operands need the contiguous (MN) extent padded to a multiple of 8 elements.
    if a_mn:
        Mp = (M + 7) // 8 * 8
        At = torch.zeros(K, Mp, device=_dev(), dtype=torch.bfloat16)
        At[:, :M] = A.t()
        A_op = At[:, :M]
    else:
        Kp = (K + 7) // 8 * 8
        Ap = torch.zeros(M, Kp, device=_dev(), dtype=torch.bfloat16)
        Ap[:, :K] = A
        A_op = Ap[:, :K]
    if b_mn:
        Np = (N + 7) // 8 * 8
        Bt = torch.zeros(K, Np, device=_dev(), dtype=torch.bfloat16)
        Bt[:, :N] = B.t()
        B_op = Bt[:, :N]
    else:
        Kp = (K + 7) // 8 * 8
        Bp = torch.zeros(N, Kp, device=_dev(), dtype=torch.bfloat16)
        Bp[:, :K] = B
        B_op = Bp[:, :K]
    return A_op, B_op, ref


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_gemm_plain(L, shape, a_mn, b_mn):
    M, N, K = shape
    A, B, ref = _operands(M, N, K, a_mn, b_mn)
    out = torch.full((M, N), float("nan"), device=_dev(), dtype=torch.float32)
    L.gemm(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, out_f32=out)
    torch.cuda.synchronize()
    assert_close(f"gemm{shape} a_mn={a_mn} b_mn={b_mn}", out, ref, rtol=2e-5, atol=1e-4)


@pytest.mark.parametrize("shape", [(256, 256, 128), (1000, 200, 72), (130, 24, 512)])
def test_gemm_simt_crosscheck(L, shape):
    M, N, K = shape
    for a_mn, b_mn in [(False, False), (True, True)]:
        A, B, ref = _operands(M, N, K, a_mn, b_mn)
        out = torch.empty((M, N), device=_dev(), dtype=torch.float32)
        L.gemm(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, out_f32=out, impl=1)
        torch.cuda.synchronize()
        assert_close(f"simt gemm{shape}", out, ref, rtol=2e-5, atol=1e-4)


def _gelu(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def _dgelu(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("shape", [(512, 2048, 512), (1000, 200, 72), (9600, 2048, 128)])
def test_gemm_epilogue_forward(L, shape, impl):
    """bias + residuals -> fp32 'pre', bf16 'pre', bf16 gelu(pre): the fused FC1/proj epilogues."""
    M, N, K = shape
    A, B, acc = _operands(M, N, K, False, False, seed=1)
    g = torch.Generator(device="cpu").manual_seed(2)
    bias = torch.randn(N, generator=g).to(_dev())
    Np = (N + 7) // 8 * 8
    r0 = torch.randn(M, Np, generator=g).to(_dev())
    r1 = torch.randn(M, Np, generator=g).to(_dev())
    out_f = torch.empty(M, Np, device=_dev())
    out_p = torch.empty(M, Np, device=_dev(), dtype=torch.bfloat16)
    out_b = torch.empty(M, Np, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, bias=bias, res0=r0[:, :N], res1=r1[:, :N], out_f32=out_f[:, :N], out_pre=out_p[:, :N],
           out_bf16=out_b[:, :N], act=L.ACT_GELU, alpha=0.5, impl=impl)
    torch.cuda.synchronize()
    pre = 0.5 * acc + bias + r0[:, :N] + r1[:, :N]
    assert_close("pre fp32", out_f[:, :N], pre, rtol=2e-5, atol=1e-4)
    assert_close("pre bf16", out_p[:, :N], pre, rtol=2 ** -8)
    assert_close("gelu bf16", out_b[:, :N], _gelu(pre), rtol=2 ** -8)


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("shape", [(512, 256, 512), (19200, 256, 128), (1000, 200, 72), (16, 256, 384)])
def test_gemm_bf16_residuals(L, shape, impl):
    """PG_ACT_RES_BF16: res0 / res1 are bf16 matrices (GatedPixelCNN's vertical-to-horizontal sums) — tensor-core kernel
    SIMT cross-check and skinny kernel."""
    M, N, K = shape
    if (impl == 2) != (M <= 32):
        pytest.skip("the skinny kernel takes M <= 32 only")
    A, B, acc = _operands(M, N, K, False, False, seed=31)
    g = torch.Generator(device="cpu").manual_seed(32)
    bias = torch.randn(N, generator=g).to(_dev())
    Np = (N + 7) // 8 * 8
    r0 = torch.randn(M, Np, generator=g).to(_dev()).bfloat16()
    r1 = torch.randn(M, Np, generator=g).to(_dev()).bfloat16()
    out_f = torch.empty(M, Np, device=_dev())
    out_b = torch.empty(M, Np, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, bias=bias, res0=r0[:, :N], res1=r1[:, :N], out_f32=out_f[:, :N], out_bf16=out_b[:, :N],
           act=L.ACT_RELU, impl=impl)
    torch.cuda.synchronize()
    pre = acc + bias + r0[:, :N].float() + r1[:, :N].float()
    assert_close("pre fp32", out_f[:, :N], pre, rtol=2e-5, atol=1e-4)
    assert_close("relu bf16", out_b[:, :N], torch.relu(pre), rtol=2 ** -8)
    out_1 = torch.empty(M, Np, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, res0=r1[:, :N], out_bf16=out_1[:, :N], impl=impl)
    torch.cuda.synchronize()
    assert_close("one bf16 residual", out_1[:, :N], acc + r1[:, :N].float(), rtol=2 ** -8)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("M", [640, 19200])
def test_gemm_epilogue_dact(L, impl, M):
    """dgrad through GELU: out = (dY·W) * gelu'(u)  (M = 19200 runs on CTA pairs)."""
    N, K = 512, 256
    A, B, acc = _operands(M, N, K, False, True, seed=3)
    u = torch.randn(M, N, generator=torch.Generator().manual_seed(4)).to(_dev()).bfloat16()
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, b_mn=True, aux=u, dact=L.ACT_GELU, out_bf16=out, impl=impl)
    torch.cuda.synchronize()
    assert_close("dact", out, acc * _dgelu(u.float()), rtol=2 ** -8)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("M", [640, 19200])
def test_gemm_stored_derivative(L, impl, M):
    """FC1 forward stores gelu'(pre) (PG_ACT_STORE_DERIV); the FC2 dgrad epilogue multiplies by it (PG_ACT_GIVEN)."""
    N, K = 512, 256
    A, B, acc = _operands(M, N, K, False, False, seed=11)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(12)).to(_dev())
    out_d = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    out_b = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, bias=bias, out_pre=out_d, out_bf16=out_b, act=L.ACT_GELU | L.ACT_STORE_DERIV, impl=impl)
    torch.cuda.synchronize()
    pre = acc + bias
    assert_close("gelu", out_b, _gelu(pre), rtol=2 ** -8)
    assert_close("gelu'", out_d, _dgelu(pre), rtol=2 ** -8, atol=2e-3)
    A2, B2, acc2 = _operands(M, N, K, False, True, seed=13)
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A2, B2, M, N, K, b_mn=True, aux=out_d, dact=L.ACT_GIVEN, out_bf16=out, impl=impl)
    torch.cuda.synchronize()
    assert_close("given", out, acc2 * out_d.float(), rtol=2 ** -8)


@pytest.mark.parametrize("split_k", [1, 3, 8])
def test_gemm_wgrad_splitk_accumulate(L, split_k):
    """wgrad shape: dW[Cout,Cin] += dYᵀ·X over P pixels, split along the pixel dimension (slices summed in order)."""
    Cout, Cin, P = 256, 192, 4096
    A, B, ref = _operands(Cout, Cin, P, True, True, seed=5)
    out = torch.ones(Cout, Cin, device=_dev())
    L.gemm(A, B, Cout, Cin, P, a_mn=True, b_mn=True, out_f32=out, accumulate=True, split_k=split_k)
    torch.cuda.synchronize()
    assert_close(f"wgrad split_k={split_k}", out, ref + 1.0, rtol=2e-5, atol=1e-3)


@pytest.mark.parametrize("Cout,Cin,P,split_k", [(256, 192, 4096, 1), (256, 192, 4096, 3), (1536, 512, 8192, 6),
                                                (24, 64, 1000, 1), (520, 128, 12352, 8), (2048, 512, 65536, 4)])
def test_gemm_wgrad_with_bias_gradient(L, Cout, Cin, P, split_k):
    """pg_gemm_epilogue.bias_grad: the weight-gradient launch also reduces the dY tiles it stages into the bias gradient
    (partial M / K tiles, split-K, several tiles per CTA); dW must be unchanged by it."""
    A, B, ref = _operands(Cout, Cin, P, True, True, seed=41)     # A = dY read MN-major: A[k, m] = dY[pixel k, cout m]
    dw = torch.zeros(Cout, Cin, device=_dev())
    db = torch.full((Cout,), -1.0, device=_dev())
    L.gemm(A, B, Cout, Cin, P, a_mn=True, b_mn=True, out_f32=dw, accumulate=True, split_k=split_k, bias_grad=db)
    torch.cuda.synchronize()
    assert_close("dW", dw, ref, rtol=2e-5, atol=1e-3 * (P / 4096) ** 0.5)
    assert_close("db", db, A.float().sum(0) - 1.0, rtol=1e-4, atol=1e-3 * (P / 4096) ** 0.5)
    with pytest.raises(RuntimeError, match="bias_grad"):  # not a weight-gradient GEMM
        L.gemm(B, B, 64, 64, 64, out_f32=torch.zeros(64, 64, device=_dev()), bias_grad=torch.zeros(64, device=_dev()))


@pytest.mark.parametrize("M,N,K", [(16, 2048, 512), (2, 96, 32), (32, 520, 2048), (5, 3, 64)])
def test_gemm_skinny_rows(L, M, N, K):
    """M <= 32 rows (the per-pixel step of incremental sampling) takes the skinny kernel: same epilogue semantics."""
    A, B, acc = _operands(M, N, K, False, False, seed=21)
    g = torch.Generator().manual_seed(22)
    bias = torch.randn(N, generator=g).to(_dev())
    r0 = torch.randn(M, N, generator=g).to(_dev())
    r1 = torch.randn(M, N, generator=g).to(_dev())
    out_f = torch.empty(M, N, device=_dev())
    out_b = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    L.gemm(A, B, M, N, K, bias=bias, res0=r0, res1=r1, out_f32=out_f, out_bf16=out_b, act=L.ACT_GELU, impl=2)
    torch.cuda.synchronize()
    pre = acc + bias + r0 + r1
    assert_close("skinny pre", out_f, pre, rtol=2e-5, atol=1e-4)
    assert_close("skinny gelu", out_b, _gelu(pre), rtol=2 ** -8)


@pytest.mark.parametrize("N,S,H,dk,dv,strict", [(3, 200, 2, 64, 64, False), (2, 64, 1, 64, 128, True), (4, 1024, 8, 64, 64, False)])
def test_attention_decode_matches_full_attention(L, N, S, H, dk, dv, strict):
    """Appending positions one at a time through the KV cache reproduces the rows of the full causal attention."""
    q, k, v, do = _attn_inputs(N, S, H, dk, dv, seed=23)
    o_ref, _, _, _, _ = _attn_ref(q, k, v, do, N, S, H, dk, dv, strict)
    kc = torch.zeros(N * S, H * dk, device=_dev(), dtype=torch.bfloat16)
    vc = torch.zeros(N * S, H * dv, device=_dev(), dtype=torch.bfloat16)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    qv, kv_, vv = q.view(N, S, -1), k.view(N, S, -1), v.view(N, S, -1)
    o = torch.empty(N, H * dv, device=_dev(), dtype=torch.bfloat16)
    steps = range(S) if S <= 256 else list(range(0, 40)) + list(range(S - 8, S))
    if S > 256:  # pre-fill the caches for the skipped positions
        kc.view(N, S, -1)[:] = kv_
        vc.view(N, S, -1)[:] = vv
    for p in steps:
        pos.fill_(p)
        L.attn_decode(qv[:, p].contiguous(), kv_[:, p].contiguous(), vv[:, p].contiguous(), kc, vc, o, pos, N, S, H, dk, dv, strict)
        torch.cuda.synchronize()
        assert_close(f"decode pos {p}", o, o_ref.view(N, S, -1)[:, p], rtol=2 ** -7, atol=2e-3)
    assert torch.equal(kc.view(N, S, -1)[:, steps[-1]], kv_[:, steps[-1]])


def test_gemm_strided_views(L):
    """q/k/v style column slices of a wider matrix as A, and a column slice as the output."""
    M, K, N = 512, 128, 192
    g = torch.Generator().manual_seed(6)
    wide = torch.randn(M, 3 * K, generator=g).to(_dev()).bfloat16()
    W = torch.randn(N, K, generator=g).to(_dev()).bfloat16()
    outw = torch.zeros(M, 2 * N, device=_dev(), dtype=torch.bfloat16)
    L.gemm(wide[:, K:2 * K], W, M, N, K, out_bf16=outw[:, N:])
    torch.cuda.synchronize()
    assert_close("strided", outw[:, N:], wide[:, K:2 * K].float() @ W.float().t(), rtol=2 ** -8)
    assert (outw[:, :N] == 0).all()


def test_colsum(L):
    x = torch.randn(3000, 200, generator=torch.Generator().manual_seed(7)).to(_dev())
    out = torch.empty(200, device=_dev())
    L.colsum(x, out)
    xb = x.bfloat16()
    outb = torch.ones(200, device=_dev())
    L.colsum(xb, outb, accumulate=True)
    torch.cuda.synchronize()
    assert_close("colsum f32", out, x.sum(0), rtol=1e-5, atol=1e-3)
    assert_close("colsum bf16", outb, xb.float().sum(0) + 1, rtol=1e-5, atol=1e-3)
    # the scalar path: C not a multiple of 8, a pitch that is not a multiple of 8 (or 4 for fp32), a base one element into
    # its allocation; one row, and rows spanning several 256-row (vector) / 512-row (scalar) strips
    g = torch.Generator().manual_seed(17)
    for P, C, ld, off in [(3000, 3, 3, 0), (1100, 100, 103, 1), (1, 100, 104, 1), (1, 8, 8, 0), (1300, 64, 64, 1)]:
        for dtype in (torch.float32, torch.bfloat16):
            buf = torch.randn(P * ld + off, generator=g).to(_dev()).to(dtype)
            xv = buf[off:].view(P, ld)[:, :C]
            o = torch.full((C,), 0.25, device=_dev())
            L.colsum(xv, o, accumulate=True)
            torch.cuda.synchronize()
            assert_close(f"colsum {dtype} P={P} C={C} ld={ld} offset={off}", o, xv.double().sum(0) + 0.25, rtol=1e-5,
                         atol=1e-3)


# --------------------------------------------------------------------------------------------------
# LayerNorm
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,C", [(1000, 512), (4096, 512), (784, 64), (300, 256), (100, 96),
                                 # the fast path's widest instance, the generic path off a multiple of 32 and above 1024,
                                 # single rows
                                 (600, 1024), (300, 1000), (200, 2048), (1, 1024), (1, 1000)])
def test_layernorm_fwd_bwd(L, P, C):
    g = torch.Generator().manual_seed(8)
    x = (torch.randn(P, C, generator=g) * 3 + 1).to(_dev())
    gamma = (torch.randn(C, generator=g) * 0.5 + 1).to(_dev())
    beta = torch.randn(C, generator=g).to(_dev())
    dy = torch.randn(P, C, generator=g).to(_dev())
    r0 = torch.randn(P, C, generator=g).to(_dev())
    r1 = torch.randn(P, C, generator=g).to(_dev())

    xr = x.clone().requires_grad_(True)
    gr = gamma.clone().requires_grad_(True)
    br = beta.clone().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xr, (C,), gr, br, 1e-5)
    yr.backward(dy)

    y_b = torch.empty(P, C, device=_dev(), dtype=torch.bfloat16)
    y_f = torch.empty(P, C, device=_dev())
    mean = torch.empty(P, device=_dev())
    rstd = torch.empty(P, device=_dev())
    L.layernorm_fwd(x, gamma, beta, 1e-5, y_bf16=y_b, y_f32=y_f, mean=mean, rstd=rstd)
    dx_f = torch.empty(P, C, device=_dev())
    dx_b = torch.empty(P, C, device=_dev(), dtype=torch.bfloat16)
    dgam = torch.zeros(C, device=_dev())
    dbet = torch.zeros(C, device=_dev())
    dxs = torch.zeros(C, device=_dev())
    L.layernorm_bwd(dy, x, gamma, mean, rstd, dres0=r0, dres1=r1, dx_f32=dx_f, dx_bf16=dx_b, dgamma=dgam, dbeta=dbet,
                    dx_colsum=dxs)
    # bf16 dy variant
    dx_f2 = torch.empty(P, C, device=_dev())
    L.layernorm_bwd(dy.bfloat16(), x, gamma, mean, rstd, dx_f32=dx_f2)
    torch.cuda.synchronize()
    assert_close("ln y f32", y_f, yr, rtol=1e-5, atol=1e-5)
    assert_close("ln y bf16", y_b, yr, rtol=2 ** -8)
    assert_close("ln dx", dx_f, xr.grad + r0 + r1, rtol=1e-5, atol=1e-5)
    assert_close("ln dx bf16", dx_b, xr.grad + r0 + r1, rtol=2 ** -8)
    assert_close("ln dgamma", dgam, gr.grad, rtol=1e-4, atol=1e-3)
    assert_close("ln dbeta", dbet, br.grad, rtol=1e-4, atol=1e-3)
    assert_close("ln colsum(dx)", dxs, (xr.grad + r0 + r1).sum(0), rtol=1e-4, atol=1e-3)
    xr2 = x.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(xr2, (C,), gamma, beta, 1e-5).backward(dy.bfloat16().float())
    assert_close("ln dx (bf16 dy)", dx_f2, xr2.grad, rtol=1e-5, atol=1e-5)


# --------------------------------------------------------------------------------------------------
# GatedActivation, BCE, converters
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["tanh", "none"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gated_activation(L, act, dtype):
    P, C = 1500, 128
    g = torch.Generator().manual_seed(9)
    x = torch.randn(P, 2 * C, generator=g).to(_dev()).to(dtype)
    dy = torch.randn(P, C, generator=g).to(_dev()).to(dtype)
    xr = x.float().requires_grad_(True)
    f = torch.tanh(xr[:, :C]) if act == "tanh" else xr[:, :C]
    yr = f * torch.sigmoid(xr[:, C:])
    yr.backward(dy.float())
    y = torch.empty(P, C, device=_dev(), dtype=dtype)
    dx = torch.empty(P, 2 * C, device=_dev(), dtype=dtype)
    L.gated_act_fwd(x, y, L.ACT_BY_NAME[act])
    L.gated_act_bwd(x, dy, dx, L.ACT_BY_NAME[act])
    torch.cuda.synchronize()
    rt = 1e-5 if dtype == torch.float32 else 2 ** -8
    assert_close("gated y", y, yr, rtol=rt, atol=1e-6)
    assert_close("gated dx", dx, xr.grad, rtol=rt, atol=1e-6)
    # the mixed-dtype combinations: the output in the other dtype; and for a bf16 x, an fp32 dy (the gated residual
    # block's backward) with a bf16 dx
    other = torch.bfloat16 if dtype == torch.float32 else torch.float32
    y_o = torch.empty(P, C, device=_dev(), dtype=other)
    L.gated_act_fwd(x, y_o, L.ACT_BY_NAME[act])
    torch.cuda.synchronize()
    assert_close(f"gated y ({dtype} -> {other})", y_o, yr, rtol=2 ** -8, atol=1e-6)
    if dtype == torch.bfloat16:
        dy_f = torch.randn(P, C, generator=g).to(_dev())
        xr2 = x.float().requires_grad_(True)
        f2 = torch.tanh(xr2[:, :C]) if act == "tanh" else xr2[:, :C]
        (f2 * torch.sigmoid(xr2[:, C:])).backward(dy_f)
        dx2 = torch.empty(P, 2 * C, device=_dev(), dtype=torch.bfloat16)
        L.gated_act_bwd(x, dy_f, dx2, L.ACT_BY_NAME[act])
        torch.cuda.synchronize()
        assert_close("gated dx (bf16 x, fp32 dy)", dx2, xr2.grad, rtol=2 ** -8, atol=1e-6)


def test_bce(L):
    Nb, D = 16, 3 * 32 * 32
    g = torch.Generator().manual_seed(10)
    logits = (torch.randn(Nb, D, generator=g) * 4).to(_dev())
    target = torch.rand(Nb, D, generator=g).to(_dev())
    lr = logits.clone().requires_grad_(True)
    loss_r = torch.nn.functional.binary_cross_entropy_with_logits(lr, target, reduction="none").sum(1).mean()
    loss_r.backward()
    loss = torch.zeros(1, device=_dev())
    dl = torch.empty_like(logits)
    L.bce_logits(logits, target, 1.0 / Nb, loss, dl)
    torch.cuda.synchronize()
    assert abs(loss.item() / Nb - loss_r.item()) <= 1e-5 * abs(loss_r.item())
    assert_close("bce dlogits", dl, lr.grad, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("N,C,H,W", [(3, 3, 32, 32), (2, 1, 28, 28), (2, 70, 7, 9)])
def test_layout_converters(L, N, C, H, W):
    x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(11)).to(_dev())
    Cp = (C + 7) // 8 * 8
    pm_f = torch.zeros(N * H * W, Cp, device=_dev())
    pm_b = torch.zeros(N * H * W, Cp, device=_dev(), dtype=torch.bfloat16)
    L.nchw_to_pm(x, pm_f[:, :C])
    L.nchw_to_pm(x, pm_b[:, :C])
    back = torch.empty_like(x)
    L.pm_to_nchw(pm_f[:, :C], back)
    back_b = torch.empty_like(x)
    L.pm_to_nchw(pm_b[:, :C], back_b)
    torch.cuda.synchronize()
    ref = x.permute(0, 2, 3, 1).reshape(N * H * W, C)
    assert torch.equal(pm_f[:, :C], ref)
    assert torch.equal(pm_b[:, :C], ref.bfloat16())
    assert torch.equal(back, x)
    assert torch.equal(back_b, x.bfloat16().float())
    assert (pm_f[:, C:] == 0).all()
    # an activation on the way out, from the fp32 and the bf16 pixel-major copies
    acts = {"relu": torch.relu, "elu": torch.nn.functional.elu, "tanh": torch.tanh,
            "gelu": torch.nn.functional.gelu}
    for name, fn in acts.items():
        for src, want in ((pm_f, x), (pm_b, x.bfloat16().float())):
            out = torch.empty_like(x)
            L.pm_to_nchw(src[:, :C], out, act=L.ACT_BY_NAME[name])
            torch.cuda.synchronize()
            if name == "relu":
                assert torch.equal(out, fn(want)), f"pm_to_nchw relu from {src.dtype}"
            else:
                assert_close(f"pm_to_nchw {name} from {src.dtype}", out, fn(want), rtol=1e-5, atol=4e-5)


# --------------------------------------------------------------------------------------------------
# Attention
# --------------------------------------------------------------------------------------------------
def _attn_ref(q, k, v, do, N, S, H, dk, dv, strict):
    """fp32 restatement of nn/attention.py:147-160 on [P, H*d] pixel-major inputs (with autograd)."""
    qf = q.float().view(N, S, H, dk).transpose(1, 2).requires_grad_(True)
    kf = k.float().view(N, S, H, dk).transpose(1, 2).requires_grad_(True)
    vf = v.float().view(N, S, H, dv).transpose(1, 2).requires_grad_(True)
    mask = torch.tril(torch.ones(S, S, device=q.device), diagonal=-int(strict)).view(1, 1, S, S)
    s = (qf @ kf.transpose(2, 3)) / math.sqrt(dk)
    s = s.masked_fill(mask == 0, float("-inf"))
    p = torch.softmax(s, dim=-1).masked_fill(mask == 0, 0)
    o = p @ vf
    out = o.transpose(1, 2).reshape(N * S, H * dv)
    out.backward(do.float())
    lse = torch.logsumexp(s, dim=-1)
    g = lambda t, d: t.grad.transpose(1, 2).reshape(N * S, H * d)
    return out.detach(), lse, g(qf, dk), g(kf, dk), g(vf, dv)


ATTN_CASES = [
    # N, S, H, dk, dv, strict
    (2, 256, 2, 64, 64, False),
    (1, 1024, 8, 64, 64, False),
    (2, 784, 4, 16, 16, False),
    (2, 1024, 1, 16, 128, True),
    (1, 64, 1, 16, 32, True),
    (3, 100, 2, 32, 32, False),
    (6, 1024, 8, 64, 64, False),   # 384 work items: several per persistent CTA of the backward kernel
    (10, 1024, 2, 16, 128, True),  # same for the 128-wide value slot (single K/V stage)
    (40, 200, 4, 64, 64, True),    # 320 short items (two tiles), ragged
]


def _attn_inputs(N, S, H, dk, dv, seed=12):
    g = torch.Generator().manual_seed(seed)
    P = N * S
    qkv = torch.randn(P, H * (2 * dk + dv), generator=g).to(_dev()).bfloat16()
    q, k, v = qkv[:, : H * dk], qkv[:, H * dk: 2 * H * dk], qkv[:, 2 * H * dk:]
    do = torch.randn(P, H * dv, generator=g).to(_dev()).bfloat16()
    return q, k, v, do


def _to_slots(t, H, d, slot):
    """[P, H*d] -> [P, H*slot] with each head in a zero-padded slot (layout of the tensor-core kernels)."""
    P = t.shape[0]
    out = torch.zeros(P, H, slot, device=t.device, dtype=t.dtype)
    out[:, :, :d] = t.reshape(P, H, d)
    return out.reshape(P, H * slot)


def _from_slots(t, H, d, slot):
    return t.reshape(t.shape[0], H, slot)[:, :, :d].reshape(t.shape[0], H * d)


@pytest.mark.parametrize("impl", [1, 0, 3])
@pytest.mark.parametrize("case", ATTN_CASES)
def test_attention_fwd_bwd(L, case, impl):
    N, S, H, dk, dv, strict = case
    q, k, v, do = _attn_inputs(N, S, H, dk, dv)
    P = N * S
    o_ref, lse_ref, dq_ref, dk_ref, dv_ref = _attn_ref(q, k, v, do, N, S, H, dk, dv, strict)
    if impl != 1:  # tensor-core kernels (0, and 3 for the backward): 64-wide q/k slots, 64/128-wide v slots, scale from the true dk
        ks, vs = 64, (64 if dv <= 64 else 128)
        q, k, v, do = _to_slots(q, H, dk, ks), _to_slots(k, H, dk, ks), _to_slots(v, H, dv, vs), _to_slots(do, H, dv, vs)
    else:
        ks, vs = dk, dv
    o = torch.full((P, H * vs), float("nan"), device=_dev(), dtype=torch.bfloat16)
    lse = torch.empty(N, H, S, device=_dev())
    L.causal_attn_fwd(q, k, v, o, lse, N, S, H, ks, vs, strict, impl=impl, dk_true=dk)
    torch.cuda.synchronize()
    assert_close("attn o", _from_slots(o, H, dv, vs), o_ref, rtol=2 ** -7, atol=1e-3)
    if strict:
        assert (o.view(N, S, -1)[:, 0] == 0).all(), "strict mask: first position must be exactly zero"
        assert_close("attn lse", lse[:, :, 1:], lse_ref[:, :, 1:], rtol=1e-3, atol=1e-3)
    else:
        assert_close("attn lse", lse, lse_ref, rtol=1e-3, atol=1e-3)
    dq = torch.full((P, H * ks), float("nan"), device=_dev(), dtype=torch.bfloat16)
    dk_ = torch.full((P, H * ks), float("nan"), device=_dev(), dtype=torch.bfloat16)
    dv_ = torch.full((P, H * vs), float("nan"), device=_dev(), dtype=torch.bfloat16)
    delta = torch.empty(N, H, S, device=_dev())
    dq_acc = torch.full((P, H * ks), 7.0, device=_dev())  # accepted by the ABI, contents ignored
    L.causal_attn_bwd(q, k, v, o, do, lse, delta, dq_acc, dq, dk_, dv_, N, S, H, ks, vs, strict, impl=impl, dk_true=dk)
    torch.cuda.synchronize()
    assert_close("attn dq", _from_slots(dq, H, dk, ks), dq_ref, rtol=2 ** -6, atol=2e-3)
    assert_close("attn dk", _from_slots(dk_, H, dk, ks), dk_ref, rtol=2 ** -6, atol=2e-3)
    assert_close("attn dv", _from_slots(dv_, H, dv, vs), dv_ref, rtol=2 ** -6, atol=2e-3)
    if impl != 1 and dk < ks:
        assert (dq.reshape(P, H, ks)[:, :, dk:] == 0).all() and (dk_.reshape(P, H, ks)[:, :, dk:] == 0).all()


# --------------------------------------------------------------------------------------------------
# Tap-loop convolution on the GEMM kernel (4-D TMA shifted boxes, no im2col buffer)
# --------------------------------------------------------------------------------------------------
def _shift(x, dy, dx):
    """out[n, h, w] = x[n, h + dy, w + dx], zero outside the image (x: [N, H, W, C])."""
    N, H, W, C = x.shape
    out = torch.zeros_like(x)
    h0, h1 = max(0, -dy), min(H, H - dy)
    w0, w1 = max(0, -dx), min(W, W - dx)
    if h1 > h0 and w1 > w0:
        out[:, h0:h1, w0:w1] = x[:, h0 + dy:h1 + dy, w0 + dx:w1 + dx]
    return out


TAPS_3x3 = [(i - 1, j - 1) for i in range(3) for j in range(3)]
CONV_GEMM_CASES = [
    # N, H, W, Cin, Cout, taps
    (4, 32, 32, 128, 256, [(0, -1), (0, 0), (0, 1)]),              # GatedPixelCNN 1x3 (vertical stack)
    (2, 32, 32, 256, 512, [(-1, -1), (-1, 0), (0, -1), (0, 0)]),   # PixelSNAIL 2x2 -> 2C
    (3, 16, 32, 64, 64, [(-2, 0), (-1, 0)]),                       # Nx1 after the front crop
    (2, 32, 32, 128, 128, TAPS_3x3),                               # wide CausalConv2d (all taps, masked by the weights)
    (40, 32, 32, 256, 256, [(-1, -1), (-1, 0), (0, -1), (0, 0)]),  # enough tiles for the 2-CTA kernel
    (2, 8, 16, 64, 192, [(0, -3), (0, -2), (0, -1), (0, 0)]),      # narrow image (W = 16), 1x4 causal
]


@pytest.mark.parametrize("case", CONV_GEMM_CASES)
def test_conv_gemm_fwd_dgrad_wgrad(L, case):
    from pytorch_generative_b200 import ops

    N, H, W, Cin, Cout, taps = case
    T, P = len(taps), N * H * W
    g = torch.Generator().manual_seed(21)
    x = torch.randn(P, Cin, generator=g).to(_dev()).bfloat16()
    wcat = (torch.randn(Cout, T * Cin, generator=g) / (T * Cin) ** 0.5).to(_dev()).bfloat16()
    bias = torch.randn(Cout, generator=g).to(_dev())
    dy = torch.randn(P, Cout, generator=g).to(_dev()).bfloat16()
    # fp32 reference of the same tap sum
    xr = x.float().view(N, H, W, Cin).requires_grad_(True)
    wr = wcat.float().requires_grad_(True)
    y_ref = bias + sum(_shift(xr, dy_, dx_).reshape(P, Cin) @ wr[:, t * Cin:(t + 1) * Cin].t() for t, (dy_, dx_) in enumerate(taps))
    y_ref.backward(dy.float())
    _, _, y = ops.conv_fwd(x, wcat, bias, N, H, W, taps, want_bf16=False, want_f32=True)
    dxb, dxf = ops.conv_dgrad(dy, wcat, Cin, N, H, W, taps, want_f32=True)
    dw = torch.zeros(Cout, T * Cin, device=_dev())
    db = torch.full((Cout,), 2.0, device=_dev())  # the bias gradient rides on the wgrad launch and accumulates
    ops.conv_wgrad(dy, x, dw, N, H, W, taps, db_out=db)
    torch.cuda.synchronize()
    assert_close("conv gemm db", db, dy.float().sum(0) + 2.0, rtol=1e-4, atol=1e-3 * (P ** 0.5))
    assert_close("conv gemm y", y, y_ref.detach(), rtol=1e-3, atol=1e-3)
    assert_close("conv gemm dx", dxf, xr.grad.reshape(P, Cin), rtol=1e-3, atol=1e-3)
    assert_close("conv gemm dx bf16", dxb, xr.grad.reshape(P, Cin), rtol=2 ** -7, atol=1e-2)
    assert_close("conv gemm dw", dw, wr.grad, rtol=1e-3, atol=2e-3 * (P ** 0.5))


# --------------------------------------------------------------------------------------------------
# Small-Cin causal conv
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pre_act", ["none", "relu", "elu"])
@pytest.mark.parametrize("N,Cin,H,W,Cout,kh,kw,ph,pw", [
    (4, 3, 32, 32, 512, 3, 3, 1, 1), (3, 1, 28, 28, 32, 7, 7, 3, 3), (2, 3, 8, 8, 24, 3, 3, 1, 1),
    (2, 1, 28, 28, 64, 3, 3, 1, 1),
    (2, 16, 28, 28, 64, 3, 3, 1, 1),   # PixelCNN's 16-channel layers (K = 144)
    (2, 3, 16, 16, 128, 7, 7, 3, 3),   # Cout * K = 18816 weight-gradient outputs: two launches of 16384
    (2, 3, 12, 20, 32, 3, 5, 1, 2),    # kh != kw
])
def test_conv_small(L, N, Cin, H, W, Cout, kh, kw, ph, pw, pre_act):
    """pg_conv_small_* (K = Cin kh kw <= 160) against torch fp32 autograd of conv2d(act(x)): the input activation is
    applied in the forward, and dx includes act'(x)."""
    g = torch.Generator().manual_seed(13)
    x = (torch.rand(N, Cin, H, W, generator=g) * 2 - 1).to(_dev())  # both signs: relu / elu are not the identity
    w = (torch.randn(Cout, Cin, kh, kw, generator=g) * 0.2).to(_dev())
    mask = torch.zeros(kh, kw, device=_dev())
    mask[: kh // 2] = 1
    mask[kh // 2, : kw // 2] = 1
    w = w * mask
    b = torch.randn(Cout, generator=g).to(_dev())
    dy = torch.randn(N * H * W, Cout, generator=g).to(_dev())
    act_fn = {"none": lambda t: t, "relu": torch.relu, "elu": torch.nn.functional.elu}[pre_act]
    act = L.ACT_BY_NAME[pre_act]
    pad = (ph, pw)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = torch.nn.functional.conv2d(act_fn(xr), wr, br, padding=pad)
    yr.backward(dy.view(N, H, W, Cout).permute(0, 3, 1, 2))
    out = torch.empty(N * H * W, Cout, device=_dev())
    out_b = torch.empty(N * H * W, Cout, device=_dev(), dtype=torch.bfloat16)
    L.conv_small_fwd(x, w, b, pad, out_f32=out, out_bf16=out_b, act_bf16=L.ACT_RELU, pre_act=act)
    dw = torch.zeros_like(w)
    db = torch.zeros_like(b)
    dx = torch.empty_like(x)
    L.conv_small_bwd(x, w, dy, pad, dw=dw, dbias=db, dx=dx, pre_act=act)
    torch.cuda.synchronize()
    ref = yr.detach().permute(0, 2, 3, 1).reshape(N * H * W, Cout)
    assert_close("conv out", out, ref, rtol=1e-5, atol=1e-5)
    assert_close("conv out relu bf16", out_b, ref.clamp_min(0), rtol=2 ** -8)
    assert_close("conv dw", dw, wr.grad, rtol=1e-4, atol=1e-3)
    assert_close("conv db", db, br.grad, rtol=1e-4, atol=1e-3)
    assert_close("conv dx", dx, xr.grad, rtol=1e-4, atol=1e-4)
