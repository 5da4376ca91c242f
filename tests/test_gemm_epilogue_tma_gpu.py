"""GEMM epilogue cases of pg_gemm_bf16's tensor-core kernel that tests/test_gemm_kernels_gpu.py does not cover: a strided
fp32 output whose padding columns must survive, bf16 residuals at a ragged N, an accumulate launch onto a non-zero
output, and the row-segment fallback taken when an fp32 pitch is not a multiple of 16 bytes (N = 3).

Operands are small integers, so every sum is exact in fp32 and the results must equal the float64 reference of
tests/_gemm_reference.py bit for bit (bf16 outputs: its bf16 rounding)."""

import pytest
import torch

import _gemm_reference as G

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
CANARY = 12288.0  # exact in fp32 and bf16


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _ints(shape, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).to(F32)


def _operands(M, N, K, seed, b_mn=False):
    A = _ints((M, K), -3, 3, seed).to(BF16)
    B = _ints((N, K), -3, 3, seed + 1).to(BF16)
    ref, _ = G.reference(A, B)
    dev = torch.device("cuda:0")
    Bd = B.t().contiguous() if b_mn else B
    return A.to(dev), Bd.to(dev), ref


@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_strided_output_keeps_padding(L, b_mn):
    M, N, K, ld = 320, 200, 256, 264  # N neither a multiple of the 128-wide tile nor of the 32-column sub-tile
    A, B, ref = _operands(M, N, K, 11, b_mn)
    dev = A.device
    bias = _ints((N,), -8, 8, 12)
    res = _ints((M, N), -50, 50, 13)
    res_buf = torch.full((M, ld), float("nan"), device=dev)
    res_buf[:, :N] = res.to(dev)
    out_buf = torch.full((M, ld), CANARY, device=dev)
    L.gemm(A, B, M, N, K, b_mn=b_mn, bias=bias.to(dev), res0=res_buf[:, :N], out_f32=out_buf[:, :N])
    torch.cuda.synchronize()
    want = ref + bias.to(F64) + res.to(F64)
    got = out_buf.cpu()
    assert torch.equal(got[:, :N].to(F64), want)
    assert bool((got[:, N:] == CANARY).all()), "the kernel wrote into the padding columns N..ld"


def test_bf16_residuals_ragged_n(L):
    M, N, K, ld = 256, 72, 192, 80
    A, B, ref = _operands(M, N, K, 21)
    dev = A.device
    r0, r1 = _ints((M, N), -20, 20, 22), _ints((M, N), -20, 20, 23)
    bufs = []
    for r in (r0, r1):
        b = torch.full((M, ld), float("nan"), device=dev, dtype=BF16)
        b[:, :N] = r.to(dev, BF16)
        bufs.append(b)
    out_f32 = torch.full((M, ld), CANARY, device=dev)
    out_bf16 = torch.full((M, ld), CANARY, device=dev, dtype=BF16)
    L.gemm(A, B, M, N, K, res0=bufs[0][:, :N], res1=bufs[1][:, :N], out_f32=out_f32[:, :N], out_bf16=out_bf16[:, :N])
    torch.cuda.synchronize()
    want = ref + r0.to(F64) + r1.to(F64)
    assert torch.equal(out_f32[:, :N].cpu().to(F64), want)
    assert torch.equal(out_bf16[:, :N].cpu(), want.to(F32).to(BF16))
    assert bool((out_f32[:, N:] == CANARY).all()) and bool((out_bf16[:, N:].float() == CANARY).all())


def test_accumulate_onto_nonzero_output(L):
    M, N, K = 384, 136, 320
    A, B, ref = _operands(M, N, K, 31)
    c0 = _ints((M, N), -1000, 1000, 32)
    out = c0.to(A.device)
    L.gemm(A, B, M, N, K, out_f32=out, accumulate=True, alpha=2.0)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu().to(F64), c0.to(F64) + 2.0 * ref)


def test_unaligned_fallback_n3(L):
    M, N, K = 1000, 3, 512  # fp32 pitch of 12 bytes: TMA cannot address it, the row-segment epilogue runs
    A, B, ref = _operands(M, N, K, 41)
    bias = _ints((N,), -8, 8, 42)
    out = torch.full((M, N), float("nan"), device=A.device)
    L.gemm(A, B, M, N, K, bias=bias.to(A.device), out_f32=out)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu().to(F64), ref + bias.to(F64))
