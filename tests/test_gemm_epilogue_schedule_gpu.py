"""Schedules of the TMA epilogue of pg_gemm_bf16's tensor-core kernel: the two consumer warpgroups' epilogues run at the
same time whenever an epilogue outlasts the other warpgroup's main loop.  Cases: an epilogue far longer than its main loop
(K = 64, aux plus two residuals, at each tile width), an odd number of work items per CTA, and M ending inside one
warp's 16 rows of a slab.

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


def _operands(M, N, K, seed):
    A = _ints((M, K), -3, 3, seed).to(BF16)
    B = _ints((N, K), -3, 3, seed + 1).to(BF16)
    ref, _ = G.reference(A, B)
    dev = torch.device("cuda:0")
    return A.to(dev), B.to(dev), ref


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("N", [32, 64, 2048], ids=["bn32", "bn64", "bn128"])
def test_epilogue_longer_than_main_loop(L, N):
    # one k-block per tile against an epilogue with five inputs and two outputs; several tiles per CTA
    K = 64
    M = 128 * (3 * _sms() if N <= 64 else 40)
    A, B, ref = _operands(M, N, K, 51)
    dev = A.device
    bias = _ints((N,), -8, 8, 52)
    aux = _ints((M, N), -3, 3, 53)
    r0, r1 = _ints((M, N), -50, 50, 54), _ints((M, N), -50, 50, 55)
    out_f32 = torch.full((M, N), float("nan"), device=dev)
    out_bf16 = torch.full((M, N), float("nan"), device=dev, dtype=BF16)
    L.gemm(A, B, M, N, K, bias=bias.to(dev), aux=aux.to(dev, BF16), dact=L.ACT_GIVEN, res0=r0.to(dev), res1=r1.to(dev),
           out_f32=out_f32, out_bf16=out_bf16)
    torch.cuda.synchronize()
    want = (ref + bias.to(F64)) * aux.to(F64) + r0.to(F64) + r1.to(F64)
    assert torch.equal(out_f32.cpu().to(F64), want)
    assert torch.equal(out_bf16.cpu(), want.to(F32).to(BF16))


@pytest.mark.parametrize("items", [1, 3, 5])
def test_odd_items_per_cta(L, items):
    # warpgroup 0 takes the CTA's last item; with K = 64 both warpgroups are in their epilogues at once
    N, K = 128, 64
    M = 128 * items * _sms()
    A, B, ref = _operands(M, N, K, 61)
    dev = A.device
    bias = _ints((N,), -8, 8, 62)
    out_f32 = torch.full((M, N), float("nan"), device=dev)
    out_bf16 = torch.full((M, N), float("nan"), device=dev, dtype=BF16)
    L.gemm(A, B, M, N, K, bias=bias.to(dev), out_f32=out_f32, out_bf16=out_bf16)
    torch.cuda.synchronize()
    want = ref + bias.to(F64)
    assert torch.equal(out_f32.cpu().to(F64), want)
    assert torch.equal(out_bf16.cpu(), want.to(F32).to(BF16))


@pytest.mark.parametrize("tail", [37, 64 + 5, 127])
def test_rows_end_inside_a_warp(L, tail):
    # the last tile ends inside warp 2's rows of slab 0 (37), warp 0's rows of slab 1 (69) or warp 3's (127)
    N, K = 192, 128
    M = 128 * 7 + tail
    A, B, ref = _operands(M, N, K, 71)
    dev = A.device
    res = _ints((M, N), -50, 50, 72)
    buf = torch.full((M + 16, N), CANARY, device=dev)
    L.gemm(A, B, M, N, K, res0=res.to(dev), out_f32=buf[:M], alpha=2.0)
    torch.cuda.synchronize()
    assert torch.equal(buf[:M].cpu().to(F64), 2.0 * ref + res.to(F64))
    assert bool((buf[M:] == CANARY).all()), "the kernel wrote rows at or past M"
