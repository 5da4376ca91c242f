"""The bias gradient that rides on weight-gradient launches (pg_gemm_bf16 with A = dY MN-major) is summed by the CTAs
of N blocks 0 .. R - 1 together, each over its share of a tile's rows (R = 1, 2 or 4 by the launch's N blocks).  Its
value must not depend on that share: for the same A, launches with 1, 2, 4 and 5 N blocks give the bits of a launch
with one N block, on the full grid and on 6 CTAs, within the float64 bound of tests/_gemm_reference.py, and exactly in
the integer regime.  M and K end in tails, and the splits run from one slice to 36."""

import zlib

import pytest
import torch

import _gemm_reference as G
from _checks import check, check_equal

pytestmark = pytest.mark.gpu

F64 = torch.float64
N_CASES = (64, 200, 256, 512, 640)  # N blocks: 1 (BN = 64), 2 (N tail), 2, 4, 5
CASES = [(200, 64 * 37 + 13, 1), (200, 64 * 37 + 13, 3), (512, 64 * 130, 2), (96, 64 * 70 + 5, 64)]


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


def _bias_grad(L, at, bt, c0, d0, M, N, K, split_k, grid):
    old = L.reserve_sms(0)
    try:
        if grid is not None:
            L.reserve_sms(L.sm_count() - grid)
        db = d0.clone()
        out = c0[:, :N].contiguous()
        L.gemm(at, bt[:, :N], M, N, K, a_mn=True, b_mn=True, out_f32=out, accumulate=True, split_k=split_k,
               bias_grad=db)
        torch.cuda.synchronize()
    finally:
        L.reserve_sms(old)
    return db


@pytest.mark.parametrize("regime", ["randn", "integer", "range"])
@pytest.mark.parametrize("M,K,split_k", CASES)
def test_bias_grad_independent_of_n_blocks(L, M, K, split_k, regime):
    dev = torch.device("cuda:0")
    A, B, c0, d0 = G.make_inputs(regime, M, max(N_CASES), K, zlib.crc32(repr((M, K, split_k, regime)).encode()),
                                 device=dev)
    at, bt = A.T.contiguous(), B.T.contiguous()  # dY [K, M] and X [K, N], both MN-major
    rs, rs_abs = G.row_sums(A)
    ref = d0.to(F64) + rs
    tag = f"M={M} K={K} split_k={split_k} {regime}"
    first = None
    for N in N_CASES:
        for grid in (None, 6):
            db = _bias_grad(L, at, bt, c0, d0, M, N, K, split_k, grid)
            label = f"{tag} N={N} grid={grid or 'all'}"
            if first is None:
                first = db
                check(f"{label}: bias gradient", db, ref, G.rowsum_bound(K, rs_abs, d0, split_k))
                if regime == "integer":
                    check(f"{label}: bias gradient exact", db, ref, G.exact_bound(ref))
            else:
                check_equal(f"{label}: bias gradient vs one N block", db, first)
