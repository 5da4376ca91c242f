"""Which pg_gemm_bf16 implementation a forward contraction of the per-pixel samplers runs on (`ops.linear_impl`): the
skinny kernel (impl 2) exactly where it takes the operands — at most 32 rows, K % 8 == 0, A ([rows, K] bf16) within
160 KiB of shared memory — and the tensor-core GEMM everywhere else."""

import pytest

from pytorch_generative_b200 import ops

SKINNY = 2
KIB160 = 160 * 1024


def test_rows():
    assert ops.linear_impl(32, 512, True) == SKINNY
    assert ops.linear_impl(1, 512, True) == SKINNY
    assert ops.linear_impl(33, 512, True) == ops.GEMM_IMPL
    assert ops.linear_impl(128, 8, True) == ops.GEMM_IMPL


@pytest.mark.parametrize("rows", [1, 16, 32])
def test_shared_memory(rows):
    k = KIB160 // (2 * rows)                 # A fills the 160 KiB exactly
    assert ops.linear_impl(rows, k, True) == SKINNY
    assert ops.linear_impl(rows, k + 8, True) == ops.GEMM_IMPL


def test_wide_image_gpt_mlp():
    """The second MLP contraction of ImageGPT's per-pixel step (K = 4C) at 32 images: skinny up to C = 640."""
    assert ops.linear_impl(32, 4 * 640, True) == SKINNY
    assert ops.linear_impl(32, 4 * 648, True) == ops.GEMM_IMPL
    assert ops.linear_impl(32, 4 * 1024, True) == ops.GEMM_IMPL
    assert ops.linear_impl(16, 4 * 1280, True) == SKINNY
    assert ops.linear_impl(16, 4 * 1288, True) == ops.GEMM_IMPL


@pytest.mark.parametrize("k", [1, 4, 12, 516])
def test_k_not_a_multiple_of_8(k):
    assert ops.linear_impl(4, k, True) == ops.GEMM_IMPL
    assert ops.linear_impl(4, k + (-k) % 8, True) == SKINNY


def test_only_on_request():
    """forward() never asks: it keeps one summation order whatever the number of rows."""
    assert ops.linear_impl(8, 64, False) == ops.GEMM_IMPL
    assert ops.GEMM_IMPL != SKINNY
