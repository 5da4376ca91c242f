"""Element-wise comparisons shared by the kernel tests (tests/_attention_reference.py, tests/_gemm_reference.py and the
test modules that use them); not a test module.  A bound is a tensor of the same shape as the reference: every element
is held to its own bound, so an error on a small element is not hidden by a large one elsewhere."""

import math

import torch

F64 = torch.float64


def violations(got, ref, bound):
    """Elements with |got - ref| > bound (NaN always counts), as a boolean tensor."""
    err = (got.to(F64) - ref.to(F64)).abs()
    return ~(err <= bound.to(F64))


def check(name, got, ref, bound):
    """|got - ref| <= bound element by element; NaN fails.  A failure names the worst element (largest error over
    bound), its index, the kernel's value and the reference value."""
    bad = violations(got, ref, bound)
    if bad.any():
        err = (got.to(F64) - ref.to(F64)).abs()
        tol = bound.to(F64).expand_as(err)
        ratio = torch.where(bad, (err / tol).nan_to_num(nan=math.inf, posinf=math.inf), torch.zeros_like(err))
        idx = tuple(int(i) for i in torch.unravel_index(ratio.reshape(-1).argmax().cpu(), got.shape))
        gv, rv = got[idx].item(), ref[idx].item()
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements outside the bound; worst at {idx}: "
                             f"got {gv!r}, ref {rv!r}, |err| {abs(gv - rv):.3e} > bound {tol[idx].item():.3e}")


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
