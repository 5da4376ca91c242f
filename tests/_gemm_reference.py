"""Float64 reference of the bf16 GEMM (pg_gemm_bf16), element-wise error bounds for its kernels, the input regimes the
GEMM tests draw from and NaN-padded operand / output views.  Shared by tests/test_gemm_kernels_gpu.py and
tests/test_gemm_bounds_cpu.py; not a test module.

Reference.  out = c0 + alpha A B^T with A [M, K] and B [N, K] the logical operands (the kernels read them K-major or
MN-major; the values are the same), computed in float64 on the device the tensors live on from the same bf16 values the
kernels read: ref = A64 B64^T, and its magnitude mag = |A64| |B64|^T.  The bias gradient of a weight-gradient launch is
d0 + sum_k A(m, k), with magnitude sum_k |A(m, k)|.

Kernel arithmetic the bounds follow (csrc/pg_gemm.cu, csrc/pg_host.cu).  Inputs are bf16, so every product is exact in
fp32; every sum is fp32.  A work item (output tile, K slice) accumulates its k-blocks of 64 in registers; the epilogue
multiplies by alpha, then stores or adds to the output (accumulate).  A split-K launch stores each slice, times alpha,
to its own scratch slice, and pg_sum_partials adds the slices in slice order (fewer than 64 slices: one thread per
element; 64 or more: 32 lanes with strided partials and a fixed butterfly) and adds the total to the output.  The bias
gradient is summed from the staged A tiles per (m block, slice), 16 k-rows per thread per k-block and two fixed
combining steps, then the same way across slices.  The skinny kernel (impl 2) and the SIMT kernel (impl 1) run one
fp32 chain per element in a different order.

Bound derivation.  U24 = 2^-24 is the unit roundoff of fp32.  A sum of n terms rounded to fp32 after each addition is
within (n - 1) U24 sum |terms| of the exact sum, whatever the order and the tree (the recursive-summation bound: every
term passes through at most n - 1 roundings; adding an exact zero rounds nothing, so padding and idle lanes add no
length).  Each further rounded operation on the way adds one U24 times the magnitudes it touches.  With
split_plan(K, split_k) = (k_iters, kps, s), kps k-blocks of 64 per slice and s slices:
  * plain, one slice:            (K + 1) U24 |alpha| mag            (K - 1 additions, the alpha multiply, one spare);
  * accumulate into c0:          (K + 2) U24 (|alpha| mag + |c0|)   (one more rounding, and |c0| joins the terms);
  * split-K, s > 1:              (64 kps + s + 1) U24 (|alpha| mag + |c0|)
      (a slice sums at most 64 kps products, alpha rounds once, the slice sum and the add to c0 take s more): far
      tighter than K when there are many short slices, which is where a lost or doubled slice has to show;
  * bias gradient:               the same chain with sum_k |A| for mag (alpha does not scale it).
The kernels' MMA accumulation is held to these bounds as stated, without a safety factor: tests/_checks.py compares
|got - ref| <= bound."""

import torch

from _checks import check_equal

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U24 = 2.0 ** -24
BK = 64   # k-block of the tensor-core kernel
BM = 128  # rows of one output tile

REGIMES = ("randn", "integer", "onehot", "range")
EXACT_REGIMES = ("integer", "onehot")  # products and sums exact in fp32: every path equals the reference


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def make_inputs(regime, M, N, K, seed, device="cpu"):
    """A [M, K], B [N, K] bf16 and an initial output c0 [M, N] / bias gradient d0 [M] (fp32), drawn on the CPU from
    `seed` and moved to `device`:
      randn    A, B, c0, d0 ~ N(0, 1);
      integer  A, B in {-3..3}, c0, d0 in {-8..8}: every partial sum is an integer (a half-integer after alpha = 1/2)
               of magnitude at most 9 K + 8, far below 2^23 at the tested K, so every summation order gives the exact
               result;
      onehot   A(m, k) = 1 iff k = (7 m + 3) mod K, B ~ N(0, 1): out(m, n) = alpha B(n, k(m)) exactly, so a slip in
               the swizzle or the k offset points at one (m, k);
      range    randn with row m of A scaled by 2^e_m and row n of B (output column n) by 2^f_n, e, f in [-40, 40]
               (c0 and d0 scaled alike): no dot product mixes magnitudes, and the bound is scale-invariant, so small
               outputs are held to the same relative accuracy as large ones."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g)
    if regime == "integer":
        ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).float()
        A, B, c0, d0 = ri(-3, 3, M, K), ri(-3, 3, N, K), ri(-8, 8, M, N), ri(-8, 8, M)
    else:
        A, B, c0, d0 = rn(M, K), rn(N, K), rn(M, N), rn(M)
        if regime == "onehot":
            A = torch.zeros(M, K)
            A[torch.arange(M), (7 * torch.arange(M) + 3) % K] = 1.0
        elif regime == "range":
            e = torch.exp2(torch.randint(-40, 41, (M,), generator=g).float())
            f = torch.exp2(torch.randint(-40, 41, (N,), generator=g).float())
            A, B, c0, d0 = A * e[:, None], B * f[:, None], c0 * e[:, None] * f[None, :], d0 * e
        else:
            assert regime == "randn", regime
    return A.to(BF16).to(device), B.to(BF16).to(device), c0.to(device), d0.to(device)


# ----------------------------------------------------------------------------------------------------------------------
# reference and bounds
# ----------------------------------------------------------------------------------------------------------------------
def split_plan(K, split_k):
    """(k_iters, kps, s) as pg_gemm_bf16 plans a launch: k-blocks, k-blocks per slice and slices.  split_k is clamped to
    [1, k_iters]; kps = ceil(k_iters / split_k) and s = ceil(k_iters / kps), so no slice is empty and the last one may be
    shorter."""
    k_iters = (K + BK - 1) // BK
    split = min(max(split_k, 1), k_iters)
    kps = (k_iters + split - 1) // split
    return k_iters, kps, (k_iters + kps - 1) // kps


def reference(A, B):
    """(ref, mag) = (A B^T, |A| |B|^T) in float64, [M, N]."""
    A64, B64 = A.to(F64), B.to(F64)
    return A64 @ B64.T, A64.abs() @ B64.abs().T


def row_sums(A):
    """(sum_k A, sum_k |A|) in float64, [M]."""
    A64 = A.to(F64)
    return A64.sum(1), A64.abs().sum(1)


def chain(K, split_k=1, accumulate=False):
    """Roundings along the longest chain of one output element (see the module docstring)."""
    _, kps, s = split_plan(K, split_k)
    if s == 1:
        return K + (2 if accumulate else 1)
    return BK * kps + s + 1


def bound(K, alpha, mag, c0=None, split_k=1):
    """Element-wise bound of alpha A B^T (+ c0): chain(K, split_k, c0 given) U24 (|alpha| mag (+ |c0|))."""
    b = abs(alpha) * mag
    if c0 is not None:
        b = b + c0.to(F64).abs()
    return chain(K, split_k, c0 is not None) * U24 * b


def rowsum_bound(K, abs_sum, d0, split_k=1):
    """Element-wise bound of the bias gradient d0 + sum_k A."""
    return chain(K, split_k, True) * U24 * (abs_sum + d0.to(F64).abs())


def exact_bound(ref):
    """A zero bound: the result must equal the reference exactly."""
    return torch.zeros_like(ref, dtype=F64)


# ----------------------------------------------------------------------------------------------------------------------
# NaN-padded views
# ----------------------------------------------------------------------------------------------------------------------
def pitched(rows, cols, dtype, device, col_off=0, fill=float("nan")):
    """(buf, view): a [rows, cols] view with unit inner stride inside a buffer filled with `fill` (NaN by default).  The
    row pitch is col_off + cols rounded up to 8, plus 8: at least 8 padding columns, a 16-byte-aligned pitch for bf16
    and fp32; three padding rows sit below the view.  col_off (a multiple of 8) starts the view part-way into each row,
    like a q / k / v column slice of a fused projection.  A kernel that read a tensor through its pitch instead of its
    extent would read NaN; one that wrote outside the view changes the buffer (see check_untouched)."""
    assert col_off % 8 == 0
    ld = (col_off + cols + 7) // 8 * 8 + 8
    buf = torch.full((rows + 3, ld), fill, dtype=dtype, device=device)
    return buf, buf[:rows, col_off:col_off + cols]


def pitched_copy(src, col_off=0):
    """src copied into a NaN-padded view (pitched); returns (buf, view)."""
    buf, view = pitched(src.shape[0], src.shape[1], src.dtype, src.device, col_off)
    view.copy_(src)
    return buf, view


def outside(buf, view):
    """Boolean mask of the elements of buf outside view."""
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask.as_strided(view.shape, view.stride(), view.storage_offset() - buf.storage_offset()).fill_(False)
    return mask


def check_untouched(name, buf, view, before):
    """Every bit of buf outside view equals the snapshot `before` (taken before the launch)."""
    m = outside(buf, view)
    check_equal(f"{name}: outside the view", buf[m], before[m])
