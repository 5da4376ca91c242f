"""Tests of the GEMM kernel tests, without a GPU: the bounds of tests/_gemm_reference.py must accept an fp32 emulation
of the kernels' arithmetic in every input regime (and equal the reference exactly where the regime makes every sum
exact), and reject the same emulation with one of nine plausible kernel bugs.

The emulation follows csrc/pg_gemm.cu and pg_sum_partials (csrc/pg_host.cu) on the CPU in fp32 from the bf16 inputs:
each work item accumulates its k-blocks of 64 in k16 steps into an fp32 accumulator, multiplies by alpha and stores
(one slice) or writes its split slice; the slices are summed in slice order (one chain below 64 slices, 32 strided
lanes and a fixed butterfly from 64 on) and added to the initial value.  The bias gradient is summed per (m block,
slice) by four k-row groups (k = g + 4 i of every k-block, read through the 128-byte swizzle), combined in a fixed
order, and then across slices the same way.  Each bug model is the emulation with one change:
  first_k16     the second k16 step of an item overwrites the accumulator (the first step's products are lost);
  swizzle       rows with row % 8 == 7 read k chunk 0 of every k-block from chunk 1, its swizzle neighbour;
  tail_block    the last k-block of a K tail dropped;
  drop_slice0   split slice 0 left out of the slice sum;
  last_partial  the per-lane sum stops one partial short (64 or more slices only);
  alpha_split   split slices stored without alpha;
  c0_twice      the initial value added twice;
  bf16_slices   split slices stored in bf16;
  rowsum_chunk  the bias-gradient threads read the 8-column chunk at swizzle position cc ^ ((k + 1) & 7) instead of
                cc ^ (k & 7)."""

import pytest
import torch

import _gemm_reference as G
from _checks import check, violations

F32 = torch.float32
BUGS = ("first_k16", "swizzle", "tail_block", "drop_slice0", "last_partial", "alpha_split", "c0_twice", "bf16_slices",
        "rowsum_chunk")


# ----------------------------------------------------------------------------------------------------------------------
# fp32 emulation
# ----------------------------------------------------------------------------------------------------------------------
def _sum_partials(parts, bug=None):
    """pg_sum_partials over the slice axis 0 of parts [s, ...] (fp32)."""
    s = parts.shape[0]
    if s < 64:
        acc = torch.zeros_like(parts[0])
        for p in range(s):
            if not (bug == "drop_slice0" and p == 0):
                acc = acc + parts[p]
        return acc
    lanes = torch.zeros((32,) + parts.shape[1:], dtype=F32)
    for p in range(s - (1 if bug == "last_partial" else 0)):
        if not (bug == "drop_slice0" and p == 0):
            lanes[p % 32] = lanes[p % 32] + parts[p]
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[idx ^ o]
    return lanes[0]


def _rowsum_item(Ab, k0, k1, bug=None):
    """Row sums of one (m block, slice) of Ab [Mp, Kp] (fp32 values of bf16, zero past M and K): four k-row groups
    g = 0..3 each add k = g + 4 i (i = 0..15) of every k-block in order, then (g0 + g1) + (g2 + g3)."""
    Mp = Ab.shape[0]
    acc = torch.zeros(4, Mp, dtype=F32)
    m = torch.arange(Mp)
    for kit in range(k0, k1):
        blk = Ab[:, kit * G.BK:(kit + 1) * G.BK]
        for i in range(16):
            for g in range(4):
                k = g + 4 * i
                rows = m
                if bug == "rowsum_chunk":  # position cc ^ ((k + 1) & 7) holds logical chunk cc ^ ((k + 1) & 7) ^ (k & 7)
                    c = (m % 128) // 8
                    cc = (c & 7) ^ ((k + 1) & 7) ^ (k & 7)
                    rows = (m // 128) * 128 + (c >> 3) * 64 + cc * 8 + m % 8
                acc[g] = acc[g] + blk[rows, k]
    return (acc[0] + acc[1]) + (acc[2] + acc[3])


def emulate(A, B, alpha=1.0, c0=None, d0=None, split_k=1, bug=None):
    """out (fp32 [M, N]) and, when d0 is given, the bias gradient (fp32 [M]) of one pg_gemm_bf16 launch on A [M, K],
    B [N, K] (bf16); c0 given = accumulate into c0."""
    M, K = A.shape
    N = B.shape[0]
    k_iters, kps, s = G.split_plan(K, split_k)
    Kp, Mp = k_iters * G.BK, (M + G.BM - 1) // G.BM * G.BM
    Af = torch.zeros(Mp, Kp, dtype=F32)
    Af[:M, :K] = A.float()
    Bf = torch.zeros(N, Kp, dtype=F32)
    Bf[:, :K] = B.float()
    Am = Af.clone()
    if bug == "swizzle":
        rows = torch.arange(M)[torch.arange(M) % 8 == 7]
        for kit in range(k_iters):
            Am[rows, kit * G.BK:kit * G.BK + 8] = Af[rows, kit * G.BK + 8:kit * G.BK + 16]
    a32 = torch.tensor(alpha, dtype=F32)
    slices, rsums = [], []
    for ks in range(s):
        k0, k1 = ks * kps, min((ks + 1) * kps, k_iters)
        acc = torch.zeros(M, N, dtype=F32)
        for kit in range(k0, k1):
            if bug == "tail_block" and K % G.BK and kit == k_iters - 1:
                continue
            for kk in range(G.BK // 16):
                c = slice(kit * G.BK + 16 * kk, kit * G.BK + 16 * kk + 16)
                prod = Am[:M, c] @ Bf[:, c].T
                acc = prod if (bug == "first_k16" and kit == k0 and kk == 1) else acc + prod
        if s > 1:
            v = acc if bug == "alpha_split" else acc * a32
            slices.append(v.to(torch.bfloat16).float() if bug == "bf16_slices" else v)
        else:
            slices.append(acc * a32)
        if d0 is not None:
            rsums.append(_rowsum_item(Af, k0, k1, bug)[:M])
    if s == 1:
        total, rtotal = slices[0], (rsums[0] if rsums else None)
    else:
        total = _sum_partials(torch.stack(slices), bug)
        rtotal = _sum_partials(torch.stack(rsums), bug) if rsums else None
    out = total if c0 is None else c0 + total
    if c0 is not None and bug == "c0_twice":
        out = out + c0
    rowsum = None if d0 is None else d0 + rtotal
    return out, rowsum


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
# name: (M, N, K, split_k, accumulate).  Every K has a tail (K % 64 != 0); M spans rows with row % 8 == 7.
CASES = {
    "plain": (136, 40, 200, 1, False),          # two m blocks, 4 k-blocks
    "accumulate": (72, 24, 1100, 1, True),      # one slice into c0, with the bias gradient
    "split3": (40, 24, 64 * 37 + 13, 3, True),  # slices of 13, 13, 12 k-blocks
    "split65": (24, 16, 64 * 64 + 8, 65, True),  # 65 slices of one k-block: the per-warp slice sum
}


def _run(regime, case, alpha, bug=None, seed=0):
    """[(name, got, ref, bound)] of one emulated launch."""
    M, N, K, split_k, acc = CASES[case]
    A, B, c0, d0 = G.make_inputs(regime, M, N, K, seed)
    ref, mag = G.reference(A, B)
    c0 = c0 if acc else None
    d0 = d0 if acc else None
    out, rowsum = emulate(A, B, alpha, c0, d0, split_k, bug)
    res = [("out", out, alpha * ref + (0 if c0 is None else c0.to(G.F64)), G.bound(K, alpha, mag, c0, split_k))]
    if d0 is not None:
        rs, rs_abs = G.row_sums(A)
        res.append(("bias gradient", rowsum, rs + d0.to(G.F64), G.rowsum_bound(K, rs_abs, d0, split_k)))
    return res


@pytest.mark.parametrize("alpha", [1.0, 0.5])
@pytest.mark.parametrize("regime", G.REGIMES)
@pytest.mark.parametrize("case", list(CASES))
def test_emulation_within_bounds(case, regime, alpha):
    """The fp32 emulation meets every bound in every regime, and is exact where the regime makes every sum exact
    (integer always; onehot without an initial value, which would round the single product once)."""
    acc = CASES[case][4]
    for name, got, ref, bound in _run(regime, case, alpha):
        tag = f"{case} {regime} alpha={alpha} {name}"
        check(tag, got, ref, bound)
        if regime == "integer" or (regime == "onehot" and not acc):
            check(f"{tag} (exact)", got, ref, G.exact_bound(ref))


def test_split_plan():
    """split_plan restates the kernel's rounding: uneven last slices, clamping to k_iters, and the slice counts the
    GPU tests rely on."""
    assert G.split_plan(64 * 37 + 13, 3) == (38, 13, 3)
    assert G.split_plan(64 * 125 + 9, 63) == (126, 2, 63)
    assert G.split_plan(64 * 127 + 9, 64) == (128, 2, 64)
    assert G.split_plan(300, 9) == (5, 1, 5)
    assert G.split_plan(50176, 98) == (784, 8, 98)
    assert G.split_plan(100352, 132) == (1568, 12, 131)
    assert G.split_plan(64 * 100 + 1, 60) == (101, 2, 51)  # 60 requested, 51 slices: the kernel's rounding


# the case and regime under which each bug model must break a bound (any one suffices; these are the ones that show it)
BUG_CASES = {
    "first_k16": ("plain", "randn"),
    "swizzle": ("plain", "randn"),
    "tail_block": ("accumulate", "integer"),
    "drop_slice0": ("split3", "randn"),
    "last_partial": ("split65", "randn"),
    "alpha_split": ("split3", "integer"),
    "c0_twice": ("accumulate", "randn"),
    "bf16_slices": ("split65", "randn"),
    "rowsum_chunk": ("accumulate", "randn"),
}


@pytest.mark.parametrize("bug", BUGS)
def test_bug_model_breaks_the_bound(bug):
    """Each bug model applied to the emulation puts elements outside a bound (alpha = 1/2, so that a missing alpha
    shows)."""
    case, regime = BUG_CASES[bug]
    failed = [name for name, got, ref, b in _run(regime, case, 0.5, bug) if violations(got, ref, b).any()]
    assert failed, f"bug model {bug} stays within every bound on {case} under {regime}"


@pytest.mark.parametrize("bug", ["first_k16", "swizzle", "tail_block", "drop_slice0", "last_partial"])
def test_bug_model_breaks_exactness(bug):
    """The main-loop and slice-sum bug models also break the exact results of the integer regime: a mutated kernel
    fails there with a plain inequality, not only a bound."""
    case = {"first_k16": "plain", "swizzle": "plain", "tail_block": "plain", "drop_slice0": "split3",
            "last_partial": "split65"}[bug]
    name, got, ref, _ = _run("integer", case, 0.5, bug)[0]
    assert violations(got, ref, G.exact_bound(ref)).any(), f"bug model {bug} keeps {case} exact"
