"""GEMM kernel tests: pg_gemm_bf16's persistent wgmma kernel (impl 0), its skinny kernel (impl 2) and SIMT kernel
(impl 1), split-K with pg_sum_partials and the bias gradient riding on weight-gradient launches, against the float64
reference of tests/_gemm_reference.py with element-wise bounds (derived in its docstring; tests/test_gemm_bounds_cpu.py
checks that they accept an emulation of the kernels and reject nine bug models).

Inputs come from the reference's regimes: randn, integer (every sum exact: results must equal the reference), onehot
(out(m, n) = alpha B(n, k(m)) exactly) and range (rows and columns scaled by 2^-40 .. 2^40).  Operands and outputs are
views inside NaN-filled buffers, some starting part-way into their rows: a tensor map or store built from the pitch
instead of the extent reads NaN or writes outside the view, and every bit outside the views is checked unchanged.
The tensor-core kernel's schedule (persistent CTAs, two consumer warpgroups taking turns) must not change a bit of the
result: the same launch is repeated and rerun on grids shrunk to 2, 4 and 6 CTAs (pg_reserve_sms)."""

import zlib

import pytest
import torch

import _gemm_reference as G
from _checks import check, check_equal

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
LAYOUTS = [(False, False), (False, True), (True, True), (True, False)]  # (a_mn, b_mn): forward, dgrad, wgrad, transposed A
LAYOUT_IDS = ["a_k-b_k", "a_k-b_mn", "a_mn-b_mn", "a_mn-b_k"]


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


@pytest.fixture
def grid(L):
    """set_grid(g): the persistent grids get g CTAs (g even; None = every SM) by reserving the other SMs.  The previous
    reservation comes back after the test, whether it passed or not."""
    old = L.reserve_sms(0)
    full = L.sm_count()

    def set_grid(g=None):
        L.reserve_sms(0 if g is None else full - g)
        assert L.sm_count() == (full if g is None else g)

    yield full, set_grid
    L.reserve_sms(old)


def _dev():
    return torch.device("cuda:0")


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _operand(X, mn, col_off=0):
    """(buf, view) of logical operand X [rows, K] as the kernel reads it: K-major X, or MN-major X^T [K, rows], inside a
    NaN-padded buffer (G.pitched)."""
    return G.pitched_copy((X.T if mn else X).contiguous(), col_off)


def _launch(L, tag, bufs, **kw):
    """L.gemm(**kw) with a snapshot of every buffer in `bufs` ({name: (buf, view)}) before it; checks after it that no
    bit outside the views changed."""
    snaps = {name: buf.clone() for name, (buf, _) in bufs.items()}
    L.gemm(**kw)
    torch.cuda.synchronize()
    for name, (buf, view) in bufs.items():
        G.check_untouched(f"{tag}{name}", buf, view, snaps[name])


# ----------------------------------------------------------------------------------------------------------------------
# a. main loop of the tensor-core kernel, every operand layout, tile edges
# ----------------------------------------------------------------------------------------------------------------------
# (M, N, K): every M in {1, 63, 64, 65, 127, 128, 129, 383}, N in {1, 8, 24, 32, 33, 64, 65, 128, 129, 200, 264} and K in
# {1, 8, 56, 64, 65, 136, 4104} at least once.  N picks the tile width (BN = 32 / 64 / 128; MN-major B takes 64 for
# N <= 32); K = 1 .. 64 is one k-block (two pipeline stages), the others end in a K tail or run 65 k-blocks.
MAIN_CASES = [
    (1, 1, 1), (63, 8, 8), (64, 24, 56), (65, 32, 64), (127, 33, 65), (128, 64, 136), (129, 65, 4104), (383, 128, 65),
    (129, 129, 136), (383, 200, 56), (65, 264, 4104), (128, 8, 4104), (383, 264, 1), (1, 200, 64),
]
SIMT_MAX_K = 136  # the SIMT kernel runs the cases up to this K


@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("M,N,K", MAIN_CASES)
def test_main_loop(L, M, N, K, a_mn, b_mn):
    """out_f32 = alpha A B^T (alpha = 1/2) within (K + 1) U24 |alpha| mag element by element, out_bf16 = bf16(out_f32)
    from the same launch bit for bit, exact in the integer and onehot regimes, nothing outside the views written; the
    SIMT kernel on the cases with K <= 136 as well."""
    alpha = 0.5
    for ri, regime in enumerate(G.REGIMES):
        A, B, _, _ = G.make_inputs(regime, M, N, K, _seed("main", M, N, K, regime), device=_dev())
        ref, mag = G.reference(A, B)
        bound = G.bound(K, alpha, mag)
        for impl in ([0, 1] if K <= SIMT_MAX_K else [0]):
            tag = f"impl {impl} {M}x{N}x{K} a_mn={a_mn} b_mn={b_mn} {regime}: "
            bufs = {"A": _operand(A, a_mn, col_off=8 * (ri & 1)), "B": _operand(B, b_mn, col_off=8 * (ri >> 1)),
                    "out_f32": G.pitched(M, N, F32, _dev(), col_off=8 * (ri & 1)),
                    "out_bf16": G.pitched(M, N, BF16, _dev(), col_off=8 * (ri >> 1))}
            of, ob = bufs["out_f32"][1], bufs["out_bf16"][1]
            _launch(L, tag, bufs, A=bufs["A"][1], B=bufs["B"][1], M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, out_f32=of,
                    out_bf16=ob, alpha=alpha, impl=impl)
            check(f"{tag}out_f32", of, alpha * ref, bound)
            if regime in G.EXACT_REGIMES:
                check(f"{tag}out_f32 exact", of, alpha * ref, G.exact_bound(ref))
            check_equal(f"{tag}out_bf16 = bf16(out_f32)", ob, of.to(BF16))


# ----------------------------------------------------------------------------------------------------------------------
# b. schedule invariance: persistent CTAs with one, two, three or dozens of work items
# ----------------------------------------------------------------------------------------------------------------------
def _run_outputs(L, tag, a, b, M, N, K, a_mn, b_mn, d0=None, c0=None, alpha=1.0, split_k=1, want_bf16=True):
    """One launch into fresh NaN-padded outputs (out_f32 = c0 and bias gradient = d0 first, when given); returns the
    output views (out_f32, out_bf16 or None, bias gradient or None) after checking the buffers around them."""
    bufs = {"A": a, "B": b, "out_f32": G.pitched(M, N, F32, _dev(), col_off=8)}
    kw = {}
    if c0 is not None:
        bufs["out_f32"][1].copy_(c0)
        kw["accumulate"] = True
    if want_bf16:
        bufs["out_bf16"] = G.pitched(M, N, BF16, _dev())
        kw["out_bf16"] = bufs["out_bf16"][1]
    if d0 is not None:
        dbuf = torch.full((M + 8,), float("nan"), device=_dev())
        bufs["bias_grad"] = (dbuf, dbuf[4:4 + M])  # 16 bytes into its allocation
        bufs["bias_grad"][1].copy_(d0)
        kw["bias_grad"] = bufs["bias_grad"][1]
    _launch(L, tag, bufs, A=a[1], B=b[1], M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, out_f32=bufs["out_f32"][1], alpha=alpha,
            split_k=split_k, **kw)
    return bufs["out_f32"][1], kw.get("out_bf16"), kw.get("bias_grad")


def _same_bits(tag, runs):
    """Every run's outputs equal the first run's bit for bit."""
    for label, outs in runs[1:]:
        for name, got, first in zip(("out_f32", "out_bf16", "bias gradient"), outs, runs[0][1]):
            if first is not None:
                check_equal(f"{tag}{name}, {label} vs {runs[0][0]}", got, first)


GRIDS = (2, 4, 6)
SCHEDULES = {  # work items (128 x 128 tiles) as a function of the full grid S
    "half_wave": lambda S: S // 2,       # one item per CTA, half the SMs idle
    "one_wave": lambda S: S,             # one item per CTA, every SM
    "wave_plus_one": lambda S: S + 1,    # CTA 0 runs two items: one per consumer warpgroup
    "three_per_cta": lambda S: 3 * S,    # an odd number of items per CTA (and 66 to 198 on the shrunk grids)
}


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)], ids=["a_k-b_k", "a_mn-b_mn"])
@pytest.mark.parametrize("schedule", list(SCHEDULES))
def test_schedule_invariance(L, grid, schedule, a_mn, b_mn):
    """M = 128 t - 37 rows of N = 128 columns (one 128-wide N block) give t work items; K = 200 ends in a K tail.  The
    launch runs twice on the full grid and once on grids of 2, 4 and 6 CTAs: out_f32, out_bf16 and (MN-major A) the bias
    gradient riding on it must be identical in every run, and the first run within its bounds."""
    full, set_grid = grid
    t = SCHEDULES[schedule](full)
    M, N, K = 128 * t - 37, 128, 200
    A, B, _, d0 = G.make_inputs("randn", M, N, K, _seed("schedule", schedule, a_mn), device=_dev())
    d0 = d0 if a_mn else None
    a, b = _operand(A, a_mn), _operand(B, b_mn)
    tag = f"{schedule} ({t} items on {full} CTAs) a_mn={a_mn}: "
    runs = [(f"run {i + 1}", _run_outputs(L, tag, a, b, M, N, K, a_mn, b_mn, d0=d0, alpha=0.5)) for i in range(2)]
    for g in GRIDS:
        set_grid(g)
        runs.append((f"{g} CTAs", _run_outputs(L, tag, a, b, M, N, K, a_mn, b_mn, d0=d0, alpha=0.5)))
    set_grid(None)
    of, _, db = runs[0][1]
    ref, mag = G.reference(A, B)
    check(f"{tag}out_f32", of, 0.5 * ref, G.bound(K, 0.5, mag))
    if d0 is not None:
        rs, rs_abs = G.row_sums(A)
        check(f"{tag}bias gradient", db, rs + d0.to(F64), G.rowsum_bound(K, rs_abs, d0))
    _same_bits(tag, runs)


@pytest.mark.parametrize("split_k", [3, 33])
def test_schedule_invariance_split(L, grid, split_k):
    """Split-K work items of different lengths in one CTA's sequence: K = 64 * 100 + 1 is 101 k-blocks, split 3 gives
    slices of 34, 34 and 33 k-blocks, split 33 gives 25 slices of 4 and one of 1; 2 x 2 tiles (M = N = 200).  Each
    consumer warpgroup steps the stage ring past the other's items by their lengths.  Repeated and on grids of 2, 4 and 6
    CTAs: out_f32 and the bias gradient identical, the first run within the split bound."""
    full, set_grid = grid
    M, N, K = 200, 200, 64 * 100 + 1
    A, B, c0, d0 = G.make_inputs("randn", M, N, K, _seed("schedule split", split_k), device=_dev())
    a, b = _operand(A, True), _operand(B, True)
    tag = f"split_k={split_k}: "
    kw = dict(d0=d0, c0=c0, alpha=0.5, split_k=split_k, want_bf16=False)
    runs = [(f"run {i + 1}", _run_outputs(L, tag, a, b, M, N, K, True, True, **kw)) for i in range(2)]
    for g in GRIDS:
        set_grid(g)
        runs.append((f"{g} CTAs", _run_outputs(L, tag, a, b, M, N, K, True, True, **kw)))
    set_grid(None)
    of, _, db = runs[0][1]
    ref, mag = G.reference(A, B)
    rs, rs_abs = G.row_sums(A)
    check(f"{tag}out_f32", of, c0.to(F64) + 0.5 * ref, G.bound(K, 0.5, mag, c0, split_k))
    check(f"{tag}bias gradient", db, d0.to(F64) + rs, G.rowsum_bound(K, rs_abs, d0, split_k))
    _same_bits(tag, runs)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)], ids=["a_k-b_k", "a_mn-b_mn"])
def test_row_extent_invariance(L, a_mn, b_mn):
    """The first M1 rows of A give the same bits as the same rows of the full launch (M = 1000), for M1 = 256 (a tile
    boundary) and M1 = 300 (inside a tile): a row's result does not depend on how many rows follow it."""
    M, N, K = 1000, 200, 136
    A, B, _, d0 = G.make_inputs("randn", M, N, K, _seed("extent", a_mn), device=_dev())
    d0 = d0 if a_mn else None
    a, b = _operand(A, a_mn), _operand(B, b_mn)
    full = _run_outputs(L, "M = 1000: ", a, b, M, N, K, a_mn, b_mn, d0=d0)
    for M1 in (256, 300):
        sub = (a[0], a[1][:, :M1] if a_mn else a[1][:M1])
        part = _run_outputs(L, f"M1 = {M1}: ", sub, b, M1, N, K, a_mn, b_mn, d0=None if d0 is None else d0[:M1])
        for name, got, whole in zip(("out_f32", "out_bf16", "bias gradient"), part, full):
            if whole is not None:
                check_equal(f"M1 = {M1} a_mn={a_mn}: {name}", got, whole[:M1])


# ----------------------------------------------------------------------------------------------------------------------
# c. split-K: slice counts either side of the per-warp slice sum, the recipes' depths, the bias gradient
# ----------------------------------------------------------------------------------------------------------------------
# name: (Cout = M, Cin = N, P = K, split_k, slices).  The weight-gradient layout (A = dY and B = X both MN-major), M and N
# tails, K not a multiple of 64.
SPLIT_CASES = {
    "split1": (24, 200, 64 * 37 + 13, 1, 1),
    "split2": (200, 200, 64 * 37 + 13, 2, 2),
    "split3": (24, 200, 64 * 37 + 13, 3, 3),       # 13, 13 and 12 k-blocks
    "slices63": (200, 200, 64 * 125 + 9, 63, 63),  # one thread per element sums the slices
    "slices64": (24, 200, 64 * 127 + 9, 64, 64),   # one warp per element
    "clamped": (200, 24, 300, 9, 5),               # split_k > k_iters: one slice per k-block
}
# The recipes' deepest weight gradients, split as ops._split_k_for plans them (98 and 131 slices on 132 SMs): ImageGPT's
# 64 x 64 weights at batch 64 of 28 x 28 images, and a 128-channel 1x1 weight gradient at batch 128.
RECIPE_CASES = {"imagegpt_64ch_b64": (64, 64, 64 * 784), "conv_128ch_b128": (128, 128, 128 * 784)}


def _split_case(case):
    if case in SPLIT_CASES:
        return SPLIT_CASES[case]
    from pytorch_generative_b200 import ops

    M, N, K = RECIPE_CASES[case]
    return M, N, K, ops._split_k_for(M, N, K), None


@pytest.mark.parametrize("regime", G.REGIMES)
@pytest.mark.parametrize("case", list(SPLIT_CASES) + list(RECIPE_CASES))
def test_split_k(L, grid, case, regime):
    """out_f32 = c0 + alpha A B^T and bias gradient = d0 + sum_k A, accumulated into random initial values, alpha 1 and
    1/2: within (64 kps + s + 1) U24 (|alpha| mag + |c0|) (and the same chain for the bias gradient); exact in the
    integer regime, where they also equal the split_k = 1 bits; identical when repeated and on a 6-CTA grid."""
    full, set_grid = grid
    M, N, K, split_k, slices = _split_case(case)
    _, kps, s = G.split_plan(K, split_k)
    if slices is None:
        assert s >= 64, f"{case}: {s} slices do not reach the per-warp slice sum"
    else:
        assert s == slices, (case, s)
    A, B, c0, d0 = G.make_inputs(regime, M, N, K, _seed("split", case, regime), device=_dev())
    a, b = _operand(A, True), _operand(B, True)
    ref, mag = G.reference(A, B)
    rs, rs_abs = G.row_sums(A)
    for alpha in (1.0, 0.5):
        tag = f"{case} ({s} slices of {kps} k-blocks) {regime} alpha={alpha}: "
        kw = dict(d0=d0, c0=c0, alpha=alpha, split_k=split_k, want_bf16=False)
        runs = [(f"run {i + 1}", _run_outputs(L, tag, a, b, M, N, K, True, True, **kw)) for i in range(2)]
        set_grid(6)
        runs.append(("6 CTAs", _run_outputs(L, tag, a, b, M, N, K, True, True, **kw)))
        set_grid(None)
        of, _, db = runs[0][1]
        out_ref, db_ref = c0.to(F64) + alpha * ref, d0.to(F64) + rs
        check(f"{tag}out_f32", of, out_ref, G.bound(K, alpha, mag, c0, split_k))
        check(f"{tag}bias gradient", db, db_ref, G.rowsum_bound(K, rs_abs, d0, split_k))
        if regime == "integer":
            check(f"{tag}out_f32 exact", of, out_ref, G.exact_bound(out_ref))
            check(f"{tag}bias gradient exact", db, db_ref, G.exact_bound(db_ref))
            if s > 1:
                runs.append(("split_k = 1", _run_outputs(L, tag, a, b, M, N, K, True, True, **dict(kw, split_k=1))))
        _same_bits(tag, runs)


# ----------------------------------------------------------------------------------------------------------------------
# d. skinny kernel (impl 2): M <= 32 rows, one warp per output column
# ----------------------------------------------------------------------------------------------------------------------
SKINNY_N = (1, 7, 8, 9, 2051)


def _skinny_case(L, M, N, K, regime):
    alpha = 0.5
    A, B, _, _ = G.make_inputs(regime, M, N, K, _seed("skinny", M, N, K, regime), device=_dev())
    ref, mag = G.reference(A, B)
    tag = f"skinny {M}x{N}x{K} {regime}: "
    bufs = {"A": _operand(A, False, col_off=8), "B": _operand(B, False), "out_f32": G.pitched(M, N, F32, _dev()),
            "out_bf16": G.pitched(M, N, BF16, _dev(), col_off=8)}
    of, ob = bufs["out_f32"][1], bufs["out_bf16"][1]
    _launch(L, tag, bufs, A=bufs["A"][1], B=bufs["B"][1], M=M, N=N, K=K, out_f32=of, out_bf16=ob, alpha=alpha, impl=2)
    check(f"{tag}out_f32", of, alpha * ref, G.bound(K, alpha, mag))
    if regime in G.EXACT_REGIMES:
        check(f"{tag}out_f32 exact", of, alpha * ref, G.exact_bound(ref))
    check_equal(f"{tag}out_bf16 = bf16(out_f32)", ob, of.to(BF16))


@pytest.mark.parametrize("K", [8, 72])
@pytest.mark.parametrize("M", [1, 2, 7, 31, 32])
def test_skinny(L, M, K):
    """out_f32 = alpha A B^T (alpha = 1/2) for N in {1, 7, 8, 9, 2051} (a partial last block of 8 warps): within
    (K + 1) U24 |alpha| mag, exact in the integer and onehot regimes, out_bf16 = bf16(out_f32) bit for bit, nothing
    outside the views written."""
    for N in SKINNY_N:
        for regime in G.REGIMES:
            _skinny_case(L, M, N, K, regime)


def test_skinny_shared_memory_limit(L):
    """M K 2 = 160 KiB, the most A rows the kernel stages in shared memory (M = 32, K = 2560)."""
    for N in (9, 2051):
        for regime in G.REGIMES:
            _skinny_case(L, 32, N, 2560, regime)


# name: (M, K, a_mn, b_mn, accumulate)
SKINNY_REFUSALS = {
    "33_rows": (33, 64, False, False, False),
    "over_160KiB": (32, 2568, False, False, False),
    "K_not_multiple_of_8": (4, 12, False, False, False),
    "A_mn_major": (4, 64, True, False, False),
    "B_mn_major": (4, 64, False, True, False),
    "accumulate": (4, 64, False, False, True),
}


@pytest.mark.parametrize("case", list(SKINNY_REFUSALS))
def test_skinny_refusals(L, case):
    """What the skinny kernel does not take comes back as a RuntimeError before any kernel is launched, and leaves the
    output as it was."""
    M, K, a_mn, b_mn, accumulate = SKINNY_REFUSALS[case]
    N = 16
    A, B, _, _ = G.make_inputs("randn", M, N, K, _seed("refusal", case), device=_dev())
    a, b = _operand(A, a_mn), _operand(B, b_mn)
    out_buf, out = G.pitched(M, N, F32, _dev())
    before, launches = out_buf.clone(), L.launch_count()
    with pytest.raises(RuntimeError, match="skinny"):
        L.gemm(a[1], b[1], M, N, K, a_mn=a_mn, b_mn=b_mn, out_f32=out, accumulate=accumulate, impl=2)
    torch.cuda.synchronize()
    assert L.launch_count() == launches, f"{case}: a kernel was launched"
    check_equal(f"{case}: output", out_buf, before)
