"""Kernel tests for the rest of the training step: LayerNorm (pg_layernorm_fwd / _bwd and the pitched _ld forms), the
small-Cin input convolution (pg_conv_small_fwd / _bwd), the recipe loss (pg_bce_logits_fwd_bwd), column sums
(pg_colsum_f32 / _bf16) and the optimizer (pg_grad_sqnorm, pg_adam_step, FusedAdam) against the float64 references of
tests/_step_reference.py, every element held to its own bound (derived in that module's docstring; tests/
test_step_bounds_cpu.py checks that the bounds accept an fp32 emulation of the kernels and reject their bug models).

Inputs come from the reference's regimes: LayerNorm rows with large means over unit spread, constant rows (y must equal
beta bit for bit wherever the fp32 mean is exact) and rows scaled by 2^-20 .. 2^20; BCE logits beyond expf's overflow
edge with hard and soft targets; Adam moments near zero.  Pitched tensors live in NaN-filled buffers: NaN in a pad
column must not reach any output, the pad columns LayerNorm writes must be +0.0 bit for bit, and rows below a view must
stay untouched.  The persistent grids are rerun shrunk through pg_reserve_sms, so each warp walks many rows and the
block partials fall on both sides of pg_sum_partials' 64-partial switch.  Reductions must give identical bits when a
launch is repeated."""

import zlib

import pytest
import torch

import _step_reference as R
from _act_reference import ELU, NONE, RELU
from _checks import check, check_equal
from _gemm_reference import check_untouched

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
NAN = float("nan")
EPS = 1e-5


@pytest.fixture(scope="module")
def L():
    from pytorch_generative_b200 import _lib

    _lib.load()
    return _lib


@pytest.fixture
def grid(L):
    """set_grid(g): the persistent grids are sized for g SMs (g even; None = every SM) by reserving the others.  The
    previous reservation comes back after the test, whether it passed or not."""
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


def _buf(P, ld, dtype=F32, fill=NAN):
    """A [P + 3, ld] buffer filled with `fill`: the kernel gets its first P rows (contiguous, pitch ld)."""
    return torch.full((P + 3, ld), fill, dtype=dtype, device=_dev())


def _into(src, ld, dtype=None):
    """src [P, C] copied into the first C columns of a NaN-filled _buf(P, ld)."""
    b = _buf(src.shape[0], ld, dtype or src.dtype)
    b[:src.shape[0], :src.shape[1]] = src.to(b.dtype)
    return b


def _sync():
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------------
FAST_C = [128 * v for v in range(1, 9)]
GENERIC_C = [1, 3, 100, 129, 1000, 1025, 2048, 4096]
LN_WIDTHS = [(C, C) for C in FAST_C + GENERIC_C] + [(3, 8), (100, 104), (129, 136), (1000, 1008)]
LN_ROWS = [1, 7, 2113, 20000]


def _fast(C, ld):
    return ld == C and C % 128 == 0 and C <= 1024


def _ln_run(L, regime, P, C, ld, seed, dy_bf16=False):
    """One forward and one backward on NaN-padded buffers of pitch ld; every check of the contract.  Returns the
    outputs (for the variant / determinism comparisons)."""
    x, gamma, beta, dy, r0, r1 = (t.to(_dev()) for t in R.ln_inputs(regime, P, C, seed))
    xb = _into(x, ld)
    gamma_, beta_ = gamma.contiguous(), beta.contiguous()
    y_f, y_b = _buf(P, ld), _buf(P, ld, BF16)
    st = torch.full((2, P + 3), NAN, device=_dev())
    snap = [t.clone() for t in (y_f, y_b, st)]
    L.layernorm_fwd(xb[:P], gamma_, beta_, EPS, y_bf16=y_b[:P], y_f32=y_f[:P], mean=st[0, :P], rstd=st[1, :P])
    _sync()
    ref = R.ln_fwd_reference(x, gamma, beta, EPS)
    tag = f"{regime} P={P} C={C} ld={ld}"
    check(f"{tag} mean", st[0, :P], ref["mean"], ref["b_mean"])
    check(f"{tag} rstd", st[1, :P], ref["rstd"], ref["b_rstd"])
    check(f"{tag} y", y_f[:P, :C], ref["y"], ref["b_y"])
    check_equal(f"{tag} y bf16", y_b[:P, :C], y_f[:P, :C].to(BF16))
    if regime == "constant" and R.ln_mean_exact(C, _fast(C, ld)):
        check_equal(f"{tag} constant rows: y == beta", y_f[:P, :C], beta.expand(P, C))
    for name, b, s in (("y", y_f, snap[0]), ("y bf16", y_b, snap[1])):
        check_equal(f"{tag} {name} pad columns", b[:P, C:], torch.zeros_like(b[:P, C:]))
        check_untouched(f"{tag} {name}", b, b[:P], s)
    check_untouched(f"{tag} mean / rstd", st, st[:, :P], snap[2])

    mean, rstd = st[0, :P].clone(), st[1, :P].clone()
    dyb = _into(dy, ld, BF16 if dy_bf16 else F32)
    r0b, r1b = _into(r0, ld), _into(r1, ld)
    dx_f, dx_b = _buf(P, ld), _buf(P, ld, BF16)
    g = torch.Generator().manual_seed(seed + 1)
    d0 = [torch.randn(C, generator=g).to(_dev()) for _ in range(3)]
    acc = [torch.full((C + 3,), NAN, device=_dev()) for _ in range(3)]
    for a, v in zip(acc, d0):
        a[:C] = v
    snap = [t.clone() for t in (dx_f, dx_b, *acc)]
    L.layernorm_bwd(dyb[:P], xb[:P], gamma_, mean, rstd, dres0=r0b[:P], dres1=r1b[:P], dx_f32=dx_f[:P],
                    dx_bf16=dx_b[:P], dgamma=acc[0][:C], dbeta=acc[1][:C], dx_colsum=acc[2][:C])
    _sync()
    dy_read = dyb[:P, :C].float()
    bref = R.ln_bwd_reference(dy_read, x, gamma, mean, rstd, r0, r1, d0)
    check(f"{tag} dx", dx_f[:P, :C], bref["dx"], bref["b_dx"])
    check_equal(f"{tag} dx bf16", dx_b[:P, :C], dx_f[:P, :C].to(BF16))
    for k, a in zip(("dgamma", "dbeta", "colsum"), acc):
        check(f"{tag} {k}", a[:C], bref[k], bref["b_" + k])
    for name, b, s in (("dx", dx_f, snap[0]), ("dx bf16", dx_b, snap[1])):
        check_equal(f"{tag} {name} pad columns", b[:P, C:], torch.zeros_like(b[:P, C:]))
        check_untouched(f"{tag} {name}", b, b[:P], s)
    for k, a, s in zip(("dgamma", "dbeta", "colsum"), acc, snap[2:]):
        check_untouched(f"{tag} {k}", a, a[:C], s)
    return dict(xb=xb, gamma=gamma_, beta=beta_, y_f=y_f, y_b=y_b, mean=mean, rstd=rstd, dyb=dyb, r0b=r0b, r1b=r1b,
                dx_f=dx_f, dx_b=dx_b, acc=acc, d0=d0)


def _ln_rows(C):
    return [P for P in LN_ROWS if P * C <= 20000 * 1024]


LN_PARAMS = [(C, ld, P) for C, ld in LN_WIDTHS for P in _ln_rows(C)]


@pytest.mark.parametrize("regime", R.LN_REGIMES)
@pytest.mark.parametrize("C,ld,P", LN_PARAMS, ids=[f"C{C}-ld{ld}-P{P}" for C, ld, P in LN_PARAMS])
def test_layernorm(L, C, ld, P, regime):
    """The fast path (C = 128 V, V = 1..8), the generic path and the pitched _ld path: y, mean, rstd, dx, dgamma, dbeta
    and colsum(dx) within their bounds, pad columns +0.0, nothing written outside the views.  A repeated launch gives
    identical bits."""
    o = _ln_run(L, regime, P, C, ld, _seed("ln", C, ld, P, regime))
    y2, st2 = _buf(P, ld), torch.empty(2, P, device=_dev())
    L.layernorm_fwd(o["xb"][:P], o["gamma"], o["beta"], EPS, y_f32=y2[:P], mean=st2[0], rstd=st2[1])
    dx2 = _buf(P, ld)
    acc2 = [v.clone() for v in o["d0"]]
    L.layernorm_bwd(o["dyb"][:P], o["xb"][:P], o["gamma"], o["mean"], o["rstd"], dres0=o["r0b"][:P], dres1=o["r1b"][:P],
                    dx_f32=dx2[:P], dgamma=acc2[0], dbeta=acc2[1], dx_colsum=acc2[2])
    _sync()
    check_equal("repeated y", y2[:P], o["y_f"][:P])
    check_equal("repeated mean / rstd", st2, torch.stack([o["mean"], o["rstd"]]))
    check_equal("repeated dx", dx2[:P], o["dx_f"][:P])
    for k, a, b in zip(("dgamma", "dbeta", "colsum"), acc2, o["acc"]):
        check_equal(f"repeated {k}", a, b[:C])


@pytest.mark.parametrize("C,ld", [(256, 256), (1024, 1024), (100, 100), (129, 136), (4096, 4096)])
def test_layernorm_variants(L, C, ld):
    """dy in bf16; each forward output alone (y_bf16 only, y_f32 only, mean / rstd NULL) gives the same bits as the full
    call; the backward with dx_f32 alone and no column sums."""
    P = 2113
    o = _ln_run(L, "randn", P, C, ld, _seed("lnv", C, ld), dy_bf16=True)
    yb = _buf(P, ld, BF16)
    L.layernorm_fwd(o["xb"][:P], o["gamma"], o["beta"], EPS, y_bf16=yb[:P])
    yf = _buf(P, ld)
    L.layernorm_fwd(o["xb"][:P], o["gamma"], o["beta"], EPS, y_f32=yf[:P])
    dx = _buf(P, ld)
    L.layernorm_bwd(o["dyb"][:P], o["xb"][:P], o["gamma"], o["mean"], o["rstd"], dx_f32=dx[:P])
    _sync()
    check_equal("y_bf16 alone", yb[:P], o["y_b"][:P])
    check_equal("y_f32 alone, no statistics", yf[:P], o["y_f"][:P])
    x = o["xb"][:P, :C]
    bref = R.ln_bwd_reference(o["dyb"][:P, :C].float(), x, o["gamma"], o["mean"], o["rstd"])
    check("dx without residuals", dx[:P, :C], bref["dx"], bref["b_dx"])
    check_equal("dx pad columns", dx[:P, C:], torch.zeros_like(dx[:P, C:]))


@pytest.mark.parametrize("sms", [2, 10, 40])
@pytest.mark.parametrize("C,ld,P", [(128, 128, 20000), (1024, 1024, 2113), (100, 104, 20000), (1000, 1000, 2113)])
def test_layernorm_shrunk_grid(L, grid, C, ld, P, sms):
    """Persistent grids sized for 2, 10 and 40 SMs: the fast backward runs 4, 20 or 80 blocks of 8 warps and the generic
    one 16, 80 or 320 one-warp blocks, so every warp walks tens to thousands of rows and the block partials fall on
    both sides of 64.  The results stay within their bounds."""
    _, set_grid = grid
    set_grid(sms)
    _ln_run(L, "offset", P, C, ld, _seed("lng", C, ld, P))


def test_layernorm_refuses_more_than_4096_generic_channels(L):
    """The generic backward keeps [3][C] partials in shared memory: C = 4097 must raise before any launch."""
    P, C = 4, 4097
    x = torch.randn(P, C, device=_dev())
    gamma = torch.ones(C, device=_dev())
    st = torch.ones(2, P, device=_dev())
    dx = torch.empty(P, C, device=_dev())
    before = L.launch_count()
    with pytest.raises(RuntimeError, match="4096"):
        L.layernorm_bwd(x, x, gamma, st[0], st[1], dx_f32=dx, dgamma=torch.zeros(C, device=_dev()))
    assert L.launch_count() == before


# ----------------------------------------------------------------------------------------------------------------------
# small-Cin convolution
# ----------------------------------------------------------------------------------------------------------------------
CONV_CASES = [  # N, Cin, H, W, Cout, kh, kw, ph, pw
    (4, 3, 32, 32, 512, 3, 3, 1, 1), (3, 1, 28, 28, 32, 7, 7, 3, 3), (2, 3, 8, 8, 24, 3, 3, 1, 1),
    (2, 1, 28, 28, 64, 3, 3, 1, 1), (2, 16, 28, 28, 64, 3, 3, 1, 1), (2, 3, 16, 16, 128, 7, 7, 3, 3),
    (2, 3, 12, 20, 32, 3, 5, 1, 2),
    (2, 2, 12, 10, 48, 3, 3, 1, 1), (2, 4, 12, 10, 48, 3, 3, 1, 1), (2, 5, 12, 10, 48, 3, 3, 1, 1),
    (2, 32, 8, 8, 64, 1, 5, 0, 2),     # K = 160 = MAX_K
    (2, 3, 9, 9, 256, 7, 7, 3, 3),     # Cout K = 37632 weight-gradient outputs: three launches of 16384
    (1, 3, 5, 7, 24, 3, 3, 1, 1),      # P = 35, not a multiple of 32
    (3, 3, 1, 1, 16, 3, 3, 1, 1),      # 1x1 images
]


@pytest.mark.parametrize("pre_act", [NONE, RELU, ELU], ids=["none", "relu", "elu"])
@pytest.mark.parametrize("case", CONV_CASES, ids=["x".join(map(str, c)) for c in CONV_CASES])
def test_conv_small(L, case, pre_act):
    """out (fp32 and bf16(relu(out))), dw and dbias onto nonzero initial values, dx (NaN-filled before the launch, so a
    channel left unwritten fails) within their bounds."""
    N, Cin, H, W, Cout, kh, kw, ph, pw = case
    x, w, b, dy, dw0, db0 = (t.to(_dev()) for t in R.conv_inputs(N, Cin, H, W, Cout, kh, kw, _seed("conv", case)))
    P = N * H * W
    out = _buf(P, Cout)
    out_b = _buf(P, Cout, BF16)
    snap = [out.clone(), out_b.clone()]
    L.conv_small_fwd(x, w, b, (ph, pw), out_f32=out[:P], out_bf16=out_b[:P], act_bf16=RELU, pre_act=pre_act)
    dw, db = dw0.clone(), db0.clone()
    dx = torch.full_like(x, NAN)
    L.conv_small_bwd(x, w, dy, (ph, pw), dw=dw, dbias=db, dx=dx, pre_act=pre_act)
    _sync()
    ref = R.conv_reference(x, w, b, dy, (ph, pw), pre_act, dw0, db0)
    check("out", out[:P], ref["out"], ref["b_out"])
    check_equal("out bf16 = bf16(relu(out))", out_b[:P], out[:P].clamp_min(0).to(BF16))
    check_untouched("out", out, out[:P], snap[0])
    check_untouched("out bf16", out_b, out_b[:P], snap[1])
    check("dw", dw, ref["dw"], ref["b_dw"])
    check("dbias", db, ref["db"], ref["b_db"])
    check("dx", dx, ref["dx"], ref["b_dx"])


def test_conv_small_refusals(L):
    """K = Cin kh kw = 161 and a dgrad weight tile over 200 KiB (with dx requested) raise before any launch."""
    x = torch.randn(1, 23, 8, 8, device=_dev())
    w = torch.randn(16, 23, 7, 1, device=_dev())  # K = 161
    dy = torch.randn(64, 16, device=_dev())
    before = L.launch_count()
    with pytest.raises(RuntimeError, match="exceeds"):
        L.conv_small_fwd(x, w, None, (3, 0), out_f32=torch.empty(64, 16, device=_dev()))
    with pytest.raises(RuntimeError, match="exceeds"):
        L.conv_small_bwd(x, w, dy, (3, 0), dw=torch.zeros_like(w), dx=torch.empty_like(x))
    x3 = torch.randn(1, 3, 8, 8, device=_dev())
    w3 = torch.randn(400, 3, 7, 7, device=_dev())  # K Cout 4 B = 235200 B
    with pytest.raises(RuntimeError, match="weight tile"):
        L.conv_small_bwd(x3, w3, torch.randn(64, 400, device=_dev()), (3, 3), dx=torch.empty_like(x3))
    assert L.launch_count() == before


# ----------------------------------------------------------------------------------------------------------------------
# BCE with logits
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hard", [False, True], ids=["soft", "hard"])
@pytest.mark.parametrize("regime", R.BCE_REGIMES)
@pytest.mark.parametrize("numel", [1, 255, 257, "sweep+1", 16 * 3 * 64 * 64])
def test_bce(L, numel, regime, hard):
    """loss onto a nonzero loss_sum and dlogits within their bounds; dlogits = NULL gives the same loss bits; a repeated
    launch gives identical bits.  "sweep+1" is one more element than the capped grid (4 blocks of 256 threads per SM)
    covers in one sweep, so one thread loops."""
    if numel == "sweep+1":
        numel = L.sm_count() * 4 * 256 + 1
    l, t = (v.to(_dev()) for v in R.bce_inputs(regime, numel, _seed("bce", numel, regime, hard), hard))
    scale, loss0 = 1.0 / 16, 2.5
    loss = torch.full((4,), NAN, device=_dev())
    loss[0] = loss0
    dl = torch.full((numel + 3,), NAN, device=_dev())
    snap = [loss.clone(), dl.clone()]
    L.bce_logits(l, t, scale, loss[:1], dl[:numel])
    loss2 = torch.full((1,), loss0, device=_dev())
    L.bce_logits(l, t, scale, loss2)
    loss3 = torch.full((1,), loss0, device=_dev())
    dl3 = torch.empty(numel, device=_dev())
    L.bce_logits(l, t, scale, loss3, dl3)
    _sync()
    ref, b, dref, db = R.bce_reference(l, t, scale, loss0)
    check("loss", loss[:1], torch.tensor([ref], dtype=F64, device=_dev()), torch.tensor([b], dtype=F64, device=_dev()))
    check("dlogits", dl[:numel], dref, db)
    check_untouched("loss", loss, loss[:1], snap[0])
    check_untouched("dlogits", dl, dl[:numel], snap[1])
    check_equal("loss with dlogits = NULL", loss2, loss[:1])
    check_equal("repeated loss", loss3, loss[:1])
    check_equal("repeated dlogits", dl3, dl[:numel])


# ----------------------------------------------------------------------------------------------------------------------
# column sums
# ----------------------------------------------------------------------------------------------------------------------
COLSUM_CASES = []
for _path, _rows in (("vec", 256), ("scalar", 512)):
    for _strips in (63, 65):
        for _C in (255, 256, 257, 264):
            if _path == "vec" and _C % 8:
                continue
            COLSUM_CASES.append((_path, _strips * _rows - (_rows // 2 if _strips == 65 else 0), _C))


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("path,P,C", COLSUM_CASES, ids=[f"{p}-P{P}-C{C}" for p, P, C in COLSUM_CASES])
def test_colsum(L, path, P, C, dtype, accumulate):
    """Strip counts either side of 64 on the vector path (strips of 256 rows) and the scalar path (512 rows, reached
    through C % 8 != 0 or a pitch that is not a multiple of 8), C at the 256-column block edges, inside NaN-padded
    buffers; accumulate onto a nonzero value or overwrite it."""
    ld = C + 8 if path == "vec" else C + 3
    g = torch.Generator().manual_seed(_seed("colsum", path, P, C))
    src = torch.randn(P, C, generator=g) * torch.exp2(torch.randint(-10, 11, (C,), generator=g).float())
    xb = _into(src.to(_dev()), ld, dtype)
    x = xb[:P, :C]
    out = torch.full((C + 3,), NAN, device=_dev())
    out[:C] = torch.randn(C, generator=g).to(_dev())
    out0 = out[:C].clone() if accumulate else None
    snap = out.clone()
    L.colsum(x, out[:C], accumulate=bool(accumulate))
    _sync()
    ref, b = R.colsum_reference(x, out0)
    check(f"colsum {path} P={P} C={C}", out[:C], ref, b)
    check_untouched("colsum", out, out[:C], snap)


# ----------------------------------------------------------------------------------------------------------------------
# optimizer: the raw ABI
# ----------------------------------------------------------------------------------------------------------------------
NO_CLIP = 3.0e38  # what FusedAdam passes for an infinite max_norm


def _adam_raw(L, ps, gs, ms, vs, chunk, max_norm, skip_above, lr, betas, eps, step, partials=None):
    """pg_grad_sqnorm (unless partials are given) and pg_adam_step over the tensors, with pointer and chunk tables built
    as FusedAdam._build_plan builds them.  Returns (partials, norm_out)."""
    numels = [p.numel() for p in ps]
    table = R.chunk_table(numels, chunk)
    n = len(table)
    ptrs = torch.tensor([[t.data_ptr() for t in ts] for ts in (ps, gs, ms, vs)], dtype=torch.int64, device=_dev())
    numel = torch.tensor(numels, dtype=torch.int64, device=_dev())
    chunks = torch.tensor(table, dtype=torch.int32, device=_dev()).contiguous()
    if partials is None:
        partials = torch.full((n,), NAN, device=_dev())
        L.grad_sqnorm(ptrs[1], numel, chunks, n, chunk, partials)
    norm_out = torch.full((2,), NAN, device=_dev())
    L.adam_step(ptrs[0], ptrs[1], ptrs[2], ptrs[3], numel, chunks, n, chunk, partials, max_norm, skip_above, lr,
                betas[0], betas[1], eps, step, norm_out)
    _sync()
    return partials, norm_out


def _on_dev(ts, offsets=None):
    """Copies of the CPU tensors ts on the GPU; with offsets, each starts offsets[i] floats into its allocation."""
    out = []
    for i, t in enumerate(ts):
        off = 0 if offsets is None else offsets[i % len(offsets)]
        b = torch.full((t.numel() + 4,), NAN, device=_dev())
        b[off:off + t.numel()] = t.to(_dev())
        out.append(b[off:off + t.numel()])
    return out


ADAM_CASES = [([1, 63, 64, 65, 1000], 64), ([7, 300 * 64 - 5, 64], 64), ([1200 * 64 + 1], 64),
              ([3 * 1024 + 1, 1023, 1025], 1024)]
HYPER = [((0.9, 0.999), 1e-8), ((0.5, 0.9), 1e-3)]


def _check_adam(tag, ps0, gs0, ms0, vs0, ps, gs, ms, vs, norm, max_norm, sc):
    for i in range(len(ps)):
        ref = R.adam_reference(ps0[i], gs0[i], ms0[i], vs0[i], norm, max_norm, sc)
        for k, got in zip("pgmv", (ps[i], gs[i], ms[i], vs[i])):
            check(f"{tag} tensor {i} {k}", got, ref[k], ref["b_" + k])


@pytest.mark.parametrize("hyper", range(len(HYPER)), ids=["default", "b0.5-0.9-eps1e-3"])
@pytest.mark.parametrize("step", [1, 2, 1000])
@pytest.mark.parametrize("max_norm", [NO_CLIP, 0.5], ids=["noclip", "clip"])
@pytest.mark.parametrize("regime", R.ADAM_REGIMES)
@pytest.mark.parametrize("case", range(len(ADAM_CASES)), ids=["mixed", "302chunks", "1202chunks", "chunk1024"])
def test_adam_raw(L, case, regime, max_norm, step, hyper):
    """Norm and update within their bounds over 5 to 1202 chunks (the re-reduction of the partials wraps above 256),
    tensors of 1 element and chunk +- 1; without clipping g is untouched bit for bit."""
    numels, chunk = ADAM_CASES[case]
    betas, eps = HYPER[hyper]
    lr = 1e-3
    cpu = R.adam_inputs(regime, numels, _seed("adam", case, regime, step))
    ps, gs, ms, vs = (_on_dev(ts) for ts in cpu)
    ps0, gs0, ms0, vs0 = ([t.clone() for t in ts] for ts in (ps, gs, ms, vs))
    n_chunks = len(R.chunk_table(numels, chunk))
    _, norm_out = _adam_raw(L, ps, gs, ms, vs, chunk, max_norm, 0.0, lr, betas, eps, step)
    nref, nb = R.sqnorm_reference(gs0, n_chunks)
    tag = f"case {case} {regime} max_norm {max_norm} step {step}"
    assert abs(norm_out[0].item() - nref) <= nb, (tag, norm_out[0].item(), nref, nb)
    assert norm_out[1].item() == 1.0
    sc = R.adam_scalars(lr, betas[0], betas[1], eps, step)
    _check_adam(tag, ps0, gs0, ms0, vs0, ps, gs, ms, vs, norm_out[0].item(), float(torch.tensor(max_norm, dtype=F32)),
                sc)
    if max_norm == NO_CLIP:
        for a, b in zip(gs, gs0):
            check_equal(f"{tag} g untouched", a, b)


@pytest.mark.parametrize("max_norm", [NO_CLIP, 0.5], ids=["noclip", "clip"])
def test_adam_misaligned(L, max_norm):
    """Tensors starting 1 to 3 floats into their allocations run the scalar loops of both kernels.  From the same
    partials the update equals the aligned run bit for bit (both paths run adam_elem); the scalar norm is within its
    bound."""
    numels, chunk = [1000, 64 * 5 + 3, 1, 4096], 64
    cpu = R.adam_inputs("randn", numels, 11)
    al = [_on_dev(ts) for ts in cpu]
    mis = [_on_dev(ts, offsets) for ts, offsets in zip(cpu, ([1, 2, 3], [2, 3, 1], [3, 1, 2], [0, 1, 3]))]
    assert all(t.data_ptr() % 16 for t in mis[0])
    partials, n_al = _adam_raw(L, *al, chunk, max_norm, 0.0, 1e-3, (0.9, 0.999), 1e-8, 3)
    _, n_mis = _adam_raw(L, *mis, chunk, max_norm, 0.0, 1e-3, (0.9, 0.999), 1e-8, 3, partials=partials.clone())
    check_equal("norm_out", n_mis, n_al)
    for name, a, b in zip("pgmv", al, mis):
        for i, (x, y) in enumerate(zip(a, b)):
            check_equal(f"misaligned {name}{i}", y, x)
    grads = _on_dev(cpu[1], [1, 2, 3])
    n_chunks = len(R.chunk_table(numels, chunk))
    parts = torch.empty(n_chunks, device=_dev())
    ptrs = torch.tensor([t.data_ptr() for t in grads], dtype=torch.int64, device=_dev())
    L.grad_sqnorm(ptrs, torch.tensor(numels, dtype=torch.int64, device=_dev()),
                  torch.tensor(R.chunk_table(numels, chunk), dtype=torch.int32, device=_dev()), n_chunks, chunk, parts)
    _sync()
    nref, nb = R.sqnorm_reference(cpu[1], n_chunks)
    assert abs(float(parts.double().sum()) ** 0.5 - nref) <= nb


@pytest.mark.parametrize("skip_above,applied", [(5.1, True), (5.0, True), (4.9, False)])
def test_adam_skip_rule(L, skip_above, applied):
    """Gradients 3 and 4 give norm 5 exactly.  The step is applied when norm <= skip_above (equal included, as the
    reference trainer's `not (norm <= skip_grad_norm)` skips); a skipped step leaves p, g, m and v unchanged bit for bit
    and sets norm_out[1] = 0."""
    ps = _on_dev([torch.tensor([1.0, -2.0])])
    gs = _on_dev([torch.tensor([3.0, 4.0])])
    ms = _on_dev([torch.tensor([0.1, 0.2])])
    vs = _on_dev([torch.tensor([0.01, 0.02])])
    before = [t[0].clone() for t in (ps, gs, ms, vs)]
    _, norm_out = _adam_raw(L, ps, gs, ms, vs, 64, 10.0, skip_above, 1e-2, (0.9, 0.999), 1e-8, 2)
    assert norm_out[0].item() == 5.0 and norm_out[1].item() == (1.0 if applied else 0.0), norm_out.tolist()
    if applied:
        assert not torch.equal(ps[0], before[0])
    else:
        for name, t, b in zip("pgmv", (ps, gs, ms, vs), before):
            check_equal(f"skipped step: {name}", t[0], b)


def _nan_grads(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    grads = [torch.randn(s, generator=g).to(_dev()) for s in shapes]
    grads[1].view(-1)[5] = NAN
    return grads


def test_adam_nan_norm_skips(L):
    """A NaN gradient norm with skip_above set skips the step, as the reference trainer does: p, g, m and v unchanged
    bit for bit, norm_out = [NaN, 0], and FusedAdam's step counter does not move."""
    from pytorch_generative_b200 import optim

    shapes = [(300,), (70001,), (1,)]
    g = torch.Generator().manual_seed(7)
    ps = [torch.randn(s, generator=g).to(_dev()).requires_grad_(True) for s in shapes]
    opt = optim.FusedAdam(ps, lr=1e-2)
    for p, gr in zip(ps, _nan_grads(shapes, 8)):
        p.grad = torch.randn_like(gr)
    opt.clip_and_step(1.0)  # one ordinary step: nonzero moments
    for p, gr in zip(ps, _nan_grads(shapes, 9)):
        p.grad = gr
    before = [(p.detach().clone(), p.grad.clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone())
              for p in ps]
    norm = opt.clip_and_step(1.0, skip_above=10.0)
    _sync()
    assert torch.isnan(norm).item()
    assert opt._plan[0]["norm_out"][1].item() == 0.0
    for p, (p0, g0, m0, v0) in zip(ps, before):
        check_equal("p", p.detach(), p0)
        check_equal("g", p.grad, g0)
        check_equal("m", opt.state[p]["exp_avg"], m0)
        check_equal("v", opt.state[p]["exp_avg_sq"], v0)
        assert float(opt.state[p]["step"]) == 1.0


@pytest.mark.parametrize("max_norm", [1e50, 1.0])
def test_adam_nan_norm_without_skip_matches_torch(L, max_norm):
    """Without a skip rule a NaN norm reaches every element as in clip_grad_norm_ + torch.optim.Adam: torch multiplies
    every gradient by clamp(max_norm / (NaN + 1e-6), max=1) = NaN, so every p, g, m and v becomes NaN."""
    from pytorch_generative_b200 import optim

    shapes = [(300,), (70001,), (1,)]
    g = torch.Generator().manual_seed(7)
    ps = [torch.randn(s, generator=g).to(_dev()).requires_grad_(True) for s in shapes]
    qs = [p.detach().clone().requires_grad_(True) for p in ps]
    fused, ref = optim.FusedAdam(ps, lr=1e-2), torch.optim.Adam(qs, lr=1e-2)
    for p, q, gr in zip(ps, qs, _nan_grads(shapes, 9)):
        p.grad, q.grad = gr.clone(), gr.clone()
    n_f = fused.clip_and_step(max_norm)
    n_r = torch.nn.utils.clip_grad_norm_(qs, max_norm)
    ref.step()
    _sync()
    assert torch.isnan(n_f).item() and torch.isnan(n_r).item()
    for p, q in zip(ps, qs):
        for name, a, b in (("p", p.detach(), q.detach()), ("g", p.grad, q.grad),
                           ("m", fused.state[p]["exp_avg"], ref.state[q]["exp_avg"]),
                           ("v", fused.state[p]["exp_avg_sq"], ref.state[q]["exp_avg_sq"])):
            assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{name}: NaN positions differ from torch"
            fin = ~torch.isnan(b)
            assert torch.allclose(a[fin], b[fin], rtol=1e-5, atol=1e-7), name
        assert float(fused.state[p]["step"]) == float(ref.state[q]["step"])


def test_fused_adam_many_chunks(L):
    """FusedAdam at its real CHUNK (65536) with 260 chunks: the re-reduction wraps above 256 partials.  Two clipped steps
    within the bounds from the kernel's own norm."""
    from pytorch_generative_b200 import optim

    numels = [257 * optim.CHUNK + 1, optim.CHUNK - 1, 1]
    g = torch.Generator().manual_seed(12)
    ps = [torch.randn(n, generator=g).to(_dev()).requires_grad_(True) for n in numels]
    opt = optim.FusedAdam(ps, lr=1e-3)
    n_chunks = len(R.chunk_table(numels, optim.CHUNK))
    assert n_chunks == 260
    for step in (1, 2):
        for p in ps:
            p.grad = torch.randn(p.shape, generator=g).to(_dev())
        snap = [(p.detach().clone(), p.grad.clone(),
                 opt.state[p]["exp_avg"].clone() if step > 1 else torch.zeros_like(p),
                 opt.state[p]["exp_avg_sq"].clone() if step > 1 else torch.zeros_like(p)) for p in ps]
        norm = opt.clip_and_step(100.0).item()
        _sync()
        nref, nb = R.sqnorm_reference([s[1] for s in snap], n_chunks)
        assert abs(norm - nref) <= nb, (norm, nref, nb)
        sc = R.adam_scalars(1e-3, 0.9, 0.999, 1e-8, step)
        _check_adam(f"FusedAdam step {step}", *zip(*snap), [p.detach() for p in ps], [p.grad for p in ps],
                    [opt.state[p]["exp_avg"] for p in ps], [opt.state[p]["exp_avg_sq"] for p in ps], norm, 100.0, sc)
