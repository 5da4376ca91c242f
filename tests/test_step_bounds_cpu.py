"""The bounds of tests/_step_reference.py checked on the CPU, without a GPU: an fp32 emulation of each kernel's arithmetic
(csrc/pg_elementwise.cu, pg_conv.cu, pg_optim.cu and pg_sum_partials in pg_host.cu: lane-strided chains and warp
butterflies, warp / block / grid-stride assignment of rows and pixels, block partials added in block order) must meet
every bound in every input regime, and each bug model below, applied alone, must break at least one of them.  A bound
that accepted a bug model would not catch that bug on the GPU either."""

import pytest
import torch

import _step_reference as R
from _act_reference import ELU, NONE, RELU
from _checks import violations

F32, F64 = torch.float32, torch.float64
SMS = 132  # the H100's SM count: the emulated persistent grids have the sizes the kernels launch with


def f32(v):
    return float(torch.tensor(v, dtype=F32))


# ----------------------------------------------------------------------------------------------------------------------
# shared reduction structure
# ----------------------------------------------------------------------------------------------------------------------
def butterfly(acc):
    """warp_sum over the last dimension (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1."""
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., idx ^ o]
    return acc[..., 0]


def lane_sum(t):
    """Row sums of t [P, C] as one warp forms them: lane l adds columns l, l + 32, ... in order, then the butterfly."""
    P, C = t.shape
    Cp = (C + 31) // 32 * 32
    v = torch.zeros(P, Cp, dtype=F32)
    v[:, :C] = t
    v = v.view(P, Cp // 32, 32)
    acc = torch.zeros(P, 32, dtype=F32)
    for k in range(Cp // 32):
        acc = acc + v[:, k]
    return butterfly(acc)


def sum_partials(part, out0):
    """pg_sum_partials: out0 + the partials [n, N] in order (fewer than 64: one chain; else 32 lanes and a butterfly)."""
    n, N = part.shape
    if n < 64:
        s = torch.zeros(N, dtype=F32)
        for p in range(n):
            s = s + part[p]
    else:
        n32 = (n + 31) // 32 * 32
        pp = torch.zeros(n32, N, dtype=F32)
        pp[:n] = part
        acc = torch.zeros(N, 32, dtype=F32)
        for k in range(n32 // 32):
            acc = acc + pp[k * 32:(k + 1) * 32].T
        s = butterfly(acc)
    return out0.to(F32) + s


def grid_for(work, threads, per_sm):
    return max(1, min((work + threads - 1) // threads, SMS * per_sm))


def warp_column_partials(terms, n_warps, warps_per_block, drop_last_row=False):
    """Column sums of terms [P, C] as ln_bwd accumulates them: warp w walks rows w, w + n_warps, ... keeping a register
    chain per column; the warps of a block add into shared memory in warp order; one partial per block."""
    P, C = terms.shape
    k = (P + n_warps - 1) // n_warps
    t = torch.zeros(k * n_warps, C, dtype=F32)
    t[:P] = terms
    if drop_last_row:  # each warp's last row left out
        rows = torch.arange(k * n_warps)
        t[(rows < P) & (rows + n_warps >= P)] = 0
    t = t.view(k, n_warps, C)
    acc = torch.zeros(n_warps, C, dtype=F32)
    for i in range(k):
        acc = acc + t[i]
    acc = acc.view(n_warps // warps_per_block, warps_per_block, C)
    part = acc[:, 0]
    for w in range(1, warps_per_block):
        part = part + acc[:, w]
    return part


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------------
def ln_fwd_emulate(x, gamma, beta, eps, fast, bug=None, ld=None):
    """(y, mean, rstd) of ln_fwd_kernel (fast) / ln_fwd_generic_kernel.  x [P, C]; with bug "ld_stats" the statistics
    run over ld columns, the pad columns C..ld holding zeros."""
    P, C = x.shape
    if bug == "ld_stats":
        xs = torch.zeros(P, ld, dtype=F32)
        xs[:, :C] = x
        n = ld
    else:
        xs, n = x, C
    s = lane_sum(xs)
    mean = s * f32(1.0 / n) if fast else s / n
    d = xs - mean[:, None]
    if bug == "one_pass":
        var = lane_sum(xs * xs) / n - mean * mean
    else:
        var = lane_sum(d * d) / (n - 1 if bug == "unbiased" else n)
    rstd = torch.rsqrt(var) + eps if bug == "eps_after_rsqrt" else torch.rsqrt(var + eps)
    y = (x - mean[:, None]) * rstd[:, None] * gamma + beta
    return y, mean, rstd


def ln_bwd_emulate(dy, x, gamma, mean, rstd, r0, r1, d0, fast, bug=None):
    """(dx, dgamma, dbeta, colsum) of ln_bwd_kernel (fast: 8 warps per block, 2 blocks per SM) / ln_bwd_generic_kernel
    (one warp per block, 8 per SM), partials through pg_sum_partials onto the initial values d0."""
    P, C = x.shape
    xh = (x - mean[:, None]) * rstd[:, None]
    gy = dy * gamma
    m1 = lane_sum(gy) * f32(1.0 / C) if fast else lane_sum(gy) / C
    s2 = lane_sum(gy * xh)
    m2 = s2 * f32(1.0 / C) if fast else s2 / C
    if bug == "no_m2":
        o = rstd[:, None] * (gy - m1[:, None])
    else:
        o = rstd[:, None] * (gy - m1[:, None] - xh * m2[:, None])
    before_res = o
    o = o + r0 + r1 if fast else (o + r0) + r1
    wpb = 8 if fast else 1
    blocks = grid_for(P * 32, 256, 2) if fast else grid_for(P * 32, 32, 8)
    nw = blocks * wpb
    dg = warp_column_partials(dy * xh, nw, wpb, drop_last_row=bug == "drop_last_row")
    db = warp_column_partials(dy, nw, wpb)
    ds = warp_column_partials(before_res if bug == "colsum_before_res" else o, nw, wpb)
    return o, sum_partials(dg, d0[0]), sum_partials(db, d0[1]), sum_partials(ds, d0[2])


LN_CASES = [(37, 128, True), (300, 256, True), (70, 384, True), (2113, 128, True), (40, 100, False), (25, 1000, False),
            (9, 3, False), (600, 129, False)]


def _ln_violations(regime, P, C, fast, bug=None, ld=None, seed=0):
    x, gamma, beta, dy, r0, r1 = R.ln_inputs(regime, P, C, seed)
    eps = 1e-5
    y, mean, rstd = ln_fwd_emulate(x, gamma, beta, eps, fast, bug, ld)
    ref = R.ln_fwd_reference(x, gamma, beta, eps)
    bad = {"y": violations(y, ref["y"], ref["b_y"]).any(), "mean": violations(mean, ref["mean"], ref["b_mean"]).any(),
           "rstd": violations(rstd, ref["rstd"], ref["b_rstd"]).any()}
    if regime == "constant" and R.ln_mean_exact(C, fast) and bug is None:
        bad["y == beta"] = not torch.equal(y, beta.expand_as(y))
    g = torch.Generator().manual_seed(seed + 1)
    d0 = tuple(torch.randn(C, generator=g) for _ in range(3))
    # the backward from the kernel's own statistics
    m32, r32 = ln_fwd_emulate(x, gamma, beta, eps, fast)[1:]
    dx, dg, db, ds = ln_bwd_emulate(dy, x, gamma, m32, r32, r0, r1, d0, fast, bug)
    bref = R.ln_bwd_reference(dy, x, gamma, m32, r32, r0, r1, d0)
    for k, got in (("dx", dx), ("dgamma", dg), ("dbeta", db), ("colsum", ds)):
        bad[k] = violations(got, bref[k], bref["b_" + k]).any()
    return {k: bool(v) for k, v in bad.items()}


@pytest.mark.parametrize("regime", R.LN_REGIMES)
@pytest.mark.parametrize("P,C,fast", LN_CASES)
def test_layernorm_emulation_meets_bounds(regime, P, C, fast):
    bad = _ln_violations(regime, P, C, fast)
    assert not any(bad.values()), bad


@pytest.mark.parametrize("bug,regime,P,C,fast,ld", [
    ("one_pass", "offset", 300, 256, True, None),
    ("unbiased", "randn", 300, 256, True, None),
    ("eps_after_rsqrt", "range", 300, 256, True, None),
    ("ld_stats", "randn", 40, 100, False, 104),
    ("no_m2", "randn", 300, 256, True, None),
    ("colsum_before_res", "randn", 300, 256, True, None),
    ("drop_last_row", "randn", 2113, 128, True, None),
    ("drop_last_row", "randn", 40, 100, False, None),
])
def test_layernorm_bug_models_break_a_bound(bug, regime, P, C, fast, ld):
    bad = _ln_violations(regime, P, C, fast, bug, ld)
    assert any(bad.values()), f"{bug}: every bound still holds"


# ----------------------------------------------------------------------------------------------------------------------
# small-Cin convolution
# ----------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in float64; one rounding of the sum (a double rounding can
    differ from the hardware's single rounding by one ulp in rare ties, far inside the bounds)."""
    return (a.to(F64) * b.to(F64) + c.to(F64)).to(F32)


def _act32(act, x):
    if act == RELU:
        return x.clamp_min(0)
    if act == ELU:
        return torch.where(x > 0, x, torch.expm1(x))
    return x


def _dact32(act, x):
    if act == RELU:
        return (x > 0).to(F32)
    if act == ELU:
        return torch.where(x > 0, torch.ones_like(x), torch.exp(x))
    return torch.ones_like(x)


def conv_emulate(x, w, b, dy, pad, pre_act, dw0, db0, bug=None):
    """(out, dw, db, dx) of conv_small_fwd_kernel (fma chain from the bias), conv_small_wgrad_kernel (32-pixel fma
    chunks, grid-stride blocks, one launch per 16384 outputs, block partials), pg_colsum_f32 and conv_small_dgrad_kernel
    (channel groups of 4, lanes over output channels, butterfly, times act'(x))."""
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = w.shape
    ph, pw = pad
    K, P = Cin * kh * kw, N * H * W
    a = _act32(pre_act, x)
    pa = torch.nn.functional.unfold(a, (kh, kw), padding=(ph, pw)).transpose(1, 2).reshape(P, K)
    wm = w.reshape(Cout, K)
    out = b.expand(P, Cout).clone()
    for k in range(K):
        out = _fma(pa[:, k:k + 1], wm[:, k], out)
    # wgrad
    blocks = min((P + 31) // 32, SMS * 2)
    n_chunks = (P + 31) // 32
    part = torch.zeros(blocks, Cout, K, dtype=F32)
    pad_p = torch.zeros(n_chunks * 32, K, dtype=F32)
    pad_p[:P] = pa
    pad_dy = torch.zeros(n_chunks * 32, Cout, dtype=F32)
    pad_dy[:P] = dy
    for c in range(n_chunks):
        s = torch.zeros(Cout, K, dtype=F32)
        for i in range(32):
            r = c * 32 + i
            s = _fma(pad_dy[r][:, None], pad_p[r][None, :], s)
        part[c % blocks] = part[c % blocks] + s
    part = part.view(blocks, Cout * K)
    if bug == "skip_second_launch":
        part[:, 16384:] = 0  # the outputs of the second launch never reach the partials
    dw = sum_partials(part, dw0.reshape(-1)).view(w.shape)
    strips = (P + 255) // 256
    sp = torch.stack([dy[s * 256:(s + 1) * 256].sum(0) for s in range(strips)])
    db = sum_partials(sp, db0)
    # dgrad: acc[p, ci, lane] over taps and output-channel groups of 32
    dyi = torch.zeros(N, H + kh, W + kw, Cout, dtype=F32)
    dyi[:, :H, :W] = dy.view(N, H, W, Cout)
    co32 = (Cout + 31) // 32 * 32
    acc = torch.zeros(N, H, W, Cin, 32, dtype=F32)
    for i in range(kh):
        for j in range(kw):
            ys, xs = torch.arange(H) - i + ph, torch.arange(W) - j + pw
            ys = torch.where((ys >= 0) & (ys < H), ys, torch.full_like(ys, H))  # row H of dyi is zero
            xs = torch.where((xs >= 0) & (xs < W), xs, torch.full_like(xs, W))
            d = torch.zeros(N, H, W, co32, dtype=F32)
            d[..., :Cout] = dyi[:, ys][:, :, xs]
            wt = torch.zeros(Cin, co32, dtype=F32)
            wt[:, :Cout] = w[:, :, i, j].T
            for cb in range(co32 // 32):
                acc = _fma(d[..., None, cb * 32:(cb + 1) * 32], wt[None, None, None, :, cb * 32:(cb + 1) * 32], acc)
    v = butterfly(acc).permute(0, 3, 1, 2)
    dx = v if bug == "no_act_deriv" or pre_act == NONE else v * _dact32(pre_act, x)
    if bug == "drop_partial_group":
        dx[:, Cin // 4 * 4:] = 0
    return out, dw, db, dx


CONV_CASES = [  # N, Cin, H, W, Cout, kh, kw, ph, pw
    (2, 3, 8, 8, 24, 3, 3, 1, 1), (1, 1, 7, 9, 32, 7, 7, 3, 3), (1, 5, 6, 5, 40, 3, 3, 1, 1),
    (1, 3, 4, 4, 130, 7, 7, 3, 3),  # Cout K = 19110 outputs: a second wgrad launch
]


def _conv_violations(case, pre_act, bug=None, seed=3):
    N, Cin, H, W, Cout, kh, kw, ph, pw = case
    x, w, b, dy, dw0, db0 = R.conv_inputs(N, Cin, H, W, Cout, kh, kw, seed)
    out, dw, db, dx = conv_emulate(x, w, b, dy, (ph, pw), pre_act, dw0, db0, bug)
    ref = R.conv_reference(x, w, b, dy, (ph, pw), pre_act, dw0, db0)
    return {k: bool(violations(got, ref[k], ref["b_" + k]).any()) for k, got in
            (("out", out), ("dw", dw), ("db", db), ("dx", dx))}


@pytest.mark.parametrize("pre_act", [NONE, RELU, ELU], ids=["none", "relu", "elu"])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_small_emulation_meets_bounds(case, pre_act):
    bad = _conv_violations(case, pre_act)
    assert not any(bad.values()), bad


@pytest.mark.parametrize("bug,case,pre_act", [
    ("skip_second_launch", CONV_CASES[3], NONE),
    ("drop_partial_group", CONV_CASES[2], NONE),
    ("no_act_deriv", CONV_CASES[0], ELU),
])
def test_conv_small_bug_models_break_a_bound(bug, case, pre_act):
    bad = _conv_violations(case, pre_act, bug)
    assert any(bad.values()), f"{bug}: every bound still holds"


# ----------------------------------------------------------------------------------------------------------------------
# BCE
# ----------------------------------------------------------------------------------------------------------------------
def bce_emulate(l, t, scale, loss0, bug=None):
    """(loss, dlogits) of bce_kernel (grid-stride threads, warp and block butterflies, one partial per block) and
    pg_sum_partials onto loss0."""
    n = l.numel()
    if bug == "no_abs_split":
        term = l - l * t + torch.log(1 + torch.exp(-l))
    else:
        term = torch.clamp_min(l, 0) - l * t + torch.log1p(torch.exp(-l.abs()))
    dl = (1 / (1 + torch.exp(-l)) - t) * scale
    G = grid_for(n, 256, 4)
    T = G * 256
    k = (n + T - 1) // T
    tt = torch.zeros(k * T, dtype=F32)
    tt[:n] = term
    acc = torch.zeros(T, dtype=F32)
    for i in range(k):
        acc = acc + tt[i * T:(i + 1) * T]
    warp = butterfly(acc.view(G, 8, 32))                        # [G, 8]
    lanes = torch.zeros(G, 32, dtype=F32)
    lanes[:, :8] = warp
    part = butterfly(lanes)                                      # [G]
    if bug == "drop_last_block":
        part = part[:-1]
    return sum_partials(part[:, None], torch.tensor([loss0]))[0], dl


BCE_SIZES = [1, 255, 257, 3000, SMS * 4 * 256 + 1]


@pytest.mark.parametrize("hard", [False, True], ids=["soft", "hard"])
@pytest.mark.parametrize("regime", R.BCE_REGIMES)
@pytest.mark.parametrize("numel", BCE_SIZES)
def test_bce_emulation_meets_bounds(numel, regime, hard):
    l, t = R.bce_inputs(regime, numel, seed=numel, hard=hard)
    loss, dl = bce_emulate(l, t, 1 / 16, 2.5)
    ref, b, dref, db = R.bce_reference(l, t, 1 / 16, 2.5)
    assert abs(float(loss) - ref) <= b, (float(loss), ref, b)
    assert not violations(dl, dref, db).any()


@pytest.mark.parametrize("bug,regime,numel", [("no_abs_split", "extreme", 255), ("drop_last_block", "randn", 257)])
def test_bce_bug_models_break_a_bound(bug, regime, numel):
    l, t = R.bce_inputs(regime, numel, seed=numel)  # the inputs test_bce_emulation_meets_bounds accepts
    loss, dl = bce_emulate(l, t, 1 / 16, 2.5, bug)
    ref, b, dref, db = R.bce_reference(l, t, 1 / 16, 2.5)
    assert not abs(float(loss) - ref) <= b or violations(dl, dref, db).any(), f"{bug}: every bound still holds"


# ----------------------------------------------------------------------------------------------------------------------
# column sums
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,C,rows", [(1, 8, 256), (300, 264, 256), (16385, 16, 256), (40000, 3, 512)])
def test_colsum_emulation_meets_bounds(P, C, rows):
    """Strips of `rows` rows (256 on the vector path, 512 on the scalar path), partials in strip order."""
    x = torch.randn(P, C, generator=torch.Generator().manual_seed(P)) * torch.exp2(torch.randint(-10, 11, (C,)).float())
    out0 = torch.randn(C)
    strips = (P + rows - 1) // rows
    part = torch.stack([x[s * rows:(s + 1) * rows].sum(0) for s in range(strips)])
    ref, b = R.colsum_reference(x, out0)
    assert not violations(sum_partials(part, out0), ref, b).any()


# ----------------------------------------------------------------------------------------------------------------------
# optimizer
# ----------------------------------------------------------------------------------------------------------------------
def adam_emulate(ps, gs, ms, vs, chunk, max_norm, lr, betas, eps, step, bug=None):
    """(norm, [(p, g, m, v)]) of grad_sqnorm_kernel (a partial per chunk) and adam_step_kernel (256 threads re-reduce
    the partials, block_sum, then adam_elem per element)."""
    parts = []
    for g in gs:
        for c in range((g.numel() + chunk - 1) // chunk):
            gc = g[c * chunk:(c + 1) * chunk]
            parts.append((gc * gc).sum())
    parts = torch.stack(parts)
    n = parts.numel()
    if bug == "norm_drops_last_partial" and n > 256:
        parts = parts[:-1]
    n32 = (parts.numel() + 255) // 256 * 256
    pp = torch.zeros(n32, dtype=F32)
    pp[:parts.numel()] = parts
    acc = torch.zeros(256, dtype=F32)
    for k in range(n32 // 256):
        acc = acc + pp[k * 256:(k + 1) * 256]
    warp = butterfly(acc.view(8, 32))
    lanes = torch.zeros(32, dtype=F32)
    lanes[:8] = warp
    norm = torch.sqrt(butterfly(lanes))
    sc = R.adam_scalars(lr, betas[0], betas[1], eps, step - 1 if bug == "bias_correction_step_minus_1" else step)
    coef = torch.tensor(f32(max_norm), dtype=F32) / (norm + torch.tensor(1e-6, dtype=F32))
    coef = torch.clamp_max(coef, 1.0)
    out = []
    for p, g, m, v in zip(ps, gs, ms, vs):
        g1 = g * coef
        gm = g if bug == "clip_after_moments" else g1
        m1 = m + sc["omb1"] * (gm - m)
        v1 = sc["beta2"] * v + sc["omb2"] * (gm * gm)
        if bug == "eps_inside_sqrt":
            denom = torch.sqrt(v1 + sc["eps"]) * sc["rsqrt_bc2"]
        else:
            denom = torch.sqrt(v1) * sc["rsqrt_bc2"] + sc["eps"]
        out.append((p - sc["lr_bc1"] * (m1 / denom), g1, m1, v1))
    return norm, out


def _adam_violations(regime, numels, chunk, max_norm, step, bug=None, betas=(0.9, 0.999), eps=1e-8, lr=1e-3):
    ps, gs, ms, vs = R.adam_inputs(regime, numels, seed=sum(numels) + step)
    n_chunks = len(R.chunk_table(numels, chunk))
    norm, out = adam_emulate(ps, gs, ms, vs, chunk, max_norm, lr, betas, eps, step, bug)
    nref, nb = R.sqnorm_reference(gs, n_chunks)
    bad = {"norm": not abs(float(norm) - nref) <= nb}
    sc = R.adam_scalars(lr, betas[0], betas[1], eps, step)
    for i, (p, g, m, v) in enumerate(zip(ps, gs, ms, vs)):
        ref = R.adam_reference(p, g, m, v, float(norm), max_norm, sc)
        for k, got in zip("pgmv", out[i]):
            bad[f"{k}{i}"] = bool(violations(got, ref[k], ref["b_" + k]).any())
    return bad


ADAM_CASES = [  # numels, chunk_elems
    ([1, 63, 64, 65, 1000], 64), ([7, 300 * 64 - 5, 64], 64), ([1200 * 64 + 1], 64), ([3 * 1024 + 1, 1024 - 1], 1024)]


@pytest.mark.parametrize("step", [1, 2, 1000])
@pytest.mark.parametrize("max_norm", [1e50, 0.5])
@pytest.mark.parametrize("regime", R.ADAM_REGIMES)
@pytest.mark.parametrize("case", range(len(ADAM_CASES)))
def test_adam_emulation_meets_bounds(case, regime, max_norm, step):
    numels, chunk = ADAM_CASES[case]
    bad = _adam_violations(regime, numels, chunk, max_norm, step)
    assert not any(bad.values()), {k: v for k, v in bad.items() if v}


@pytest.mark.parametrize("bug,max_norm,step", [
    ("bias_correction_step_minus_1", 1e50, 2),
    ("bias_correction_step_minus_1", 1e50, 1000),
    ("eps_inside_sqrt", 1e50, 2),
    ("clip_after_moments", 0.5, 2),
    ("norm_drops_last_partial", 1e50, 2),
])
def test_adam_bug_models_break_a_bound(bug, max_norm, step):
    numels, chunk = ADAM_CASES[1]  # 302 chunks, the last one full
    regime = "tiny_moments" if bug == "eps_inside_sqrt" else "randn"
    bad = _adam_violations(regime, numels, chunk, max_norm, step, bug)
    assert any(bad.values()), f"{bug}: every bound still holds"
