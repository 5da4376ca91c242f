"""Float64 references, element-wise error bounds and input regimes for the kernels every training step runs besides the
GEMM and attention: LayerNorm (pg_layernorm_fwd / _bwd and their pitched _ld forms), the small-Cin input convolution
(pg_conv_small_fwd / _bwd), the recipe loss (pg_bce_logits_fwd_bwd), column sums (pg_colsum_f32 / _bf16) and the
optimizer (pg_grad_sqnorm, pg_adam_step).  Shared by tests/test_step_kernels_gpu.py and tests/test_step_bounds_cpu.py;
not a test module.

Every reference is computed in float64 from the exact fp32 (or bf16) values the kernel reads, on the device the tensors
live on.  The bounds follow the kernels' arithmetic (csrc/pg_elementwise.cu, pg_conv.cu, pg_optim.cu, pg_host.cu) and are
used as derived here, without a safety factor (tests/_checks.py compares |got - ref| <= bound).

Bound derivation.  U = U24 = 2^-24 is the unit roundoff of fp32.
  * A sum of n terms rounded to fp32 after each addition is within (n - 1) U sum|terms| of the exact sum, in any order
    and any tree (recursive summation: every term passes through at most n - 1 roundings; adding an exact zero rounds
    nothing).  Block partials, warp butterflies and pg_sum_partials only regroup the same terms, so a column sum over P
    rows added to an initial value c0 is within (P + 2) U (sum|terms| + |c0|) (one spare rounding).
  * Each further rounded fp32 operation costs one U times the magnitudes it touches.  An fma rounds once.
  * Transcendentals cost their documented error (CUDA math API): expf 2 ulp, log1pf 1 ulp, rsqrtf 2 ulp; one ulp is at
    most 2U relative.  sqrtf and '/' are IEEE-rounded: the library is built without --use_fast_math.

LayerNorm forward, row of C values x (the first C columns of a row of pitch ld).  mu and var are the float64 two-pass
statistics, S = sum|x|.  The kernel's mean m = fl(sum x) / C (or * fl(1/C) on the fast path) is within
e_mean = (C + 2) U S / C of mu.  Its variance sums (x - m)^2 = (x - mu)^2 + ... over the fp32 mean, which adds
(mu - m)^2 <= e_mean^2 to var; the sum, the scaling and the + eps take (C + 5) U relative, so var + eps carries
r_var = ((C + 5) U (var + e_mean^2 + eps) + e_mean^2) / (var + eps) relative, and rstd = rsqrtf(.) carries
r_var / 2 + r_var^2 + 5 U (rsqrtf's 2 ulp and one spare).  y = (x - m) rstd gamma + beta: with D = |x - mu| + e_mean,
  |y - y64| <= |gamma| (e_mean rstd + D |drstd| + 3 U D rstd') + U (|gamma| D rstd' + |beta|),    rstd' = rstd + |drstd|.
The mean's error enters as e_mean rstd |gamma|: the bound grows with |mean| / std.  That is honest, not slack: the fp32
mean of a row at mean 2^8 over unit spread is only known to about C U 2^8, and the kernel subtracts it.  A one-pass
variance E[x^2] - E[x]^2 loses (2^8)^2 U relative to a unit variance and breaks the rstd bound.

LayerNorm backward.  The reference takes the mean and rstd handed to the kernel (they are inputs of the ABI), so the
statistics' error stays out of these bounds.  xh = (x - mean) rstd, gy = dy gamma, m1 = sum gy / C, m2 = sum gy xh / C,
  dx = rstd (gy - m1 - xh m2) + dres0 + dres1.
The kernel's xh carries 2 U, gy U, m1 (C + 2) U sum|gy| / C, m2 (C + 4) U sum|gy xh| / C; the two subtractions, the
product xh m2 and the scaling by rstd add one U each on what they touch, and the two residual adds one U each on
|dx| + |dres0| + |dres1|.  dgamma = d0 + sum_p dy xh (terms carry 3 U: (P + 5) U), dbeta = d0 + sum_p dy, and
colsum(dx) = c0 + sum_p dx: the chain bound plus the sum of the per-row dx bounds.

Small-Cin convolution.  a = act(x) is the pre-activation input (act_err of tests/_act_reference.py: ELU 2^-22 relative).
  forward  out = b + sum_k w a: an fma chain of K = Cin kh kw terms from the bias: (K + 1) U (|b| + sum|w a|) plus
           r_act sum|w a|.
  wgrad    dw = d0 + sum_p dy a: 32-pixel fma chunks, block accumulation and pg_sum_partials regroup P terms:
           (P + 2) U (sum|dy a| + |d0|) plus r_act sum|dy a|.
  dgrad    dx = act'(x) sum_{co,i,j} dy w: n = kh kw Cout terms through lane fma chains and a warp butterfly, then one
           multiply by act'(x) (deriv_err): |act'| (n + 2) U T + (r' |act'| + a') T with T = sum|dy w|.

BCE with logits.  term = max(l, 0) - l t + log1pf(expf(-|l|)), dlogits = (1 / (1 + expf(-l)) - t) scale.
  dlogits  the sigmoid s carries expf's 4 U on e = exp(-l) (times e / (1 + e) <= 1), the add and the division: 6 U s,
           plus 2^-126 absolute where e overflows or s is subnormal (|l| >= 87); then s - t and the scale:
           |scale| (6 U s + 2^-126 + U |s - t|) + U |dlogits|.
  loss     (numel + 2) U (sum|terms| + |loss0|) plus, per term, 3 U (max(l, 0) + |l t| + log1p(e)) + 4 U e + 2^-149
           (the product, the subtraction, log1pf's 1 ulp, the last add; expf's 2 ulp moves log1p by at most 4 U e).

Column sums: (P + 2) U (sum|x| + |out0|).

Optimizer.  The squared norm sums numel products g^2 (one rounding each) into n_chunks block partials that every block of
pg_adam_step re-reduces: a chain of numel + n_chunks terms, (numel + n_chunks + 1) U sum g^2; sqrtf halves the relative
error and adds U.  The update reference takes the kernel's own norm (norm_out[0]) and the host scalars as pg_adam_step
rounds them (lr / bc1 and 1 / sqrt(bc2) in double, then to float; 1 - beta in double, then to float):
  coef = min(1, max_norm / (norm + 1e-6f)) carries 2 U when it clips (exact 1 otherwise); g' = g coef: 3 U;
  m' = m + (1 - b1) (g' - m):   (1 - b1) (3 U |g'| + 2 U |g' - m|) + U |m'|;
  v' = b2 v + (1 - b2) g'^2:    8 U (1 - b2) g'^2 + 2 U b2 v + U |v'|;
  denom = sqrtf(v') rsqrt_bc2 + eps: relative (r_v / 2 + 2 U) sqrt(v') rsqrt_bc2 / denom + U, r_v the relative bound of v';
  p' = p - lr_bc1 m' / denom:    lr_bc1 (|dm'| + |m'| (r_d + 2 U)) / denom + U |p'|."""

import math

import torch

from _act_reference import NONE, act64, act_err, dact64, deriv_err

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U24 = 2.0 ** -24
TINY = 2.0 ** -126  # smallest normal fp32

LN_REGIMES = ("randn", "offset", "constant", "range")
BCE_REGIMES = ("randn", "extreme")
ADAM_REGIMES = ("randn", "tiny_moments")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ----------------------------------------------------------------------------------------------------------------------
def ln_inputs(regime, P, C, seed):
    """x [P, C], gamma, beta [C], dy, dres0, dres1 [P, C] fp32 on the CPU.
      randn     x ~ N(0, 1);
      offset    x = N(0, 1) + s 2^e per row, s = +-1, e in {6, 7, 8}: large row means over unit spread;
      constant  every row holds one integer in [-8, 8]: variance 0, only eps remains, and the fp32 mean is exact
                whenever the kernel's scaling is (the generic path divides; the fast path multiplies by fl(1/C));
      range     N(0, 1) rows scaled by 2^e, e in [-20, 20]: eps dominates the small rows."""
    g = _gen(seed)
    x = torch.randn(P, C, generator=g)
    if regime == "offset":
        e = torch.randint(6, 9, (P, 1), generator=g).float()
        s = torch.randint(0, 2, (P, 1), generator=g).float() * 2 - 1
        x = x + s * torch.exp2(e)
    elif regime == "constant":
        x = torch.randint(-8, 9, (P, 1), generator=g).float().expand(P, C).contiguous()
    elif regime == "range":
        x = x * torch.exp2(torch.randint(-20, 21, (P, 1), generator=g).float())
    else:
        assert regime == "randn", regime
    gamma = torch.randn(C, generator=g) * 0.5 + 1
    beta = torch.randn(C, generator=g)
    dy = torch.randn(P, C, generator=g)
    r0 = torch.randn(P, C, generator=g)
    r1 = torch.randn(P, C, generator=g)
    return x, gamma, beta, dy, r0, r1


def ln_mean_exact(C, fast):
    """Whether the fp32 mean of a row of equal integers is exact: the generic path divides by C (exact), the fast path
    multiplies by fl(1/C) (exact when C is a power of two)."""
    return not fast or (C & (C - 1)) == 0


def ln_fwd_reference(x, gamma, beta, eps):
    """x [P, C] (the first C columns), gamma, beta [C] -> dict of float64 references and bounds:
    mean, rstd [P] and y [P, C], with b_mean, b_rstd, b_y."""
    x64, g64, b64 = x.to(F64), gamma.to(F64), beta.to(F64)
    C = x64.shape[1]
    mu = x64.mean(1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    e_mean = (C + 2) * U24 * x64.abs().sum(1, keepdim=True) / C
    r_var = ((C + 5) * U24 * (var + e_mean ** 2 + eps) + e_mean ** 2) / (var + eps)
    b_rstd = rstd * (r_var / 2 + r_var ** 2 + 5 * U24)
    D = (x64 - mu).abs() + e_mean
    rstd_hi = rstd + b_rstd
    y = (x64 - mu) * rstd * g64 + b64
    b_y = g64.abs() * (e_mean * rstd + D * b_rstd + 3 * U24 * D * rstd_hi) + U24 * (g64.abs() * D * rstd_hi + b64.abs())
    return dict(mean=mu[:, 0], rstd=rstd[:, 0], y=y, b_mean=e_mean[:, 0], b_rstd=b_rstd[:, 0], b_y=b_y)


def ln_bwd_reference(dy, x, gamma, mean, rstd, dres0=None, dres1=None, d0=None):
    """Backward of LayerNorm from the statistics the kernel is given (mean, rstd [P] fp32) -> dict of float64 references
    and bounds: dx [P, C], dgamma, dbeta, colsum [C] (each onto its initial value in d0 = (dgamma0, dbeta0, colsum0)),
    with b_dx, b_dgamma, b_dbeta, b_colsum."""
    dy64, x64, g64 = dy.to(F64), x.to(F64), gamma.to(F64)
    P, C = x64.shape
    mean64, rstd64 = mean.to(F64)[:, None], rstd.to(F64)[:, None]
    xh = (x64 - mean64) * rstd64
    gy = dy64 * g64
    m1 = gy.sum(1, keepdim=True) / C
    m2 = (gy * xh).sum(1, keepdim=True) / C
    b_m1 = (C + 2) * U24 * gy.abs().sum(1, keepdim=True) / C
    b_m2 = (C + 4) * U24 * (gy * xh).abs().sum(1, keepdim=True) / C
    t = gy - m1 - xh * m2
    inner = (U24 * gy.abs() + b_m1 + xh.abs() * b_m2 + 2 * U24 * xh.abs() * (m2.abs() + b_m2)
             + U24 * xh.abs() * m2.abs() + 2 * U24 * (gy.abs() + m1.abs() + xh.abs() * m2.abs()))
    o = rstd64 * t
    b_o = rstd64 * inner + U24 * (o.abs() + rstd64 * inner)
    res = [d.to(F64) for d in (dres0, dres1) if d is not None]
    dx = o + sum(res) if res else o
    rmag = sum(r.abs() for r in res) if res else 0.0
    b_dx = b_o + 2 * U24 * (dx.abs() + o.abs() + rmag + b_o)
    z = torch.zeros(C, dtype=F64, device=x64.device)
    d0 = tuple(z if v is None else v.to(F64) for v in (d0 or (None, None, None)))
    dg_terms, db_terms = dy64 * xh, dy64
    out = dict(dx=dx, b_dx=b_dx)
    out["dgamma"] = d0[0] + dg_terms.sum(0)
    out["b_dgamma"] = (P + 5) * U24 * (dg_terms.abs().sum(0) + d0[0].abs())
    out["dbeta"] = d0[1] + db_terms.sum(0)
    out["b_dbeta"] = (P + 2) * U24 * (db_terms.abs().sum(0) + d0[1].abs())
    out["colsum"] = d0[2] + dx.sum(0)
    out["b_colsum"] = b_dx.sum(0) + (P + 2) * U24 * ((dx.abs() + b_dx).sum(0) + d0[2].abs())
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Small-Cin convolution (NCHW image in, pixel-major [P, Cout] out)
# ----------------------------------------------------------------------------------------------------------------------
def conv_inputs(N, Cin, H, W, Cout, kh, kw, seed):
    """x [N, Cin, H, W] in [-1, 1) (both signs: ReLU / ELU are not the identity), a causally masked weight, bias, dy
    [N H W, Cout] and initial values dw0 / db0 for the accumulating gradients; fp32 on the CPU."""
    g = _gen(seed)
    x = torch.rand(N, Cin, H, W, generator=g) * 2 - 1
    w = torch.randn(Cout, Cin, kh, kw, generator=g) * 0.2
    mask = torch.zeros(kh, kw)
    mask[: kh // 2] = 1
    mask[kh // 2, : kw // 2 + 1] = 1
    w = w * mask
    b = torch.randn(Cout, generator=g)
    dy = torch.randn(N * H * W, Cout, generator=g)
    dw0 = torch.randn(Cout, Cin, kh, kw, generator=g)
    db0 = torch.randn(Cout, generator=g)
    return x, w, b, dy, dw0, db0


def _patches(a64, kh, kw, ph, pw):
    """[N H W, Cin kh kw] float64 patches of a [N, Cin, H, W] (zero padding), k = ci kh kw + i kw + j as the kernel."""
    N, Cin, H, W = a64.shape
    cols = torch.nn.functional.unfold(a64, (kh, kw), padding=(ph, pw))  # [N, Cin kh kw, L]
    Ho, Wo = H + 2 * ph - kh + 1, W + 2 * pw - kw + 1
    assert (Ho, Wo) == (H, W), "the small-Cin kernels compute a same-size output"
    return cols.transpose(1, 2).reshape(N * H * W, Cin * kh * kw)


def conv_reference(x, w, b, dy, pad, pre_act=NONE, dw0=None, db0=None):
    """dict of float64 references and bounds for pg_conv_small_fwd / _bwd: out [P, Cout], dw [Cout, Cin, kh, kw] (onto
    dw0), db [Cout] (onto db0), dx [N, Cin, H, W]."""
    Cout, Cin, kh, kw = w.shape
    ph, pw = pad
    N, _, H, W = x.shape
    x64, w64, b64, dy64 = x.to(F64), w.to(F64), b.to(F64), dy.to(F64)
    a64 = act64(pre_act, x64)
    r_act, _ = act_err(pre_act, x64)
    K = Cin * kh * kw
    P = N * H * W
    pa = _patches(a64, kh, kw, ph, pw)
    wm = w64.reshape(Cout, K)
    out = pa @ wm.T + b64
    mag = pa.abs() @ wm.abs().T
    b_out = (K + 1) * U24 * (b64.abs() + mag) + r_act * mag
    dw0 = torch.zeros_like(w64) if dw0 is None else dw0.to(F64)
    db0 = torch.zeros_like(b64) if db0 is None else db0.to(F64)
    dwm = dy64.T @ pa
    dw_mag = dy64.abs().T @ pa.abs()
    dw = dw0 + dwm.reshape(w.shape)
    b_dw = ((P + 2) * U24 * (dw_mag + dw0.reshape(Cout, K).abs()) + r_act * dw_mag).reshape(w.shape)
    db = db0 + dy64.sum(0)
    b_db = (P + 2) * U24 * (dy64.abs().sum(0) + db0.abs())
    # dgrad: the transposed convolution of dy (NCHW) with w, times act'(x)
    dy_nchw = dy64.reshape(N, H, W, Cout).permute(0, 3, 1, 2)
    flip = (kh - 1 - ph, kw - 1 - pw)
    wt = w64.flip(2, 3).transpose(0, 1)
    s = torch.nn.functional.conv2d(dy_nchw, wt, padding=flip)
    T = torch.nn.functional.conv2d(dy_nchw.abs(), wt.abs(), padding=flip)
    d = dact64(pre_act, x64)
    rd, ad = deriv_err(pre_act, x64)
    n = kh * kw * Cout
    dx = s * d
    b_dx = d.abs() * (n + 2) * U24 * T + (rd * d.abs() + ad) * T
    return dict(out=out, b_out=b_out, dw=dw, b_dw=b_dw, db=db, b_db=b_db, dx=dx, b_dx=b_dx)


# ----------------------------------------------------------------------------------------------------------------------
# BCE with logits
# ----------------------------------------------------------------------------------------------------------------------
def bce_inputs(regime, numel, seed, hard=False):
    """logits and targets [numel] fp32 on the CPU.
      randn    4 N(0, 1);
      extreme  |l| uniform in [80, 100] with both signs, plus +-88.7 (expf's overflow edge), +-87.3 and exactly 0 at
               fixed positions;
    targets: soft U(0, 1), or hard (exactly 0 or 1)."""
    g = _gen(seed)
    if regime == "extreme":
        l = (torch.rand(numel, generator=g) * 20 + 80) * (torch.randint(0, 2, (numel,), generator=g).float() * 2 - 1)
        special = torch.tensor([88.7, -88.7, 87.3, -87.3, 0.0, 100.0, -100.0])
        k = min(numel, special.numel())
        l[:k] = special[:k]
        if numel > 16:
            l[numel // 2] = 0.0
            l[-1] = -88.7
    else:
        assert regime == "randn", regime
        l = torch.randn(numel, generator=g) * 4
    t = torch.randint(0, 2, (numel,), generator=g).float() if hard else torch.rand(numel, generator=g)
    return l, t


def bce_reference(logits, target, scale, loss0=0.0):
    """(loss, b_loss, dl, b_dl): the float64 summed loss onto loss0 and its bound, the float64 dlogits and their bound."""
    l, t = logits.to(F64), target.to(F64)
    e = torch.exp(-l.abs())
    lp = torch.log1p(e)
    mx = l.clamp_min(0)
    terms = mx - l * t + lp
    n = l.numel()
    loss = loss0 + float(terms.sum())
    term_err = 3 * U24 * (mx + (l * t).abs() + lp) + 4 * U24 * e + 2.0 ** -149
    b_loss = (n + 2) * U24 * (float(terms.abs().sum()) + abs(loss0)) + float(term_err.sum())
    s = torch.sigmoid(l)
    dl = (s - t) * scale
    b_dl = abs(scale) * (6 * U24 * s + TINY + U24 * (s - t).abs()) + U24 * dl.abs()
    return loss, b_loss, dl, b_dl


# ----------------------------------------------------------------------------------------------------------------------
# column sums
# ----------------------------------------------------------------------------------------------------------------------
def colsum_reference(x, out0=None):
    """(ref, bound) of out0 + sum over the rows of x [P, C] (any dtype), float64 [C]."""
    x64 = x.to(F64)
    P = x64.shape[0]
    o = torch.zeros(x64.shape[1], dtype=F64, device=x64.device) if out0 is None else out0.to(F64)
    return o + x64.sum(0), (P + 2) * U24 * (x64.abs().sum(0) + o.abs())


# ----------------------------------------------------------------------------------------------------------------------
# optimizer
# ----------------------------------------------------------------------------------------------------------------------
def adam_scalars(lr, beta1, beta2, eps, step):
    """The fp32 scalars pg_adam_step hands its kernel, rounded as it rounds them."""
    f = lambda v: float(torch.tensor(v, dtype=F32))
    bc1 = 1.0 - math.pow(beta1, step)
    bc2 = 1.0 - math.pow(beta2, step)
    return dict(lr_bc1=f(lr / bc1), rsqrt_bc2=f(1.0 / math.sqrt(bc2)), beta1=f(beta1), beta2=f(beta2),
                omb1=f(1.0 - beta1), omb2=f(1.0 - beta2), eps=f(eps))


def adam_inputs(regime, numels, seed):
    """Lists (p, g, m, v) of fp32 tensors of the given sizes on the CPU.
      randn         p, g ~ N(0, 1), m ~ 0.1 N(0, 1), v ~ 0.01 U(0, 1);
      tiny_moments  as randn, but a third of the elements have g, m and v near 0 (g ~ 1e-6 N, m ~ 1e-7 N,
                    v ~ 1e-14 U, some exactly 0): the denominator is dominated by eps."""
    g = _gen(seed)
    ps, gs, ms, vs = [], [], [], []
    for n in numels:
        p = torch.randn(n, generator=g)
        gr = torch.randn(n, generator=g)
        m = torch.randn(n, generator=g) * 0.1
        v = torch.rand(n, generator=g) * 0.01
        if regime == "tiny_moments":
            sel = torch.rand(n, generator=g) < 1 / 3
            gr = torch.where(sel, gr * 1e-6, gr)
            m = torch.where(sel, m * 1e-6, m)
            v = torch.where(sel, v * 1e-12, v)
            zero = torch.rand(n, generator=g) < 0.05
            gr, m, v = (torch.where(zero, torch.zeros_like(t), t) for t in (gr, m, v))
        else:
            assert regime == "randn", regime
        ps.append(p), gs.append(gr), ms.append(m), vs.append(v)
    return ps, gs, ms, vs


def sqnorm_reference(grads, n_chunks):
    """(norm, bound) of sqrt(sum g^2) over every tensor, float64."""
    s = sum(float(g.to(F64).pow(2).sum()) for g in grads)
    n = sum(g.numel() for g in grads)
    norm = math.sqrt(s)
    return norm, norm * ((n + n_chunks + 1) * U24 / 2 + U24)


def adam_reference(p, g, m, v, norm, max_norm, sc):
    """Float64 Adam update of one tensor from the kernel's fp32 norm and the fp32 scalars sc (adam_scalars).  Returns a
    dict of references and bounds: p, g (after clipping), m, v and b_p, b_g, b_m, b_v."""
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    eps6 = float(torch.tensor(1e-6, dtype=F32))
    coef = max_norm / (float(norm) + eps6)
    clips = coef < 1.0
    coef = min(coef, 1.0)
    g1 = g64 * coef
    b_g = 3 * U24 * g1.abs() if clips else torch.zeros_like(g1)
    m1 = m64 + sc["omb1"] * (g1 - m64)
    b_m = sc["omb1"] * (b_g + 2 * U24 * (g1 - m64).abs() + U24 * g1.abs()) + U24 * m1.abs()
    v1 = sc["beta2"] * v64 + sc["omb2"] * g1 * g1
    b_v = sc["omb2"] * (8 * U24 * g1 * g1 + 2 * g1.abs() * b_g) + 2 * U24 * sc["beta2"] * v64 + U24 * v1.abs()
    sq = v1.sqrt() * sc["rsqrt_bc2"]
    denom = sq + sc["eps"]
    r_v = torch.where(v1 > 0, b_v / v1.clamp_min(1e-300), torch.zeros_like(v1))
    r_d = (r_v / 2 + r_v ** 2 + 2 * U24) * sq / denom + U24
    stepv = sc["lr_bc1"] * m1 / denom
    p1 = p64 - stepv
    b_p = sc["lr_bc1"] * (b_m + m1.abs() * (r_d + 2 * U24)) / denom + U24 * (p1.abs() + stepv.abs())
    return dict(p=p1, g=g1, m=m1, v=v1, b_p=b_p, b_g=b_g, b_m=b_m, b_v=b_v)


def chunk_table(numels, chunk_elems):
    """[(tensor, chunk)] as FusedAdam._build_plan builds it."""
    return [(t, c) for t, n in enumerate(numels) for c in range((n + chunk_elems - 1) // chunk_elems)]
