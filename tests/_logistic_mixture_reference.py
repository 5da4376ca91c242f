"""Float64 restatement of the discretised logistic mixture likelihood (losses.logistic_mixture_nll,
models.logistic_mixture_sample_fn) and the per-element bounds its fp32 kernels are held to.  This module is the spec.

Layout: preds [N, M * G, *spatial], G = (C + 1)(C + 2) / 2, T = C (C - 1) / 2; mixture logit pi_m at channel m, mean
mu_{m,c} at M + m C + c, raw log-scale ls_{m,c} at M + M C + m C + c, raw coupling coefficient r_{m,t} at
M + 2 M C + m T + t, t = c (c - 1) / 2 + j for j < c.  Bin of x: k = rint(clamp(x, 0, 1) (K - 1)) in fp32, centre
x'_k = 2k / (K - 1) - 1, half-width h = 1 / (K - 1).  log_s = max(ls, -7), mu' = mu + sum_{j<c} tanh(r) x'_{k_j},
a = (x' - mu' + h) e^-log_s, b = (x' - mu' - h) e^-log_s, lp = -softplus(-a) (bin 0), -softplus(b) (bin K - 1),
-softplus(-a) - softplus(b) + log(-expm1(-(a - b))) otherwise; NLL = -logsumexp_m(log_softmax(pi)_m + sum_c lp).

U = 2^-24, the unit roundoff of fp32.  The CUDA library functions the kernel calls are within 1 ulp (logf, log1pf,
expm1f) or 2 ulp (expf, tanhf, __fdividef in its range); an ulp is at most 2 U relative, so they are taken as 2 U and
4 U relative.  IEEE operations round once: U relative."""

import math

import torch

F64 = torch.float64
U = 2.0 ** -24
LOG_SCALE_MIN = -7.0
BUGS = ("half_width_1_over_K", "no_clamp", "wrong_coupling", "swapped_edges")


def groups(C):
    return (C + 1) * (C + 2) // 2


def coef_index(c, j):
    return c * (c - 1) // 2 + j


def target(x, K):
    """Bin of each input value, computed in fp32 as the kernel does (losses.categorical_target's rule)."""
    return torch.round(x.float().clamp(0, 1) * float(K - 1)).long()


def centre(k, K):
    """Exact bin centre 2k / (K - 1) - 1 in float64."""
    return 2.0 * k.to(F64) / (K - 1) - 1.0


def split(preds, C):
    """(pi [N, M, P], mu [N, M, C, P], ls [N, M, C, P], r [N, M, T, P]) of preds [N, M * G, *spatial], float64."""
    N = preds.shape[0]
    p = preds.to(F64).reshape(N, preds.shape[1], -1)
    G, T = groups(C), C * (C - 1) // 2
    M = preds.shape[1] // G
    P = p.shape[-1]
    pi = p[:, :M]
    mu = p[:, M:M + M * C].reshape(N, M, C, P)
    ls = p[:, M + M * C:M + 2 * M * C].reshape(N, M, C, P)
    r = p[:, M + 2 * M * C:].reshape(N, M, T, P)
    return pi, mu, ls, r


def softplus(z):
    return z.clamp(min=0) + torch.log1p(torch.exp(-z.abs()))


def _terms(preds, x, K, bug=None):
    """Per-(image, component, channel, pixel) float64 quantities of the convention, as a dict; `bug` names one of the
    BUGS, a deliberately wrong variant the bounds must see."""
    N, C = x.shape[:2]
    pi, mu, ls, r = split(preds, C)
    k = target(x, K).reshape(N, 1, C, -1).to(pi.device)
    xc = centre(k, K)  # [N, 1, C, P]
    h = 1.0 / K if bug == "half_width_1_over_K" else 1.0 / (K - 1)
    log_s = ls if bug == "no_clamp" else ls.clamp(min=LOG_SCALE_MIN)
    th = torch.tanh(r)
    mups, coupling = [], []
    for c in range(C):
        m_c, s_c = mu[:, :, c], mu[:, :, c].abs()
        for j in range(c):
            jj = min(j + 1, C - 1) if bug == "wrong_coupling" else j
            t = th[:, :, coef_index(c, j)]
            m_c = m_c + t * xc[:, :, jj]
            s_c = s_c + (t * xc[:, :, jj]).abs()
        mups.append(m_c)
        coupling.append(s_c)
    mup = torch.stack(mups, dim=2)
    coupling = torch.stack(coupling, dim=2)
    inv = torch.exp(-log_s)
    d = xc - mup
    a, b = inv * (d + h), inv * (d - h)
    D = inv * (2 * h)
    lo, hi = k > 0, k < K - 1  # not bin 0, not bin K - 1
    if bug == "swapped_edges":
        lo, hi = k < K - 1, k > 0
    spa, spb = softplus(-a), softplus(b)
    lg = torch.log(-torch.expm1(-D))
    mid = lo & hi
    lp = torch.where(mid, -spa - spb + lg, torch.where(hi, -spa, -spb))
    L = lp.sum(dim=2)
    z = pi + L
    nll = torch.logsumexp(pi, dim=1) - torch.logsumexp(z, dim=1)
    return dict(pi=pi, mu=mu, ls=ls, r=r, th=th, k=k, xc=xc, h=h, log_s=log_s, mup=mup, S=coupling, inv=inv, d=d,
                a=a, b=b, D=D, lo=lo, hi=hi, mid=mid, spa=spa, spb=spb, lg=lg, lp=lp, L=L, z=z, nll=nll)


def nll(preds, x, K, bug=None):
    """Per (image, pixel) NLL in nats, float64, [N, *spatial]."""
    return _terms(preds, x, K, bug)["nll"].reshape(x.shape[0], *x.shape[2:])


def loss(preds, x, K):
    """(mean over images of the summed NLL, bits/dim) in float64."""
    per_image = nll(preds, x, K).reshape(x.shape[0], -1).sum(dim=1)
    value = per_image.mean()
    return value, value / (x[0].numel() * math.log(2.0))


def _sigmoid(z):
    return torch.sigmoid(z)


def _grad_parts(t):
    """d lp / d mu' (g) and d lp / d log_s (q) per (image, component, channel, pixel), from the closed forms."""
    a, b, D, inv, lo, hi, mid = t["a"], t["b"], t["D"], t["inv"], t["lo"], t["hi"], t["mid"]
    sa = torch.where(hi, _sigmoid(-a), torch.zeros_like(a))
    sb = torch.where(lo, _sigmoid(b), torch.zeros_like(b))
    f = torch.where(mid, D / torch.expm1(D), torch.zeros_like(D))
    g = -inv * (sa - sb)
    q = -a * sa + b * sb - f
    return g, q, sa, sb, f


def dpreds(preds, x, K, grad_scale, bug=None):
    """d (grad_scale * sum NLL) / d preds in float64, in preds' layout, from the closed forms of the convention.
    bug="one_minus_tanh2": the coefficient gradients with 1 - tanh(r)^2 evaluated in fp32 instead of sech^2."""
    t = _terms(preds, x, K)
    N, C = x.shape[:2]
    M = t["pi"].shape[1]
    w = torch.softmax(t["z"], dim=1)
    soft = torch.softmax(t["pi"], dim=1)
    g, q, *_ = _grad_parts(t)
    dpi = (soft - w) * grad_scale
    ws = (w * grad_scale).unsqueeze(2)
    dmu = -ws * g
    dls = torch.where(t["ls"] >= LOG_SCALE_MIN, -ws * q, torch.zeros_like(q))
    T = C * (C - 1) // 2
    dr = torch.zeros_like(t["r"])
    for c in range(C):
        for j in range(c):
            i = coef_index(c, j)
            r = t["r"][:, :, i]
            if bug == "one_minus_tanh2":
                t32 = torch.tanh(r).float()
                sech2 = (1.0 - t32 * t32).to(F64)
            else:
                sech2 = 1.0 / torch.cosh(r) ** 2
            dr[:, :, i] = dmu[:, :, c] * sech2 * t["xc"][:, 0, j].unsqueeze(1)
    P = t["pi"].shape[-1]
    out = torch.cat([dpi, dmu.reshape(N, M * C, P), dls.reshape(N, M * C, P), dr.reshape(N, M * T, P)], dim=1)
    return out.reshape(preds.shape)


# ------------------------------------------------------------------------------------------------
# fp32 error bounds of the loss kernel
# ------------------------------------------------------------------------------------------------
def sum_relative_bound(M):
    """Relative error bound of an fp32 online sum s = sum_m exp(l_m - max) over M terms (s >= 1): each expf within
    2 ulp plus the rounding of its argument (U |l - max| relative, and |l - max| e^(l - max) <= 1/e), one rounding per
    addition and per rescale of the running sum (pg_categorical.cu's bound, M terms)."""
    return (3 * M + 16) * U


def _error_terms(preds, x, K):
    """Absolute fp32 error bounds of every intermediate the kernel forms, first order, per (image, component, channel,
    pixel) unless stated:
      x'      fmaf(2k, fl(1 / (K - 1)), -1): h within U relative, so 2k h within 2 U; plus the fma: 3 U.
      mu'     c fmas onto mu, each rounding U |partial| <= U S (S = |mu| + sum |tanh r x'|); tanhf 4 U relative and x'
              3 U absolute per term: (c + 5) U S + 3 U sum |tanh r|.
      d       x' - mu': e_mu' + 3 U + U |d|;  d +- h: e_d + U h + U |d +- h|.
      inv     expf(-log_s), log_s exact: 4 U relative.
      a, b    inv e(d +- h) + 5 U |a| (inv's 4 U and the product's U).
      D       fl(inv * fl(2 / (K - 1))): 6 U relative.
      softplus(z) = max(z, 0) + log1pf(expf(-|z|)): expf 4 U e^-|z|, log1pf 2 U, the addition U softplus; with
              e^-|z| <= softplus(z) / ln 2, at most 10 U softplus(z) own error, plus sigmoid(z) e_z from its input.
      log(-expm1(-D)): input error e_D / expm1(D) <= 6 U, expm1f 2 U relative (2 U absolute after the log), logf
              2 U |lg|: 8 U + 2 U |lg|.
      lp      the terms' errors plus 2 U |.| for the two additions of a middle bin.
      L       sum over c of e_lp plus (C - 1) U sum |lp|;  z = pi + L: e_L + U |z|."""
    t = _terms(preds, x, K)
    C = x.shape[1]
    S, th, xc = t["S"], t["th"], t["xc"]
    e_mup = []
    for c in range(C):
        extra = sum((th[:, :, coef_index(c, j)].abs() for j in range(c)), torch.zeros_like(S[:, :, c]))
        e_mup.append((c + 5) * U * S[:, :, c] + 3 * U * extra)
    e_mup = torch.stack(e_mup, dim=2)
    d, h, inv, a, b, D = t["d"], t["h"], t["inv"], t["a"], t["b"], t["D"]
    e_d = e_mup + 3 * U + U * d.abs()
    e_a = inv * (e_d + U * h + U * (d + h).abs()) + 5 * U * a.abs()
    e_b = inv * (e_d + U * h + U * (d - h).abs()) + 5 * U * b.abs()
    e_D = 6 * U * D
    sa_full, sb_full = _sigmoid(-a), _sigmoid(b)
    e_spa = sa_full * e_a + 10 * U * t["spa"]
    e_spb = sb_full * e_b + 10 * U * t["spb"]
    e_lg = 8 * U + 2 * U * t["lg"].abs()
    mid, lo, hi = t["mid"], t["lo"], t["hi"]
    e_lp = torch.where(mid, e_spa + e_spb + e_lg + 2 * U * (t["spa"] + t["spb"] + t["lg"].abs()),
                       torch.where(hi, e_spa, e_spb))
    e_L = e_lp.sum(dim=2) + (C - 1) * U * t["lp"].abs().sum(dim=2)
    e_z = e_L + U * t["z"].abs()
    return t, dict(e_mup=e_mup, e_d=e_d, e_a=e_a, e_b=e_b, e_D=e_D, e_z=e_z)


def nll_bound(preds, x, K):
    """Per (image, pixel) bound of the kernel's NLL = (m_pi - m_z) + (log s_pi - log s_z): the responsibilities'
    weighted errors of z (first order: d NLL / d z_m = -w_m, and pi is exact), both sums' relative errors carried
    through the logs, the logs' own 1 ulp, and the roundings of m_pi - m_z, of the log difference and of the final
    addition; doubled for slack."""
    t, e = _error_terms(preds, x, K)
    pi, z = t["pi"], t["z"]
    M = pi.shape[1]
    w = torch.softmax(z, dim=1)
    m1, m2 = pi.max(dim=1).values, z.max(dim=1).values
    ls1 = torch.log(torch.exp(pi - m1.unsqueeze(1)).sum(dim=1))
    ls2 = torch.log(torch.exp(z - m2.unsqueeze(1)).sum(dim=1))
    b = ((w * e["e_z"]).sum(dim=1) + 2 * 1.01 * sum_relative_bound(M) + 3 * U * (ls1.abs() + ls2.abs())
         + 3 * U * (m1 - m2).abs() + 2 * U * t["nll"].abs())
    return (2 * b + 1e-30).reshape(x.shape[0], *x.shape[2:])


def image_sum_bound(preds, x, K, n_blocks):
    """Bound of the per-image sums: every element's bound plus the fp32 additions of the reduction (a 5-level warp
    butterfly, a 2-level block butterfly over 4 warps, then at most n_blocks sequential additions of the partials)."""
    N = x.shape[0]
    b = nll_bound(preds, x, K).reshape(N, -1).sum(dim=1)
    v = nll(preds, x, K).abs().reshape(N, -1).sum(dim=1)
    return b + 1.1 * (12 + n_blocks) * U * v


def dpreds_bound(preds, x, K, grad_scale):
    """Per-element bound of the kernel's dpreds, in preds' layout, first order in U:
      softmax(pi)_m = expf(pi - m1) * fl(1 / s1): 4 U + U |pi - m1| + the sum's relative error + 2 U.
      w_m = expf(z_m - m2) * fl(1 / s2): as above, plus e_z_m + sum_j w_j e_z_j from the errors of z.
      d pi = (soft - w) gs: both relative errors, the subtraction and the scale (gs is fp32: one more U).
      sigmoid(z) (expf, one addition, __fdividef): 9 U relative, plus sigmoid(z) sigmoid(-z) e_z from its input.
      g = -inv (sigmoid(-a) - sigmoid(b)) (or one of them at an edge bin): inv e(diff) + 5 U |g|.
      q = (-a sigmoid(-a) + b sigmoid(b)) - D / expm1(D): products |a| e_sig + sig e_a + U, D / expm1(D) by
          __fdividef within 6 U plus its input error (slope <= 1/2) 3 U D, two additions; 1e-35 absolute where
          expm1(D) passes 2^126 and __fdividef gives 0.
      d mu = -(w gs) g, d log_s = -(w gs) q (0 exactly below -7), d r = (d mu * sech^2(r)) * x'_j with sech^2 by
          expf, one addition, one square and __fdividef: 10 U relative, plus 2^-126 where it underflows.
    Doubled, plus 1e-40 absolute."""
    t, e = _error_terms(preds, x, K)
    N, C = x.shape[:2]
    pi, z = t["pi"], t["z"]
    M = pi.shape[1]
    P = pi.shape[-1]
    gs = abs(grad_scale)
    srb = sum_relative_bound(M)
    w = torch.softmax(z, dim=1)
    soft = torch.softmax(pi, dim=1)
    m1, m2 = pi.max(dim=1, keepdim=True).values, z.max(dim=1, keepdim=True).values
    e_z = e["e_z"]
    rel_soft = 6 * U + U * (pi - m1).abs() + srb
    rel_w = e_z + (w * e_z).sum(dim=1, keepdim=True) + 6 * U + U * (z - m2).abs() + srb
    b_pi = gs * (soft * rel_soft + w * rel_w + 2 * U * (soft - w).abs())
    g, q, sa, sb, f = _grad_parts(t)
    a, b, inv, D, lo, hi, mid = t["a"], t["b"], t["inv"], t["D"], t["lo"], t["hi"], t["mid"]
    e_sa = torch.where(hi, sa * (9 * U + _sigmoid(a) * e["e_a"]), torch.zeros_like(a))
    e_sb = torch.where(lo, sb * (9 * U + _sigmoid(-b) * e["e_b"]), torch.zeros_like(b))
    e_g = inv * (e_sa + e_sb + U * (sa - sb).abs()) + 5 * U * g.abs()
    e_asa = a.abs() * e_sa + sa * e["e_a"] + U * (a * sa).abs()
    e_bsb = b.abs() * e_sb + sb * e["e_b"] + U * (b * sb).abs()
    e_f = torch.where(mid, 3 * U * D + 6 * U * f + 1e-35, torch.zeros_like(D))
    e_q = e_asa + e_bsb + e_f + 2 * U * ((a * sa).abs() + (b * sb).abs() + f)
    ws = (w * gs).unsqueeze(2)
    rel_ws = (rel_w + 2 * U).unsqueeze(2)
    dmu = ws * g
    b_mu = ws * e_g + dmu.abs() * rel_ws + U * dmu.abs()
    b_ls = torch.where(t["ls"] >= LOG_SCALE_MIN, ws * e_q + (ws * q).abs() * (rel_ws + U), torch.zeros_like(q))
    T = C * (C - 1) // 2
    b_r = torch.zeros_like(t["r"])
    for c in range(C):
        for j in range(c):
            i = coef_index(c, j)
            r = t["r"][:, :, i]
            s2 = 1.0 / torch.cosh(r) ** 2
            xj = t["xc"][:, 0, j].unsqueeze(1).abs()
            gm = dmu[:, :, c].abs()
            b_r[:, :, i] = (s2 * xj * b_mu[:, :, c] + gm * xj * (10 * U * s2 + 2.0 ** -126) + gm * s2 * 3 * U
                            + 2 * U * gm * s2 * xj)
    out = torch.cat([b_pi, b_mu.reshape(N, M * C, P), b_ls.reshape(N, M * C, P), b_r.reshape(N, M * T, P)], dim=1)
    return (2 * out + 1e-40).reshape(preds.shape)


# ------------------------------------------------------------------------------------------------
# sampling
# ------------------------------------------------------------------------------------------------
def inverse_map(preds, u, K):
    """Float64 draw of each row of preds [n, M * G] under uniforms u [n, 1 + C]: the first component whose cumulative
    softmax(pi) reaches u[:, 0], then for c ascending k_c = rint(clamp((v + 1) / 2, 0, 1) (K - 1)) with
    v = mu' + e^log_s (log u - log1p(-u)), mu' coupled to the drawn bins' centres.  Returns (k [n, C] int64,
    near [n] bool): near marks rows where u[:, 0] is within the fp32 bound of a component boundary, or a channel's
    (v + 1) / 2 (K - 1) is within its fp32 bound of a bin edge (a half-integer), so the kernel's draw may differ
    there (and, through the coupling, in the later channels)."""
    n = preds.shape[0]
    C = u.shape[1] - 1
    p = preds.to(F64)
    u = u.to(F64)
    pi, mu, ls, r = split(p.reshape(n, -1, 1), C)
    pi, mu, ls, r = pi[..., 0], mu[..., 0], ls[..., 0], r[..., 0]
    M = pi.shape[1]
    cum = torch.softmax(pi, dim=1).cumsum(dim=1)
    m = (cum < u[:, :1]).sum(dim=1).clamp(max=M - 1)
    near = ((cum[:, :-1] - u[:, :1]).abs() <= 4 * sum_relative_bound(M)).any(dim=1)
    rows = torch.arange(n)
    k = torch.zeros(n, C, dtype=torch.long)
    for c in range(C):
        mup = mu[rows, m, c]
        S = mup.abs()
        for j in range(c):
            t = torch.tanh(r[rows, m, coef_index(c, j)]) * centre(k[:, j], K)
            mup = mup + t
            S = S + t.abs()
        uc = u[:, 1 + c]
        lu = torch.log(uc) - torch.log1p(-uc)
        s = torch.exp(ls[rows, m, c].clamp(min=LOG_SCALE_MIN))
        v = mup + s * lu
        kv = (v + 1) / 2 * (K - 1)
        k[:, c] = torch.round(kv.clamp(0, K - 1)).long()
        finite = torch.isfinite(lu)
        e_v = (c + 8) * U * S + 3 * U * c + s * lu.abs().nan_to_num(0, 0, 0) * 10 * U + U * v.abs().nan_to_num(0, 0, 0)
        e_k = (K - 1) / 2 * (e_v + U * (v + 1).abs().nan_to_num(0, 0, 0)) + U * kv.abs().nan_to_num(0, 0, 0)
        edge = torch.floor(kv.nan_to_num(0, 0, 0)) + 0.5
        dist = (kv - edge).abs()
        inside = (kv > 0.5 - 4 * e_k) & (kv < K - 1.5 + 4 * e_k)
        near = near | (finite & inside & (dist <= 4 * e_k))
    return k, near


def joint_probabilities(row, C, K):
    """Float64 probability of every cell (k_0, ..., k_{C-1}) of one pixel's bins under the parameters row [M * G]:
    exp(-NLL) of the image holding that cell, as a tensor [K] * C."""
    cells = torch.cartesian_prod(*[torch.arange(K)] * C).reshape(-1, C) if C > 1 else torch.arange(K).reshape(-1, 1)
    x = (cells.to(F64) / (K - 1)).float().reshape(-1, C, 1, 1)
    preds = row.reshape(1, -1, 1, 1).expand(cells.shape[0], -1, 1, 1)
    return torch.exp(-nll(preds, x, K)).reshape([K] * C)
