"""Float64 reference of causal softmax attention, element-wise error bounds for its CUDA kernels, and the input regimes
the attention tests draw from.  Shared by tests/test_attention_kernels_gpu.py and tests/test_attention_bounds_cpu.py;
not a test module.

Reference.  Per (image, head), on the device the tensors live on, from the same bf16 values the kernels read, with no
autograd and nothing in fp32:  s = c q k^T with c = 1/sqrt(dk_true), keys j <= i visible (j < i when strict);
p = softmax(s) over the visible keys, o = p v, lse = log sum_j exp(s_ij); dv = p^T dO, dP = dO v^T,
D_i = sum_d dO_id o_id, dS = p (dP - D), dq = c dS k, dk = c dS^T q.  A strict row 0 has no keys: the kernels define
its o and its lse as 0.

Kernel arithmetic the bounds follow (csrc/pg_attention_tc.cuh; the SIMT and decode kernels of csrc/pg_attention.cu do
the same steps with P kept in fp32, so the same bounds hold for them).  Inputs are bf16, so every product of two inputs
is exact in fp32.  Scores are fp32 sums of dk_slot products (padded slot columns add exact zeros); the softmax runs
online over 128-key tiles: p = ex2.approx.ftz(s c log2(e) - m c log2(e)) against the running max m, O and l rescaled by
alpha = ex2(m_old - m_new) whenever the max moves; P is rounded to bf16 as the A operand of O += P V; o = bf16(O / l),
lse = m c + __logf(l).  The backward recomputes p = ex2(s c log2(e) - lse log2(e)) from the forward's own lse, takes
delta from the forward's own o, and rounds P and dS = p (dP - delta) to bf16 as A operands; all sums are fp32.

Bound derivation.  U8 = 2^-8 is the unit roundoff of bf16 (round to nearest), U24 = 2^-24 that of fp32; an fp32 sum
is charged U23 = 2^-23 per addition along its longest chain times the sum of the absolute values of its terms (the
worst case of recursive summation in any order, doubled because tensor-core accumulation may truncate).  Every term is
a float64 product of non-negative matrices or an element-wise expression: no term depends on a maximum over a tensor;
row quantities (E_i, R_i, n_i) are maxima or counts over one row's visible keys.
  * Exponent error of p_ij, natural-log units:  e_ij = dk_slot U23 c sum_d |q_id k_jd|  (the fp32 score)
      + 2^-20 R_i, R_i = max_j |c s_ij| over the row's visible keys: the fp32 roundings of c, c log2(e), the running
        maxima times c log2(e), the fma argument and the alpha arguments, each at most U24 (2 R_i), 13 of them;
      + (T_i + 1) EX2: the ex2.approx error of p and of one alpha per 128-key tile (T_i = i // 128 + 1 tiles).  An
        alpha multiplies O and l alike, but only the terms already summed, so its error reweights those terms.
    E_i = max_j e_ij.
  * Forward:  |o~_id - o_id| <= U8 |o_id| + (U8 + 2 E_i + 2 g_i + 2^-22) M_id + FLUSH sum_j |v_jd|
      M_id = sum_j p_ij |v_jd|; U8 |o| is the output rounding, the U8 in the bracket the rounding of P; E_i once for the
      numerator's p and once for l; g_i = (n_i + 2 T_i + 4) U23 for the fp32 sums of O and l (n_i visible keys, two
      roundings per tile for the rescale) and 2^-22 for 1 / l and the final product.  FLUSH covers ex2.approx.ftz
      flushing a p or an alpha below 2^-126 to zero (l >= 1 after the final max, so the normalised error is below
      2^-125 per key).
  * lse:  E_i + g_i + LG2 (1 + log n_i) + 2^-22 (R_i + |lse_i|)  (the exponent error of l, its sum, __logf, and the
      roundings of m c and of the final sum).
  * Backward, propagating the forward's own o~ and lse errors:
      eps_ij = e_ij + B_lse_i + 2^-20 (R_i + |lse_i|) + 2^-21: relative error of the recomputed p (score, lse, the
        roundings of lse log2(e) and of the fma argument, ex2, and the two fp32 roundings of p (dP - delta));
      e'_ij = dv_slot U23 sum_d |dO_id v_jd|: the fp32 dP;
      dD_i = sum_d |dO_id| B^o_id + dv_slot U23 sum_d |dO_id| (|o_id| + B^o_id): delta from o~ in fp32;
      G_ij = (U8 + eps_ij) |dS_ij| + p_ij (1 + eps_ij) (e'_ij + dD_i) + FLUSH (|dP_ij - D_i| + e'_ij + dD_i):
        the error of the bf16 dS the kernels multiply;
      dv_jd <= U8 |dv_jd| + sum_i ((U8 + eps_ij) p_ij + FLUSH) |dO_id| + g'_j sum_i p_ij |dO_id|
      dk_jd <= U8 |dk_jd| + c sum_i G_ij |q_id| + g'_j c sum_i (|dS_ij| + G_ij) |q_id|
      dq_id <= U8 |dq_id| + c sum_j G_ij |k_jd| + g''_i c sum_j (|dS_ij| + G_ij) |k_jd|
      with g'_j = (n'_j + 8) U23 (n'_j queries see key j) and g''_i = (n_i + 8) U23 for the fp32 sums and the final
      multiply by c.
Higher-order products of these small terms are covered by one safety factor, SAFETY = 2, applied to every bound here
and nowhere else.  `check` applies it."""

import math

import torch

import _checks
from _checks import check_equal  # noqa: F401  (re-exported for the attention tests)

U24 = 2.0 ** -24
U23 = 2.0 ** -23
U8 = 2.0 ** -8
EX2 = 2.0 ** -22    # relative error of ex2.approx.f32 (2 ulp); __expf is ex2.approx of x log2(e)
LG2 = 2.0 ** -21    # absolute error of __logf (lg2.approx times ln 2) at l >= 1, per unit of log l beyond 1
FLUSH = 2.0 ** -120  # absolute error of a p or alpha flushed to zero below 2^-126, with margin for the normalisation
SAFETY = 2.0
F64, BF16 = torch.float64, torch.bfloat16

REGIMES = ("randn", "peaked", "rising", "sink", "diagonal", "ties", "extreme")


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def make_inputs(regime, N, H, S, dk, dv, seed, device="cpu"):
    """q, k: [N, H, S, dk] and v, dO: [N, H, S, dv], bf16 on `device`, drawn on the CPU from `seed`.  dk is the true
    head width, so c q.k has the stated spread for c = 1/sqrt(dk):
      randn     q, k, v, dO ~ N(0, 1): c q.k ~ N(0, 1), p nearly uniform;
      peaked    c q.k ~ N(0, 64): a few keys hold the mass, many p flush to zero;
      rising    c q.k_j = 3 j / 128 + N(0, 0.09): the row max moves into every 128-key tile (and every decode split);
      sink      c q.k_0 = 20, the rest N(0, 0.09): the max stays in tile 0, later tiles add e^-20-sized terms;
      diagonal  q_i = 16 k_i / sqrt(dk): c q_i.k_i ~ 16, c q_i.k_j ~ N(0, 256 / dk), each row's own key dominates;
      ties      q = 0: p exactly uniform, o_i the mean of the visible v;
      extreme   c q.k ~ N(0, 625): |c s| up to about 80."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g)
    q, k = rn(N, H, S, dk), rn(N, H, S, dk)
    rd = math.sqrt(dk)
    if regime == "peaked":
        q, k = q * math.sqrt(8.0), k * math.sqrt(8.0)
    elif regime == "extreme":
        q, k = q * 5.0, k * 5.0
    elif regime in ("rising", "sink"):
        u = torch.where(rn(N, H, 1, dk) >= 0, 1.0, -1.0)  # |u|^2 = dk, exact in bf16
        j = torch.arange(S, dtype=torch.float32).view(1, 1, S, 1)
        t = 3.0 * j / 128 if regime == "rising" else 20.0 * (j == 0).float()
        k = t / rd * u + 0.3 * k
        q = u.expand(N, H, S, dk).clone()
    elif regime == "diagonal":
        q = k * (16.0 / rd)
    elif regime == "ties":
        q = torch.zeros_like(q)
    else:
        assert regime == "randn", regime
    v, do = rn(N, H, S, dv), rn(N, H, S, dv)
    return tuple(t.to(BF16).to(device) for t in (q, k, v, do))


# ----------------------------------------------------------------------------------------------------------------------
# reference and bounds
# ----------------------------------------------------------------------------------------------------------------------
def _head(q, k, v, do, qpos, c, strict, ks, vs, backward):
    """One (image, head): q [Sq, dk] at positions qpos, k [Sk, dk], v [Sk, dv], do [Sq, dv] -> dict of float64."""
    q, k, v = q.to(F64), k.to(F64), v.to(F64)
    Sk = k.shape[0]
    vis = torch.arange(Sk, device=q.device).view(1, -1) <= (qpos.view(-1, 1) - int(strict))
    visf = vis.to(F64)
    n = visf.sum(1)
    has = n > 0
    s = c * (q @ k.T)
    sm = s.masked_fill(~vis, -math.inf)
    mx = torch.where(has, sm.amax(1), torch.zeros_like(n))
    ex = torch.exp(sm - mx[:, None])
    l = ex.sum(1)
    p = torch.where(has[:, None], ex / torch.where(has, l, torch.ones_like(l))[:, None], torch.zeros_like(ex))
    lse = torch.where(has, mx + torch.log(torch.where(has, l, torch.ones_like(l))), torch.zeros_like(l))
    o = p @ v

    A = c * (q.abs() @ k.abs().T)
    R = (s.abs() * visf).amax(1)
    T = (qpos // 128 + 1).to(F64)
    e = visf * (ks * U23 * A + 2.0 ** -20 * R[:, None] + ((T + 1) * EX2)[:, None])
    E = e.amax(1)
    gam = (n + 2 * T + 4) * U23
    M = p @ v.abs()
    b_o = U8 * o.abs() + (U8 + 2 * E + 2 * gam + 2.0 ** -22)[:, None] * M + FLUSH * (visf @ v.abs())
    b_lse = E + gam + LG2 * (1 + torch.log(n.clamp_min(1))) + 2.0 ** -22 * (R + lse.abs())
    out = dict(o=o, lse=lse, b_o=b_o, b_lse=b_lse, has=has)
    if not backward:
        return out

    dO = do.to(F64)
    dP = dO @ v.T
    D = (dO * o).sum(1)
    dS = p * (dP - D[:, None])
    eps = visf * (e + (b_lse + 2.0 ** -20 * (R + lse.abs()) + 2.0 ** -21)[:, None])
    e2 = vs * U23 * (dO.abs() @ v.abs().T)
    dD = (dO.abs() * b_o).sum(1) + vs * U23 * (dO.abs() * (o.abs() + b_o)).sum(1)
    G = (U8 + eps) * dS.abs() + p * (1 + eps) * (e2 + dD[:, None]) + FLUSH * visf * ((dP - D[:, None]).abs() + e2 + dD[:, None])
    g_k = (visf.sum(0) + 8) * U23
    g_q = (n + 8) * U23
    dSa = dS.abs() + G
    dq, dk, dv = c * (dS @ k), c * (dS.T @ q), p.T @ dO
    out.update(
        D=D, dq=dq, dk=dk, dv=dv,
        b_dv=U8 * dv.abs() + ((U8 + eps) * p + FLUSH * visf).T @ dO.abs() + g_k[:, None] * (p.T @ dO.abs()),
        b_dk=U8 * dk.abs() + c * (G.T @ q.abs()) + g_k[:, None] * c * (dSa.T @ q.abs()),
        b_dq=U8 * dq.abs() + c * (G @ k.abs()) + g_q[:, None] * c * (dSa @ k.abs()),
    )
    return out


def attention(q, k, v, do, strict, dk_true, ks, vs, backward=True):
    """Reference and bounds for full causal attention.  q, k: [N, H, S, dk_true]; v, do: [N, H, S, dv_true] (bf16);
    ks, vs: the slot widths the kernel sums over.  Returns a dict of float64 tensors stacked to [N, H, S(, d)]."""
    N, H, S, _ = q.shape
    c = 1.0 / math.sqrt(dk_true)
    qpos = torch.arange(S, device=q.device)
    heads = [_head(q[n, h], k[n, h], v[n, h], do[n, h], qpos, c, strict, ks, vs, backward)
             for n in range(N) for h in range(H)]
    return {key: torch.stack([r[key] for r in heads]).view(N, H, *heads[0][key].shape) for key in heads[0]}


def decode_row(q, k, v, pos, strict, dk_true, ks):
    """Reference and forward bounds of one KV-cached step: q [N, H, dk] at position pos against keys k [N, H, S, dk]
    and values v [N, H, S, dv] (rows past pos are never visible).  Returns o, b_o: [N, H, dv]."""
    N, H = q.shape[:2]
    c = 1.0 / math.sqrt(dk_true)
    qpos = torch.tensor([pos], device=q.device)
    rows = [_head(q[n, h].unsqueeze(0), k[n, h, :pos + 1], v[n, h, :pos + 1], None, qpos, c, strict, ks, 0, False)
            for n in range(N) for h in range(H)]
    return (torch.stack([r["o"][0] for r in rows]).view(N, H, -1),
            torch.stack([r["b_o"][0] for r in rows]).view(N, H, -1))


# ----------------------------------------------------------------------------------------------------------------------
# comparisons
# ----------------------------------------------------------------------------------------------------------------------
def violations(got, ref, bound):
    """Elements with |got - ref| > SAFETY bound (NaN always counts), as a boolean tensor."""
    return _checks.violations(got, ref, SAFETY * bound)


def check(name, got, ref, bound):
    """|got - ref| <= SAFETY bound element by element (tests/_checks.py); NaN fails."""
    _checks.check(name, got, ref, SAFETY * bound)
