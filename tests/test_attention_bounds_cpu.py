"""Tests of the attention kernel tests, without a GPU: the bounds of tests/_attention_reference.py must accept an fp32
emulation of the kernels' arithmetic and reject the same emulation with one of seven plausible kernel bugs.

The emulation follows csrc/pg_attention_tc.cuh and csrc/pg_attention.cu step by step, on the CPU in fp32 from the
bf16 inputs: forward over 128-query tiles and 128-key tiles with an online max, exp2 of s c log2(e) - m c log2(e), the
alpha rescaling of O and l, P rounded to bf16 for O += P V and fp32 sums; backward dK / dV over 64-query tiles and dQ
over 128-key tiles with p recomputed from the emulated lse, delta from the emulated bf16 o, and P and dS rounded to
bf16; the KV-cached decode over 1024-key splits and their merge.  Each bug model is the emulation with one change,
each a masking or arithmetic slip a kernel edit can plausibly make:
  mask_shift   the diagonal-tile mask one key too far (j <= i - strict + 1) on query tiles after the first;
  l_no_alpha   l not rescaled by alpha when the running max moves;
  scale_slot   the scale 1/sqrt(slot width) instead of 1/sqrt(dk_true);
  drop_tile    key tile 0 dropped for the last query tile;
  late_qtile   the dK / dV loop skipping its first 64-query tile for key tiles after the first;
  delta_pair   dQ taking delta from the other row of the thread's pair (row r ^ 8 of the 128-row tile);
  merge_f1     the decode merge weighting every split by f = 1 instead of exp(m_s - m)."""

import math

import pytest
import torch

import _attention_reference as R

F32 = torch.float32
LOG2E = 1.4426950408889634
BUGS = ("mask_shift", "l_no_alpha", "scale_slot", "drop_tile", "late_qtile", "delta_pair", "merge_f1")


def _bf(x):
    return x.to(torch.bfloat16).to(F32)


def _f32(x):
    return torch.tensor(x, dtype=F32)


# ----------------------------------------------------------------------------------------------------------------------
# fp32 emulations of one (image, head)
# ----------------------------------------------------------------------------------------------------------------------
def emu_forward(q, k, v, scale, strict, bug=None):
    """o (bf16 values as fp32) and lse of attn_fwd_tc_kernel for q, k [S, dk], v [S, dv]."""
    S = q.shape[0]
    qf, kf, vf = q.float(), k.float(), v.float()
    c = _f32(scale)
    sl2 = c * _f32(LOG2E)
    T = (S + 127) // 128
    o = torch.zeros(S, v.shape[1])
    lse = torch.zeros(S)
    for i in range(T):
        rows = torch.arange(i * 128, min(S, i * 128 + 128))
        qlim = rows - int(strict) + (1 if bug == "mask_shift" and i > 0 else 0)
        m = torch.full((len(rows),), -math.inf)
        l = torch.zeros(len(rows))
        O = torch.zeros(len(rows), v.shape[1])
        for j in range(i + 1):
            keys = torch.arange(j * 128, min(S, j * 128 + 128))
            s = qf[rows] @ kf[keys].T
            if j == i:
                s = s.masked_fill(keys[None, :] > qlim[:, None], -math.inf)
            if bug == "drop_tile" and i == T - 1 and j == 0 and T > 1:
                s = torch.full_like(s, -math.inf)
            mx = torch.maximum(m, s.amax(1))
            mu = torch.where(mx == -math.inf, torch.zeros_like(mx), mx)
            alpha = torch.exp2((m - mu) * sl2)
            P = torch.exp2(s * sl2 - (mu * sl2)[:, None])
            l = (l if bug == "l_no_alpha" else l * alpha) + P.sum(1)
            m = mx
            O = O * alpha[:, None] + _bf(P) @ vf[keys]
        inv = torch.where(l > 0, 1 / l, torch.zeros_like(l))
        o[rows] = _bf(O * inv[:, None])
        lse[rows] = torch.where(l > 0, m * c + torch.log(l), torch.zeros_like(l))
    return o, lse


def emu_backward(q, k, v, o, do, lse, scale, strict, bug=None):
    """dq, dk, dv (bf16 values as fp32) and delta of the delta kernel, attn_bwd_tc_kernel and attn_dq_tc_kernel."""
    S = q.shape[0]
    qf, kf, vf, dof = q.float(), k.float(), v.float(), do.float()
    c = _f32(scale)
    sl2 = c * _f32(LOG2E)
    delta = (dof * o).sum(1)
    lse2 = lse * _f32(LOG2E)
    T, TQ = (S + 127) // 128, (S + 63) // 64
    dq, dk, dv = torch.zeros_like(qf), torch.zeros_like(kf), torch.zeros_like(vf)
    for j in range(T):
        keys = torch.arange(j * 128, min(S, j * 128 + 128))
        dV, dK = torch.zeros(len(keys), v.shape[1]), torch.zeros(len(keys), q.shape[1])
        for it in range(2 * j, TQ):
            qs = torch.arange(it * 64, min(S, it * 64 + 64))
            vis = keys[:, None] <= qs[None, :] - int(strict)
            if bug == "late_qtile" and j > 0 and it == 2 * j:
                vis = torch.zeros_like(vis)
            p = torch.where(vis, torch.exp2(kf[keys] @ qf[qs].T * sl2 - lse2[qs][None, :]), torch.zeros(()))
            ds = p * (vf[keys] @ dof[qs].T - delta[qs][None, :])
            dV += _bf(p) @ dof[qs]
            dK += _bf(ds) @ qf[qs]
        dv[keys], dk[keys] = _bf(dV), _bf(dK * c)
    for i in range(T):
        rows = torch.arange(i * 128, min(S, i * 128 + 128))
        dl = delta[rows]
        if bug == "delta_pair":
            partner = rows ^ 8
            dl = torch.where(partner < S, delta[partner.clamp_max(S - 1)], torch.zeros(()))
        dQ = torch.zeros(len(rows), q.shape[1])
        for j in range(i + 1):
            keys = torch.arange(j * 128, min(S, j * 128 + 128))
            vis = keys[None, :] <= rows[:, None] - int(strict)
            p = torch.where(vis, torch.exp2(qf[rows] @ kf[keys].T * sl2 - lse2[rows][:, None]), torch.zeros(()))
            dQ += _bf(p * (dof[rows] @ vf[keys].T - dl[:, None])) @ kf[keys]
        dq[rows] = _bf(dQ * c)
    return dq, dk, dv, delta


def emu_decode(q, k, v, pos, scale, strict, bug=None, split=1024):
    """attn_decode_kernel<SPLIT> and attn_decode_merge_kernel for one (image, head): q [dk] at position pos against the
    cache rows k [S, dk], v [S, dv]."""
    S = k.shape[0]
    qf, kf, vf = q.float(), k.float(), v.float()
    c = _f32(scale)
    nkeys = pos + (0 if strict else 1)
    parts = []
    for s0 in range(0, S, split):
        keys = torch.arange(s0, max(s0, min(nkeys, s0 + split)))
        if len(keys) == 0:
            parts.append((_f32(-math.inf), _f32(0.0), torch.zeros(v.shape[1])))
            continue
        sc = (kf[keys] @ qf) * c
        m = sc.max()
        p = torch.exp(sc - m)
        parts.append((m, p.sum(), p @ vf[keys]))
    m = max(pm for pm, _, _ in parts)
    l, acc = _f32(0.0), torch.zeros(v.shape[1])
    for pm, pl, po in parts:
        f = _f32(1.0) if (pm == m or bug == "merge_f1") else torch.exp(pm - m)
        l = l + pl * f
        acc = acc + po * f
    return _bf(acc * (1 / l if nkeys > 0 else 0.0))


# ----------------------------------------------------------------------------------------------------------------------
# running the emulation against the bounds
# ----------------------------------------------------------------------------------------------------------------------
FULL_CASES = [  # S, slot widths and true widths: one 64-slot and one 128-slot head, both narrower than their slots
    (300, 64, 40, 64, 48),
    (300, 128, 72, 128, 100),
]
DECODE_S, DECODE_POS = 2100, (0, 1, 1023, 1024, 1500, 2099)


def _full(regime, strict, case, bug=None, seed=0):
    """Emulated outputs and references of one head; returns [(name, got, ref, bound)]."""
    S, ks, dk, vs, dv = case
    q, k, v, do = (t[0, 0] for t in R.make_inputs(regime, 1, 1, S, dk, dv, seed))
    ref = R.attention(*(t.view(1, 1, S, -1) for t in (q, k, v, do)), strict, dk, ks, vs)
    ref = {key: t[0, 0] for key, t in ref.items()}
    scale = 1 / math.sqrt(ks if bug == "scale_slot" else dk)
    o, lse = emu_forward(q, k, v, scale, strict, bug)
    dq, dk_, dv_, _ = emu_backward(q, k, v, o, do, lse, scale, strict, bug)
    return [("o", o, ref["o"], ref["b_o"]), ("lse", lse, ref["lse"], ref["b_lse"]),
            ("dq", dq, ref["dq"], ref["b_dq"]), ("dk", dk_, ref["dk"], ref["b_dk"]), ("dv", dv_, ref["dv"], ref["b_dv"])]


def _decode(regime, strict, bug=None, seed=0):
    dk, ks, dv = 16, 64, 64
    q, k, v, _ = (t[0, 0] for t in R.make_inputs(regime, 1, 1, DECODE_S, dk, dv, seed))
    out = []
    for pos in DECODE_POS:
        o = emu_decode(q[pos], k, v, pos, 1 / math.sqrt(ks if bug == "scale_slot" else dk), strict, bug)
        ref, b = R.decode_row(q[pos].view(1, 1, -1), k.view(1, 1, DECODE_S, -1), v.view(1, 1, DECODE_S, -1), pos,
                              strict, dk, ks)
        out.append((f"decode pos {pos}", o, ref[0, 0], b[0, 0]))
    return out


def _fails(results):
    return [name for name, got, ref, b in results if R.violations(got, ref, b).any()]


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("regime", R.REGIMES)
@pytest.mark.parametrize("case", FULL_CASES)
def test_emulation_within_bounds(regime, strict, case):
    """The fp32 emulation of the tensor-core forward and backward meets every bound, in every input regime."""
    for name, got, ref, bound in _full(regime, strict, case):
        R.check(f"{regime} strict={strict} {case} {name}", got, ref, bound)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("regime", ["peaked", "rising", "sink"])
def test_decode_emulation_within_bounds(regime, strict):
    """The fp32 emulation of the split decode and its merge meets the forward bound on both sides of a split edge."""
    for name, got, ref, bound in _decode(regime, strict):
        R.check(f"{regime} strict={strict} {name}", got, ref, bound)


def _bug_results(bug, regime, strict):
    if bug == "merge_f1":
        return _decode(regime, strict, bug)
    return [r for case in FULL_CASES for r in _full(regime, strict, case, bug)]


# the regime under which each bug model must break the bound (any one suffices; these are the ones that show it)
BUG_REGIMES = {
    "mask_shift": ("diagonal", True),
    "l_no_alpha": ("rising", False),
    "scale_slot": ("peaked", False),
    "drop_tile": ("sink", False),
    "late_qtile": ("diagonal", False),
    "delta_pair": ("randn", False),
    "merge_f1": ("rising", False),
}


@pytest.mark.parametrize("bug", BUGS)
def test_bug_model_breaks_the_bound(bug):
    """Each bug model applied to the emulation puts elements outside the bound."""
    regime, strict = BUG_REGIMES[bug]
    failed = _fails(_bug_results(bug, regime, strict))
    assert failed, f"bug model {bug} stays within every bound under {regime} strict={strict}"
